// Parameter gradients of the fine-tuning path (`unfreeze_model`, ddpm.py:1450-1452: the UNet and the CLIP text encoder
// train next to the embedding): convolution weight gradients on the cb_gemm wgmma main loop, bias and per-image column
// sums, GroupNorm / LayerNorm affine gradients and the token-embedding gradient.  Every sum is taken in a fixed order, so
// each result is bit-identical from run to run.
#include <string.h>

#include <cooperative_groups.h>

#include "cb_common.cuh"

namespace cb {

// ---- tap gather for the convolution weight gradient ---------------------------------------------------------------
// col[p][ci*K*K + t] = x[n][oh*stride + ky - pad][ow*stride + kx - pad][ci] (0 outside the image) for output pixel
// p = (n, oh, ow) in raster order and tap t = ky*K + kx.  A row of col is ordered like a row of the nn.Parameter
// [Cout][Cin][kh][kw], so the GEMM dW = dy^T col writes the parameter layout directly.  One thread per (pixel, 8 channels):
// a 16-byte load per tap (the element bits are copied, whatever the 16-bit type), a register transpose, and K*K 16-byte
// stores of the 8*K*K contiguous elements.
template <int K>
__global__ void __launch_bounds__(256)
wgrad_gather_kernel(const unsigned short* __restrict__ x, long long ldx, unsigned short* __restrict__ col, int H, int W,
                    int cin, int OH, int OW, int stride, int pad, long long total) {
    pdl_sync();
    constexpr int T = K * K;
    const int groups = cin >> 3;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long p = i / groups;
        const int cg = (int)(i - p * groups);
        const int ow = (int)(p % OW);
        const long long q = p / OW;
        const int oh = (int)(q % OH);
        const long long n = q / OH;
        uint32_t in[T][4];
#pragma unroll
        for (int t = 0; t < T; ++t) {
            const int ih = oh * stride + t / K - pad, iw = ow * stride + t % K - pad;
            uint4 v = make_uint4(0u, 0u, 0u, 0u);
            if (ih >= 0 && ih < H && iw >= 0 && iw < W)
                v = *reinterpret_cast<const uint4*>(x + ((n * H + ih) * W + iw) * ldx + cg * 8);
            in[t][0] = v.x; in[t][1] = v.y; in[t][2] = v.z; in[t][3] = v.w;
        }
        // element e = j*T + t of the output run is channel j of tap t
        uint32_t out[T * 4];
#pragma unroll
        for (int w = 0; w < T * 4; ++w) {
            const int e0 = 2 * w, e1 = 2 * w + 1;
            const uint32_t lo = (in[e0 % T][(e0 / T) >> 1] >> (16 * ((e0 / T) & 1))) & 0xFFFFu;
            const uint32_t hi = (in[e1 % T][(e1 / T) >> 1] >> (16 * ((e1 / T) & 1))) & 0xFFFFu;
            out[w] = lo | (hi << 16);
        }
        uint4* dst = reinterpret_cast<uint4*>(col + p * (long long)cin * T + (long long)cg * 8 * T);
#pragma unroll
        for (int t = 0; t < T; ++t) dst[t] = make_uint4(out[4 * t], out[4 * t + 1], out[4 * t + 2], out[4 * t + 3]);
    }
}

// ---- column sums ----------------------------------------------------------------------------------------------------
// A thread-block cluster of S CTAs (1, S, 1) owns 32 columns; each CTA has 32 row lanes (warps), so row lane
// L = rank*32 + w adds rows L, L + 32*S, ... in order.  Each CTA adds its 32 lane sums in order, then rank 0 adds the S CTA
// sums in rank order through distributed shared memory.  S depends on the row count only (row_split), so the order of
// every sum is fixed by the shape.
constexpr int kRedLanes = 32;
constexpr int kMaxRowSplit = 8;     // portable cluster size

// CTAs per column tile: enough rows for every warp of the cluster to add at least 32 of them
static inline int row_split(long long rows) {
    long long s = rows / (32LL * kRedLanes);
    return (int)(s < 1 ? 1 : (s > kMaxRowSplit ? kMaxRowSplit : s));
}

// in-order sum of the 32 lane partials of each column, then of the cluster's CTAs in rank order; result valid in rank 0,
// warp 0.  Called by every thread of every CTA of the cluster.
template <int NV>
__device__ __forceinline__ void cluster_colsum(float (&v)[NV], float (*s_lane)[kRedLanes][33], float (*s_cta)[32]) {
    namespace cg = cooperative_groups;
    cg::cluster_group cl = cg::this_cluster();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < NV; ++k) s_lane[k][w][lane] = v[k];
    __syncthreads();
    if (w == 0) {
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            float t = 0.f;
#pragma unroll 8
            for (int i = 0; i < kRedLanes; ++i) t += s_lane[k][i][lane];
            s_cta[k][lane] = t;
        }
    }
    cl.sync();
    if (cl.block_rank() == 0 && w == 0) {
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            float t = 0.f;
            for (unsigned q = 0; q < cl.num_blocks(); ++q) t += cl.map_shared_rank(&s_cta[k][0], q)[lane];
            v[k] = t;
        }
    }
    cl.sync();      // the other CTAs keep their shared memory until rank 0 has read it
}

template <typename T>
__global__ void __launch_bounds__(1024)
colsum_kernel(const T* __restrict__ x, long long ldx, float* __restrict__ out, long long rows_per_group, int C,
              float alpha) {
    pdl_sync();
    __shared__ float s_lane[1][kRedLanes][33];
    __shared__ float s_cta[1][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + lane;
    const int L = blockIdx.y * kRedLanes + w, stride = gridDim.y * kRedLanes;
    const T* xg = x + (long long)blockIdx.z * rows_per_group * ldx;
    float acc[1] = {0.f};
    if (c < C)
        for (long long r = L; r < rows_per_group; r += stride) acc[0] += cvt<T>::to_f(xg[r * ldx + c]);
    cluster_colsum<1>(acc, s_lane, s_cta);
    if (blockIdx.y == 0 && w == 0 && c < C) out[(long long)blockIdx.z * C + c] = alpha * acc[0];
}

// ---- GroupNorm / LayerNorm affine gradients -------------------------------------------------------------------------
// dgamma[c] = alpha * sum dz * xh, dbeta[c] = alpha * sum dz over every row, xh = (x - mean) * rstd with the forward's
// saved statistics, dz = dy (times silu'(xh*gamma + beta) where the forward fused SiLU).  GN = true: rows are N images of
// HW pixels and the statistics are [N][G]; GN = false (LayerNorm): one statistic per row.  Same thread map and order as
// colsum_kernel; GroupNorm visits the rows image by image.
template <typename TG, typename TX, bool GN>
__global__ void __launch_bounds__(1024)
norm_affine_bwd_kernel(const TG* __restrict__ dy, const TX* __restrict__ x, const float* __restrict__ gamma,
                       const float* __restrict__ beta, const float* __restrict__ mean, const float* __restrict__ rstd,
                       float* __restrict__ dgamma, float* __restrict__ dbeta, int N, int HW, int C, int G, int silu,
                       float alpha) {
    pdl_sync();
    __shared__ float s_lane[2][kRedLanes][33];
    __shared__ float s_cta[2][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + lane;
    const int L = blockIdx.y * kRedLanes + w, stride = gridDim.y * kRedLanes;
    float acc[2] = {0.f, 0.f};      // dgamma, dbeta
    if (c < C) {
        const float ga = silu ? gamma[c] : 0.f, be = silu ? beta[c] : 0.f;
        const int g = GN ? c / (C / G) : 0;
        // GroupNorm: every lane visits each image and takes its pixels L, L+stride, ...; LayerNorm: rows L, L+stride, ...
        for (int n = GN ? 0 : L; n < N; n += GN ? 1 : stride) {
            const float m = mean[GN ? n * G + g : n], rs = rstd[GN ? n * G + g : n];
            for (int r = GN ? L : 0; r < HW; r += GN ? stride : 1) {
                const long long off = ((long long)n * HW + r) * C + c;
                const float xh = (cvt<TX>::to_f(x[off]) - m) * rs;
                float d = cvt<TG>::to_f(dy[off]);
                if (silu) d *= silu_grad(xh * ga + be);
                acc[0] += d * xh;
                acc[1] += d;
            }
        }
    }
    cluster_colsum<2>(acc, s_lane, s_cta);
    if (blockIdx.y == 0 && w == 0 && c < C) {
        if (dgamma) dgamma[c] = alpha * acc[0];
        if (dbeta) dbeta[c] = alpha * acc[1];
    }
}

// ---- token-embedding gradient ---------------------------------------------------------------------------------------
// One CTA per token i.  Only the first token of each id writes: it adds the rows of every token with that id in token
// order (no atomics, so repeated ids give the same bits every run).
__device__ __forceinline__ long long clamp_id(long long id, int V) { return id < 0 ? 0 : (id >= V ? V - 1 : id); }

__global__ void __launch_bounds__(256)
embedding_bwd_kernel(const long long* __restrict__ ids, const float* __restrict__ dout, long long ld,
                     float* __restrict__ dtable, int n, int D, int V, float alpha) {
    pdl_sync();
    const int i = blockIdx.x;
    const long long v = clamp_id(ids[i], V);
    int dup = 0;
    for (int j = threadIdx.x; j < i; j += blockDim.x) dup |= clamp_id(ids[j], V) == v;
    if (__syncthreads_or(dup)) return;
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
        float acc = 0.f;
        for (int j = i; j < n; ++j)
            if (clamp_id(ids[j], V) == v) acc += dout[(long long)j * ld + d];
        dtable[v * D + d] = alpha * acc;
    }
}

// split-K slices of the weight-gradient GEMM: about two CTAs per SM (the 3-stage ring), at least 8 k-iterations per slice;
// 1 when cb_gemm could not split this shape
static int wgrad_splits(int cout, int n_cols, long long P) {
    const long long tiles = (long long)ceil_div(n_cols, 128) * ceil_div(cout, 128);
    const long long kiters = ceil_div64(P, 64);
    long long sp = 2LL * device_sm_count() / tiles;
    if (sp > 8) sp = 8;
    if (sp > kiters / 8) sp = kiters / 8;
    if (sp < 2 || gemm_splitk_ws_bytes(n_cols, ceil_div(cout, 128), 1, 2) < 0) return 1;
    return gemm_split_count((int)kiters, (int)sp);
}

}  // namespace cb

using namespace cb;

#define CB_WG_DISPATCH(dtype, T, ...)                                              \
    do {                                                                           \
        if ((dtype) == CB_F32) { using T = float; __VA_ARGS__; }                   \
        else if ((dtype) == CB_F16) { using T = __half; __VA_ARGS__; }             \
        else if ((dtype) == CB_BF16) { using T = __nv_bfloat16; __VA_ARGS__; }     \
        else CB_REQUIRE(false, CB_ERR_ARG, "bad dtype %d", (int)(dtype));         \
    } while (0)

static bool conv_wgrad_geometry(int N, int H, int W, int cin, int cout, int k, int stride, int pad, int* OH, int* OW) {
    if (N <= 0 || H <= 0 || W <= 0 || cin <= 0 || cout <= 0 || (k != 1 && k != 3) || stride < 1 || pad < 0) return false;
    *OH = (H + 2 * pad - k) / stride + 1;
    *OW = (W + 2 * pad - k) / stride + 1;
    return *OH > 0 && *OW > 0 && H + 2 * pad >= k && W + 2 * pad >= k;
}

extern "C" int cb_conv_wgrad_ws_bytes(int N, int H, int W, int cin, int cout, int k, int stride, int pad,
                                      long long* col_bytes, long long* splitk_bytes) {
    int OH, OW;
    CB_REQUIRE(conv_wgrad_geometry(N, H, W, cin, cout, k, stride, pad, &OH, &OW) && col_bytes && splitk_bytes, CB_ERR_ARG,
               "conv_wgrad_ws_bytes: bad geometry");
    const long long P = (long long)N * OH * OW;
    const int n_cols = cin * k * k;
    const bool direct = k == 1 && stride == 1 && pad == 0;
    const int sp = wgrad_splits(cout, n_cols, P);
    *col_bytes = direct ? 0 : P * n_cols * 2;
    *splitk_bytes = gemm_splitk_ws_bytes(n_cols, ceil_div(cout, 128), 1, sp);
    return 0;
}

extern "C" int cb_conv_wgrad(const void* x, long long ldx, const void* dy, long long lddy, int dtype, int N, int H, int W,
                             int cin, int cout, int k, int stride, int pad, float alpha, float* dW, void* col,
                             void* splitk_ws, long long splitk_ws_bytes, void* stream) {
    int OH, OW;
    CB_REQUIRE(conv_wgrad_geometry(N, H, W, cin, cout, k, stride, pad, &OH, &OW), CB_ERR_ARG, "conv_wgrad: bad geometry");
    CB_REQUIRE(dtype == CB_F16 || dtype == CB_BF16, CB_ERR_ARG, "conv_wgrad: dtype must be f16 or bf16");
    CB_REQUIRE(x && dy && dW, CB_ERR_ARG, "conv_wgrad: NULL x / dy / dW");
    CB_REQUIRE(cin % 8 == 0 && cout % 8 == 0 && ldx >= cin && lddy >= cout && ldx % 8 == 0 && lddy % 8 == 0, CB_ERR_ALIGN,
               "conv_wgrad: channels and row pitches must be multiples of 8");
    CB_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dW) |
                 reinterpret_cast<uintptr_t>(col)) & 15u) == 0,
               CB_ERR_ALIGN, "conv_wgrad: x, dy, dW and col must be 16-byte aligned");
    long long col_need, sk_need;
    int rc = cb_conv_wgrad_ws_bytes(N, H, W, cin, cout, k, stride, pad, &col_need, &sk_need);
    if (rc) return rc;
    CB_REQUIRE(col_need == 0 || col, CB_ERR_ARG, "conv_wgrad: this geometry needs the col buffer");
    CB_REQUIRE(sk_need == 0 || (splitk_ws && splitk_ws_bytes >= sk_need), CB_ERR_ARG,
               "conv_wgrad: split-K workspace of %lld bytes needed", sk_need);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long P = (long long)N * OH * OW;
    const int n_cols = cin * k * k;
    if (col_need) {
        const long long total = P * (cin / 8);
        const long long want = (total + 255) / 256;
        const unsigned grid = (unsigned)(want < 65535LL * 8 ? want : 65535LL * 8);
        if (k == 3)
            CB_CUDA(CB_LAUNCH((wgrad_gather_kernel<3>), grid, 256, 0, st, (const unsigned short*)x, ldx,
                              (unsigned short*)col, H, W, cin, OH, OW, stride, pad, total));
        else
            CB_CUDA(CB_LAUNCH((wgrad_gather_kernel<1>), grid, 256, 0, st, (const unsigned short*)x, ldx,
                              (unsigned short*)col, H, W, cin, OH, OW, stride, pad, total));
        count_launches(1);
    }
    CB_REQUIRE(P <= 0x7FFFFFFF, CB_ERR_ARG, "conv_wgrad: too many output pixels");
    cb_gemm_desc d;
    memset(&d, 0, sizeof(d));
    d.M = cout;
    d.N = n_cols;
    d.K = (int32_t)P;
    d.batch = 1;
    d.ab_dtype = dtype;
    d.A = dy;
    d.lda = lddy;
    d.a_major = CB_MAJOR_MN;
    d.B = col_need ? col : x;
    d.ldb = col_need ? n_cols : ldx;
    d.b_major = CB_MAJOR_MN;
    d.D = dW;
    d.d_dtype = CB_F32;
    d.ldd = n_cols;
    d.alpha = alpha;
    d.act = CB_ACT_NONE;
    const int sp = wgrad_splits(cout, n_cols, P);
    if (sp > 1) {
        d.splitk_ws = splitk_ws;
        d.splitk_ws_bytes = splitk_ws_bytes;
        d.splits = sp;
    } else {
        d.splits = 1;
    }
    return cb_gemm(&d, stream);
}

extern "C" int cb_colsum(const void* x, int x_dtype, long long ldx, float* out, long long rows, int C, int groups,
                         float alpha, void* stream) {
    CB_REQUIRE(x && out && rows > 0 && C > 0 && ldx >= C && groups > 0 && groups <= 65535 && rows % groups == 0,
               CB_ERR_ARG, "colsum: bad shape");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int S = row_split(rows / groups);
    const dim3 grid((unsigned)ceil_div(C, 32), (unsigned)S, (unsigned)groups);
    CB_WG_DISPATCH(x_dtype, T, CB_CUDA(launch_kernel_cluster((colsum_kernel<T>), grid, dim3(1024), dim3(1, S, 1), 0, st,
                                                             (const T*)x, ldx, out, rows / groups, C, alpha)));
    count_launches(1);
    return 0;
}

#define CB_NORM_AFFINE_LAUNCH(GN)                                                                                          \
    const int S = row_split((long long)N * HW);                                                                            \
    CB_WG_DISPATCH(dy_dtype, TG, CB_WG_DISPATCH(x_dtype, TX, CB_CUDA(launch_kernel_cluster(                                \
        (norm_affine_bwd_kernel<TG, TX, GN>), dim3((unsigned)ceil_div(C, 32), (unsigned)S), dim3(1024), dim3(1, S, 1), 0,  \
        st, (const TG*)dy, (const TX*)x, gamma, beta, mean, rstd, dgamma, dbeta, N, HW, C, G, silu, alpha))))

extern "C" int cb_groupnorm_affine_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, const float* gamma,
                                       const float* beta, const float* mean, const float* rstd, float* dgamma,
                                       float* dbeta, int N, int HW, int C, int G, int act_silu, float alpha,
                                       void* stream) {
    CB_REQUIRE(dy && x && mean && rstd && (dgamma || dbeta), CB_ERR_ARG, "groupnorm_affine_bwd: NULL pointer");
    CB_REQUIRE(N > 0 && HW > 0 && C > 0 && G > 0 && C % G == 0, CB_ERR_ARG, "groupnorm_affine_bwd: bad shape");
    const int silu = act_silu & 1;
    CB_REQUIRE(!silu || (gamma && beta), CB_ERR_ARG, "groupnorm_affine_bwd: the SiLU route needs gamma and beta");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    CB_NORM_AFFINE_LAUNCH(true);
    count_launches(1);
    return 0;
}

extern "C" int cb_layernorm_affine_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, const float* mean,
                                       const float* rstd, float* dgamma, float* dbeta, int M, int C, float alpha,
                                       void* stream) {
    CB_REQUIRE(dy && x && mean && rstd && (dgamma || dbeta), CB_ERR_ARG, "layernorm_affine_bwd: NULL pointer");
    CB_REQUIRE(M > 0 && C > 0, CB_ERR_ARG, "layernorm_affine_bwd: bad shape");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int N = M, HW = 1, G = 1, silu = 0;
    const float* gamma = nullptr;
    const float* beta = nullptr;
    CB_NORM_AFFINE_LAUNCH(false);
    count_launches(1);
    return 0;
}

extern "C" int cb_embedding_bwd(const long long* ids, const float* dout, long long ld, float* dtable, int n, int D, int V,
                                float alpha, void* stream) {
    CB_REQUIRE(ids && dout && dtable && n > 0 && D > 0 && V > 0 && ld >= D, CB_ERR_ARG, "embedding_bwd: bad shape");
    CB_CUDA(CB_LAUNCH((embedding_bwd_kernel), n, 256, 0, reinterpret_cast<cudaStream_t>(stream), ids, dout, ld, dtable, n,
                      D, V, alpha));
    count_launches(1);
    return 0;
}
