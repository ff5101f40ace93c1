// LayerNorm forward / backward for fp32 residual-stream rows (ldm/modules/attention.py:199-215 norm1..3, the CLIP text
// layers' layer_norm1/2 and final_layer_norm): 128-bit accesses, register arrays sized for the row, and -- when there are
// few rows (16x16 / 8x8 UNet levels, the 77 CLIP tokens) -- four warps per row so the launch still covers the SMs.
// Rows whose shape this file does not cover fall back to the one-warp-per-row kernels in cb_norm.cu.
#include "cb_common.cuh"

namespace cb {

template <typename T> struct Q4;
template <> struct Q4<float> {
    static __device__ __forceinline__ void ld(const float* p, float (&f)[4]) {
        const float4 v = *reinterpret_cast<const float4*>(p);
        f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
    }
    static __device__ __forceinline__ void st(float* p, const float (&f)[4]) {
        *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
    }
};
template <> struct Q4<__half> {
    static __device__ __forceinline__ void ld(const __half* p, float (&f)[4]) {
        const uint2 u = *reinterpret_cast<const uint2*>(p);
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
        const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
        f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y;
    }
    static __device__ __forceinline__ void st(__half* p, const float (&f)[4]) {
        uint2 u;
        *reinterpret_cast<__half2*>(&u.x) = __floats2half2_rn(f[0], f[1]);
        *reinterpret_cast<__half2*>(&u.y) = __floats2half2_rn(f[2], f[3]);
        *reinterpret_cast<uint2*>(p) = u;
    }
};
template <> struct Q4<__nv_bfloat16> {
    static __device__ __forceinline__ void ld(const __nv_bfloat16* p, float (&f)[4]) {
        const uint2 u = *reinterpret_cast<const uint2*>(p);
        const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
        const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
        f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y;
    }
    static __device__ __forceinline__ void st(__nv_bfloat16* p, const float (&f)[4]) {
        uint2 u;
        *reinterpret_cast<__nv_bfloat162*>(&u.x) = __floats2bfloat162_rn(f[0], f[1]);
        *reinterpret_cast<__nv_bfloat162*>(&u.y) = __floats2bfloat162_rn(f[2], f[3]);
        *reinterpret_cast<uint2*>(p) = u;
    }
};

// two sums over the WPR warps that share one row (WPR = 1: plain warp reduction)
template <int WPR>
__device__ __forceinline__ void row_sum2(float& a, float& b, float (*s_red)[2], int wir) {
    a = warp_sum(a);
    b = warp_sum(b);
    if (WPR > 1) {
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        if (lane == 0) { s_red[warp][0] = a; s_red[warp][1] = b; }
        __syncthreads();
        const int w0 = warp - wir;
        a = 0.f; b = 0.f;
#pragma unroll
        for (int i = 0; i < WPR; ++i) { a += s_red[w0 + i][0]; b += s_red[w0 + i][1]; }
        __syncthreads();
    }
}

// block = 128 threads = 4 warps; WPR warps per row; lane l of warp-in-row w owns quads (w*32 + l) + i*32*WPR, i < MAXQ
template <typename TY, int WPR, int MAXQ>
__global__ void __launch_bounds__(128)
ln_fwd_q_kernel(const float* __restrict__ x, TY* __restrict__ y, const float* __restrict__ gamma,
                const float* __restrict__ beta, float* __restrict__ mean_out, float* __restrict__ rstd_out, int M, int C,
                float eps) {
    __shared__ float s_red[4][2];
    pdl_sync();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wir = warp % WPR;
    int row = blockIdx.x * (4 / WPR) + warp / WPR;
    const bool live = row < M;
    if (!live) row = M - 1;               // keep every warp in the block barriers; results are discarded
    const int nq = C >> 2;
    const float* xr = x + (size_t)row * C;
    float v[MAXQ][4];
    float s = 0.f, dummy = 0.f;
#pragma unroll
    for (int i = 0; i < MAXQ; ++i) {
        const int q = wir * 32 + lane + i * 32 * WPR;
        if (q < nq) {
            Q4<float>::ld(xr + 4 * q, v[i]);
            s += (v[i][0] + v[i][1]) + (v[i][2] + v[i][3]);
        }
    }
    row_sum2<WPR>(s, dummy, s_red, wir);
    const float mean = s / C;
    float qs = 0.f;
#pragma unroll
    for (int i = 0; i < MAXQ; ++i) {
        const int q = wir * 32 + lane + i * 32 * WPR;
        if (q < nq) {
#pragma unroll
            for (int k = 0; k < 4; ++k) { const float a = v[i][k] - mean; qs += a * a; }
        }
    }
    dummy = 0.f;
    row_sum2<WPR>(qs, dummy, s_red, wir);
    const float rstd = rsqrtf(qs / C + eps);
    if (!live) return;
    if (lane == 0 && wir == 0) {
        mean_out[row] = mean;
        rstd_out[row] = rstd;
    }
    TY* yr = y + (size_t)row * C;
#pragma unroll
    for (int i = 0; i < MAXQ; ++i) {
        const int q = wir * 32 + lane + i * 32 * WPR;
        if (q < nq) {
            float g[4], b[4], o[4];
            Q4<float>::ld(gamma + 4 * q, g);
            Q4<float>::ld(beta + 4 * q, b);
#pragma unroll
            for (int k = 0; k < 4; ++k) o[k] = (v[i][k] - mean) * rstd * g[k] + b[k];
            Q4<TY>::st(yr + 4 * q, o);
        }
    }
}

template <typename TG, typename TD, int WPR, int MAXQ>
__global__ void __launch_bounds__(128)
ln_bwd_q_kernel(const TG* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ gamma,
                const float* __restrict__ mean, const float* __restrict__ rstd, TD* __restrict__ dx,
                TG* __restrict__ dx_lp, int M, int C, int accumulate) {
    __shared__ float s_red[4][2];
    pdl_sync();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wir = warp % WPR;
    int row = blockIdx.x * (4 / WPR) + warp / WPR;
    const bool live = row < M;
    if (!live) row = M - 1;
    const int nq = C >> 2;
    const float m = mean[row], rs = rstd[row];
    const float* xr = x + (size_t)row * C;
    const TG* dr = dy + (size_t)row * C;
    float xh[MAXQ][4], t[MAXQ][4];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < MAXQ; ++i) {
        const int q = wir * 32 + lane + i * 32 * WPR;
        if (q < nq) {
            float xv[4], d[4], g[4];
            Q4<float>::ld(xr + 4 * q, xv);
            Q4<TG>::ld(dr + 4 * q, d);
            Q4<float>::ld(gamma + 4 * q, g);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                xh[i][k] = (xv[k] - m) * rs;
                t[i][k] = d[k] * g[k];
                s1 += t[i][k];
                s2 += t[i][k] * xh[i][k];
            }
        }
    }
    row_sum2<WPR>(s1, s2, s_red, wir);
    if (!live) return;
    s1 /= C;
    s2 /= C;
    TD* orow = dx + (size_t)row * C;
#pragma unroll
    for (int i = 0; i < MAXQ; ++i) {
        const int q = wir * 32 + lane + i * 32 * WPR;
        if (q < nq) {
            float o[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) o[k] = rs * (t[i][k] - s1 - xh[i][k] * s2);
            if (accumulate) {
                float p[4];
                Q4<TD>::ld(orow + 4 * q, p);
#pragma unroll
                for (int k = 0; k < 4; ++k) o[k] += p[k];
            }
            Q4<TD>::st(orow + 4 * q, o);
            if (dx_lp) Q4<TG>::st(dx_lp + (size_t)row * C + 4 * q, o);   // 16-bit copy for the GEMM that consumes dx next
        }
    }
}

// (WPR, MAXQ) for a shape, or false when the legacy kernel has to take it
static bool ln_plan(int M, int C, int& wpr, int& maxq) {
    if (C % 4 != 0) return false;
    wpr = (M <= 1024 && C >= 512) || M <= 256 ? 4 : 1;
    const int q = ceil_div(C / 4, 32 * wpr);
    if (q <= 3) maxq = 3;
    else if (q <= 10) maxq = 10;
    else if (wpr == 1 && ceil_div(C / 4, 128) <= 10) { wpr = 4; maxq = ceil_div(C / 4, 128) <= 3 ? 3 : 10; }
    else return false;
    return true;
}

}  // namespace cb

using namespace cb;

#define CB_LN_DISPATCH16(dtype, T, ...)                                          \
    if ((dtype) == CB_F32) { using T = float; __VA_ARGS__; }                     \
    else if ((dtype) == CB_F16) { using T = __half; __VA_ARGS__; }               \
    else { using T = __nv_bfloat16; __VA_ARGS__; }

#define CB_LN_PLAN(WPR_, MAXQ_, ...)                                             \
    if (wpr == 1 && maxq == 3) { constexpr int WPR_ = 1, MAXQ_ = 3; __VA_ARGS__; }        \
    else if (wpr == 1) { constexpr int WPR_ = 1, MAXQ_ = 10; __VA_ARGS__; }               \
    else if (maxq == 3) { constexpr int WPR_ = 4, MAXQ_ = 3; __VA_ARGS__; }               \
    else { constexpr int WPR_ = 4, MAXQ_ = 10; __VA_ARGS__; }

extern "C" int cb_layernorm_fwd(const void* x, int x_dtype, void* y, int y_dtype, const float* gamma, const float* beta,
                                int M, int C, float eps, float* mean_out, float* rstd_out, void* stream) {
    int wpr = 1, maxq = 3;
    const bool aligned = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) |
                           reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta)) & 15u) == 0;
    if (x_dtype != CB_F32 || !aligned || M <= 0 || !ln_plan(M, C, wpr, maxq))
        return layernorm_fwd_legacy(x, x_dtype, y, y_dtype, gamma, beta, M, C, eps, mean_out, rstd_out, stream);
    CB_REQUIRE(y_dtype >= CB_F16 && y_dtype <= CB_F32, CB_ERR_ARG, "layernorm: bad y dtype");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    dim3 grid(ceil_div(M, 4 / wpr));
    CB_LN_DISPATCH16(y_dtype, TY, CB_LN_PLAN(W, Q,
        CB_LAUNCH((ln_fwd_q_kernel<TY, W, Q>), grid, 128, 0, st, (const float*)x, (TY*)y, gamma, beta, mean_out, rstd_out, M, C, eps)));
    CB_CUDA(cudaGetLastError());
    count_launches(1);
    return 0;
}

extern "C" int cb_layernorm_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, const float* gamma,
                                const float* mean, const float* rstd, void* dx, int dx_dtype, void* dx_lp, int M, int C,
                                int accumulate, void* stream) {
    int wpr = 1, maxq = 3;
    const bool aligned = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dx) |
                           reinterpret_cast<uintptr_t>(dx_lp) | reinterpret_cast<uintptr_t>(gamma)) & 15u) == 0;
    if (x_dtype != CB_F32 || !aligned || M <= 0 || !ln_plan(M, C, wpr, maxq))
        return layernorm_bwd_legacy(dy, dy_dtype, x, x_dtype, gamma, mean, rstd, dx, dx_dtype, dx_lp, M, C, accumulate, stream);
    // CB_LN_DISPATCH16 takes any other value for bf16: refuse it here, as the fallback route does
    CB_REQUIRE(dy_dtype >= CB_F16 && dy_dtype <= CB_F32, CB_ERR_ARG, "layernorm_bwd: bad dy dtype");
    CB_REQUIRE(dx_dtype == CB_F32 || dx_dtype == dy_dtype, CB_ERR_ARG, "layernorm_bwd: dx dtype must be f32 or equal dy dtype");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    dim3 grid(ceil_div(M, 4 / wpr));
    if (dx_dtype == CB_F32) {
        CB_LN_DISPATCH16(dy_dtype, TG, CB_LN_PLAN(W, Q,
            CB_LAUNCH((ln_bwd_q_kernel<TG, float, W, Q>), grid, 128, 0, st, (const TG*)dy, (const float*)x, gamma, mean, rstd, (float*)dx, (TG*)dx_lp, M, C, accumulate)));
    } else {
        CB_LN_DISPATCH16(dy_dtype, TG, CB_LN_PLAN(W, Q,
            CB_LAUNCH((ln_bwd_q_kernel<TG, TG, W, Q>), grid, 128, 0, st, (const TG*)dy, (const float*)x, gamma, mean, rstd, (TG*)dx, (TG*)dx_lp, M, C, accumulate)));
    }
    CB_CUDA(cudaGetLastError());
    count_launches(1);
    return 0;
}
