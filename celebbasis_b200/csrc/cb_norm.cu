// GroupNorm(+SiLU) and LayerNorm, forward and activation-gradient backward, channels-last.
//
// Replaces ldm/modules/diffusionmodules/util.py:199-216 (GroupNorm32 / normalization),
// ldm/modules/attention.py:76-77 + ldm/modules/diffusionmodules/model.py:38-39 (Normalize, eps 1e-6),
// the nn.SiLU that follows them in ResBlock (openaimodel.py:201-241) and nn.LayerNorm in
// BasicTransformerBlock (attention.py:196-215) / CLIP layers.  HBM-bound: every kernel reads its
// input once (2-wide / 4-wide vector loads, channel index fastest => fully coalesced rows) and the
// statistics pass keeps per-thread partials in registers, adds them per group in a fixed order in
// shared memory, and combines the CTAs' (sum, sumsq) partials in a fixed order: through distributed
// shared memory inside a thread-block cluster, or as one partial per (CTA, group) in the workspace
// that the apply kernel adds up in CTA order.
//
// GroupNorm dispatch: forward = cluster kernel where the rows fit in shared memory, else the TMA-streamed
// statistics + apply pair; backward = cluster kernel, else the statistics + apply pair.
#include "cb_common.cuh"

namespace cb {

template <typename T> struct Vec2;
template <> struct Vec2<float> {
    static __device__ __forceinline__ float2 ld(const float* p) { return *reinterpret_cast<const float2*>(p); }
    static __device__ __forceinline__ void st(float* p, float2 v) { *reinterpret_cast<float2*>(p) = v; }
};
template <> struct Vec2<__half> {
    static __device__ __forceinline__ float2 ld(const __half* p) {
        return __half22float2(*reinterpret_cast<const __half2*>(p));
    }
    static __device__ __forceinline__ void st(__half* p, float2 v) {
        *reinterpret_cast<__half2*>(p) = __floats2half2_rn(v.x, v.y);
    }
};
template <> struct Vec2<__nv_bfloat16> {
    static __device__ __forceinline__ float2 ld(const __nv_bfloat16* p) {
        return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p));
    }
    static __device__ __forceinline__ void st(__nv_bfloat16* p, float2 v) {
        *reinterpret_cast<__nv_bfloat162*>(p) = __floats2bfloat162_rn(v.x, v.y);
    }
};

__device__ __forceinline__ float silu_grad(float z) {
    const float s = __fdividef(1.0f, 1.0f + __expf(-z));
    return s * (1.0f + z * (1.0f - s));
}

// Per-group accumulation into shared memory in a fixed order, so that the statistics are bit-identical from run to run:
// lanes of a warp that hold the same group add up with shuffles (a tree over a contiguous run, else in lane order), the
// run's first lane adds the result into its warp's slot, and group_acc_flush() adds the slots into s_a / s_b in warp
// order.  group_accumulate must be called by all live lanes of the warp (uniform control flow); group_acc_begin() and
// group_acc_flush() by every thread of the block.
constexpr int kGnSlotWarps = 32;          // up to 1024 threads
struct GnSlots { float2 v[kGnSlotWarps][64]; };
__device__ __forceinline__ GnSlots& gn_slots() {
    __shared__ GnSlots s;
    return s;
}
__device__ __forceinline__ void group_acc_begin() {
    float2* v = &gn_slots().v[0][0];
    for (int i = threadIdx.x; i < kGnSlotWarps * 64; i += blockDim.x) v[i] = make_float2(0.f, 0.f);
    __syncthreads();
}
__device__ __forceinline__ void group_accumulate(float* s_a, float* s_b, int g, float v1, float v2) {
    (void)s_a; (void)s_b;
    const unsigned act = __activemask();
    const unsigned peers = __match_any_sync(act, g);
    const int lane = threadIdx.x & 31;
    const int first = __ffs(peers) - 1, last = 31 - __clz(peers);
    const unsigned run = peers >> first;
    const bool contiguous = (run & (run + 1)) == 0;
    if (__all_sync(act, contiguous)) {
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const float t1 = __shfl_down_sync(act, v1, off);
            const float t2 = __shfl_down_sync(act, v2, off);
            if (lane + off <= last) { v1 += t1; v2 += t2; }
        }
    } else {
        float t1 = 0.f, t2 = 0.f;
        for (int l = 0; l < 32; ++l) {
            if (!((act >> l) & 1u)) continue;
            const float u1 = __shfl_sync(act, v1, l), u2 = __shfl_sync(act, v2, l);
            if ((peers >> l) & 1u) { t1 += u1; t2 += u2; }
        }
        v1 = t1; v2 = t2;
    }
    if (lane == first) {
        float2& sl = gn_slots().v[threadIdx.x >> 5][g];
        sl = make_float2(sl.x + v1, sl.y + v2);
    }
    __syncwarp(act);
}
// after a __syncthreads(): s_a[g] += sum over warps (in warp order) of the slots, for g < n
__device__ __forceinline__ void group_acc_flush(float* s_a, float* s_b, int n) {
    if ((int)threadIdx.x < n) {
        float a = 0.f, b = 0.f;
        const int nw = (blockDim.x + 31) >> 5;
        for (int w = 0; w < nw; ++w) { const float2 v = gn_slots().v[w][threadIdx.x]; a += v.x; b += v.y; }
        s_a[threadIdx.x] += a;
        s_b[threadIdx.x] += b;
    }
    __syncthreads();
}
// statistics + apply kernel pairs: the statistics kernel publishes one (sum, sum2) partial per CTA and group, the apply kernel
// (same grid) adds them up in CTA order
__device__ __forceinline__ void publish_block_partials(double* ws, const float* s_a, const float* s_b, int G) {
    if ((int)threadIdx.x < G)
        reinterpret_cast<float2*>(ws)[((size_t)blockIdx.y * gridDim.x + blockIdx.x) * G + threadIdx.x] =
            make_float2(s_a[threadIdx.x], s_b[threadIdx.x]);
}
__device__ __forceinline__ double2 sum_block_partials(const double* ws, int G, int g) {
    const float2* part = reinterpret_cast<const float2*>(ws);
    double a = 0.0, b = 0.0;
    for (int k = 0; k < (int)gridDim.x; ++k) {
        const float2 v = part[((size_t)blockIdx.y * gridDim.x + k) * G + g];
        a += v.x;
        b += v.y;
    }
    return make_double2(a, b);
}

constexpr int kGnMaxDynSmem = 184 * 1024;  // dynamic shared memory of the staged variants (+ GnSlots + statics <= 227 KiB)
constexpr int kGnThreads = 256;           // upper bound; the launch uses PW*RY threads (see gn_shape)
constexpr int kGnMaxChunks = 8;           // channel-pair chunks per thread: C <= 2*PW*8

// Thread mapping shared by the statistics + apply GroupNorm kernels: a block is a (RY x PW) grid of threads; tx owns channel
// pairs {tx + j*PW}, ty strides over the rows of the block's row range.  PW is the largest divisor of C/2 that is
// <= 256, so every thread is busy for C = 128 (PW 64, RY 4) as well as C = 320 (PW 160, RY 1) or C = 2560 (PW 256).
struct GnShape { int pw, ry, chunks; };
static inline GnShape gn_shape(int C) {
    const int npairs = C >> 1;
    int pw = npairs < 256 ? npairs : 256;
    while (npairs % pw) --pw;
    GnShape s;
    s.pw = pw;
    s.ry = 256 / pw > 0 ? 256 / pw : 1;
    s.chunks = npairs / pw;
    return s;
}

// ---- GroupNorm forward for tensors whose rows do not fit the cluster kernel's shared memory (VAE 512^2 / 256^2 maps, large
// batches): a statistics pass and an apply pass, with the rows streaming through a 3-stage ring of 32 KiB
// cp.async.bulk (TMA 1-D) chunks, so every CTA keeps ~64-96 KiB in flight instead of a few 8-byte loads per thread.
constexpr int kGnTmaStages = 3;
constexpr int kGnTmaChunkBytes = 32768;

template <typename TX, typename F>
__device__ __forceinline__ void gn_tma_row_stream(const TX* __restrict__ xrows, int nrows, int C, int rows_per_chunk,
                                                  unsigned char* smem, unsigned long long* bars, F&& consume) {
    const int nchunks = (nrows + rows_per_chunk - 1) / rows_per_chunk;
    auto issue = [&](int ci) {
        const int rows = min(rows_per_chunk, nrows - ci * rows_per_chunk);
        const uint32_t bytes = (uint32_t)((size_t)rows * C * sizeof(TX));
        const int stg = ci % kGnTmaStages;
        const uint32_t bar = smem_u32(&bars[stg]);
        mbar_arrive_expect_tx(bar, bytes);
        tma_bulk_g2s(smem_u32(smem + (size_t)stg * kGnTmaChunkBytes), xrows + (size_t)ci * rows_per_chunk * C, bytes, bar);
    };
    if (threadIdx.x == 0)
        for (int ci = 0; ci < min(kGnTmaStages, nchunks); ++ci) issue(ci);
    for (int ci = 0; ci < nchunks; ++ci) {
        const int stg = ci % kGnTmaStages;
        mbar_wait(smem_u32(&bars[stg]), (ci / kGnTmaStages) & 1);
        const int rows = min(rows_per_chunk, nrows - ci * rows_per_chunk);
        consume(reinterpret_cast<const TX*>(smem + (size_t)stg * kGnTmaChunkBytes), ci * rows_per_chunk, rows);
        __syncthreads();                                   // every thread is done with this stage
        if (threadIdx.x == 0 && ci + kGnTmaStages < nchunks) issue(ci + kGnTmaStages);
    }
}

template <typename TX>
__global__ void __launch_bounds__(kGnThreads)
gn_stats_tma_kernel(const TX* __restrict__ x, double* __restrict__ ws, int HW, int C, int G, int rows_per_block,
                    int rows_per_chunk, int PW, int RY, int chunks) {
    extern __shared__ __align__(128) unsigned char gn_smem[];
    __shared__ float s_sum[64], s_sq[64];
    __shared__ __align__(8) unsigned long long s_bars[kGnTmaStages];
    const int n = blockIdx.y;
    const int tx = threadIdx.x % PW, ty = threadIdx.x / PW;
    const int r0 = blockIdx.x * rows_per_block;
    const int r1 = min(HW, r0 + rows_per_block);
    const int cpg = C / G;
    if (threadIdx.x == 0) {
        for (int i = 0; i < kGnTmaStages; ++i) mbar_init(smem_u32(&s_bars[i]), 1);
        mbar_fence_init();
        fence_proxy_async_smem();
    }
    if (threadIdx.x < 64) { s_sum[threadIdx.x] = 0.f; s_sq[threadIdx.x] = 0.f; }
    group_acc_begin();
    __syncthreads();
    pdl_sync();
    float a1[kGnMaxChunks], a2[kGnMaxChunks];
#pragma unroll
    for (int j = 0; j < kGnMaxChunks; ++j) { a1[j] = 0.f; a2[j] = 0.f; }
    if (r1 > r0) {
        gn_tma_row_stream<TX>(x + ((size_t)n * HW + r0) * C, r1 - r0, C, rows_per_chunk, gn_smem, s_bars,
                              [&](const TX* sx, int, int rows) {
#pragma unroll 4
            for (int r = ty; r < rows; r += RY) {
                const TX* sr = sx + (size_t)r * C + 2 * tx;
#pragma unroll
                for (int j = 0; j < kGnMaxChunks; ++j) {
                    if (j < chunks) {
                        const float2 v = Vec2<TX>::ld(sr + 2 * j * PW);
                        a1[j] += v.x + v.y;
                        a2[j] += v.x * v.x + v.y * v.y;
                    }
                }
            }
        });
    }
#pragma unroll
    for (int j = 0; j < kGnMaxChunks; ++j) {
        if (j < chunks) {
            const int g = (2 * (tx + j * PW)) / cpg;
            group_accumulate(s_sum, s_sq, g, a1[j], a2[j]);
        }
    }
    __syncthreads();
    group_acc_flush(s_sum, s_sq, 64);
    publish_block_partials(ws, s_sum, s_sq, G);
}

template <typename TX, typename TY>
__global__ void __launch_bounds__(kGnThreads)
gn_apply_tma_kernel(const TX* __restrict__ x, TY* __restrict__ y, const float* __restrict__ gamma,
                    const float* __restrict__ beta, const double* __restrict__ ws, float* __restrict__ mean_out,
                    float* __restrict__ rstd_out, int HW, int C, int G, float eps, int act, int rows_per_block,
                    int rows_per_chunk, int PW, int RY, int chunks) {
    extern __shared__ __align__(128) unsigned char gn_smem[];
    __shared__ float s_mean[64], s_rstd[64];
    __shared__ __align__(8) unsigned long long s_bars[kGnTmaStages];
    const int n = blockIdx.y;
    const int tx = threadIdx.x % PW, ty = threadIdx.x / PW;
    const int cpg = C / G;
    if (threadIdx.x == 0) {
        for (int i = 0; i < kGnTmaStages; ++i) mbar_init(smem_u32(&s_bars[i]), 1);
        mbar_fence_init();
        fence_proxy_async_smem();
    }
    __syncthreads();
    pdl_sync();
    if (threadIdx.x < G) {
        const double cnt = (double)HW * cpg;
        const double2 sums = sum_block_partials(ws, G, threadIdx.x);
        const double m = sums.x / cnt;
        double var = sums.y / cnt - m * m;
        if (var < 0) var = 0;
        const float rs = (float)(1.0 / sqrt(var + (double)eps));
        s_mean[threadIdx.x] = (float)m;
        s_rstd[threadIdx.x] = rs;
        if (blockIdx.x == 0) {
            mean_out[n * G + threadIdx.x] = (float)m;
            rstd_out[n * G + threadIdx.x] = rs;
        }
    }
    __syncthreads();
    const int r0 = blockIdx.x * rows_per_block;
    const int r1 = min(HW, r0 + rows_per_block);
    if (r1 <= r0) return;
    // per-thread affine of its channel pairs: y = x * ga + be
    float ga0[kGnMaxChunks], ga1[kGnMaxChunks], be0[kGnMaxChunks], be1[kGnMaxChunks];
#pragma unroll
    for (int j = 0; j < kGnMaxChunks; ++j) {
        if (j < chunks) {
            const int c = 2 * (tx + j * PW);
            const int g = c / cpg;
            const float m = s_mean[g], rs = s_rstd[g];
            ga0[j] = gamma[c] * rs; ga1[j] = gamma[c + 1] * rs;
            be0[j] = beta[c] - m * ga0[j]; be1[j] = beta[c + 1] - m * ga1[j];
        }
    }
    TY* yb = y + ((size_t)n * HW + r0) * C + 2 * tx;
    gn_tma_row_stream<TX>(x + ((size_t)n * HW + r0) * C, r1 - r0, C, rows_per_chunk, gn_smem, s_bars,
                          [&](const TX* sx, int row_base, int rows) {
#pragma unroll 4
        for (int r = ty; r < rows; r += RY) {
            const TX* sr = sx + (size_t)r * C + 2 * tx;
            TY* yr = yb + (size_t)(row_base + r) * C;
#pragma unroll
            for (int j = 0; j < kGnMaxChunks; ++j) {
                if (j < chunks) {
                    float2 v = Vec2<TX>::ld(sr + 2 * j * PW);
                    v.x = v.x * ga0[j] + be0[j];
                    v.y = v.y * ga1[j] + be1[j];
                    if (act) { v.x = silu_f(v.x); v.y = silu_f(v.y); }
                    Vec2<TY>::st(yr + 2 * j * PW, v);
                }
            }
        }
    });
}

// ---- GroupNorm backward statistics: ws += {sum dz*gamma, sum dz*gamma*xhat} ---------------------------
template <typename TX, typename TG>
__global__ void __launch_bounds__(kGnThreads)
gn_bwd_stats_kernel(const TG* __restrict__ dy, const TX* __restrict__ x, const float* __restrict__ gamma,
                    const float* __restrict__ beta, const float* __restrict__ mean, const float* __restrict__ rstd,
                    double* __restrict__ ws, int HW, int C, int G, int act, int rows_per_block, int PW, int RY,
                    int chunks) {
    pdl_sync();
    __shared__ float s_1[64], s_2[64];
    const int n = blockIdx.y;
    const int tx = threadIdx.x % PW, ty = threadIdx.x / PW;
    const int cpg = C / G;
    if (threadIdx.x < 64) { s_1[threadIdx.x] = 0.f; s_2[threadIdx.x] = 0.f; }
    group_acc_begin();
    __syncthreads();
    const int r0 = blockIdx.x * rows_per_block;
    const int r1 = min(HW, r0 + rows_per_block);
    const size_t base = ((size_t)n * HW) * C;
    for (int j = 0; j < chunks; ++j) {
        const int c = 2 * (tx + j * PW);
        const int g = c / cpg;
        const float m = mean[n * G + g], rs = rstd[n * G + g];
        const float ga0 = gamma[c], ga1 = gamma[c + 1], be0 = beta[c], be1 = beta[c + 1];
        float a1 = 0.f, a2 = 0.f;
#pragma unroll 4
        for (int r = r0 + ty; r < r1; r += RY) {
            const size_t off = base + (size_t)r * C + c;
            const float2 xv = Vec2<TX>::ld(x + off);
            float2 d = Vec2<TG>::ld(dy + off);
            const float xh0 = (xv.x - m) * rs, xh1 = (xv.y - m) * rs;
            if (act) {
                d.x *= silu_grad(xh0 * ga0 + be0);
                d.y *= silu_grad(xh1 * ga1 + be1);
            }
            const float t0 = d.x * ga0, t1 = d.y * ga1;
            a1 += t0 + t1;
            a2 += t0 * xh0 + t1 * xh1;
        }
        group_accumulate(s_1, s_2, g, a1, a2);
    }
    __syncthreads();
    group_acc_flush(s_1, s_2, 64);
    publish_block_partials(ws, s_1, s_2, G);
}

// ---- GroupNorm backward apply: dx (+)= rstd*(dz*gamma - s1/cnt - xhat*s2/cnt) ----------------------------
template <typename TX, typename TG, typename TD>
__global__ void __launch_bounds__(kGnThreads)
gn_bwd_apply_kernel(const TG* __restrict__ dy, const TX* __restrict__ x, const float* __restrict__ gamma,
                    const float* __restrict__ beta, const float* __restrict__ mean, const float* __restrict__ rstd,
                    const double* __restrict__ ws, TD* __restrict__ dx, TG* __restrict__ dx_lp, int HW, int C, int G, int act,
                    int accumulate, int rows_per_block, int PW, int RY, int chunks) {
    pdl_sync();
    __shared__ float s_1[64], s_2[64];
    const int n = blockIdx.y;
    const int tx = threadIdx.x % PW, ty = threadIdx.x / PW;
    const int cpg = C / G;
    if (threadIdx.x < G) {
        const double cnt = (double)HW * cpg;
        const double2 sums = sum_block_partials(ws, G, threadIdx.x);
        s_1[threadIdx.x] = (float)(sums.x / cnt);
        s_2[threadIdx.x] = (float)(sums.y / cnt);
    }
    __syncthreads();
    const int r0 = blockIdx.x * rows_per_block;
    const int r1 = min(HW, r0 + rows_per_block);
    const size_t base = ((size_t)n * HW) * C;
    for (int j = 0; j < chunks; ++j) {
        const int c = 2 * (tx + j * PW);
        const int g = c / cpg;
        const float m = mean[n * G + g], rs = rstd[n * G + g];
        const float ga0 = gamma[c], ga1 = gamma[c + 1], be0 = beta[c], be1 = beta[c + 1];
        const float m1 = s_1[g], m2 = s_2[g];
#pragma unroll 4
        for (int r = r0 + ty; r < r1; r += RY) {
            const size_t off = base + (size_t)r * C + c;
            const float2 xv = Vec2<TX>::ld(x + off);
            float2 d = Vec2<TG>::ld(dy + off);
            const float xh0 = (xv.x - m) * rs, xh1 = (xv.y - m) * rs;
            if (act) {
                d.x *= silu_grad(xh0 * ga0 + be0);
                d.y *= silu_grad(xh1 * ga1 + be1);
            }
            float2 o;
            o.x = rs * (d.x * ga0 - m1 - xh0 * m2);
            o.y = rs * (d.y * ga1 - m1 - xh1 * m2);
            if (accumulate) {
                const float2 p = Vec2<TD>::ld(dx + off);
                o.x += p.x;
                o.y += p.y;
            }
            Vec2<TD>::st(dx + off, o);
            if (dx_lp) Vec2<TG>::st(dx_lp + off, o);      // 16-bit copy for the dgrad GEMM that consumes dx next
        }
    }
}

// ---- GroupNorm on thread-block clusters: one launch, x read once ------------------------------------------------------
// A cluster owns a SLAB of `gpc` consecutive groups (cw = gpc * C/G channels) of one image for ALL rows; its S CTAs split
// the rows.  Every CTA stages its rows x cw sub-matrix in shared memory (read once), the per-group partial sums of the S
// CTAs meet through distributed shared memory (each CTA stores its gpc (sum, sumsq) pairs into every peer: S*gpc 8-byte
// remote stores, one cluster barrier), and the normalised rows are written straight from shared memory.  CTAs wait only on
// the peers of their own cluster, which the hardware co-schedules, so the grid needs no global barrier and need not be
// resident at once (util.py:199-216 GroupNorm32, openaimodel.py:201-241).
constexpr int kGnClThreads = 512;
constexpr int kGnClMaxS = 16;

// 4 consecutive channels (16 bytes of fp32, 8 bytes of a 16-bit type) per access
template <typename T> struct Vec4;
template <> struct Vec4<float> {
    static __device__ __forceinline__ float4 ld(const float* p) { return *reinterpret_cast<const float4*>(p); }
    static __device__ __forceinline__ void st(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
};
template <> struct Vec4<__half> {
    static __device__ __forceinline__ float4 ld(const __half* p) {
        const uint2 u = *reinterpret_cast<const uint2*>(p);
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
        const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
        return make_float4(a.x, a.y, b.x, b.y);
    }
    static __device__ __forceinline__ void st(__half* p, float4 v) {
        uint2 u;
        *reinterpret_cast<__half2*>(&u.x) = __floats2half2_rn(v.x, v.y);
        *reinterpret_cast<__half2*>(&u.y) = __floats2half2_rn(v.z, v.w);
        *reinterpret_cast<uint2*>(p) = u;
    }
};
template <> struct Vec4<__nv_bfloat16> {
    static __device__ __forceinline__ float4 ld(const __nv_bfloat16* p) {
        const uint2 u = *reinterpret_cast<const uint2*>(p);
        const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
        const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
        return make_float4(a.x, a.y, b.x, b.y);
    }
    static __device__ __forceinline__ void st(__nv_bfloat16* p, float4 v) {
        uint2 u;
        *reinterpret_cast<__nv_bfloat162*>(&u.x) = __floats2bfloat162_rn(v.x, v.y);
        *reinterpret_cast<__nv_bfloat162*>(&u.y) = __floats2bfloat162_rn(v.z, v.w);
        *reinterpret_cast<uint2*>(p) = u;
    }
};

// thread -> (channel quad `cq` of the slab, first row `ry`); rows advance by RY.  nq = quads per slab row.  The two channel
// pairs of a quad may belong to different groups (C/G is even, not necessarily a multiple of 4): gA / gB.
struct GnClMap { int cq, ry, RY, gA, gB; bool on; };
__device__ __forceinline__ GnClMap gn_cl_map(int nq, int cpg) {
    GnClMap m;
    m.RY = kGnClThreads / nq;
    m.cq = threadIdx.x % nq;
    m.ry = threadIdx.x / nq;
    m.on = m.ry < m.RY;
    m.gA = (4 * m.cq) / cpg;
    m.gB = (4 * m.cq + 2) / cpg;
    return m;
}

// exchange of per-group partial pairs inside the cluster; returns the cluster totals in s_t1/s_t2 (double, [gpc])
__device__ __forceinline__ void gn_cl_allreduce(float* s_a, float* s_b, float2 (*s_recv)[32], double* s_t1, double* s_t2,
                                                int gpc, int S, int rank) {
    __syncthreads();                               // s_a / s_b complete
    cluster_wait();                                // (arrive was issued at kernel entry) every CTA of the cluster runs
    for (int t = threadIdx.x; t < S * gpc; t += kGnClThreads) {
        const int peer = t / gpc, g = t - peer * gpc;
        st_cluster_f32x2(smem_u32(&s_recv[rank][g]), (uint32_t)peer, s_a[g], s_b[g]);
    }
    cluster_sync_all();                            // release our stores / acquire everyone else's
    if (threadIdx.x < gpc) {
        double t1 = 0.0, t2 = 0.0;
        for (int r = 0; r < S; ++r) { t1 += (double)s_recv[r][threadIdx.x].x; t2 += (double)s_recv[r][threadIdx.x].y; }
        s_t1[threadIdx.x] = t1;
        s_t2[threadIdx.x] = t2;
    }
    __syncthreads();
}

template <typename TX, typename TY>
__global__ void __launch_bounds__(kGnClThreads)
gn_cluster_fwd_kernel(const TX* __restrict__ x, TY* __restrict__ y, const float* __restrict__ gamma,
                      const float* __restrict__ beta, float* __restrict__ mean_out, float* __restrict__ rstd_out, int HW,
                      int C, int G, float eps, int act, int gpc, int rows_per_cta) {
    extern __shared__ __align__(128) unsigned char gn_smem[];
    TX* sx = reinterpret_cast<TX*>(gn_smem);
    __shared__ float s_a[32], s_b[32];
    __shared__ __align__(8) float2 s_recv[kGnClMaxS][32];
    __shared__ double s_t1[32], s_t2[32];
    cluster_arrive_relaxed();
    const int S = gridDim.x, rank = blockIdx.x, slab = blockIdx.y, n = blockIdx.z;
    const int cpg = C / G, cw = gpc * cpg, nq = cw >> 2, c0 = slab * cw;
    const int r0 = rank * rows_per_cta, r1 = min(HW, r0 + rows_per_cta);
    if (threadIdx.x < 32) { s_a[threadIdx.x] = 0.f; s_b[threadIdx.x] = 0.f; }
    group_acc_begin();
    __syncthreads();
    pdl_sync();
    const GnClMap m = gn_cl_map(nq, cpg);
    const size_t base = ((size_t)n * HW) * C + c0 + 4 * m.cq;
    if (m.on) {
        float a1 = 0.f, a2 = 0.f, b1 = 0.f, b2 = 0.f;
#pragma unroll 8
        for (int r = r0 + m.ry; r < r1; r += m.RY) {
            const float4 v = Vec4<TX>::ld(x + base + (size_t)r * C);
            Vec4<TX>::st(sx + (size_t)(r - r0) * cw + 4 * m.cq, v);
            a1 += v.x + v.y;
            a2 += v.x * v.x + v.y * v.y;
            b1 += v.z + v.w;
            b2 += v.z * v.z + v.w * v.w;
        }
        if (m.gA == m.gB) { a1 += b1; a2 += b2; b1 = 0.f; b2 = 0.f; }
        group_accumulate(s_a, s_b, m.gA, a1, a2);
        group_accumulate(s_a, s_b, m.gB, b1, b2);
    }
    __syncthreads();
    group_acc_flush(s_a, s_b, 32);
    gn_cl_allreduce(s_a, s_b, s_recv, s_t1, s_t2, gpc, S, rank);
    if (threadIdx.x < gpc) {
        const double cnt = (double)HW * cpg;
        const double mu = s_t1[threadIdx.x] / cnt;
        double var = s_t2[threadIdx.x] / cnt - mu * mu;
        if (var < 0) var = 0;
        const float rs = (float)(1.0 / sqrt(var + (double)eps));
        s_a[threadIdx.x] = (float)mu;
        s_b[threadIdx.x] = rs;
        if (rank == 0) {
            mean_out[n * G + slab * gpc + threadIdx.x] = (float)mu;
            rstd_out[n * G + slab * gpc + threadIdx.x] = rs;
        }
    }
    __syncthreads();
    if (m.on) {
        const int c = c0 + 4 * m.cq;
        const float muA = s_a[m.gA], rsA = s_b[m.gA], muB = s_a[m.gB], rsB = s_b[m.gB];
        const float g0 = gamma[c] * rsA, g1 = gamma[c + 1] * rsA, g2 = gamma[c + 2] * rsB, g3 = gamma[c + 3] * rsB;
        const float b0 = beta[c] - muA * g0, b1 = beta[c + 1] - muA * g1, b2 = beta[c + 2] - muB * g2, b3 = beta[c + 3] - muB * g3;
#pragma unroll 4
        for (int r = r0 + m.ry; r < r1; r += m.RY) {
            float4 v = Vec4<TX>::ld(sx + (size_t)(r - r0) * cw + 4 * m.cq);
            v.x = v.x * g0 + b0;
            v.y = v.y * g1 + b1;
            v.z = v.z * g2 + b2;
            v.w = v.w * g3 + b3;
            if (act) { v.x = silu_f(v.x); v.y = silu_f(v.y); v.z = silu_f(v.z); v.w = silu_f(v.w); }
            Vec4<TY>::st(y + base + (size_t)r * C, v);
        }
    }
}

template <typename TX, typename TG, typename TD>
__global__ void __launch_bounds__(kGnClThreads)
gn_cluster_bwd_kernel(const TG* __restrict__ dy, const TX* __restrict__ x, const float* __restrict__ gamma,
                      const float* __restrict__ beta, const float* __restrict__ mean, const float* __restrict__ rstd,
                      TD* __restrict__ dx, TG* __restrict__ dx_lp, int HW, int C, int G, int act, int accumulate, int gpc,
                      int rows_per_cta) {
    // x and dy of this CTA's rows x slab are staged once; xhat and dz * gamma are recomputed from them in both passes
    extern __shared__ __align__(128) unsigned char gn_smem[];
    const int cpg = C / G, cw = gpc * cpg, nq = cw >> 2;
    TX* sx = reinterpret_cast<TX*>(gn_smem);
    TG* sdy = reinterpret_cast<TG*>(gn_smem + (((size_t)rows_per_cta * cw * sizeof(TX) + 127) & ~(size_t)127));
    __shared__ float s_a[32], s_b[32];
    __shared__ __align__(8) float2 s_recv[kGnClMaxS][32];
    __shared__ double s_t1[32], s_t2[32];
    cluster_arrive_relaxed();
    const int S = gridDim.x, rank = blockIdx.x, slab = blockIdx.y, n = blockIdx.z;
    const int c0 = slab * cw;
    const int r0 = rank * rows_per_cta, r1 = min(HW, r0 + rows_per_cta);
    if (threadIdx.x < 32) { s_a[threadIdx.x] = 0.f; s_b[threadIdx.x] = 0.f; }
    group_acc_begin();
    __syncthreads();
    pdl_sync();
    const GnClMap m = gn_cl_map(nq, cpg);
    const size_t base = ((size_t)n * HW) * C + c0 + 4 * m.cq;
    float mu[2] = {0.f, 0.f}, rs[2] = {0.f, 0.f}, ga[4] = {0.f, 0.f, 0.f, 0.f}, be[4] = {0.f, 0.f, 0.f, 0.f};
    // dz * gamma and xhat of one quad (activation gradient recomputed from xhat)
    auto terms = [&](const float4& xv, const float4& dv, float (&t)[4], float (&xh)[4]) {
        const float xs[4] = {xv.x, xv.y, xv.z, xv.w};
        float d[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            xh[k] = (xs[k] - mu[k >> 1]) * rs[k >> 1];
            if (act) d[k] *= silu_grad(xh[k] * ga[k] + be[k]);
            t[k] = d[k] * ga[k];
        }
    };
    if (m.on) {
        const int c = c0 + 4 * m.cq;
        mu[0] = mean[n * G + slab * gpc + m.gA]; rs[0] = rstd[n * G + slab * gpc + m.gA];
        mu[1] = mean[n * G + slab * gpc + m.gB]; rs[1] = rstd[n * G + slab * gpc + m.gB];
#pragma unroll
        for (int k = 0; k < 4; ++k) { ga[k] = gamma[c + k]; be[k] = beta[c + k]; }
        float a1 = 0.f, a2 = 0.f, b1 = 0.f, b2 = 0.f;
#pragma unroll 4
        for (int r = r0 + m.ry; r < r1; r += m.RY) {
            const float4 xv = Vec4<TX>::ld(x + base + (size_t)r * C);
            const float4 dv = Vec4<TG>::ld(dy + base + (size_t)r * C);
            const size_t so = (size_t)(r - r0) * cw + 4 * m.cq;
            Vec4<TX>::st(sx + so, xv);
            Vec4<TG>::st(sdy + so, dv);
            float t[4], xh[4];
            terms(xv, dv, t, xh);
            a1 += t[0] + t[1];
            a2 += t[0] * xh[0] + t[1] * xh[1];
            b1 += t[2] + t[3];
            b2 += t[2] * xh[2] + t[3] * xh[3];
        }
        if (m.gA == m.gB) { a1 += b1; a2 += b2; b1 = 0.f; b2 = 0.f; }
        group_accumulate(s_a, s_b, m.gA, a1, a2);
        group_accumulate(s_a, s_b, m.gB, b1, b2);
    }
    __syncthreads();
    group_acc_flush(s_a, s_b, 32);
    gn_cl_allreduce(s_a, s_b, s_recv, s_t1, s_t2, gpc, S, rank);
    if (threadIdx.x < gpc) {
        const double cnt = (double)HW * cpg;
        s_a[threadIdx.x] = (float)(s_t1[threadIdx.x] / cnt);
        s_b[threadIdx.x] = (float)(s_t2[threadIdx.x] / cnt);
    }
    __syncthreads();
    if (m.on) {
        const float m1[2] = {s_a[m.gA], s_a[m.gB]}, m2[2] = {s_b[m.gA], s_b[m.gB]};
#pragma unroll 4
        for (int r = r0 + m.ry; r < r1; r += m.RY) {
            const size_t so = (size_t)(r - r0) * cw + 4 * m.cq;
            const float4 xv = Vec4<TX>::ld(sx + so);
            const float4 dv = Vec4<TG>::ld(sdy + so);
            float t[4], xh[4], o[4];
            terms(xv, dv, t, xh);
#pragma unroll
            for (int k = 0; k < 4; ++k) o[k] = rs[k >> 1] * (t[k] - m1[k >> 1] - xh[k] * m2[k >> 1]);
            const size_t off = base + (size_t)r * C;
            if (accumulate) {
                const float4 p = Vec4<TD>::ld(dx + off);
                o[0] += p.x; o[1] += p.y; o[2] += p.z; o[3] += p.w;
            }
            const float4 ov = make_float4(o[0], o[1], o[2], o[3]);
            Vec4<TD>::st(dx + off, ov);
            if (dx_lp) Vec4<TG>::st(dx_lp + off, ov);      // 16-bit copy for the dgrad GEMM that consumes dx next
        }
    }
}

// cluster shape for (N images, HW rows, C channels, G groups): slabs of gpc groups, S CTAs per slab.  Returns false when
// the staged rows do not fit in shared memory (the statistics + apply kernel pairs take over).
static bool g_gn_cluster_unavailable = false;     // set when a cluster launch was refused: the kernel pairs take over
struct GnClPlan { int S, gpc, rows_per_cta; size_t smem; };
static inline bool gn_cluster_plan(int N, int HW, int C, int G, size_t bytes_per_elem, GnClPlan* out) {
    if (G > 32) return false;
    const int cpg = C / G;
    const int sms = device_sm_count();
    for (int gpc : {4, 8, 2, 16, 1, 32}) {
        if (G % gpc) continue;
        const int cw = gpc * cpg;
        const int nq = cw / 4;
        if (cw % 4 || C % 4 || nq < 2 || nq > kGnClThreads) continue;      // thread map: 4-channel accesses, >= 1 row lane per quad
        const long long slabs = (long long)N * (G / gpc);
        int S = kGnClMaxS;
        while (S > 1 && slabs * S > sms) S >>= 1;
        if (slabs * S > 2 * sms) continue;
        if (S > HW) S = 1;
        const int rows = ceil_div(HW, S);
        const size_t smem = (((size_t)rows * cw * bytes_per_elem) + 255) & ~(size_t)127;
        if (smem > kGnMaxDynSmem) continue;
        out->S = S; out->gpc = gpc; out->rows_per_cta = rows; out->smem = smem;
        return true;
    }
    return false;
}

// ---- LayerNorm: one warp per row ------------------------------------------------------------------------
constexpr int kLnMaxPairsPerLane = 32;  // C <= 2048

template <typename TX, typename TY>
__global__ void __launch_bounds__(128)
ln_fwd_kernel(const TX* __restrict__ x, TY* __restrict__ y, const float* __restrict__ gamma,
              const float* __restrict__ beta, float* __restrict__ mean_out, float* __restrict__ rstd_out, int M, int C,
              float eps) {
    pdl_sync();
    const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (row >= M) return;
    const int lane = threadIdx.x & 31;
    const int npairs = C >> 1;
    const TX* xr = x + (size_t)row * C;
    float2 v[kLnMaxPairsPerLane];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < kLnMaxPairsPerLane; ++i) {
        const int pr = lane + i * 32;
        if (pr < npairs) {
            v[i] = Vec2<TX>::ld(xr + 2 * pr);
            s += v[i].x + v[i].y;
        }
    }
    const float mean = warp_sum(s) / C;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < kLnMaxPairsPerLane; ++i) {
        const int pr = lane + i * 32;
        if (pr < npairs) {
            const float a = v[i].x - mean, b = v[i].y - mean;
            q += a * a + b * b;
        }
    }
    const float rstd = rsqrtf(warp_sum(q) / C + eps);
    if (lane == 0) {
        mean_out[row] = mean;
        rstd_out[row] = rstd;
    }
    TY* yr = y + (size_t)row * C;
#pragma unroll
    for (int i = 0; i < kLnMaxPairsPerLane; ++i) {
        const int pr = lane + i * 32;
        if (pr < npairs) {
            const int c = 2 * pr;
            float2 o;
            o.x = (v[i].x - mean) * rstd * gamma[c] + beta[c];
            o.y = (v[i].y - mean) * rstd * gamma[c + 1] + beta[c + 1];
            Vec2<TY>::st(yr + c, o);
        }
    }
}

template <typename TX, typename TG, typename TD>
__global__ void __launch_bounds__(128)
ln_bwd_kernel(const TG* __restrict__ dy, const TX* __restrict__ x, const float* __restrict__ gamma,
              const float* __restrict__ mean, const float* __restrict__ rstd, TD* __restrict__ dx, TG* __restrict__ dx_lp,
              int M, int C, int accumulate) {
    pdl_sync();
    const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (row >= M) return;
    const int lane = threadIdx.x & 31;
    const int npairs = C >> 1;
    const float m = mean[row], rs = rstd[row];
    const TX* xr = x + (size_t)row * C;
    const TG* dr = dy + (size_t)row * C;
    float2 xh[kLnMaxPairsPerLane], t[kLnMaxPairsPerLane];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < kLnMaxPairsPerLane; ++i) {
        const int pr = lane + i * 32;
        if (pr < npairs) {
            const int c = 2 * pr;
            const float2 xv = Vec2<TX>::ld(xr + c);
            const float2 d = Vec2<TG>::ld(dr + c);
            xh[i].x = (xv.x - m) * rs;
            xh[i].y = (xv.y - m) * rs;
            t[i].x = d.x * gamma[c];
            t[i].y = d.y * gamma[c + 1];
            s1 += t[i].x + t[i].y;
            s2 += t[i].x * xh[i].x + t[i].y * xh[i].y;
        }
    }
    s1 = warp_sum(s1) / C;
    s2 = warp_sum(s2) / C;
    TD* or_ = dx + (size_t)row * C;
#pragma unroll
    for (int i = 0; i < kLnMaxPairsPerLane; ++i) {
        const int pr = lane + i * 32;
        if (pr < npairs) {
            const int c = 2 * pr;
            float2 o;
            o.x = rs * (t[i].x - s1 - xh[i].x * s2);
            o.y = rs * (t[i].y - s1 - xh[i].y * s2);
            if (accumulate) {
                const float2 p = Vec2<TD>::ld(or_ + c);
                o.x += p.x;
                o.y += p.y;
            }
            Vec2<TD>::st(or_ + c, o);
            if (dx_lp) Vec2<TG>::st(dx_lp + (size_t)row * C + c, o);     // 16-bit copy for the GEMM that consumes dx next
        }
    }
}

// CTAs per image whose (sum, sumsq) partials (float2 per group) fit the caller's workspace.  The last 8 bytes stay out of
// the budget: the partials are added in CTA order, so a different CTA count would change the results' bits.
static inline int gn_max_blocks(int N, int G) { return std::max(1, (int)((CB_GN_WS_BYTES - 8) / (8 * (size_t)G * N))); }
static inline int gn_rows_per_block(int HW, int N, int G) {
    const int target_blocks = 8 * device_sm_count();     // 256-thread blocks: 8 per SM keep 2048 threads x 8 loads in flight
    int per_img = std::min(ceil_div(target_blocks, N), gn_max_blocks(N, G));
    if (per_img < 1) per_img = 1;
    int rpb = ceil_div(HW, per_img);
    if (rpb < 1) rpb = 1;
    return rpb;
}

}  // namespace cb

using namespace cb;

#define CB_DISPATCH_2(dtype, T, ...)                                             \
    if ((dtype) == CB_F32) { using T = float; __VA_ARGS__; }                     \
    else if ((dtype) == CB_F16) { using T = __half; __VA_ARGS__; }               \
    else if ((dtype) == CB_BF16) { using T = __nv_bfloat16; __VA_ARGS__; }       \
    else { cb::set_error("unsupported dtype %d", (int)(dtype)); return CB_ERR_ARG; }

static int gn_check(int N, int HW, int C, int G) {
    CB_REQUIRE(N > 0 && HW > 0 && C > 0 && G > 0 && G <= 64 && C % G == 0, CB_ERR_ARG, "groupnorm: bad shape N=%d HW=%d C=%d G=%d", N, HW, C, G);
    CB_REQUIRE((C / G) % 2 == 0, CB_ERR_ARG, "groupnorm: channels per group must be even (C=%d G=%d)", C, G);
    CB_REQUIRE(gn_shape(C).chunks <= kGnMaxChunks, CB_ERR_ARG, "groupnorm: C=%d not supported by the thread mapping", C);
    return 0;
}

extern "C" int cb_groupnorm_cluster_plan(int N, int HW, int C, int G, int bytes_per_elem, int* plan) {
    int rc = gn_check(N, HW, C, G);
    if (rc) return rc;
    CB_REQUIRE(plan != nullptr && bytes_per_elem > 0, CB_ERR_ARG, "cb_groupnorm_cluster_plan: bad arguments");
    GnClPlan pl;
    if (!gn_cluster_plan(N, HW, C, G, (size_t)bytes_per_elem, &pl)) return 0;
    plan[0] = pl.S; plan[1] = pl.gpc; plan[2] = pl.rows_per_cta; plan[3] = (int)pl.smem;
    return 1;
}

extern "C" int cb_groupnorm_fwd(const void* x, int x_dtype, void* y, int y_dtype, const float* gamma, const float* beta,
                                int N, int HW, int C, int G, float eps, int act_silu, float* mean_out, float* rstd_out,
                                double* ws, void* stream) {
    int rc = gn_check(N, HW, C, G);
    if (rc) return rc;
    // checked before any launch: the streaming pair dispatches y_dtype only after its statistics kernel is launched
    CB_REQUIRE(x_dtype >= CB_F16 && x_dtype <= CB_F32 && y_dtype >= CB_F16 && y_dtype <= CB_F32, CB_ERR_ARG,
               "groupnorm_fwd: unsupported dtype (x %d, y %d)", x_dtype, y_dtype);
    // the streaming pair stages whole rows with cp.async.bulk, whose sizes and addresses are multiples of 16 bytes;
    // checked here, before any launch, so that a shape is accepted or refused the same way on every device
    const size_t row_bytes = (size_t)C * (x_dtype == CB_F32 ? 4 : 2);
    CB_REQUIRE(row_bytes % 16 == 0, CB_ERR_ARG, "groupnorm_fwd: rows must be multiples of 16 bytes (C=%d, x dtype %d)", C,
               x_dtype);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    // flags: bit 0 = fuse SiLU; bits 8..23: upper bound on the CTAs of the streaming two-kernel path (0 = two per SM): a
    // front end that shares the device with a latency-bound chain of small launches leaves the other SMs to it
    const int cta_cap = (act_silu >> 8) & 0xFFFF;
    act_silu &= 1;
    {
        // cluster path: slabs of groups, statistics through distributed shared memory
        GnClPlan pl;
        if (!g_gn_cluster_unavailable && gn_cluster_plan(N, HW, C, G, x_dtype == CB_F32 ? 4 : 2, &pl)) {
            dim3 gridc((unsigned)pl.S, (unsigned)(G / pl.gpc), (unsigned)N);
            cudaError_t le = cudaSuccess;
            CB_DISPATCH_2(x_dtype, TX, CB_DISPATCH_2(y_dtype, TY, {
                auto kern = gn_cluster_fwd_kernel<TX, TY>;
                static bool set = false;
                if (!set) {
                    le = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kGnMaxDynSmem);
                    if (le == cudaSuccess) le = cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
                    set = le == cudaSuccess;
                }
                if (le == cudaSuccess)
                    le = launch_kernel_cluster(kern, gridc, dim3(kGnClThreads), dim3((unsigned)pl.S, 1, 1), pl.smem, st,
                                               (const TX*)x, (TY*)y, gamma, beta, mean_out, rstd_out, HW, C, G, eps, act_silu,
                                               pl.gpc, pl.rows_per_cta);
            }));
            if (le == cudaSuccess) {
                CB_CUDA(cudaGetLastError());
                cb::count_launches(1);
                return 0;
            }
            // this device cannot co-schedule the cluster (or refuses the attributes): clear the launch error and use the
            // streaming pair from now on
            (void)cudaGetLastError();
            g_gn_cluster_unavailable = true;
        }
    }
    // streaming (TMA-staged) pair.  ws: one (sum, sumsq) float2 partial per (image, CTA, group), added up in CTA order.
    // gn_check bounds C to 4096, so a row is at most 16 KiB and a 32 KiB stage holds at least two.
    const GnShape gs = gn_shape(C);
    const int nthr = gs.pw * gs.ry;
    const int rpc = (int)(kGnTmaChunkBytes / row_bytes);
    const int ctas = cta_cap > 0 ? std::min(cta_cap, 2 * device_sm_count()) : 2 * device_sm_count();
    const int nb = std::max(1, std::min(ctas / N, gn_max_blocks(N, G)));
    const int rpbt = ceil_div(HW, nb);
    dim3 gridt(ceil_div(HW, rpbt), N);
    const size_t smem = (size_t)kGnTmaStages * kGnTmaChunkBytes;
    CB_DISPATCH_2(x_dtype, TX, {
        auto kern = gn_stats_tma_kernel<TX>;
        static bool set = false;
        if (!set) { CB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); set = true; }
        CB_LAUNCH((kern), gridt, nthr, smem, st, (const TX*)x, ws, HW, C, G, rpbt, rpc, gs.pw, gs.ry, gs.chunks);
    });
    CB_DISPATCH_2(x_dtype, TX, CB_DISPATCH_2(y_dtype, TY, {
        auto kern = gn_apply_tma_kernel<TX, TY>;
        static bool set = false;
        if (!set) { CB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); set = true; }
        CB_LAUNCH((kern), gridt, nthr, smem, st, (const TX*)x, (TY*)y, gamma, beta, ws, mean_out, rstd_out, HW, C, G, eps, act_silu, rpbt, rpc, gs.pw, gs.ry, gs.chunks);
    }));
    CB_CUDA(cudaGetLastError());
    cb::count_launches(2);
    return 0;
}

extern "C" int cb_groupnorm_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, const float* gamma,
                                const float* beta, const float* mean, const float* rstd, void* dx, int dx_dtype,
                                void* dx_lp, int N, int HW, int C, int G, int act_silu, int accumulate, double* ws,
                                void* stream) {
    int rc = gn_check(N, HW, C, G);
    if (rc) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const GnShape gs = gn_shape(C);
    const int nthr = gs.pw * gs.ry;
    CB_REQUIRE(dx_dtype == CB_F32 || dx_dtype == dy_dtype, CB_ERR_ARG, "groupnorm_bwd: dx dtype must be f32 or equal dy dtype");
    act_silu &= 1;
    {
        GnClPlan pl;
        if (!g_gn_cluster_unavailable && gn_cluster_plan(N, HW, C, G, (x_dtype == CB_F32 ? 4 : 2) + (dy_dtype == CB_F32 ? 4 : 2), &pl)) {
            dim3 gridc((unsigned)pl.S, (unsigned)(G / pl.gpc), (unsigned)N);
            cudaError_t le = cudaSuccess;
#define CB_GN_BWD_CLUSTER(TDX)                                                                                                    \
            CB_DISPATCH_2(x_dtype, TX, CB_DISPATCH_2(dy_dtype, TG, {                                                              \
                auto kern = gn_cluster_bwd_kernel<TX, TG, TDX>;                                                                   \
                static bool set = false;                                                                                          \
                if (!set) {                                                                                                       \
                    le = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kGnMaxDynSmem);                     \
                    if (le == cudaSuccess) le = cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);    \
                    set = le == cudaSuccess;                                                                                      \
                }                                                                                                                 \
                if (le == cudaSuccess)                                                                                            \
                    le = launch_kernel_cluster(kern, gridc, dim3(kGnClThreads), dim3((unsigned)pl.S, 1, 1), pl.smem, st,          \
                                               (const TG*)dy, (const TX*)x, gamma, beta, mean, rstd, (TDX*)dx, (TG*)dx_lp, HW, C, \
                                               G, act_silu, accumulate, pl.gpc, pl.rows_per_cta);                                 \
            }))
            if (dx_dtype == CB_F32) { CB_GN_BWD_CLUSTER(float); }
            else { CB_GN_BWD_CLUSTER(TG); }
#undef CB_GN_BWD_CLUSTER
            if (le == cudaSuccess) {
                CB_CUDA(cudaGetLastError());
                cb::count_launches(1);
                return 0;
            }
            (void)cudaGetLastError();            // see cb_groupnorm_fwd
            g_gn_cluster_unavailable = true;
        }
    }
    // statistics + apply pair.  ws: one (sum, sumsq) float2 partial per (image, CTA, group), added up in CTA order
    const int rpb = gn_rows_per_block(HW, N, G);
    dim3 grid(ceil_div(HW, rpb), N);
    CB_DISPATCH_2(x_dtype, TX, CB_DISPATCH_2(dy_dtype, TG,
CB_LAUNCH((gn_bwd_stats_kernel<TX, TG>), grid, nthr, 0, st, (const TG*)dy, (const TX*)x, gamma, beta, mean, rstd, ws, HW, C, G, act_silu, rpb, gs.pw, gs.ry, gs.chunks)));
    // dx dtype: f32 or the gradient dtype
    if (dx_dtype == CB_F32) {
        CB_DISPATCH_2(x_dtype, TX, CB_DISPATCH_2(dy_dtype, TG,
CB_LAUNCH((gn_bwd_apply_kernel<TX, TG, float>), grid, nthr, 0, st, (const TG*)dy, (const TX*)x, gamma, beta, mean, rstd, ws, (float*)dx, (TG*)dx_lp, HW, C, G, act_silu, accumulate, rpb, gs.pw, gs.ry, gs.chunks)));
    } else {
        CB_REQUIRE(dx_dtype == dy_dtype, CB_ERR_ARG, "groupnorm_bwd: dx dtype must be f32 or equal dy dtype");
        CB_DISPATCH_2(x_dtype, TX, CB_DISPATCH_2(dy_dtype, TG,
CB_LAUNCH((gn_bwd_apply_kernel<TX, TG, TG>), grid, nthr, 0, st, (const TG*)dy, (const TX*)x, gamma, beta, mean, rstd, ws, (TG*)dx, (TG*)dx_lp, HW, C, G, act_silu, accumulate, rpb, gs.pw, gs.ry, gs.chunks)));
    }
    CB_CUDA(cudaGetLastError());
    cb::count_launches(2);
    return 0;
}

int cb::layernorm_fwd_legacy(const void* x, int x_dtype, void* y, int y_dtype, const float* gamma, const float* beta,
                             int M, int C, float eps, float* mean_out, float* rstd_out, void* stream) {
    CB_REQUIRE(M > 0 && C > 0 && C % 2 == 0 && C <= 64 * kLnMaxPairsPerLane, CB_ERR_ARG, "layernorm: bad shape M=%d C=%d", M, C);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    dim3 grid(ceil_div(M, 4));
    CB_DISPATCH_2(x_dtype, TX, CB_DISPATCH_2(y_dtype, TY,
CB_LAUNCH((ln_fwd_kernel<TX, TY>), grid, 128, 0, st, (const TX*)x, (TY*)y, gamma, beta, mean_out, rstd_out, M, C, eps)));
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

int cb::layernorm_bwd_legacy(const void* dy, int dy_dtype, const void* x, int x_dtype, const float* gamma,
                             const float* mean, const float* rstd, void* dx, int dx_dtype, void* dx_lp, int M, int C,
                             int accumulate, void* stream) {
    CB_REQUIRE(M > 0 && C > 0 && C % 2 == 0 && C <= 64 * kLnMaxPairsPerLane, CB_ERR_ARG, "layernorm_bwd: bad shape M=%d C=%d", M, C);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    dim3 grid(ceil_div(M, 4));
    if (dx_dtype == CB_F32) {
        CB_DISPATCH_2(x_dtype, TX, CB_DISPATCH_2(dy_dtype, TG,
CB_LAUNCH((ln_bwd_kernel<TX, TG, float>), grid, 128, 0, st, (const TG*)dy, (const TX*)x, gamma, mean, rstd, (float*)dx, (TG*)dx_lp, M, C, accumulate)));
    } else {
        CB_REQUIRE(dx_dtype == dy_dtype, CB_ERR_ARG, "layernorm_bwd: dx dtype must be f32 or equal dy dtype");
        CB_DISPATCH_2(x_dtype, TX, CB_DISPATCH_2(dy_dtype, TG,
CB_LAUNCH((ln_bwd_kernel<TX, TG, TG>), grid, 128, 0, st, (const TG*)dy, (const TX*)x, gamma, mean, rstd, (TG*)dx, (TG*)dx_lp, M, C, accumulate)));
    }
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}
