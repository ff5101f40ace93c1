// cb_gemm — wgmma GEMM / implicit-GEMM convolution for sm_90a.
//
// One CTA computes one 128 x BN output tile:
//   thread 0         : TMA producer (cp.async.bulk.tensor, SWIZZLE_128B boxes, mbarrier complete_tx)
//   warpgroups 1, 2  : wgmma.mma_async on 64 rows each, fp32 accumulators in registers
//   warpgroup 0      : row metadata and bias row of the tile during the k-loop
//   all 384 threads  : epilogue (staged accumulator tile -> alpha/bias/act/residual -> HBM), 8-column units
// Convolutions never materialise im2col: each (tap, 64-channel) k-iteration loads a SHIFTED
// [box_i][box_h][box_w][64ch] box of the NHWC image straight into the K-major A tile; padding is
// the TMA out-of-bounds zero fill, stride-2 is the tensor-map traversal stride.
#include <algorithm>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "cb_common.cuh"

namespace cb {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int kThreads = 384;

struct GemmParams {
    int M, N, K;
    int kchunks, taps, kw;
    int ksteps_last;  // MMA k-steps (of 16) in the last 64-chunk of each tap
    int conv;
    int out_h, out_w, img_n;
    int box_w, box_h, box_i;
    int tiles_w, tiles_h;
    int stride, pad_top, pad_left;
    int b_tap_rows, flip_taps;
    void* D;
    int d_dtype;
    long long ldd, d_bs, d_bs2;
    void* D2;          // optional second destination (same value, own dtype / row pitch)
    int d2_dtype;
    long long ldd2;
    int glu;                   // GEGLU epilogue: column chunks come in (value, gate) pairs; D2 = value * gelu(gate)
    const float* act_param;    // CB_ACT_PRELU: per-column negative slope
    const float* d2_scale;     // optional per-column affine applied to the D2 copy only: D2 = v * scale[col] + shift[col]
    const float* d2_shift;
    int batch_inner;
    int d_transposed;
    int vec_ok;
    int force_stages;  // 0 auto / 3 / 6 (cb_gemm_desc.stages)
    const float* bias;
    int bias_row_div;
    long long ldbias;
    const void* R;
    int r_dtype;
    long long ldr, r_bs, r_bs2;
    float alpha;
    int act;
    int bf16;                 // operands are bf16 (else fp16)
    unsigned a_bytes, b_bytes;
    // split-K: the k-iterations of one output tile are spread over `splits` CTAs which store their fp32 partials into
    // the tile's slices of `ws`; the last CTA to arrive (per-tile counter) sums them in slice order and runs the epilogue.
    int splits, kiters_per_split;
    float* ws;
    unsigned* counters;
    int cluster_sk;           // split-K through distributed shared memory: the `splits` CTAs of a tile form a cluster (1,1,splits)
    int dbg_mode;             // tuning aid (env CB_GEMM_DBG_MODE): 1 exit after setup, 2 skip epilogue, 3 exit at once
    unsigned long long* dbg;  // optional per-CTA timeline (8 x u64 globaltimer ns per CTA), NULL in production
};

template <int BN, int kStages>
struct TileCfg {
    static constexpr int kTmemCols = BN <= 64 ? 64 : (BN <= 128 ? 128 : 256);
    static constexpr int kABytes = BM * BK * 2;
    static constexpr int kBBytes = BN * BK * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kSmemBytes = kStages * kStageBytes + 1024 + 256;
    static_assert(kStages * kStageBytes >= BM * (BN + 4) * 4, "the accumulator tile is staged in the TMA ring");
};

__device__ __forceinline__ unsigned long long gtimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ float apply_act(float v, int act) {
    switch (act) {
        case CB_ACT_SILU: return silu_f(v);
        case CB_ACT_GELU: return gelu_f(v);
        case CB_ACT_QUICK_GELU: return quick_gelu_f(v);
        default: return v;
    }
}

// activation of 8 consecutive columns starting at `col` (PReLU reads its per-column slopes)
__device__ __forceinline__ void apply_act8(float (&f)[8], int act, const float* act_param, int col, int ncols = 8) {
    if (act == CB_ACT_PRELU) {
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (j < ncols) f[j] = f[j] > 0.f ? f[j] : f[j] * __ldg(act_param + col + j);
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] = apply_act(f[j], act);
    }
}
// second destination: optional per-column affine (eval BatchNorm of the consumer folded into the producer's epilogue)
__device__ __forceinline__ void d2_affine8(float (&g)[8], const float (&f)[8], const float* sc, const float* sh, int col,
                                           int ncols = 8) {
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] = (sc && j < ncols) ? f[j] * __ldg(sc + col + j) + __ldg(sh + col + j) : f[j];
}

template <typename T>
__device__ __forceinline__ void load8(const T* p, float (&f)[8]);
template <>
__device__ __forceinline__ void load8<__half>(const __half* p, float (&f)[8]) {
    uint4 u = *reinterpret_cast<const uint4*>(p);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float2 t = __half22float2(h[i]);
        f[2 * i] = t.x;
        f[2 * i + 1] = t.y;
    }
}
template <>
__device__ __forceinline__ void load8<__nv_bfloat16>(const __nv_bfloat16* p, float (&f)[8]) {
    uint4 u = *reinterpret_cast<const uint4*>(p);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float2 t = __bfloat1622float2(h[i]);
        f[2 * i] = t.x;
        f[2 * i + 1] = t.y;
    }
}
template <>
__device__ __forceinline__ void load8<float>(const float* p, float (&f)[8]) {
    float4 a = *reinterpret_cast<const float4*>(p);
    float4 b = *reinterpret_cast<const float4*>(p + 4);
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
    f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

template <typename T>
__device__ __forceinline__ void store8(T* p, const float (&f)[8]);
template <>
__device__ __forceinline__ void store8<__half>(__half* p, const float (&f)[8]) {
    uint4 u;
    __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
    *reinterpret_cast<uint4*>(p) = u;
}
template <>
__device__ __forceinline__ void store8<__nv_bfloat16>(__nv_bfloat16* p, const float (&f)[8]) {
    uint4 u;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
    *reinterpret_cast<uint4*>(p) = u;
}
template <>
__device__ __forceinline__ void store8<float>(float* p, const float (&f)[8]) {
    *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
    *reinterpret_cast<float4*>(p + 4) = make_float4(f[4], f[5], f[6], f[7]);
}

__device__ __forceinline__ float load_any(const void* base, int dtype, long long idx) {
    if (dtype == CB_F32) return reinterpret_cast<const float*>(base)[idx];
    if (dtype == CB_F16) return __half2float(reinterpret_cast<const __half*>(base)[idx]);
    return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(base)[idx]);
}
__device__ __forceinline__ void store_any(void* base, int dtype, long long idx, float v) {
    if (dtype == CB_F32) reinterpret_cast<float*>(base)[idx] = v;
    else if (dtype == CB_F16) reinterpret_cast<__half*>(base)[idx] = __float2half_rn(v);
    else reinterpret_cast<__nv_bfloat16*>(base)[idx] = __float2bfloat16_rn(v);
}

// 8 consecutive values -> 16-byte aligned destination of any output dtype (second destination D2)
__device__ __forceinline__ void store8_any(void* base, int dtype, long long idx, const float (&f)[8]) {
    if (dtype == CB_F32) store8<float>(reinterpret_cast<float*>(base) + idx, f);
    else if (dtype == CB_F16) store8<__half>(reinterpret_cast<__half*>(base) + idx, f);
    else store8<__nv_bfloat16>(reinterpret_cast<__nv_bfloat16*>(base) + idx, f);
}

// Residual of one 8-column unit as raw 16-byte words (two for fp32, one for fp16 / bf16), loaded a few units before the
// accumulator needs it.  D may alias R: every element is read and then written by the same thread, so the early load
// never sees a value this launch stored.
__device__ __forceinline__ void residual_load8(const GemmParams& p, long long idx, uint4 (&v)[2]) {
    if (p.r_dtype == CB_F32) {
        const uint4* s = reinterpret_cast<const uint4*>(reinterpret_cast<const float*>(p.R) + idx);
        v[0] = s[0];
        v[1] = s[1];
    } else {
        v[0] = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(p.R) + idx);
    }
}
__device__ __forceinline__ void residual_unpack8(const GemmParams& p, const uint4 (&v)[2], float (&r)[8]) {
    if (p.r_dtype == CB_F32) {
        const uint4 a = v[0], b = v[1];
        r[0] = __uint_as_float(a.x); r[1] = __uint_as_float(a.y); r[2] = __uint_as_float(a.z); r[3] = __uint_as_float(a.w);
        r[4] = __uint_as_float(b.x); r[5] = __uint_as_float(b.y); r[6] = __uint_as_float(b.z); r[7] = __uint_as_float(b.w);
    } else {
        const uint32_t w[4] = {v[0].x, v[0].y, v[0].z, v[0].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float2 t;
            if (p.r_dtype == CB_F16) t = __half22float2(*reinterpret_cast<const __half2*>(&w[j]));
            else t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[j]));
            r[2 * j] = t.x; r[2 * j + 1] = t.y;
        }
    }
}

// Epilogue of one 8-column unit of one output row: alpha is applied by the caller; bias, activation, residual, store D,
// then D2 with its affine.  kExt is the instantiation that carries the rarely used features (second destination, PReLU
// slopes, D2 affine, GEGLU), so the common instantiation does not carry their code.
template <bool kExt>
__device__ __forceinline__ void epilogue_group8(const GemmParams& p, float (&f)[8], long long grow, long long brow, int col,
                                             long long d_off, long long r_off, int ncols, const float* rpre = nullptr,
                                             const float* sbias = nullptr) {
    if (sbias) {       // this tile's bias row, staged in shared memory before the accumulator was ready
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] += sbias[j];
    } else if (p.bias) {
        if (ncols == 8 && p.vec_ok) {      // vec_ok: 16-byte aligned bias rows
            float b[8];
            load8<float>(p.bias + brow * p.ldbias + col, b);
#pragma unroll
            for (int j = 0; j < 8; ++j) f[j] += b[j];
        } else {
            for (int j = 0; j < ncols; ++j) f[j] += p.bias[brow * p.ldbias + col + j];
        }
    }
    if (p.act != CB_ACT_NONE) {
        if constexpr (kExt) {
            apply_act8(f, p.act, p.act_param, col, ncols);
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) f[j] = apply_act(f[j], p.act);
        }
    }
    if (ncols == 8 && p.vec_ok && !p.d_transposed) {
        if (rpre) {
#pragma unroll
            for (int j = 0; j < 8; ++j) f[j] += rpre[j];
        } else if (p.R) {
            float r[8];
            const long long ridx = r_off + grow * p.ldr + col;
            if (p.r_dtype == CB_F32) load8<float>(reinterpret_cast<const float*>(p.R) + ridx, r);
            else if (p.r_dtype == CB_F16) load8<__half>(reinterpret_cast<const __half*>(p.R) + ridx, r);
            else load8<__nv_bfloat16>(reinterpret_cast<const __nv_bfloat16*>(p.R) + ridx, r);
#pragma unroll
            for (int j = 0; j < 8; ++j) f[j] += r[j];
        }
        const long long didx = d_off + grow * p.ldd + col;
        if (p.d_dtype == CB_F32) store8<float>(reinterpret_cast<float*>(p.D) + didx, f);
        else if (p.d_dtype == CB_F16) store8<__half>(reinterpret_cast<__half*>(p.D) + didx, f);
        else store8<__nv_bfloat16>(reinterpret_cast<__nv_bfloat16*>(p.D) + didx, f);
        if constexpr (kExt) {
            if (p.D2) {
                float g2[8];
                d2_affine8(g2, f, p.d2_scale, p.d2_shift, col);
                store8_any(p.D2, p.d2_dtype, grow * p.ldd2 + col, g2);
            }
        }
    } else {
        for (int j = 0; j < ncols; ++j) {
            float v = f[j];
            if (p.R) v += load_any(p.R, p.r_dtype, r_off + grow * p.ldr + col + j);
            const long long didx = p.d_transposed ? (d_off + (long long)(col + j) * p.ldd + grow)
                                                  : (d_off + grow * p.ldd + col + j);
            store_any(p.D, p.d_dtype, didx, v);
            if constexpr (kExt) {
                if (p.D2) store_any(p.D2, p.d2_dtype, grow * p.ldd2 + col + j,
                                    p.d2_scale ? v * p.d2_scale[col + j] + p.d2_shift[col + j] : v);
            }
        }
    }
}

// Warp roles (384 threads, one CTA per SM):
//   warpgroup 0 : thread 0 is the TMA producer; the other threads stage the tile's row metadata and bias row meanwhile
//   warpgroups 1, 2 : wgmma consumers, rows [0, 64) and [64, 128) of the tile, fp32 accumulators in registers
// Once the last k-iteration has retired, the consumers park their accumulators in the (then idle) TMA ring as a row-major
// fp32 tile of pitch BN + 4 floats, and all 384 threads run the epilogue on it (epilogue_units).
template <int BN>
struct StageCfg {
    static constexpr int kPitch = BN + 4;
    static constexpr int kBytes = ((BM * kPitch * 4) + 1023) / 1024 * 1024;
};

// 8 consecutive accumulator columns of the staged tile, times alpha
__device__ __forceinline__ void stage_ld8(const float* src, float alpha, float (&f)[8]) {
    const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
    f[0] = a.x * alpha; f[1] = a.y * alpha; f[2] = a.z * alpha; f[3] = a.w * alpha;
    f[4] = b.x * alpha; f[5] = b.y * alpha; f[6] = b.z * alpha; f[7] = b.w * alpha;
}

// ---- split-K hand-off through L2 (all 384 threads): every CTA stores its fp32 partial tile into its own slice of the
//      tile's workspace (slice = k-slice index); the last CTA to arrive (per-tile counter) adds the slices up in slice order,
//      starting from zero -- the same order as the cluster exchange, so the result does not depend on which CTA finishes
//      last --, writes the sum back over its staged tile for the ordinary epilogue and re-zeroes the counter.
//      Slice layout: float4 group g (= 4 columns) of row r is float4 number g * BM + r, so consecutive threads touch
//      consecutive 16-byte words.  The reduction keeps kU float4 per thread and the next slice's loads in flight while it
//      adds the current one: the last CTA reads S partial tiles (up to S x 80 KiB) and is bound by L2 latency, not by adds.
//      Returns false in every CTA but the last one of the tile.
template <int BN>
__device__ __forceinline__ bool splitk_reduce_to_stage(const GemmParams& p, unsigned tile_id, int sp, float* stage,
                                                       int ncols_tile) {
    constexpr int kPitch = StageCfg<BN>::kPitch;
    constexpr int kSlice4 = BM * BN / 4;
    constexpr int kU = 8;
    const int n4 = ((ncols_tile + 3) >> 2) * BM;        // float4 groups that hold output columns
    const float4* slices = reinterpret_cast<const float4*>(p.ws) + static_cast<size_t>(tile_id) * p.splits * kSlice4;
    float4* mine = reinterpret_cast<float4*>(p.ws) + (static_cast<size_t>(tile_id) * p.splits + sp) * kSlice4;
    for (int i = threadIdx.x; i < n4; i += kThreads)
        __stcg(mine + i, *reinterpret_cast<const float4*>(stage + (i % BM) * kPitch + 4 * (i / BM)));
    __threadfence();
    __syncthreads();
    __shared__ unsigned s_last;
    if (threadIdx.x == 0) {
        const unsigned prev = atomicAdd(p.counters + tile_id, 1u);
        s_last = (prev == static_cast<unsigned>(p.splits) - 1u) ? 1u : 0u;
    }
    __syncthreads();
    if (s_last == 0u) return false;
    __threadfence();
    for (int i0 = threadIdx.x; i0 < n4; i0 += kU * kThreads) {
        float4 sum[kU], cur[kU], nxt[kU];
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            sum[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            nxt[u] = sum[u];
            cur[u] = i0 + u * kThreads < n4 ? __ldcg(slices + i0 + u * kThreads) : sum[u];
        }
#pragma unroll 1
        for (int s = 0; s < p.splits; ++s) {
            if (s + 1 < p.splits) {
                const float4* src = slices + static_cast<size_t>(s + 1) * kSlice4;
#pragma unroll
                for (int u = 0; u < kU; ++u)
                    if (i0 + u * kThreads < n4) nxt[u] = __ldcg(src + i0 + u * kThreads);
            }
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                sum[u].x += cur[u].x; sum[u].y += cur[u].y; sum[u].z += cur[u].z; sum[u].w += cur[u].w;
                cur[u] = nxt[u];
            }
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            const int i = i0 + u * kThreads;
            if (i < n4) *reinterpret_cast<float4*>(stage + (i % BM) * kPitch + 4 * (i / BM)) = sum[u];
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) p.counters[tile_id] = 0u;   // self-cleaning for the next launch
    return true;
}

// One k-iteration of a consumer warpgroup: KSTEPS k16 MMAs over the stage at (a_src, b_src), issued as one wgmma group.
// Straight-line code between one fence and one commit lets ptxas put a single warpgroup.arrive in front of the batch and
// the scoreboard wait (gsb0) on its last MMA only; an MMA in a branch of its own gets an injected arrive (C7519) and waits
// for the one before it.
template <int BN, bool A_MN, bool B_MN, bool BF16, int KSTEPS>
__device__ __forceinline__ void mma_batch(float (&acc)[BN / 2], uint32_t a_src, uint32_t b_src) {
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < KSTEPS; ++k) {
        const uint64_t adesc = A_MN ? gmma_desc_sw128(a_src + k * 2048, 8192, 1024) : gmma_desc_sw128(a_src + k * 32, 16, 1024);
        const uint64_t bdesc = B_MN ? gmma_desc_sw128(b_src + k * 2048, 8192, 1024) : gmma_desc_sw128(b_src + k * 32, 16, 1024);
        Wgmma<BN, BF16, A_MN, B_MN>::mma(acc, adesc, bdesc, 1u);
    }
    wgmma_commit();
}

// ksteps < 4 only in the last 64-chunk of a tap (K % 64 != 0); it gets exactly that many MMAs, never zero-filled extra
// ones: a +0 product would turn a -0.0 accumulator into +0.0
template <int BN, bool A_MN, bool B_MN, bool BF16>
__device__ __forceinline__ void mma_kiter(float (&acc)[BN / 2], uint32_t a_src, uint32_t b_src, int ksteps) {
    switch (ksteps) {
        case 4: mma_batch<BN, A_MN, B_MN, BF16, 4>(acc, a_src, b_src); break;
        case 3: mma_batch<BN, A_MN, B_MN, BF16, 3>(acc, a_src, b_src); break;
        case 2: mma_batch<BN, A_MN, B_MN, BF16, 2>(acc, a_src, b_src); break;
        default: mma_batch<BN, A_MN, B_MN, BF16, 1>(acc, a_src, b_src); break;
    }
}

// ---- epilogue, all 384 threads.  The work unit is 8 consecutive columns of one row of the staged fp32 tile
//      (epilogue_group8).  Unit u of the tile is row u / (BN / 8), column group u % (BN / 8), so the lanes of a warp cover
//      consecutive column groups of the same rows: every D / D2 store and residual load of a warp writes or reads whole
//      rows of the tile (two rows per warp at BN = 128, four at BN = 64).  Thread t takes units t, t + 384, ...
//      - transposed D: unit u is row u % 128 of column group u / 128, so the lanes store consecutive rows of one column;
//      - GEGLU: the unit is one 8-column slice of the 32 value columns of a 64-column group and the matching 8 gate columns;
//      - the residual of a thread's next kResAhead units is in flight while it works on the current one;
//      - cluster split-K: every thread sends units of its partial tile to their owner CTAs, then sums the units it owns
//        over the senders in sender order 0..S-1 and finishes them like the ordinary path.  Both phases map the lanes to
//        consecutive rows of one group, so the exchange slots a warp writes and reads are contiguous.
template <int BN, bool kExt>
__device__ __forceinline__ void epilogue_units(const GemmParams& p, const float* stage, const long long* s_grow,
                                               const int* s_brow, const float* s_bias, int n0, int ncols_tile, int zo,
                                               int zi, int sp, uint32_t xbuf, unsigned long long* dbg) {
    constexpr int kPitch = StageCfg<BN>::kPitch;
    constexpr int G = BN / 8;             // column groups per tile row
    constexpr int kResAhead = 2;
    const long long d_off = (long long)zo * p.d_bs2 + (long long)zi * p.d_bs;
    const long long r_off = (long long)zo * p.r_bs2 + (long long)zi * p.r_bs;
    const int tid = threadIdx.x;
    auto sbias_of = [&](int row, int col) { return p.bias && s_brow[row] < 0 ? s_bias + col : nullptr; };

    if (p.cluster_sk) {
        const int S = p.splits;
        const int GI = (G + S - 1) / S;                      // groups a CTA can own: group g -> CTA g % S
        fence_proxy_async_smem();                            // the ring was written / read through the async proxy
        cluster_sync_all();                                  // #1: every CTA of the cluster has staged its accumulator
        for (int u = tid; u < BM * G; u += kThreads) {
            const int row = u % BM, g = u / BM;              // lanes: consecutive rows, i.e. consecutive 32-byte slots
            if (g * 8 < ncols_tile) {
                const float* src = stage + row * kPitch + g * 8;
                const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
                const uint32_t v[8] = {__float_as_uint(a.x), __float_as_uint(a.y), __float_as_uint(a.z), __float_as_uint(a.w),
                                       __float_as_uint(b.x), __float_as_uint(b.y), __float_as_uint(b.z), __float_as_uint(b.w)};
                st_cluster_f32x8(xbuf + static_cast<uint32_t>(((sp * GI + g / S) * BM + row) * 32), static_cast<uint32_t>(g % S), v);
            }
        }
        cluster_sync_all();                                  // #2: all partial groups have landed in their owners
#pragma unroll 1
        for (int u = tid; u < BM * GI; u += kThreads) {
            const int row = u % BM, gi = u / BM;             // an owner's groups are S apart: no row-contiguous stores
            const int g = gi * S + sp;
            const long long grow = s_grow[row];
            if (g * 8 >= ncols_tile || grow < 0) continue;
            float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
            for (int s2 = 0; s2 < S; ++s2) {
                const uint32_t a = xbuf + static_cast<uint32_t>(((s2 * GI + gi) * BM + row) * 32);
                const float4 lo = ld_shared_f32x4(a), hi = ld_shared_f32x4(a + 16);
                f[0] += lo.x; f[1] += lo.y; f[2] += lo.z; f[3] += lo.w;
                f[4] += hi.x; f[5] += hi.y; f[6] += hi.z; f[7] += hi.w;
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) f[j] *= p.alpha;
            epilogue_group8<kExt>(p, f, grow, s_brow[row], n0 + g * 8, d_off, r_off, min(8, ncols_tile - g * 8), nullptr,
                                  sbias_of(row, g * 8));
        }
        return;
    }

    if constexpr (kExt) {
        if (p.glu) {
            // column group c64 of the tile holds 32 value columns, then their 32 gate columns (N % 64 == 0, no per-image
            // bias: the bias row is always the staged one)
            constexpr int GQ = BN / 16;
#pragma unroll 1
            for (int u = tid; u < BM * GQ; u += kThreads) {
                const int row = u / GQ, q = u % GQ;
                const int vcol = (q >> 2) * 64 + (q & 3) * 8;
                const long long grow = s_grow[row];
                if (vcol >= ncols_tile || grow < 0) continue;
                float fv[8], fg[8];
                stage_ld8(stage + row * kPitch + vcol, p.alpha, fv);
                stage_ld8(stage + row * kPitch + vcol + 32, p.alpha, fg);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    fv[j] += p.bias ? s_bias[vcol + j] : 0.f;
                    fg[j] += p.bias ? s_bias[vcol + 32 + j] : 0.f;
                }
                if (p.D) {
                    store8_any(p.D, p.d_dtype, grow * p.ldd + n0 + vcol, fv);
                    store8_any(p.D, p.d_dtype, grow * p.ldd + n0 + vcol + 32, fg);
                }
                float h[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) h[j] = fv[j] * gelu_f(fg[j]);
                store8_any(p.D2, p.d2_dtype, grow * p.ldd2 + ((n0 + (q >> 2) * 64) >> 1) + (q & 3) * 8, h);
            }
            return;
        }
    }

    // residual fast path (whole aligned units of a row-major D): raw residual of this thread's units k .. k + kResAhead
    const bool r_pre = p.R && p.vec_ok && !p.d_transposed;
    uint4 rq[kResAhead + 1][2];
    auto res_fetch = [&](int k, uint4 (&v)[2]) {
        const int u = tid + k * kThreads;
        if (u >= BM * G) return;
        const int row = u / G, col = (u % G) * 8;
        const long long grow = s_grow[row];
        if (grow >= 0 && col + 8 <= ncols_tile) residual_load8(p, r_off + grow * p.ldr + n0 + col, v);
    };
    if (r_pre) {
#pragma unroll
        for (int k = 0; k < kResAhead; ++k) res_fetch(k, rq[k]);
    }
    const int nunits = (BM * G - tid + kThreads - 1) / kThreads;
#pragma unroll 1
    for (int k = 0; k < nunits; ++k) {
        if (r_pre) res_fetch(k + kResAhead, rq[kResAhead]);
        const int u = tid + k * kThreads;
        const int row = p.d_transposed ? u % BM : u / G;
        const int col = (p.d_transposed ? u / BM : u % G) * 8;
        const long long grow = s_grow[row];
        if (col < ncols_tile && grow >= 0) {
            const int ncols = min(8, ncols_tile - col);
            float f[8], r[8];
            stage_ld8(stage + row * kPitch + col, p.alpha, f);
            if (r_pre && ncols == 8) residual_unpack8(p, rq[0], r);
            epilogue_group8<kExt>(p, f, grow, s_brow[row], n0 + col, d_off, r_off, ncols, r_pre && ncols == 8 ? r : nullptr,
                                  sbias_of(row, col));
        }
        if (dbg && k == 0 && tid == 64) dbg[6] = clock64();
        if (r_pre) {
#pragma unroll
            for (int j = 0; j < kResAhead; ++j) { rq[j][0] = rq[j + 1][0]; rq[j][1] = rq[j + 1][1]; }
        }
    }
}

template <int BN, bool A_MN, bool B_MN, int kStages, bool kExt>
__global__ void __launch_bounds__(kThreads, 1)
cb_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ GemmParams p) {
    using Cfg = TileCfg<BN, kStages>;
    using SCfg = StageCfg<BN>;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;  // SWIZZLE_128B needs 1 KiB alignment
    float* stage = reinterpret_cast<float*>(smem_raw + (smem_base - smem_u32(smem_raw)));
    const uint32_t bar_base = smem_base + kStages * Cfg::kStageBytes;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (kStages + s); };

    __shared__ long long s_grow[BM];           // global output row of each tile row, -1 past the edge of D
    __shared__ int s_brow[BM];                 // bias row of each tile row, -1 for the tile's first (staged) one
    __shared__ __align__(16) float s_bias[BN];
    const int warp = threadIdx.x >> 5;
    // warp-uniform as far as the compiler can tell: with a plain threadIdx-derived index the consumer branch counts as
    // divergent, and ptxas serialises every wgmma.mma_async in it (C7520), waiting for each MMA before issuing the next
    const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);
    if (p.dbg_mode == 3) { pdl_sync(); return; }
    unsigned long long* dbg = p.dbg ? p.dbg + 8ull * ((blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) : nullptr;
    if (dbg && threadIdx.x == 0) { dbg[0] = clock64(); dbg[7] = gtimer(); }
    const int n0 = blockIdx.x * BN;
    const int m_tile = blockIdx.y;
    const int sp = blockIdx.z % p.splits;
    const int bz = blockIdx.z / p.splits;
    const int zi = bz % p.batch_inner;
    const int zo = bz / p.batch_inner;

    // tile origin
    int m0 = 0, ow0 = 0, oh0 = 0, img0 = 0;
    if (p.conv) {
        const int tw = m_tile % p.tiles_w;
        const int th = (m_tile / p.tiles_w) % p.tiles_h;
        const int ti = m_tile / (p.tiles_w * p.tiles_h);
        ow0 = tw * p.box_w;
        oh0 = th * p.box_h;
        img0 = ti * p.box_i;
    } else {
        m0 = m_tile * BM;
    }

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < kStages; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), 8);       // lane 0 of each of the 8 consumer warps releases the stage
        }
        mbar_fence_init();
        fence_proxy_async_smem();
    }
    __syncthreads();
    if (dbg && threadIdx.x == 0) dbg[1] = clock64();
    pdl_sync();   // barrier init / descriptor prefetch above overlap the previous kernel's tail

    const int kiters_all = p.dbg_mode == 1 ? 0 : p.taps * p.kchunks;
    const int it0 = sp * p.kiters_per_split;
    const int it1 = min(kiters_all, it0 + p.kiters_per_split);

    if (wg == 0) {
        if (threadIdx.x == 0) {
            // ===================== TMA producer =====================
            // ring slot, its phase bit and the (tap row r, tap column sx, 64-chunk kc) of the k-iteration are counters
            // stepped once per iteration: no integer division in the loop
            int s = 0;
            uint32_t ph = 0;
            int tap = it0 / p.kchunks;
            int kc = it0 - tap * p.kchunks;
            int r = tap / p.kw;
            int sx = tap - r * p.kw;
            for (int it = it0; it < it1; ++it) {
                mbar_wait(empty_bar(s), ph ^ 1u);
                mbar_arrive_expect_tx(full_bar(s), p.a_bytes + p.b_bytes);
                const uint32_t a_dst = smem_base + s * Cfg::kStageBytes;
                const uint32_t b_dst = a_dst + Cfg::kABytes;
                const int tap_b = p.flip_taps ? (p.taps - 1 - tap) : tap;
                if (p.conv) {
                    tma_load_4d(a_dst, &tmA, full_bar(s), kc * BK, ow0 * p.stride + sx - p.pad_left,
                                oh0 * p.stride + r - p.pad_top, img0);
                } else if (A_MN) {
                    tma_load_4d(a_dst, &tmA, full_bar(s), m0, kc * BK, zi, zo);
                    tma_load_4d(a_dst + 8192, &tmA, full_bar(s), m0 + 64, kc * BK, zi, zo);
                } else {
                    tma_load_4d(a_dst, &tmA, full_bar(s), kc * BK, m0, zi, zo);
                }
                if (B_MN) {
#pragma unroll
                    for (int j = 0; j < BN / 64; ++j)
                        tma_load_4d(b_dst + j * 8192, &tmB, full_bar(s), n0 + j * 64,
                                    tap_b * p.b_tap_rows + kc * BK, zi, zo);
                } else {
                    tma_load_4d(b_dst, &tmB, full_bar(s), kc * BK, tap_b * p.b_tap_rows + n0, zi, zo);
                }
                if (++s == kStages) { s = 0; ph ^= 1u; }
                if (++kc == p.kchunks) {
                    kc = 0;
                    ++tap;
                    if (++sx == p.kw) { sx = 0; ++r; }
                }
            }
        }
        __syncwarp();
        // while the consumers run the k-loop: global row (or -1 past the edge) and bias row of every tile row, and the bias
        // row of the tile's first output row in shared memory.  Conv tiles are [box_i][box_h][box_w] pixel boxes.
        const int r = threadIdx.x;
        long long grow;
        bool row_valid;
        if (p.conv) {
            const int per_img = p.box_h * p.box_w;
            const int bi = r / per_img;
            const int rem = r - bi * per_img;
            const int bh = rem / p.box_w;
            const int bw = rem - bh * p.box_w;
            const int img = img0 + bi, oh = oh0 + bh, ow = ow0 + bw;
            row_valid = (bi < p.box_i) && (img < p.img_n) && (oh < p.out_h) && (ow < p.out_w);
            grow = ((long long)img * p.out_h + oh) * p.out_w + ow;
        } else {
            grow = m0 + r;
            row_valid = grow < p.M;
        }
        s_grow[r] = row_valid ? grow : -1;
        if (p.bias) {
            const long long tile_row0 = p.conv ? (((long long)img0 * p.out_h + oh0) * p.out_w + ow0) : (long long)m0;
            const long long brow0 = p.bias_row_div > 0 ? tile_row0 / p.bias_row_div : 0;
            const long long brow = p.bias_row_div > 0 ? grow / p.bias_row_div : 0;
            s_brow[r] = brow == brow0 ? -1 : static_cast<int>(brow);
            const int ncols = min(BN, p.N - n0);
            for (int i = r; i < BN; i += 128) s_bias[i] = i < ncols ? p.bias[brow0 * p.ldbias + n0 + i] : 0.f;
        }
    } else {
        // ===================== wgmma consumers =====================
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        const uint32_t a_half = static_cast<uint32_t>(wg - 1) * 8192u;     // this warpgroup's 64 rows of the A tile
        // wgmma.wait_group is warp-collective, so once it returns one lane's arrival releases the stage for its warp
        const bool releaser = (threadIdx.x & 31) == 0;
        int s = 0, s_prev = 0;
        uint32_t ph = 0;
        int kc = it0 % p.kchunks;
        for (int it = it0; it < it1; ++it) {
            mbar_wait(full_bar(s), ph);
            if (dbg && it == it0 && threadIdx.x == 128) dbg[2] = clock64();
            const uint32_t a_src = smem_base + s * Cfg::kStageBytes + a_half;
            const uint32_t b_src = smem_base + s * Cfg::kStageBytes + Cfg::kABytes;
            const int ksteps = (kc == p.kchunks - 1) ? p.ksteps_last : (BK / 16);
            wgmma_fence_regs(acc);
            if (p.bf16) mma_kiter<BN, A_MN, B_MN, true>(acc, a_src, b_src, ksteps);
            else mma_kiter<BN, A_MN, B_MN, false>(acc, a_src, b_src, ksteps);
            // keep one k-iteration of MMAs in flight: the previous stage is released once its group has retired
            wgmma_wait<1>();
            wgmma_fence_regs(acc);
            if (it > it0 && releaser) mbar_arrive(empty_bar(s_prev));
            s_prev = s;
            if (++s == kStages) { s = 0; ph ^= 1u; }
            if (++kc == p.kchunks) kc = 0;
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        if (it1 > it0 && releaser) mbar_arrive(empty_bar(s_prev));
        if (dbg && threadIdx.x == 128) dbg[3] = clock64();
        named_bar(4, 256);          // both warpgroups' MMAs have read the ring for the last time
        const int l = threadIdx.x & 31, w = warp & 3;
        float* srow = stage + ((wg - 1) * 64 + w * 16 + (l >> 2)) * SCfg::kPitch + 2 * (l & 3);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            *reinterpret_cast<float2*>(srow + 8 * j) = make_float2(acc[4 * j], acc[4 * j + 1]);
            *reinterpret_cast<float2*>(srow + 8 * SCfg::kPitch + 8 * j) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
    }
    named_bar(2, kThreads);        // accumulator tile, row metadata and bias row staged
    const int ncols_tile = min(BN, p.N - n0);
    if (p.splits > 1 && !p.cluster_sk && p.dbg_mode == 0) {
        const unsigned tile_id = (static_cast<unsigned>(bz) * gridDim.y + m_tile) * gridDim.x + blockIdx.x;
        if (!splitk_reduce_to_stage<BN>(p, tile_id, sp, stage, ncols_tile)) return;
    }
    if (p.dbg_mode == 1 || p.dbg_mode == 2) return;
    if (dbg && threadIdx.x == 64) dbg[4] = clock64();
    epilogue_units<BN, kExt>(p, stage, s_grow, s_brow, s_bias, n0, ncols_tile, zo, zi, sp, smem_base + SCfg::kBytes, dbg);
    if (dbg && threadIdx.x == 64) dbg[5] = clock64();
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess) {
            fn = reinterpret_cast<EncodeTiledFn>(p);
        }
    }
    return fn;
}

int make_tmap(CUtensorMap* out, int dtype, int rank, const void* ptr, const uint64_t* dims,
              const uint64_t* strides_bytes /* rank-1 */, const uint32_t* box, const uint32_t* estr) {
    EncodeTiledFn fn = get_encode_fn();
    CB_REQUIRE(fn != nullptr, CB_ERR_DRIVER, "cuTensorMapEncodeTiled entry point unavailable");
    CB_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15u) == 0, CB_ERR_ALIGN, "tensor base %p not 16B aligned", ptr);
    for (int i = 0; i < rank - 1; ++i)
        CB_REQUIRE((strides_bytes[i] & 15u) == 0, CB_ERR_ALIGN, "tensor stride[%d]=%llu bytes not multiple of 16", i,
                   (unsigned long long)strides_bytes[i]);
    CUtensorMapDataType dt = dtype == CB_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    CUresult rc = fn(out, dt, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides_bytes, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CB_REQUIRE(rc == CUDA_SUCCESS, CB_ERR_DRIVER,
               "cuTensorMapEncodeTiled failed rc=%d rank=%d dims=[%llu,%llu,%llu,%llu] box=[%u,%u,%u,%u]", (int)rc,
               rank, (unsigned long long)dims[0], (unsigned long long)dims[1],
               (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0), box[0],
               box[1], rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
    return 0;
}

static inline bool needs_ext(const GemmParams& p) { return p.D2 != nullptr || p.act == CB_ACT_PRELU || p.glu; }

template <int BN, bool A_MN, bool B_MN, int kStages, bool kExt>
static int launch_se(const CUtensorMap& tA, const CUtensorMap& tB, const GemmParams& p, dim3 grid, cudaStream_t st) {
    using Cfg = TileCfg<BN, kStages>;
    static bool attr_done = false;
    auto kern = cb_gemm_kernel<BN, A_MN, B_MN, kStages, kExt>;
    if (!attr_done) {
        CB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
        attr_done = true;
    }
    if (p.cluster_sk) {
        // the k-slices of a tile are one cluster (1,1,splits); the exchange buffer lives in the idle TMA ring behind the
        // staged accumulator tile (cluster_sk_fits)
        const int S = p.splits;
        CB_REQUIRE(S >= 2 && S <= 16 && grid.z % S == 0, CB_ERR_ARG, "cb_gemm(cluster split-K): %d slices not in [2,16]", S);
        static bool np_done = false;
        if (S > 8 && !np_done) {
            CB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
            np_done = true;
        }
        CB_CUDA(launch_kernel_cluster(kern, grid, dim3(kThreads), dim3(1, 1, (unsigned)S), (size_t)Cfg::kSmemBytes, st, tA, tB, p));
        CB_CUDA(cudaGetLastError());
        count_launches(1);
        return 0;
    }
CB_LAUNCH((kern), grid, kThreads, Cfg::kSmemBytes, st, tA, tB, p);
    CB_CUDA(cudaGetLastError());
    count_launches(1);
    return 0;
}

template <int BN, bool A_MN, bool B_MN, int kStages>
static int launch_s(const CUtensorMap& tA, const CUtensorMap& tB, const GemmParams& p, dim3 grid, cudaStream_t st) {
    return needs_ext(p) ? launch_se<BN, A_MN, B_MN, kStages, true>(tA, tB, p, grid, st)
                        : launch_se<BN, A_MN, B_MN, kStages, false>(tA, tB, p, grid, st);
}

// ring depth the launch below picks for this tile width / grid
static int ring_stages(int bn, const GemmParams& p, long long ctas) {
    if (bn == 256) return 4;
    static const int env_force = getenv("CB_GEMM_STAGES") ? atoi(getenv("CB_GEMM_STAGES")) : 0;   // tuning aid
    const int force = p.force_stages ? p.force_stages : env_force;
    if (force == 3) return 3;
    if (force == 6 || ctas <= device_sm_count()) return 6;
    return 3;
}
// cluster split-K exchanges partial tiles through the part of the TMA ring behind the staged accumulator tile
static bool cluster_sk_fits(int bn, int splits, int stages) {
    const long long stage_bytes = ((long long)BM * (bn + 4) * 4 + 1023) / 1024 * 1024;
    const long long ring = (long long)stages * (BM * BK * 2 + bn * BK * 2);
    const long long gi = (bn / 8 + splits - 1) / splits;
    return stage_bytes + (long long)splits * gi * BM * 32 <= ring;
}

template <int BN, bool A_MN, bool B_MN>
static int launch(const CUtensorMap& tA, const CUtensorMap& tB, const GemmParams& p, dim3 grid, cudaStream_t st) {
    if constexpr (BN == 256) {
        return launch_s<BN, A_MN, B_MN, 4>(tA, tB, p, grid, st);   // 48 KiB stages: 4-deep ring, one CTA per SM
    } else {
        const long long ctas = (long long)grid.x * grid.y * grid.z;
        if (ring_stages(BN, p, ctas) == 6) return launch_s<BN, A_MN, B_MN, 6>(tA, tB, p, grid, st);
        return launch_s<BN, A_MN, B_MN, 3>(tA, tB, p, grid, st);
    }
}

// Cost model of one launch: a k-iteration of a 128 x BN tile is taken to be bound by the operand bytes one SM pulls out
// of L2 (~(128+BN)*128 B at ~80 GB/s per SM), a split-K reduction to cost ~1 ns per 150 fp32 adds in L2 plus ~3 us of
// hand-off.  The constants are estimates, not measurements; the tile width and the split minimise the estimate for the
// launch at hand, and the host autotuner (ops.py) times the real candidates.
static double tile_time_us(int bn, long long tiles, int kiters, int sms) {
    const double t_iter = (128.0 + bn) * 128.0 / 80e3;          // us per k-iteration per CTA
    const long long waves = (tiles + sms - 1) / sms;
    return (double)waves * kiters * t_iter;
}

// requested = false: the library's own choice, ignoring desc.tile_n and CB_GEMM_BN
static int pick_bn(const cb_gemm_desc& d, int m_tiles, int kiters, bool requested = true) {
    const int N = d.N;
    const int sms = device_sm_count();
    int cands[3];
    int nc = 0;
    if (d.b_major == CB_MAJOR_MN) {
        if (N <= 64) return 64;
        cands[nc++] = 128;
        cands[nc++] = 64;
    } else {
        if (N <= 64) return 64;
        cands[nc++] = 160;
        cands[nc++] = 128;
        cands[nc++] = 64;
    }
    static const int env_bn = getenv("CB_GEMM_BN") ? atoi(getenv("CB_GEMM_BN")) : 0;   // tuning aid
    const int force_bn = !requested ? 0 : (d.tile_n > 0 ? d.tile_n : env_bn);
    // 128x256 tile: only on request (per-shape autotuner / caller), and only with K-major A -- there is no MN-major-A
    // instantiation of that width, so such a request falls through to the model below
    if (force_bn == 256 && N >= 256 && d.a_major != CB_MAJOR_MN) return 256;
    for (int i = 0; i < nc; ++i)
        if (cands[i] == force_bn) return force_bn;
    int best = cands[0];
    double best_t = 1e30;
    for (int i = 0; i < nc; ++i) {
        const int bn = cands[i];
        const long long tiles = (long long)ceil_div(N, bn) * m_tiles * d.batch;
        double t = tile_time_us(bn, tiles, kiters, sms) + 0.02 * ceil_div(N, bn);   // tie-break: fewer, wider tiles
        if (t < best_t) { best_t = t; best = bn; }
    }
    return best;
}

}  // namespace cb

using namespace cb;

extern "C" int cb_gemm(const cb_gemm_desc* dp, void* stream) {
    CB_REQUIRE(dp != nullptr, CB_ERR_ARG, "cb_gemm: null desc");
    const cb_gemm_desc& d = *dp;
    CB_REQUIRE(d.ab_dtype == CB_F16 || d.ab_dtype == CB_BF16, CB_ERR_ARG, "cb_gemm: ab_dtype must be f16/bf16");
    CB_REQUIRE(d.A && d.B && (d.D || (d.glu && d.D2)), CB_ERR_ARG, "cb_gemm: null A/B/D");
    if (d.glu) {
        CB_REQUIRE(d.D2 && d.N % 64 == 0 && d.batch == 1 && !d.d_transposed && !d.R && d.act == CB_ACT_NONE &&
                       d.bias_row_div == 0,
                   CB_ERR_ARG, "cb_gemm(glu): needs D2, N %% 64 == 0, batch 1, no residual / activation / per-image bias");
    }
    CB_REQUIRE(d.N > 0 && d.K > 0 && d.batch > 0, CB_ERR_ARG, "cb_gemm: bad N/K/batch");
    CB_REQUIRE(d.d_dtype >= CB_F16 && d.d_dtype <= CB_F32, CB_ERR_ARG, "cb_gemm: bad d_dtype");
    const int es = 2;
    const bool a_mn = d.a_major == CB_MAJOR_MN, b_mn = d.b_major == CB_MAJOR_MN;
    CB_REQUIRE(!(d.conv && a_mn), CB_ERR_ARG, "cb_gemm: conv mode needs K-major A (NHWC)");
    CB_REQUIRE(!(a_mn && !b_mn), CB_ERR_ARG, "cb_gemm: (A MN-major, B K-major) is not instantiated");

    const int b_in = d.batch_inner > 0 ? d.batch_inner : d.batch;
    CB_REQUIRE(d.batch % b_in == 0, CB_ERR_ARG, "cb_gemm: batch %d not a multiple of batch_inner %d", d.batch, b_in);
    const int b_out = d.batch / b_in;
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.batch_inner = b_in;
    p.N = d.N;
    p.K = d.K;
    p.kchunks = ceil_div(d.K, BK);
    p.ksteps_last = ceil_div(d.K - (p.kchunks - 1) * BK, 16);
    p.conv = d.conv;
    p.taps = 1;
    p.kw = 1;
    p.b_tap_rows = d.b_tap_rows;
    p.flip_taps = d.flip_taps;

    CUtensorMap tA, tB;
    int m_tiles;
    if (d.conv) {
        CB_REQUIRE(d.img_n > 0 && d.img_h > 0 && d.img_w > 0 && d.out_h > 0 && d.out_w > 0 && d.kh > 0 && d.kw > 0,
                   CB_ERR_ARG, "cb_gemm(conv): bad geometry");
        CB_REQUIRE(d.stride == 1 || d.stride == 2, CB_ERR_ARG, "cb_gemm(conv): stride must be 1 or 2");
        CB_REQUIRE(d.batch == 1, CB_ERR_ARG, "cb_gemm(conv): batch must be 1 (images are rows)");
        p.taps = d.kh * d.kw;
        p.kw = d.kw;
        p.M = d.img_n * d.out_h * d.out_w;
        p.out_h = d.out_h;
        p.out_w = d.out_w;
        p.img_n = d.img_n;
        p.stride = d.stride;
        p.pad_top = d.pad_top;
        p.pad_left = d.pad_left;
        // pixel box: <=128 output pixels as [box_i][box_h][box_w]
        int bw = d.out_w < BM ? d.out_w : BM;
        int bh = BM / bw;
        if (bh > d.out_h) bh = d.out_h;
        int bi = BM / (bw * bh);
        if (bi > d.img_n) bi = d.img_n;
        if (bi < 1) bi = 1;
        p.box_w = bw;
        p.box_h = bh;
        p.box_i = bi;
        p.tiles_w = ceil_div(d.out_w, bw);
        p.tiles_h = ceil_div(d.out_h, bh);
        m_tiles = p.tiles_w * p.tiles_h * ceil_div(d.img_n, bi);
        p.a_bytes = (unsigned)(bw * bh * bi) * BK * es;
        const uint64_t C = (uint64_t)d.K;
        const uint64_t rowstride = (uint64_t)d.lda;  // elements between consecutive pixels (>= K)
        uint64_t dims[4] = {C, (uint64_t)d.img_w, (uint64_t)d.img_h, (uint64_t)d.img_n};
        uint64_t strides[3] = {rowstride * es, rowstride * es * d.img_w, rowstride * es * d.img_w * d.img_h};
        uint32_t box[4] = {BK, (uint32_t)(bw * d.stride), (uint32_t)(bh * d.stride), (uint32_t)bi};
        uint32_t estr[4] = {1, (uint32_t)d.stride, (uint32_t)d.stride, 1};
        CB_REQUIRE(box[1] <= 256 && box[2] <= 256, CB_ERR_ARG, "cb_gemm(conv): box too large");
        int rc = make_tmap(&tA, d.ab_dtype, 4, d.A, dims, strides, box, estr);
        if (rc) return rc;
    } else {
        CB_REQUIRE(d.M > 0, CB_ERR_ARG, "cb_gemm: bad M");
        p.M = d.M;
        m_tiles = ceil_div(d.M, BM);
        p.a_bytes = BM * BK * es;
        const uint64_t dflt = (uint64_t)(a_mn ? d.lda * (int64_t)d.K : d.lda * (int64_t)d.M);
        const uint64_t bs = (uint64_t)(b_in > 1 ? d.a_batch_stride : dflt);
        const uint64_t bs2 = (uint64_t)(b_out > 1 ? d.a_batch_stride2 : dflt);
        if (a_mn) {
            uint64_t dims[4] = {(uint64_t)d.M, (uint64_t)d.K, (uint64_t)b_in, (uint64_t)b_out};
            uint64_t strides[3] = {(uint64_t)d.lda * es, bs * es, bs2 * es};
            uint32_t box[4] = {64, BK, 1, 1};
            uint32_t estr[4] = {1, 1, 1, 1};
            int rc = make_tmap(&tA, d.ab_dtype, 4, d.A, dims, strides, box, estr);
            if (rc) return rc;
        } else {
            uint64_t dims[4] = {(uint64_t)d.K, (uint64_t)d.M, (uint64_t)b_in, (uint64_t)b_out};
            uint64_t strides[3] = {(uint64_t)d.lda * es, bs * es, bs2 * es};
            uint32_t box[4] = {BK, BM, 1, 1};
            uint32_t estr[4] = {1, 1, 1, 1};
            int rc = make_tmap(&tA, d.ab_dtype, 4, d.A, dims, strides, box, estr);
            if (rc) return rc;
        }
    }

    // desc.cta_pair asks for large-M tiles of desc.tile_n; every tile is one CTA (sm_90 has no two-CTA MMA)
    int BN = pick_bn(d, m_tiles, p.taps * p.kchunks);
    if (d.glu && BN % 64 != 0) BN = 128;        // (value, gate) column pairs live in 64-column groups
    const int b_box_rows = BN;
    p.b_bytes = (unsigned)b_box_rows * BK * es;
    {
        const uint64_t brows_total = (uint64_t)(d.conv ? (int64_t)p.taps * d.b_tap_rows : (b_mn ? d.K : d.N));
        const uint64_t dflt = (uint64_t)(d.ldb * (int64_t)brows_total);
        const uint64_t bs = (uint64_t)(b_in > 1 ? d.b_batch_stride : dflt);
        const uint64_t bs2 = (uint64_t)(b_out > 1 ? d.b_batch_stride2 : dflt);
        uint32_t estr[4] = {1, 1, 1, 1};
        if (b_mn) {
            uint64_t dims[4] = {(uint64_t)d.N, brows_total, (uint64_t)b_in, (uint64_t)b_out};
            uint64_t strides[3] = {(uint64_t)d.ldb * es, bs * es, bs2 * es};
            uint32_t box[4] = {64, BK, 1, 1};
            int rc = make_tmap(&tB, d.ab_dtype, 4, d.B, dims, strides, box, estr);
            if (rc) return rc;
        } else {
            uint64_t dims[4] = {(uint64_t)d.K, brows_total, (uint64_t)b_in, (uint64_t)b_out};
            uint64_t strides[3] = {(uint64_t)d.ldb * es, bs * es, bs2 * es};
            uint32_t box[4] = {BK, (uint32_t)b_box_rows, 1, 1};
            int rc = make_tmap(&tB, d.ab_dtype, 4, d.B, dims, strides, box, estr);
            if (rc) return rc;
        }
    }

    p.D = d.D;
    p.d_dtype = d.d_dtype;
    p.ldd = d.ldd;
    p.d_bs = d.d_batch_stride;
    p.d_bs2 = d.d_batch_stride2;
    p.d_transposed = d.d_transposed;
    p.D2 = d.D2;
    p.d2_dtype = d.d2_dtype;
    p.ldd2 = d.ldd2;
    if (d.D2) {
        CB_REQUIRE(d.batch == 1 && !d.d_transposed, CB_ERR_ARG, "cb_gemm: D2 needs batch == 1 and a non-transposed D");
        CB_REQUIRE(d.d2_dtype >= CB_F16 && d.d2_dtype <= CB_F32, CB_ERR_ARG, "cb_gemm: bad d2_dtype");
        const int es2 = d.d2_dtype == CB_F32 ? 4 : 2;
        CB_REQUIRE((reinterpret_cast<uintptr_t>(d.D2) & 15u) == 0 && (d.ldd2 * es2) % 16 == 0 &&
                       d.ldd2 >= (d.glu ? d.N / 2 : d.N),
                   CB_ERR_ALIGN, "cb_gemm: D2 must be 16-byte aligned with a 16-byte multiple row pitch >= N (N/2 with glu)");
    }
    p.glu = d.glu;
    p.act_param = d.act_param;
    p.d2_scale = d.d2_scale;
    p.d2_shift = d.d2_shift;
    CB_REQUIRE(d.act != CB_ACT_PRELU || d.act_param != nullptr, CB_ERR_ARG, "cb_gemm: CB_ACT_PRELU needs act_param (slopes)");
    CB_REQUIRE((d.d2_scale == nullptr) == (d.d2_shift == nullptr), CB_ERR_ARG, "cb_gemm: d2_scale and d2_shift go together");
    p.bias = d.bias;
    p.bias_row_div = d.bias_row_div;
    p.ldbias = d.ldbias;
    p.R = d.R;
    p.r_dtype = d.r_dtype;
    p.ldr = d.ldr;
    p.r_bs = d.r_batch_stride;
    p.r_bs2 = d.r_batch_stride2;
    p.alpha = d.alpha;
    p.act = d.act;
    p.dbg = reinterpret_cast<unsigned long long*>(d.debug_timeline);
    {
        static const int mode = getenv("CB_GEMM_DBG_MODE") ? atoi(getenv("CB_GEMM_DBG_MODE")) : 0;
        p.dbg_mode = mode;
    }
    p.bf16 = d.ab_dtype == CB_BF16 ? 1 : 0;
    {
        const int des = d.d_dtype == CB_F32 ? 4 : 2;
        bool ok = ((reinterpret_cast<uintptr_t>(d.D) & 15u) == 0) && ((d.ldd * des) % 16 == 0) &&
                  ((d.d_batch_stride * des) % 16 == 0) && ((d.d_batch_stride2 * des) % 16 == 0);
        if (d.R) {
            const int res = d.r_dtype == CB_F32 ? 4 : 2;
            ok = ok && ((reinterpret_cast<uintptr_t>(d.R) & 15u) == 0) && ((d.ldr * res) % 16 == 0) &&
                 ((d.r_batch_stride * res) % 16 == 0) && ((d.r_batch_stride2 * res) % 16 == 0);
        }
        if (d.bias) ok = ok && ((reinterpret_cast<uintptr_t>(d.bias) & 15u) == 0) && ((d.ldbias * 4) % 16 == 0);
        p.vec_ok = ok ? 1 : 0;
    }

    // ---- split-K heuristic: fill the SMs when the tile grid alone cannot (bs=1 low-resolution layers) ----
    p.force_stages = (d.stages == 3 || d.stages == 6) ? d.stages : 0;
    p.splits = 1;
    p.kiters_per_split = p.taps * p.kchunks;
    {
        const int kiters = p.taps * p.kchunks;
        const int sms = device_sm_count();
        // The split is a function of the shape (or an explicit desc.splits) alone, never of the tile width a caller or the
        // autotuner asks for: every configuration of a shape then adds its k-slices in the same order and the results are
        // bit-identical whichever configuration wins the timing.
        const int bn_s = pick_bn(d, m_tiles, kiters, false);
        const long long tiles_s = (long long)ceil_div(d.N, bn_s) * m_tiles * d.batch;
        const long long counters_bytes = 65536;
        const long long avail = d.splitk_ws_bytes - counters_bytes;
        // workspace bounds valid for every tile width: tiles <= ceil(N / 64) * ..., tiles * BN <= (N + 255) * ...
        const long long tiles_max = (long long)ceil_div(d.N, 64) * m_tiles * d.batch;
        const long long slice_bytes = (long long)(d.N + 255) * m_tiles * d.batch * BM * 4;
        if (d.splitk_ws != nullptr && !d.glu && tiles_max <= counters_bytes / 4 &&
            (d.splits > 0 || (tiles_s < sms && kiters >= 8))) {
            const double out_elems = (double)p.M * d.batch * d.N;
            double best_t = tile_time_us(bn_s, tiles_s, kiters, sms);
            int best_sp = 1;
            if (d.splits > 0) {
                best_sp = d.splits < kiters ? d.splits : kiters;       // caller-tuned
            } else {
                const int max_sp = (int)(sms / tiles_s) < 64 ? (int)(sms / tiles_s) : 64;
                for (int sp = 2; sp <= max_sp; ++sp) {
                    const int per = ceil_div(kiters, sp);
                    if (per < 4) break;
                    const double t = per * ((128.0 + bn_s) * 128.0 / 80e3) + out_elems * sp / 150e3 + 3.0;
                    if (t < best_t) { best_t = t; best_sp = sp; }
                }
            }
            if (best_sp > 1) {
                const int per = ceil_div(kiters, best_sp);
                const int splits = ceil_div(kiters, per);
                if (slice_bytes * splits <= avail) {                       // one partial-tile slice per k-slice
                    p.splits = splits;
                    p.kiters_per_split = per;
                    p.counters = reinterpret_cast<unsigned*>(d.splitk_ws);
                    p.ws = reinterpret_cast<float*>(reinterpret_cast<char*>(d.splitk_ws) + counters_bytes);
                }
            }
        }
    }
    // split-K through distributed shared memory instead of the global workspace (desc.splitk_cluster, host autotuner), where
    // the exchange buffer fits the ring the launch runs with
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    dim3 grid((unsigned)ceil_div(d.N, BN), (unsigned)m_tiles, (unsigned)(d.batch * p.splits));
    p.cluster_sk = (d.splitk_cluster == 1 && p.splits >= 2 && p.splits <= 16 && p.dbg_mode == 0 &&
                    cluster_sk_fits(BN, p.splits, ring_stages(BN, p, (long long)grid.x * grid.y * grid.z))) ? 1 : 0;
    if (!a_mn && !b_mn) {
        if (BN == 64) return launch<64, false, false>(tA, tB, p, grid, st);
        if (BN == 128) return launch<128, false, false>(tA, tB, p, grid, st);
        if (BN == 256) return launch<256, false, false>(tA, tB, p, grid, st);
        return launch<160, false, false>(tA, tB, p, grid, st);
    } else if (!a_mn && b_mn) {
        if (BN == 64) return launch<64, false, true>(tA, tB, p, grid, st);
        if (BN == 256) return launch<256, false, true>(tA, tB, p, grid, st);
        return launch<128, false, true>(tA, tB, p, grid, st);
    } else {
        if (BN == 64) return launch<64, true, true>(tA, tB, p, grid, st);
        return launch<128, true, true>(tA, tB, p, grid, st);
    }
}
