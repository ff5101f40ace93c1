// cb_gemm — wgmma GEMM / implicit-GEMM convolution for sm_90a.
//
// One CTA computes one 128 x BN output tile:
//   thread 0         : TMA producer (cp.async.bulk.tensor, SWIZZLE_128B boxes, mbarrier complete_tx)
//   warpgroups 1, 2  : wgmma.mma_async on 64 rows each, fp32 accumulators in registers
//   warpgroup 0      : epilogue (staged accumulator rows -> alpha/bias/act/residual -> HBM)
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
    int vec32_ok;     // D (and R) rows are 32-byte aligned: one 32-byte sector per lane and chunk in the epilogue
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
    int ws_tr;                // accumulator-tile layout in ws: 1 = float4-group-major (coalesced warp requests), 0 = row-major
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

// Epilogue for 8 consecutive columns of one output row (one thread).  Kept deliberately small: the epilogue runs once
// per CTA, so its cost is dominated by cold instruction fetch (~300 cycles per 128 B line of straight-line code).
// Residual values of one 32-column chunk of this thread's row, fetched as raw 16-byte words BEFORE the accumulator is
// needed (the loads are in flight while the MMAs / the previous chunk's stores run; D may alias R, so the compiler could
// never hoist them itself).
struct ResidualChunk { uint4 v[8]; };
// one 32-byte sector as two 16-byte accesses (sm_90 has no 256-bit global load / store)
__device__ __forceinline__ void ldg256(const void* ptr, uint4& a, uint4& b) {
    a = reinterpret_cast<const uint4*>(ptr)[0];
    b = reinterpret_cast<const uint4*>(ptr)[1];
}
__device__ __forceinline__ void stg256(void* ptr, const uint4& a, const uint4& b) {
    reinterpret_cast<uint4*>(ptr)[0] = a;
    reinterpret_cast<uint4*>(ptr)[1] = b;
}
__device__ __forceinline__ void residual_prefetch(const GemmParams& p, long long ridx, ResidualChunk& rc) {
    if (p.r_dtype == CB_F32) {
        const float* s = reinterpret_cast<const float*>(p.R) + ridx;
        if (p.vec32_ok) {
#pragma unroll
            for (int j = 0; j < 4; ++j) ldg256(s + 8 * j, rc.v[2 * j], rc.v[2 * j + 1]);
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) rc.v[j] = reinterpret_cast<const uint4*>(s)[j];
        }
    } else {
        const __half* s = reinterpret_cast<const __half*>(p.R) + ridx;
        if (p.vec32_ok) {
#pragma unroll
            for (int j = 0; j < 2; ++j) ldg256(s + 16 * j, rc.v[2 * j], rc.v[2 * j + 1]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) rc.v[j] = reinterpret_cast<const uint4*>(s)[j];
        }
    }
}
__device__ __forceinline__ void residual_unpack8(const GemmParams& p, const ResidualChunk& rc, int g, float (&r)[8]) {
    if (p.r_dtype == CB_F32) {
        const uint4 a = rc.v[2 * g], b = rc.v[2 * g + 1];
        r[0] = __uint_as_float(a.x); r[1] = __uint_as_float(a.y); r[2] = __uint_as_float(a.z); r[3] = __uint_as_float(a.w);
        r[4] = __uint_as_float(b.x); r[5] = __uint_as_float(b.y); r[6] = __uint_as_float(b.z); r[7] = __uint_as_float(b.w);
    } else {
        const uint4 a = rc.v[g];
        const uint32_t w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float2 t;
            if (p.r_dtype == CB_F16) t = __half22float2(*reinterpret_cast<const __half2*>(&w[j]));
            else t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[j]));
            r[2 * j] = t.x; r[2 * j + 1] = t.y;
        }
    }
}

// kExt: the instantiation that carries the rarely used epilogue features (second destination, PReLU slopes, D2 affine).
// They are compiled OUT of the common instantiation: the epilogue runs once per CTA and its cost is cold instruction
// fetch, so every extra line of straight-line code is paid by all 700+ GEMM launches of the step.
template <bool kExt>
__device__ __forceinline__ void epilogue_group8(const GemmParams& p, float (&f)[8], long long grow, long long brow, int col,
                                             long long d_off, long long r_off, int ncols, const float* rpre = nullptr,
                                             const float* sbias = nullptr) {
    if (sbias) {       // this tile's bias row, staged in shared memory before the accumulator was ready
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] += sbias[j];
    } else if (p.bias) {
        if (ncols == 8) {
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

// GEGLU (attention.py:37-45) inside the FF-in projection's epilogue.  The weight rows are interleaved at load time so that
// every 64-column group of the GEMM output holds 32 value columns followed by their 32 gate columns; this thread's row of
// such a group arrives as two accumulator chunks.  D (optional) keeps the pre-activations for the backward pass, D2
// receives value * gelu(gate) at column (group * 32).
__device__ __forceinline__ void epilogue_glu64(const GemmParams& p, float (&fv)[32], float (&fg)[32], long long grow, int col,
                                               const float* sbias) {
    uint4 pk[4];
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        float(&f)[32] = half ? fg : fv;
#pragma unroll
        for (int g = 0; g < 4; ++g) {
            float b[8];
            if (sbias) {
#pragma unroll
                for (int j = 0; j < 8; ++j) b[j] = sbias[half * 32 + g * 8 + j];
            } else if (p.bias) {
                load8<float>(p.bias + col + half * 32 + g * 8, b);
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) b[j] = 0.f;
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) f[g * 8 + j] += b[j];
            if (p.D) {
                float t[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) t[j] = f[g * 8 + j];
                store8_any(p.D, p.d_dtype, grow * p.ldd + col + half * 32 + g * 8, t);
            }
        }
    }
#pragma unroll
    for (int g = 0; g < 4; ++g) {
        float u[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) u[j] = fv[g * 8 + j] * gelu_f(fg[g * 8 + j]);
        store8_any(p.D2, p.d2_dtype, grow * p.ldd2 + (col >> 1) + g * 8, u);
    }
    (void)pk;
}

// Full 32-column chunk of one output row on the aligned fast path: bias / activation / residual on registers, then
// 256-bit stores (one full 32-byte sector per lane and instruction) when the rows are 32-byte aligned.
template <bool kExt>
__device__ __forceinline__ void epilogue_chunk32(const GemmParams& p, const float (&fin)[32], long long grow, long long brow,
                                                 int col, long long d_off, long long r_off, const ResidualChunk* rc,
                                                 const float* sbias) {
    const long long didx = d_off + grow * p.ldd + col;
    uint4 pk[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
        float f[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] = fin[g * 8 + j];
        if (sbias) {
#pragma unroll
            for (int j = 0; j < 8; ++j) f[j] += sbias[g * 8 + j];
        } else if (p.bias) {
            float b[8];
            load8<float>(p.bias + brow * p.ldbias + col + g * 8, b);
#pragma unroll
            for (int j = 0; j < 8; ++j) f[j] += b[j];
        }
        if (p.act != CB_ACT_NONE) {
            if constexpr (kExt) {
                apply_act8(f, p.act, p.act_param, col + g * 8);
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) f[j] = apply_act(f[j], p.act);
            }
        }
        if (rc) {
            float r[8];
            residual_unpack8(p, *rc, g, r);
#pragma unroll
            for (int j = 0; j < 8; ++j) f[j] += r[j];
        } else if (p.R) {
            float r[8];
            const long long ridx = r_off + grow * p.ldr + col + g * 8;
            if (p.r_dtype == CB_F32) load8<float>(reinterpret_cast<const float*>(p.R) + ridx, r);
            else if (p.r_dtype == CB_F16) load8<__half>(reinterpret_cast<const __half*>(p.R) + ridx, r);
            else load8<__nv_bfloat16>(reinterpret_cast<const __nv_bfloat16*>(p.R) + ridx, r);
#pragma unroll
            for (int j = 0; j < 8; ++j) f[j] += r[j];
        }
        if constexpr (kExt) {
            if (p.D2) {
                float g2[8];
                d2_affine8(g2, f, p.d2_scale, p.d2_shift, col + g * 8);
                store8_any(p.D2, p.d2_dtype, grow * p.ldd2 + col + g * 8, g2);
            }
        }
        if (p.d_dtype == CB_F32) {
            float* dst = reinterpret_cast<float*>(p.D) + didx + g * 8;
            const uint4 a = make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3]));
            const uint4 b = make_uint4(__float_as_uint(f[4]), __float_as_uint(f[5]), __float_as_uint(f[6]), __float_as_uint(f[7]));
            if (p.vec32_ok) stg256(dst, a, b);
            else { reinterpret_cast<uint4*>(dst)[0] = a; reinterpret_cast<uint4*>(dst)[1] = b; }
        } else {
            if (p.d_dtype == CB_F16) {
                __half2* h = reinterpret_cast<__half2*>(&pk[g]);
#pragma unroll
                for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
            } else {
                __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&pk[g]);
#pragma unroll
                for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
            }
            if (g & 1) {
                uint16_t* dst = reinterpret_cast<uint16_t*>(p.D) + didx + (g - 1) * 8;
                if (p.vec32_ok) stg256(dst, pk[g - 1], pk[g]);
                else { reinterpret_cast<uint4*>(dst)[0] = pk[g - 1]; reinterpret_cast<uint4*>(dst)[1] = pk[g]; }
            }
        }
    }
}

// ---- split-K hand-off (epilogue warpgroup, 128 threads): every CTA stores its fp32 partial tile into its own slice of
//      the tile's workspace (slice = k-slice index); the last CTA to arrive (per-tile counter) adds the slices up in slice
//      order -- the same order as the cluster exchange, so the result does not depend on which CTA finishes last --, runs
//      the epilogue and re-zeroes the counter for the next launch.
//      slice layout (p.ws_tr): float4 group g (= 4 columns) of row r lives at ((g * BM) + r) * 4 floats, so the 32 lanes of
//      a warp (32 consecutive rows) touch 512 contiguous bytes per store / load -- four full 128-byte lines instead of 32
//      half-sectors of 32 different lines; ws_tr = 0 keeps the row-major tile (row pitch BN floats).
__device__ __forceinline__ void stage_ld32(const float* row, int c, uint32_t (&acc)[32]);
template <int BN, bool kExt>
__device__ __forceinline__ void splitk_reduce_epilogue(const GemmParams& p, unsigned tile_id, int sp, const float* trow, int r,
                                                       bool row_valid, long long grow, long long brow, int n0, int ncols_tile,
                                                       long long d_off, long long r_off, const float* sb, bool r_fast,
                                                       long long r_row) {
    const int rs = p.ws_tr ? 4 : BN;             // floats between consecutive rows of one float4 group
    const int gs = p.ws_tr ? BM * 4 : 4;         // floats between consecutive float4 groups of one row
    float* slices = p.ws + static_cast<size_t>(tile_id) * p.splits * (BM * BN) + static_cast<size_t>(r) * rs;
    float* mine = slices + static_cast<size_t>(sp) * (BM * BN);
#pragma unroll 1
    for (int c = 0; c * 32 < ncols_tile; ++c) {
        uint32_t acc[32];
        stage_ld32(trow, c, acc);
        if (row_valid) {
#pragma unroll
            for (int j = 0; j < 32; j += 4)
                __stcg(reinterpret_cast<float4*>(mine + (c * 8 + (j >> 2)) * gs),
                       make_float4(__uint_as_float(acc[j]), __uint_as_float(acc[j + 1]), __uint_as_float(acc[j + 2]),
                                   __uint_as_float(acc[j + 3])));
        }
    }
    __threadfence();
    asm volatile("bar.sync 1, 128;" ::: "memory");
    __shared__ unsigned s_last;
    if (threadIdx.x == 64) {
        const unsigned prev = atomicAdd(p.counters + tile_id, 1u);
        s_last = (prev == static_cast<unsigned>(p.splits) - 1u) ? 1u : 0u;
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    const bool last = s_last != 0u;
    if (!last) return;
    __threadfence();
    if (row_valid) {
        ResidualChunk rc_cur;
#pragma unroll 1
        for (int c = 0; c * 32 < ncols_tile; ++c) {
            const bool pre = r_fast && ncols_tile - c * 32 >= 32;
            if (pre) residual_prefetch(p, r_row + c * 32, rc_cur);
            float4 v[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
            for (int s2 = 0; s2 < p.splits; ++s2) {
                const float* src = slices + static_cast<size_t>(s2) * (BM * BN);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float4 t = __ldcg(reinterpret_cast<const float4*>(src + (c * 8 + j) * gs));
                    v[j].x += t.x; v[j].y += t.y; v[j].z += t.z; v[j].w += t.w;
                }
            }
            if (p.vec_ok && !p.d_transposed && ncols_tile - c * 32 >= 32) {
                float f[32];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    f[4 * j] = v[j].x * p.alpha; f[4 * j + 1] = v[j].y * p.alpha;
                    f[4 * j + 2] = v[j].z * p.alpha; f[4 * j + 3] = v[j].w * p.alpha;
                }
                epilogue_chunk32<kExt>(p, f, grow, brow, n0 + c * 32, d_off, r_off, pre ? &rc_cur : nullptr, sb ? sb + c * 32 : nullptr);
            } else {
#pragma unroll
                for (int g = 0; g < 4; ++g) {
                    const int nc = min(8, ncols_tile - c * 32 - g * 8);
                    if (nc > 0) {
                        const float4 lo = v[2 * g], hi = v[2 * g + 1];
                        float f[8] = {lo.x * p.alpha, lo.y * p.alpha, lo.z * p.alpha, lo.w * p.alpha,
                                      hi.x * p.alpha, hi.y * p.alpha, hi.z * p.alpha, hi.w * p.alpha};
                        epilogue_group8<kExt>(p, f, grow, brow, n0 + c * 32 + g * 8, d_off, r_off, nc, nullptr, sb ? sb + c * 32 + g * 8 : nullptr);
                    }
                }
            }
        }
    }
    if (threadIdx.x == 64) p.counters[tile_id] = 0u;   // self-cleaning for the next launch
}

// Warp roles (384 threads, one CTA per SM):
//   warpgroup 0 : thread 0 is the TMA producer; after the main loop all 128 threads run the epilogue, one output row each
//   warpgroups 1, 2 : wgmma consumers, rows [0, 64) and [64, 128) of the tile, fp32 accumulators in registers
// Once the last k-iteration has retired, the consumers park their accumulators in the (then idle) TMA ring as a row-major
// fp32 tile of pitch BN + 4 floats (conflict-free 16-byte row reads), so the epilogue reads one row per thread.
template <int BN>
struct StageCfg {
    static constexpr int kPitch = BN + 4;
    static constexpr int kBytes = ((BM * kPitch * 4) + 1023) / 1024 * 1024;
};

// 32 consecutive accumulator columns of this thread's row from the staged tile
__device__ __forceinline__ void stage_ld32(const float* row, int c, uint32_t (&acc)[32]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float4 v = *reinterpret_cast<const float4*>(row + c * 32 + 4 * j);
        acc[4 * j] = __float_as_uint(v.x); acc[4 * j + 1] = __float_as_uint(v.y);
        acc[4 * j + 2] = __float_as_uint(v.z); acc[4 * j + 3] = __float_as_uint(v.w);
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

    const int warp = threadIdx.x >> 5;
    const int wg = warp >> 2;
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
            mbar_init(empty_bar(s), 256);     // every consumer thread releases the stage
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
            for (int it = it0; it < it1; ++it) {
                const int li = it - it0;
                const int s = li % kStages;
                const uint32_t ph = (li / kStages) & 1;
                mbar_wait(empty_bar(s), ph ^ 1u);
                mbar_arrive_expect_tx(full_bar(s), p.a_bytes + p.b_bytes);
                const int tap = it / p.kchunks;
                const int kc = it - tap * p.kchunks;
                const uint32_t a_dst = smem_base + s * Cfg::kStageBytes;
                const uint32_t b_dst = a_dst + Cfg::kABytes;
                const int tap_b = p.flip_taps ? (p.taps - 1 - tap) : tap;
                if (p.conv) {
                    const int r = tap / p.kw, sx = tap - r * p.kw;
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
            }
        }
        __syncwarp();
    } else {
        // ===================== wgmma consumers =====================
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        const uint32_t a_half = static_cast<uint32_t>(wg - 1) * 8192u;     // this warpgroup's 64 rows of the A tile
        for (int it = it0; it < it1; ++it) {
            const int li = it - it0;
            const int s = li % kStages;
            mbar_wait(full_bar(s), (li / kStages) & 1);
            if (dbg && li == 0 && threadIdx.x == 128) dbg[2] = clock64();
            const uint32_t a_src = smem_base + s * Cfg::kStageBytes + a_half;
            const uint32_t b_src = smem_base + s * Cfg::kStageBytes + Cfg::kABytes;
            const int kc = it % p.kchunks;
            const int ksteps = (kc == p.kchunks - 1) ? p.ksteps_last : (BK / 16);
            wgmma_fence_regs(acc);
            wgmma_fence();
            for (int k = 0; k < ksteps; ++k) {
                const uint64_t adesc = A_MN ? gmma_desc_sw128(a_src + k * 2048, 8192, 1024) : gmma_desc_sw128(a_src + k * 32, 16, 1024);
                const uint64_t bdesc = B_MN ? gmma_desc_sw128(b_src + k * 2048, 8192, 1024) : gmma_desc_sw128(b_src + k * 32, 16, 1024);
                wgmma_any<BN, A_MN, B_MN>(p.bf16 != 0, acc, adesc, bdesc, 1u);
            }
            wgmma_commit();
            // keep one k-iteration of MMAs in flight: the previous stage is released once its group has retired
            wgmma_wait<1>();
            wgmma_fence_regs(acc);
            if (li > 0) mbar_arrive(empty_bar((li - 1) % kStages));
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        if (it1 > it0) mbar_arrive(empty_bar((it1 - it0 - 1) % kStages));
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
    named_bar(2, kThreads);        // accumulator tile staged
    if (p.cluster_sk && wg != 0) { cluster_sync_all(); cluster_sync_all(); }   // the two cluster barriers of the epilogue

    if (wg == 0) {
        // ===================== epilogue: one output row per thread =====================
        const int r = threadIdx.x;
        bool row_valid;
        long long grow;
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
        const long long brow = p.bias_row_div > 0 ? grow / p.bias_row_div : 0;
        const long long d_off = (long long)zo * p.d_bs2 + (long long)zi * p.d_bs;
        const long long r_off = (long long)zo * p.r_bs2 + (long long)zi * p.r_bs;
        const int ncols_tile = min(BN, p.N - n0);
        // bias row of this tile -> shared memory (global bias loads in the store loop would each wait a full L2 round
        // trip behind the previous chunk's stores)
        __shared__ __align__(16) float s_bias[BN + 8];
        const float* sb = nullptr;
        if (p.bias) {
            const long long tile_row0 = p.conv ? (((long long)img0 * p.out_h + oh0) * p.out_w + ow0) : (long long)m0;
            const long long brow0 = p.bias_row_div > 0 ? tile_row0 / p.bias_row_div : 0;
            for (int i = threadIdx.x; i < BN; i += 128) s_bias[i] = i < ncols_tile ? p.bias[brow0 * p.ldbias + n0 + i] : 0.f;
            named_bar(3, 128);
            if (brow == brow0) sb = s_bias;
        }
        // residual fast path: whole 32-column chunks, 16-byte aligned rows
        const bool r_fast = p.R && p.vec_ok && !p.d_transposed && row_valid;
        const long long r_row = r_off + grow * p.ldr + n0;
        ResidualChunk rc_cur, rc_next;
        if (r_fast && p.splits == 1 && ncols_tile >= 32) residual_prefetch(p, r_row, rc_cur);
        if (dbg && threadIdx.x == 64) dbg[4] = clock64();
        const float* trow = stage + r * SCfg::kPitch;
        if (p.dbg_mode == 1 || p.dbg_mode == 2) {
        } else if (p.splits == 1) {
#pragma unroll 1
            for (int c = 0; c * 32 < ncols_tile; ++c) {
                uint32_t acc[32];
                if constexpr (kExt) {
                    if (p.glu) {
                        uint32_t acc2[32];
                        stage_ld32(trow, c, acc);
                        stage_ld32(trow, c + 1, acc2);
                        if (row_valid) {
                            float fv[32], fg[32];
#pragma unroll
                            for (int j = 0; j < 32; ++j) { fv[j] = __uint_as_float(acc[j]) * p.alpha; fg[j] = __uint_as_float(acc2[j]) * p.alpha; }
                            epilogue_glu64(p, fv, fg, grow, n0 + c * 32, sb ? sb + c * 32 : nullptr);
                        }
                        ++c;
                        continue;
                    }
                }
                stage_ld32(trow, c, acc);
                const bool pre = r_fast && ncols_tile - c * 32 >= 32;
                if (r_fast && ncols_tile - (c + 1) * 32 >= 32) residual_prefetch(p, r_row + (c + 1) * 32, rc_next);
                if (row_valid && p.vec_ok && !p.d_transposed && ncols_tile - c * 32 >= 32) {
                    float f[32];
#pragma unroll
                    for (int j = 0; j < 32; ++j) f[j] = __uint_as_float(acc[j]) * p.alpha;
                    epilogue_chunk32<kExt>(p, f, grow, brow, n0 + c * 32, d_off, r_off, pre ? &rc_cur : nullptr, sb ? sb + c * 32 : nullptr);
                } else if (row_valid) {
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        const int nc = min(8, ncols_tile - c * 32 - g * 8);
                        if (nc > 0) {
                            float f[8];
#pragma unroll
                            for (int j = 0; j < 8; ++j) f[j] = __uint_as_float(acc[g * 8 + j]) * p.alpha;
                            epilogue_group8<kExt>(p, f, grow, brow, n0 + c * 32 + g * 8, d_off, r_off, nc, nullptr, sb ? sb + c * 32 + g * 8 : nullptr);
                        }
                    }
                }
                rc_cur = rc_next;
            }
        } else if (p.cluster_sk) {
            // ---- split-K inside a thread-block cluster: the `splits` CTAs of this tile are the cluster (1,1,splits), rank =
            //      k-slice.  The 8-column groups of the tile are dealt round-robin to the CTAs (group g -> CTA g % S); every CTA
            //      sends each group of its partial accumulator into the owner's exchange buffer (the part of the idle TMA ring
            //      behind the staged tile), slot [sender][g / S][row] of 32 bytes, then sums its own groups over the S senders
            //      and runs the epilogue for them.  Two cluster barriers replace the L2 reductions, the __threadfence, the
            //      arrival counter and the read-back of the global-workspace path.
            const int S = p.splits;
            const int GI = (BN / 8 + S - 1) / S;                 // groups a CTA can own
            const uint32_t xbuf = smem_base + SCfg::kBytes;
            fence_proxy_async_smem();                            // the ring was written / read through the async proxy
            cluster_sync_all();                                  // #1: every CTA of the cluster has staged its accumulator
#pragma unroll 1
            for (int c = 0; c * 32 < ncols_tile; ++c) {
                uint32_t acc[32];
                stage_ld32(trow, c, acc);
#pragma unroll
                for (int gq = 0; gq < 4; ++gq) {
                    const int g = c * 4 + gq;
                    if (g * 8 < ncols_tile)
                        st_cluster_f32x8(xbuf + static_cast<uint32_t>(((sp * GI + g / S) * BM + r) * 32),
                                         static_cast<uint32_t>(g % S), &acc[gq * 8]);
                }
            }
            cluster_sync_all();                                  // #2: all partial groups have landed in their owners
            for (int gi = 0; gi < GI; ++gi) {
                const int g = gi * S + sp;
                if (g * 8 >= ncols_tile) break;
                float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
                for (int s2 = 0; s2 < S; ++s2) {
                    const uint32_t a = xbuf + static_cast<uint32_t>(((s2 * GI + gi) * BM + r) * 32);
                    const float4 lo = ld_shared_f32x4(a), hi = ld_shared_f32x4(a + 16);
                    f[0] += lo.x; f[1] += lo.y; f[2] += lo.z; f[3] += lo.w;
                    f[4] += hi.x; f[5] += hi.y; f[6] += hi.z; f[7] += hi.w;
                }
                if (row_valid) {
#pragma unroll
                    for (int j = 0; j < 8; ++j) f[j] *= p.alpha;
                    epilogue_group8<kExt>(p, f, grow, brow, n0 + g * 8, d_off, r_off, min(8, ncols_tile - g * 8), nullptr,
                                          sb ? sb + g * 8 : nullptr);
                }
            }
        } else {
            const unsigned tile_id = (static_cast<unsigned>(bz) * gridDim.y + m_tile) * gridDim.x + blockIdx.x;
            splitk_reduce_epilogue<BN, kExt>(p, tile_id, sp, trow, r, row_valid, grow, brow, n0, ncols_tile, d_off, r_off, sb,
                                             r_fast, r_row);
        }
        if (dbg && threadIdx.x == 64) dbg[5] = clock64();
    }
    if (dbg && threadIdx.x == 0) dbg[6] = clock64();
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
    if (force_bn == 256 && N >= 256) return 256;    // 128x256 tile: only on request (per-shape autotuner / caller)
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
        bool ok32 = ok && ((reinterpret_cast<uintptr_t>(d.D) & 31u) == 0) && ((d.ldd * des) % 32 == 0) &&
                    ((d.d_batch_stride * des) % 32 == 0) && ((d.d_batch_stride2 * des) % 32 == 0);
        if (d.R) {
            const int res = d.r_dtype == CB_F32 ? 4 : 2;
            ok32 = ok32 && ((reinterpret_cast<uintptr_t>(d.R) & 31u) == 0) && ((d.ldr * res) % 32 == 0) &&
                   ((d.r_batch_stride * res) % 32 == 0) && ((d.r_batch_stride2 * res) % 32 == 0);
        }
        p.vec32_ok = ok32 ? 1 : 0;
    }

    // ---- split-K heuristic: fill the SMs when the tile grid alone cannot (bs=1 low-resolution layers) ----
    p.force_stages = (d.stages == 3 || d.stages == 6) ? d.stages : 0;
    {
        static const int ws_tr = getenv("CB_GEMM_WS_TR") ? atoi(getenv("CB_GEMM_WS_TR")) : 1;   // A/B aid
        p.ws_tr = ws_tr;
    }
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
