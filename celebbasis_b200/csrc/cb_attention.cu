// cb_attention_fwd — fused scaled-dot-product attention forward for sm_90a (flash style).
//
// Replaces the materialised `sim = einsum(q,k)*scale; attn = sim.softmax(-1); out = einsum(attn, v)` of
// ldm/modules/attention.py:178-191 (and the CLIP layers' masked variant, encoders/modules.py:24-31): the
// (heads x N x N) score tensor -- 512 MiB fp32 per 4096-token block in the reference -- never reaches HBM unless
// the caller asks for the probabilities (training keeps them for the backward pass).
//
// One CTA = 128 query rows of one (image, head), three warpgroups:
//   warpgroup 0   : TMA producer (one elected thread) -- Q once, then K_j / V_j blocks of 64 keys through a 4-stage
//                   mbarrier ring.  It hands most of its registers to the consumers (setmaxnreg).
//   warpgroups 1,2: query rows [0, 64) / [64, 128).  Per block: S_j = Q K_j^T with wgmma (fp32 in registers), online
//                   softmax on the register fragment (running max / sum per row, exp2 with the scale folded in, row
//                   reductions across the four lanes that share a row), P_j written as a K-major SWIZZLE_128B A tile in
//                   shared memory, O += P_j V_j with wgmma (V read MN-major straight from its [keys][d] layout, O in
//                   registers); finally O / l -> HBM and logsumexp.
//                   Pipelined within the warpgroup: O += P_{j-1} V_{j-1} is queued behind S_j and stays in flight while
//                   the softmax of block j runs, so the tensor cores and the exp unit work at the same time.
// Head dims 40 / 64 / 80 / 128 (any multiple of 8 up to 128): the tensor maps declare the head's d columns as the
// K extent, so TMA zero-fills the rest of each 64-column box and the MMAs run on 16-column multiples.  The number of
// those k16 steps is a template parameter, so every MMA group is one straight-line batch.
#include <string.h>

#include <type_traits>

#include "cb_common.cuh"

namespace cb {

constexpr int kAttnConsumers = 256;                  // two wgmma warpgroups
constexpr int kAttnThreads = kAttnConsumers + 128;   // + the TMA producer warpgroup
// Register split of the 384-thread CTA (65,536 registers): ptxas budgets 168 per thread for three warpgroups; the
// producer drops to 24 and the two consumer warpgroups rise to 240 (128 * 24 + 256 * 240 = 64,512).
constexpr int kAttnProducerRegs = 24;
constexpr int kAttnConsumerRegs = 240;
constexpr int kBQ = 128;    // query rows per CTA
constexpr int kBKV = 64;    // keys per block

struct AttnParams {
    int nq, nk, heads, images;
    int d;                  // head dim
    int causal;
    int two_pass;           // pass A: row max / sum only; pass B: normalised probabilities (needed when P is stored)
    float scale_log2e;      // scale * log2(e)
    void* O;
    long long ldo;          // elements between consecutive query rows of O
    float* lse;             // [images][heads][nq] natural-log sum-exp (scaled scores), or NULL
    void* P;                // optional probabilities [images*heads][nq][ldp] (same 16-bit dtype as the operands)
    long long ldp;
    int is_bf16;            // operands, O and P are bf16 (else fp16)
};

template <int DBOX>  // number of 64-column boxes of the head dim (1: d <= 64, 2: d <= 128)
struct AttnCfg {
    static constexpr int kQBytes = DBOX * kBQ * 128;
    static constexpr int kKBytes = DBOX * kBKV * 128;
    static constexpr int kVBytes = DBOX * kBKV * 128;
    static constexpr int kPBytes = kBQ * 128;              // 64 keys = one 128-byte chunk per query row
    // K_j / V_j stay resident until O += P_j V_j retires during block j+1; the other stages are the producer's lead
    static constexpr int kStages = 4;
    static constexpr int kSmemBytes = kQBytes + kStages * (kKBytes + kVBytes) + 2 * kPBytes + 1024 + 256;   // two P buffers
};

// Consumer-side mbarrier wait.  Unlike mbar_wait it has no __trap() hang guard: a trap reachable from the consumer
// region makes ptxas ignore the setmaxnreg.inc budget and allocate the consumers within the 168 registers of a
// 384-thread CTA, which spills the backward's dK/dV accumulators and serialises their wgmmas (C7512).
__device__ __forceinline__ void mbar_wait_consumer(uint32_t bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}

template <uint32_t R>
__device__ __forceinline__ void regs_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R>
__device__ __forceinline__ void regs_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// acc[64 x 64] (+)= A B^T over KS k16 steps, one wgmma group: A = 64 rows at a, B = 64 rows at b, both K-major
// SWIZZLE_128B with the head dim split into 64-column boxes a_box / b_box bytes apart.  k = 0 overwrites acc.
// Straight-line code between one fence and one commit gets one warpgroup.arrive for the whole batch; an MMA in a
// branch of its own gets an injected arrive (C7519) and waits for the one before it.
template <int KS, bool BF16>
__device__ __forceinline__ void mma_rows(float (&acc)[32], uint32_t a, uint32_t a_box, uint32_t b, uint32_t b_box) {
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < KS; ++k)
        Wgmma<64, BF16, 0, 0>::mma(acc, gmma_desc_sw128(a + (k >> 2) * a_box + (k & 3) * 32, 16, 1024),
                                   gmma_desc_sw128(b + (k >> 2) * b_box + (k & 3) * 32, 16, 1024), k > 0 ? 1u : 0u);
    wgmma_commit();
}
template <int KS>
__device__ __forceinline__ void mma_rows_any(bool bf16, float (&acc)[32], uint32_t a, uint32_t a_box, uint32_t b,
                                             uint32_t b_box) {
    if (bf16) mma_rows<KS, true>(acc, a, a_box, b, b_box);
    else mma_rows<KS, false>(acc, a, a_box, b, b_box);
}
// acc[64 x NO] (+)= A Y over one 64-item block, one wgmma group: A = [64 rows][64 items] K-major at a (16-item step k),
// Y = [64 items][NO] MN-major at y (16 items = 2 groups of 8 rows, SBO 1024; 64-column chunks at LBO).
// acc_in = 0 overwrites acc with the first product.
template <int NO, bool BF16>
__device__ __forceinline__ void mma_block(float (&acc)[NO / 2], uint32_t a, uint32_t y, uint32_t acc_in) {
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBKV / 16; ++k)
        Wgmma<NO, BF16, 0, 1>::mma(acc, gmma_desc_sw128(a + k * 32, 16, 1024), gmma_desc_sw128(y + k * 2048, kBKV * 128, 1024),
                                   k > 0 ? 1u : acc_in);
    wgmma_commit();
}
template <int NO>
__device__ __forceinline__ void mma_block_any(bool bf16, float (&acc)[NO / 2], uint32_t a, uint32_t y, uint32_t acc_in) {
    if (bf16) mma_block<NO, true>(acc, a, y, acc_in);
    else mma_block<NO, false>(acc, a, y, acc_in);
}

__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t pack2(float a, float b, bool bf16) {
    if (bf16) {
        __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&h);
    }
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
// two consecutive 16-bit values at (row r, column col) of a [128 rows][64 columns] K-major SWIZZLE_128B A tile
__device__ __forceinline__ void st_a_pair(uint32_t tile, int r, int col, uint32_t v) {
    const uint32_t dst = tile + r * 128 + ((((uint32_t)col >> 3) ^ ((uint32_t)r & 7u)) << 4) + (col & 7) * 2;
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(dst), "r"(v) : "memory");
}
__device__ __forceinline__ float quad_max(float v) {
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

template <int KS>   // k16 steps of the head dim: ceil(d / 16)
__global__ void __launch_bounds__(kAttnThreads, 1)
cb_attention_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                        const __grid_constant__ CUtensorMap tmV, const __grid_constant__ AttnParams p) {
    constexpr int DBOX = (KS + 3) / 4;
    using Cfg = AttnCfg<DBOX>;
    constexpr int kSt = Cfg::kStages;
    constexpr int NO = DBOX * 64;                 // output columns (zero-filled past d)
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t sQ = base;
    const uint32_t sKV = sQ + Cfg::kQBytes;                                 // stage s: K at sKV + s*(K+V), V after K
    const uint32_t sP = sKV + kSt * (Cfg::kKBytes + Cfg::kVBytes);          // P of block j in buffer j & 1
    const uint32_t bars = sP + 2 * Cfg::kPBytes;
    const uint32_t bar_q = bars;
    auto bar_kv_full = [&](int s) { return bars + 8u * (1 + s); };
    auto bar_kv_empty = [&](int s) { return bars + 8u * (1 + kSt + s); };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // warp-uniform as far as the compiler can tell (a plain threadIdx-derived index makes the role branch divergent)
    const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);
    const int q0 = blockIdx.x * kBQ;
    const int head = blockIdx.y, img = blockIdx.z;
    int nblk = (p.nk + kBKV - 1) / kBKV;
    if (p.causal) nblk = min(nblk, (min(q0 + kBQ, p.nq) + kBKV - 1) / kBKV);
    const int nstat = p.two_pass ? nblk : 0;      // leading statistics-only virtual blocks
    const int nv = nstat + nblk;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmQ);
        tma_prefetch_desc(&tmK);
        tma_prefetch_desc(&tmV);
        mbar_init(bar_q, 1);
        for (int s = 0; s < kSt; ++s) {
            mbar_init(bar_kv_full(s), 1);
            mbar_init(bar_kv_empty(s), kAttnConsumers);
        }
        mbar_fence_init();
        fence_proxy_async_smem();
    }
    __syncthreads();
    pdl_sync();

    if (wg == 0) {
        regs_dealloc<kAttnProducerRegs>();
        if (threadIdx.x == 0) {
            // ============================ TMA producer ============================
            mbar_arrive_expect_tx(bar_q, Cfg::kQBytes);
#pragma unroll
            for (int b = 0; b < DBOX; ++b) tma_load_4d(sQ + b * (kBQ * 128), &tmQ, bar_q, b * 64, q0, head, img);
            for (int vj = 0; vj < nv; ++vj) {
                const int s = vj % kSt;
                const uint32_t ph = (vj / kSt) & 1;
                const bool full = vj >= nstat;
                const int j = full ? vj - nstat : vj;
                mbar_wait(bar_kv_empty(s), ph ^ 1u);
                mbar_arrive_expect_tx(bar_kv_full(s), Cfg::kKBytes + (full ? Cfg::kVBytes : 0));
                const uint32_t dK = sKV + s * (Cfg::kKBytes + Cfg::kVBytes), dV = dK + Cfg::kKBytes;
#pragma unroll
                for (int b = 0; b < DBOX; ++b) {
                    tma_load_4d(dK + b * (kBKV * 128), &tmK, bar_kv_full(s), b * 64, j * kBKV, head, img);
                    if (full) tma_load_4d(dV + b * (kBKV * 128), &tmV, bar_kv_full(s), b * 64, j * kBKV, head, img);
                }
            }
        }
        return;
    }
    regs_alloc<kAttnConsumerRegs>();

    // ============================ consumers: 64 query rows per warpgroup ============================
    const int cw = wg - 1;
    const int rl = cw * 64 + (warp & 3) * 16 + (lane >> 2);   // tile row of fragment half 0 (half 1: rl + 8)
    const int cq = 2 * (lane & 3);                             // this thread's first column in every 8-column group
    const bool bf16 = p.is_bf16 != 0;
    const uint32_t qoff = static_cast<uint32_t>(cw) * 8192u;   // this warpgroup's 64 rows of a 128-row tile
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f}, inv_l[2] = {1.f, 1.f};
    float o[NO / 2];
#pragma unroll
    for (int i = 0; i < NO / 2; ++i) o[i] = 0.f;

    // Per block vj: S_vj = Q K_vj^T is issued, then O += P_{vj-1} V_{vj-1} behind it; the softmax of block vj runs once
    // S_vj has retired, while the PV group is still on the tensor cores.  That group retires before O is rescaled and
    // P_vj is handed to the next block; only then is the K/V stage of block vj-1 released.
    // Whether a PV group is pending is known at compile time in each of the three loops below: a wgmma wait under a
    // runtime condition counts as divergent, and ptxas then serialises the MMAs (C7518).
    int pv_stage = 0, pv_j = 0;                    // P_{vj-1} in shared memory, waiting for its PV group
    auto issue_pv = [&]() {
        wgmma_fence_regs(o);
        mma_block_any<NO>(bf16, o, sP + (pv_j & 1) * Cfg::kPBytes + qoff,
                          sKV + pv_stage * (Cfg::kKBytes + Cfg::kVBytes) + Cfg::kKBytes, 1u);
    };
    float sc[32];
    auto block = [&](int vj, auto pv_pending_c) {
        constexpr bool pv_pending = decltype(pv_pending_c)::value;
        const bool full = vj >= nstat;
        const int j = full ? vj - nstat : vj;
        const int s = vj % kSt;
        mbar_wait_consumer(bar_kv_full(s), (vj / kSt) & 1);
        mma_rows_any<KS>(bf16, sc, sQ + qoff, kBQ * 128, sKV + s * (Cfg::kKBytes + Cfg::kVBytes), kBKV * 128);
        if constexpr (pv_pending) {
            issue_pv();
            wgmma_wait<1>();                       // S_vj has retired; O += P_{vj-1} V_{vj-1} may still run
        } else {
            wgmma_wait<0>();
        }
        wgmma_fence_regs(sc);
        if (!full) mbar_arrive(bar_kv_empty(s));          // statistics pass: the K stage is free once S is done
        const int kbase = j * kBKV;
        // masked keys -> -inf, then the row maxima on the raw scores (scale > 0 commutes with max)
        float mx[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            int kvalid = min(kBKV, p.nk - kbase);
            if (p.causal) kvalid = min(kvalid, q0 + rl + 8 * h - kbase + 1);
            float mh = -INFINITY;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    float& v = sc[4 * jj + 2 * h + c];
                    if (jj * 8 + cq + c >= kvalid) v = -INFINITY;
                    mh = fmaxf(mh, v);
                }
            mx[h] = quad_max(mh) * p.scale_log2e;
        }
        const bool online = !(p.two_pass && full);      // running max / sum still being built
        float m_use[2], corr[2] = {1.f, 1.f};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            if (online) {
                // Lazy rescale: the reference maximum only moves when the block maximum exceeds it by more than 2^8
                // (probabilities stay <= 256, exact in fp16/fp32).
                const float m_new = fmaxf(m[h], mx[h]);
                if (m[h] == -INFINITY) {
                    m[h] = m_new;                            // first block: nothing accumulated yet (l = 0, O zero)
                } else if (m_new > m[h] + 8.f) {
                    corr[h] = fast_exp2(m[h] - m_new);
                    m[h] = m_new;
                }
                l[h] *= corr[h];
            }
            m_use[h] = (m[h] == -INFINITY) ? 0.f : m[h];  // (fully masked so far: the exponent argument stays -inf)
        }
        if (!full) {                                    // statistics pass: accumulate the row sums only
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float rs = 0.f;
#pragma unroll
                for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                    for (int c = 0; c < 2; ++c) rs += fast_exp2(fmaf(sc[4 * jj + 2 * h + c], p.scale_log2e, -m_use[h]));
                l[h] += rs;
                if (vj == nstat - 1) {
                    l[h] = quad_sum(l[h]);
                    inv_l[h] = l[h] > 0.f ? 1.f / l[h] : 0.f;
                }
            }
            return;
        }
        // P = exp2(s - m) (normalised by 1/l in two-pass mode): swizzled K-major A tile in smem (+ optional HBM copy).
        // Buffer j & 1 was last read by O += P_{j-2} V_{j-2}, which retired in the previous block.
        const uint32_t tile = sP + (j & 1) * Cfg::kPBytes;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int qrow = q0 + rl + 8 * h;
            uint32_t* prow = (p.P && qrow < p.nq)
                                 ? reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.P) +
                                                               ((static_cast<long long>(img) * p.heads + head) * p.nq + qrow) * p.ldp + kbase + cq)
                                 : nullptr;
            const float pscale = p.two_pass ? inv_l[h] : 1.f;
            float rs = 0.f;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                const float e0 = fast_exp2(fmaf(sc[4 * jj + 2 * h], p.scale_log2e, -m_use[h])) * pscale;
                const float e1 = fast_exp2(fmaf(sc[4 * jj + 2 * h + 1], p.scale_log2e, -m_use[h])) * pscale;
                rs += e0 + e1;
                const uint32_t v = pack2(e0, e1, bf16);
                st_a_pair(tile, rl + 8 * h, jj * 8 + cq, v);
                if (prow && kbase + jj * 8 < p.ldp) prow[jj * 4] = v;
            }
            if (online) l[h] += rs;
        }
        if constexpr (pv_pending) {
            wgmma_wait<0>();                       // O += P_{vj-1} V_{vj-1} has retired
            wgmma_fence_regs(o);
            mbar_arrive(bar_kv_empty(pv_stage));   // K_{vj-1} / V_{vj-1} stage reusable
        }
        if (online) {                              // x * 1.0f is exact: rows whose maximum did not move keep their bits
#pragma unroll
            for (int jj = 0; jj < NO / 8; ++jj)
#pragma unroll
                for (int h = 0; h < 2; ++h) { o[4 * jj + 2 * h] *= corr[h]; o[4 * jj + 2 * h + 1] *= corr[h]; }
        }
        fence_proxy_async_smem();       // generic-proxy smem writes -> visible to the tensor core (async proxy)
        named_bar(1 + cw, 128);         // this warpgroup's 64 rows of P are complete
        pv_stage = s;
        pv_j = j;
    };
    mbar_wait_consumer(bar_q, 0);
    int vj = 0;
    for (; vj < nstat; ++vj) block(vj, std::false_type{});     // statistics pass (two-pass mode)
    block(vj++, std::false_type{});                            // first full block: nothing to accumulate yet
    for (; vj < nv; ++vj) block(vj, std::true_type{});
    issue_pv();                                                // there is always at least one full block
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    // ---- epilogue: O / l, logsumexp ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        if (!p.two_pass) l[h] = quad_sum(l[h]);
        const int qrow = q0 + rl + 8 * h;
        if (qrow >= p.nq) continue;
        const float inv = p.two_pass ? 1.f : (l[h] > 0.f ? 1.f / l[h] : 0.f);
        if (p.lse && (lane & 3) == 0)
            p.lse[(static_cast<long long>(img) * p.heads + head) * p.nq + qrow] = (m[h] + log2f(l[h])) * 0.6931471805599453f;
        uint16_t* orow = reinterpret_cast<uint16_t*>(p.O) + (static_cast<long long>(img) * p.nq + qrow) * p.ldo +
                         static_cast<long long>(head) * p.d;
#pragma unroll
        for (int jj = 0; jj < NO / 8; ++jj) {
            const int col = jj * 8 + cq;
            if (col < p.d)
                *reinterpret_cast<uint32_t*>(orow + col) = pack2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv, bf16);
        }
    }
}

// Causal forward with P export: a query tile only visits the key blocks up to its last query, so the forward kernel never
// writes P for the blocks past them.  Those probabilities are zero; this kernel writes them (up to the row pitch), one P
// row per warp at a time.  It is a launch of its own because code added to the forward kernel moves ptxas's schedule of
// the forward's main loop: at d = 40 that cost 3 % of the forward's time (H100 80GB HBM3, 400 W).
__global__ void __launch_bounds__(128) cb_attention_p_tail_kernel(const __grid_constant__ AttnParams p) {
    pdl_sync();
    const int q0 = blockIdx.x * kBQ, head = blockIdx.y, img = blockIdx.z;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nvis = (min(q0 + kBQ, p.nq) + kBKV - 1) / kBKV;       // the forward's last visited key block + 1
    const long long c1 = min(static_cast<long long>((p.nk + kBKV - 1) / kBKV) * kBKV, p.ldp);
    for (int r = warp; r < min(kBQ, p.nq - q0); r += 4) {
        uint16_t* prow = reinterpret_cast<uint16_t*>(p.P) + ((static_cast<long long>(img) * p.heads + head) * p.nq + q0 + r) * p.ldp;
        for (long long c = static_cast<long long>(nvis) * kBKV + lane * 8; c < c1; c += 32 * 8)
            *reinterpret_cast<uint4*>(prow + c) = make_uint4(0u, 0u, 0u, 0u);
    }
}

int make_tmap(CUtensorMap* out, int dtype, int rank, const void* ptr, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* estr);

template <int KS>
static int launch_attn(const CUtensorMap& q, const CUtensorMap& k, const CUtensorMap& v, const AttnParams& p, dim3 grid,
                       cudaStream_t st) {
    using Cfg = AttnCfg<(KS + 3) / 4>;
    static bool done = false;
    auto kern = cb_attention_fwd_kernel<KS>;
    if (!done) {
        CB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
        done = true;
    }
    CB_LAUNCH((kern), grid, kAttnThreads, Cfg::kSmemBytes, st, q, k, v, p);
    CB_CUDA(cudaGetLastError());
    count_launches(1);
    return 0;
}


// =================================================================================================================
// Backward.  Two launches of one kernel template, both without atomics and without the (heads x N x N) tensors:
//   MODE 0 (dQ)    : CTA = 128 query rows.  X1 = Q, X2 = dO stationary; per 64-key block Y1 = K_j, Y2 = V_j.
//   MODE 1 (dK,dV) : CTA = 128 key rows.    X1 = K, X2 = V  stationary; per 64-query block Y1 = Q_j, Y2 = dO_j.
// Every block, per warpgroup of 64 stationary rows: T1 = X1 Y1^T (scores, or their transpose) and T2 = X2 Y2^T (dP, or
// its transpose) with wgmma into registers; P = exp2(T1*scale*log2e - lse*log2e) and dS = P o (T2 - delta) * scale with
// the forward's log-sum-exp and delta = rowsum(dO o O) (indexed by row in MODE 0, by column in MODE 1) are written as
// K-major SWIZZLE_128B A tiles; then  MODE 0: acc += dS Y1 (= dS K);  MODE 1: accV += P^T Y2 (= P^T dO),
// accK += dS^T Y1 (= dS^T Q) with the streamed tiles read MN-major, exactly like V in the forward kernel.
// MODE 0 also computes delta (it owns dO and reads O) and stores it for the MODE 1 launch that follows it in stream order.
// The CTA layout and register split are the forward kernel's.  T1 and T2 are issued back to back, so P is computed
// while T2 runs; the accumulation group of block j stays in flight until block j+1's T1 has retired.
struct AttnBwdParams {
    int n_stat, n_stream, heads, images;     // rows of the stationary / streamed operands (nq,nk in MODE 0; nk,nq in MODE 1)
    int d, causal;
    float scale, scale_log2e;
    const float* lse;        // [images][heads][nq]
    float* delta;            // [images][heads][nq]   (written by MODE 0, read by MODE 1)
    const void* O;           // MODE 0 only: forward output, for delta
    const void* dO;
    long long ldo, lddo;
    void* out1;              // MODE 0: dQ ; MODE 1: dV
    void* out2;              // MODE 1: dK
    long long ld1, ld2;
    int is_bf16;
    int nq;                  // query count (lse / delta row pitch)
    void* dS;                // MODE 0, optional: dS = P o (dP - delta) * scale exported as [images*heads][nq][ldds] (16-bit)
    long long ldds;
};

template <int DBOX, int MODE>
struct AttnBwdCfg {
    static constexpr int kXBytes = DBOX * kBQ * 128;        // one stationary tile
    static constexpr int kYBytes = DBOX * kBKV * 128;       // one streamed tile
    static constexpr int kABytes = kBQ * 128;               // one A tile (128 rows x 64 block items)
    static constexpr int kNumA = MODE == 0 ? 1 : 2;
    static constexpr int kNumAcc = MODE == 0 ? 1 : 2;
    static constexpr int kSmemBytes = 2 * kXBytes + 2 * 2 * kYBytes + kNumA * kABytes + 1024 + 256;
};

// MODE 1's two accumulations of one block as one wgmma group (k-order within each accumulator as in mma_block)
template <int NO, bool BF16>
__device__ __forceinline__ void mma_block2(float (&acc0)[NO / 2], uint32_t a0, uint32_t y0, float (&acc1)[NO / 2],
                                           uint32_t a1, uint32_t y1, uint32_t acc_in) {
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBKV / 16; ++k) {
        Wgmma<NO, BF16, 0, 1>::mma(acc0, gmma_desc_sw128(a0 + k * 32, 16, 1024), gmma_desc_sw128(y0 + k * 2048, kBKV * 128, 1024),
                                   k > 0 ? 1u : acc_in);
        Wgmma<NO, BF16, 0, 1>::mma(acc1, gmma_desc_sw128(a1 + k * 32, 16, 1024), gmma_desc_sw128(y1 + k * 2048, kBKV * 128, 1024),
                                   k > 0 ? 1u : acc_in);
    }
    wgmma_commit();
}

template <int KS, int MODE>   // KS: k16 steps of the head dim, ceil(d / 16)
__global__ void __launch_bounds__(kAttnThreads, 1)
cb_attention_bwd_kernel(const __grid_constant__ CUtensorMap tmX1, const __grid_constant__ CUtensorMap tmX2,
                        const __grid_constant__ CUtensorMap tmY1, const __grid_constant__ CUtensorMap tmY2,
                        const __grid_constant__ AttnBwdParams p) {
    constexpr int DBOX = (KS + 3) / 4;
    using Cfg = AttnBwdCfg<DBOX, MODE>;
    constexpr int NO = DBOX * 64;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t sX1 = base, sX2 = base + Cfg::kXBytes;
    const uint32_t sY = sX2 + Cfg::kXBytes;                       // stage s: Y1 at sY + s*2*kYBytes, Y2 right after
    const uint32_t sA = sY + 4 * Cfg::kYBytes;                    // A tile 0 (dS in MODE 0, P^T in MODE 1), tile 1 (dS^T)
    const uint32_t bars = sA + Cfg::kNumA * Cfg::kABytes;
    const uint32_t bar_x = bars;
    auto bar_y_full = [&](int s) { return bars + 8u * (1 + s); };
    auto bar_y_empty = [&](int s) { return bars + 8u * (3 + s); };
    __shared__ float2 s_stat[2][kBKV];         // MODE 1: (lse*log2e, delta*scale) of the streamed queries, per warpgroup

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);
    const int x0 = blockIdx.x * kBQ;
    const int head = blockIdx.y, img = blockIdx.z;
    // streamed block range (causal: keys <= query)
    int jbeg = 0, jend = (p.n_stream + kBKV - 1) / kBKV;
    if (p.causal) {
        if (MODE == 0) jend = min(jend, (min(x0 + kBQ, p.n_stat) + kBKV - 1) / kBKV);     // keys up to the last query row
        else jbeg = x0 / kBKV;                                                            // queries from the first key row
    }
    const int nit = max(0, jend - jbeg);

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmX1); tma_prefetch_desc(&tmX2); tma_prefetch_desc(&tmY1); tma_prefetch_desc(&tmY2);
        mbar_init(bar_x, 1);
        for (int s = 0; s < 2; ++s) { mbar_init(bar_y_full(s), 1); mbar_init(bar_y_empty(s), kAttnConsumers); }
        mbar_fence_init();
        fence_proxy_async_smem();
    }
    __syncthreads();
    pdl_sync();

    if (wg == 0) {
        regs_dealloc<kAttnProducerRegs>();
        if (threadIdx.x == 0) {
            mbar_arrive_expect_tx(bar_x, 2 * Cfg::kXBytes);
#pragma unroll
            for (int b = 0; b < DBOX; ++b) {
                tma_load_4d(sX1 + b * (kBQ * 128), &tmX1, bar_x, b * 64, x0, head, img);
                tma_load_4d(sX2 + b * (kBQ * 128), &tmX2, bar_x, b * 64, x0, head, img);
            }
            for (int it = 0; it < nit; ++it) {
                const int s = it & 1;
                mbar_wait(bar_y_empty(s), ((it >> 1) & 1) ^ 1u);
                mbar_arrive_expect_tx(bar_y_full(s), 2 * Cfg::kYBytes);
                const uint32_t d1 = sY + s * 2 * Cfg::kYBytes, d2 = d1 + Cfg::kYBytes;
#pragma unroll
                for (int b = 0; b < DBOX; ++b) {
                    tma_load_4d(d1 + b * (kBKV * 128), &tmY1, bar_y_full(s), b * 64, (jbeg + it) * kBKV, head, img);
                    tma_load_4d(d2 + b * (kBKV * 128), &tmY2, bar_y_full(s), b * 64, (jbeg + it) * kBKV, head, img);
                }
            }
        }
        return;
    }
    regs_alloc<kAttnConsumerRegs>();

    // ====================== consumers: 64 stationary rows per warpgroup ======================
    const int cw = wg - 1;
    const int rl = cw * 64 + (warp & 3) * 16 + (lane >> 2);   // tile row of fragment half 0 (half 1: rl + 8)
    const int cq = 2 * (lane & 3);
    const int et = threadIdx.x & 127;                          // thread index inside the warpgroup
    const bool bf16 = p.is_bf16 != 0;
    const uint32_t xoff = static_cast<uint32_t>(cw) * 8192u;
    const long long stat_base = (static_cast<long long>(img) * p.heads + head) * p.nq;
    const float kLog2e = 1.4426950408889634f;
    float lse_r[2] = {0.f, 0.f}, delta_r[2] = {0.f, 0.f};     // MODE 0: this thread's query rows' statistics
    if (MODE == 0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int xrow = x0 + rl + 8 * h;
            float acc = 0.f;
            if (xrow < p.n_stat) {
                lse_r[h] = p.lse[stat_base + xrow] * kLog2e;
                const uint16_t* orow = reinterpret_cast<const uint16_t*>(p.O) + (static_cast<long long>(img) * p.n_stat + xrow) * p.ldo + static_cast<long long>(head) * p.d;
                const uint16_t* grow = reinterpret_cast<const uint16_t*>(p.dO) + (static_cast<long long>(img) * p.n_stat + xrow) * p.lddo + static_cast<long long>(head) * p.d;
                for (int c = (lane & 3) * 8; c < p.d; c += 32) {       // the four lanes of a row split its 8-column groups
                    const uint4 a = *reinterpret_cast<const uint4*>(orow + c), b = *reinterpret_cast<const uint4*>(grow + c);
                    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        float2 fa, fb;
                        if (bf16) {
                            fa = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&aw[i]));
                            fb = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&bw[i]));
                        } else {
                            fa = __half22float2(*reinterpret_cast<const __half2*>(&aw[i]));
                            fb = __half22float2(*reinterpret_cast<const __half2*>(&bw[i]));
                        }
                        acc += fa.x * fb.x + fa.y * fb.y;
                    }
                }
            }
            acc = quad_sum(acc);
            delta_r[h] = acc * p.scale;            // used as fma(T2, scale, -delta*scale)
            if (xrow < p.n_stat && (lane & 3) == 0) p.delta[stat_base + xrow] = acc;
        }
    }
    // acc1: MODE 1 only.  Neither is initialised: the first block's MMAs overwrite them (scale_d = 0), and an accumulator
    // written by ordinary instructions would make ptxas serialise every wgmma of the loop.  For the same reason P lives in
    // registers of its own, not in T1's accumulator.
    float acc0[NO / 2], acc1[NO / 2];
    mbar_wait_consumer(bar_x, 0);
    for (int it = 0; it < nit; ++it) {
        const int j = jbeg + it;
        const int cbase = j * kBKV;
        const int s = it & 1;
        if (MODE == 1 && et < kBKV) {
            const int qc = cbase + et;
            s_stat[cw][et] = qc < p.n_stream ? make_float2(p.lse[stat_base + qc] * kLog2e, p.delta[stat_base + qc] * p.scale)
                                             : make_float2(0.f, 0.f);
        }
        named_bar(1 + cw, 128);                    // the statistics are in place
        mbar_wait_consumer(bar_y_full(s), (it >> 1) & 1);
        const uint32_t y1 = sY + s * 2 * Cfg::kYBytes, y2 = y1 + Cfg::kYBytes;
        // groups in flight: [accumulation of block j-1], T1, T2
        float t[32], t2[32];
        mma_rows_any<KS>(bf16, t, sX1 + xoff, kBQ * 128, y1, kBKV * 128);
        mma_rows_any<KS>(bf16, t2, sX2 + xoff, kBQ * 128, y2, kBKV * 128);
        // valid streamed items of this block for each of this thread's rows
        int cvalid[2], cfirst[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int xrow = x0 + rl + 8 * h;
            cvalid[h] = min(kBKV, p.n_stream - cbase);      // columns past the end of the streamed operand
            cfirst[h] = 0;
            if (p.causal) {
                if (MODE == 0) cvalid[h] = min(cvalid[h], xrow - cbase + 1);      // keys <= this query
                else cfirst[h] = max(0, xrow - cbase);                            // queries >= this key
            }
            if (MODE == 0 && xrow >= p.n_stat) cvalid[h] = 0;
        }
        wgmma_wait<1>();                           // T1 and the accumulation of block j-1 have retired
        wgmma_fence_regs(t);
        if (it > 0) mbar_arrive(bar_y_empty(s ^ 1));   // Y_{j-1} stage reusable
        // P = ex2(fma(T1, scale*log2e, -lse*log2e)), zero outside the valid block items, computed while T2 runs
        float pr[32];
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int col = jj * 8 + cq + c;
                    const float l2 = MODE == 0 ? lse_r[h] : s_stat[cw][col].x;
                    const float pv = fast_exp2(fmaf(t[4 * jj + 2 * h + c], p.scale_log2e, -l2));
                    pr[4 * jj + 2 * h + c] = (col < cvalid[h] && col >= cfirst[h]) ? pv : 0.f;
                }
        // The A tiles were last read by the accumulation group of block j-1, which wgmma_wait<1> above retired.  A
        // wgmma group completes as one warpgroup-wide operation, so once this warp has seen it retire, none of the
        // group's reads of all 64 rows is still pending, and no warpgroup barrier is needed before the tiles are rewritten.
        if (MODE == 1) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                for (int h = 0; h < 2; ++h) st_a_pair(sA, rl + 8 * h, jj * 8 + cq, pack2(pr[4 * jj + 2 * h], pr[4 * jj + 2 * h + 1], bf16));
        }
        wgmma_wait<0>();
        wgmma_fence_regs(t2);
        // dS = P * fma(T2, scale, -delta*scale)
        const uint32_t ds_tile = MODE == 0 ? sA : sA + Cfg::kABytes;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int xrow = x0 + rl + 8 * h;
            uint32_t* dsrow = (MODE == 0 && p.dS && xrow < p.n_stat)
                                  ? reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.dS) + (stat_base + xrow) * p.ldds + cbase + cq)
                                  : nullptr;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                float ds[2];
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const float dl = MODE == 0 ? delta_r[h] : s_stat[cw][jj * 8 + cq + c].y;
                    ds[c] = pr[4 * jj + 2 * h + c] * fmaf(t2[4 * jj + 2 * h + c], p.scale, -dl);
                }
                const uint32_t v = pack2(ds[0], ds[1], bf16);
                st_a_pair(ds_tile, rl + 8 * h, jj * 8 + cq, v);
                if (dsrow && cbase + jj * 8 < p.ldds) dsrow[jj * 4] = v;
            }
        }
        fence_proxy_async_smem();
        named_bar(1 + cw, 128);                    // this warpgroup's 64 rows of the A tiles are complete
        wgmma_fence_regs(acc0);
        if constexpr (MODE == 1) wgmma_fence_regs(acc1);
        const uint32_t acc_in = it > 0 ? 1u : 0u;
        if constexpr (MODE == 0) {
            mma_block_any<NO>(bf16, acc0, sA + xoff, y1, acc_in);
        } else {
            if (bf16) mma_block2<NO, true>(acc0, sA + xoff, y2, acc1, sA + Cfg::kABytes + xoff, y1, acc_in);
            else mma_block2<NO, false>(acc0, sA + xoff, y2, acc1, sA + Cfg::kABytes + xoff, y1, acc_in);
        }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc0);
    if constexpr (MODE == 1) wgmma_fence_regs(acc1);
    if (MODE == 0 && p.dS) {
        // causal: key blocks past this tile's last query were never visited -- their dS is zero
        const int nblk_all = (p.n_stream + kBKV - 1) / kBKV;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int xrow = x0 + rl + 8 * h;
            if (xrow >= p.n_stat) continue;
            uint16_t* dsrow = reinterpret_cast<uint16_t*>(p.dS) + (stat_base + xrow) * p.ldds;
            for (int jb = jend; jb < nblk_all; ++jb)
                for (int key8 = lane & 3; key8 < 8; key8 += 4)
                    if (jb * kBKV + key8 * 8 < p.ldds) *reinterpret_cast<uint4*>(dsrow + jb * kBKV + key8 * 8) = make_uint4(0u, 0u, 0u, 0u);
        }
    }
    // ---- epilogue: accumulators -> HBM ----
    auto store_acc = [&](const float (&acc)[NO / 2], void* out, long long ldout) {
        uint16_t* outp = reinterpret_cast<uint16_t*>(out);
        if (outp == nullptr) return;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int xrow = x0 + rl + 8 * h;
            if (xrow >= p.n_stat) continue;
            uint16_t* orow = outp + (static_cast<long long>(img) * p.n_stat + xrow) * ldout + static_cast<long long>(head) * p.d;
#pragma unroll
            for (int jj = 0; jj < NO / 8; ++jj) {
                const int col = jj * 8 + cq;
                if (col < p.d)                                 // no streamed block (causal corner): the result is zero
                    *reinterpret_cast<uint32_t*>(orow + col) =
                        nit > 0 ? pack2(acc[4 * jj + 2 * h], acc[4 * jj + 2 * h + 1], bf16) : 0u;
            }
        }
    };
    store_acc(acc0, p.out1, p.ld1);
    if constexpr (MODE == 1) store_acc(acc1, p.out2, p.ld2);
}

template <int KS, int MODE>
static int launch_attn_bwd(const CUtensorMap& x1, const CUtensorMap& x2, const CUtensorMap& y1, const CUtensorMap& y2,
                           const AttnBwdParams& p, dim3 grid, cudaStream_t st) {
    using Cfg = AttnBwdCfg<(KS + 3) / 4, MODE>;
    static bool done = false;
    auto kern = cb_attention_bwd_kernel<KS, MODE>;
    if (!done) {
        CB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
        done = true;
    }
    CB_LAUNCH((kern), grid, kAttnThreads, Cfg::kSmemBytes, st, x1, x2, y1, y2, p);
    CB_CUDA(cudaGetLastError());
    count_launches(1);
    return 0;
}

// the head dim's k16 step count as a template argument: d is a multiple of 8 up to 128, so ks = ceil(d / 16) is 1..8
template <int MODE>
static int launch_attn_bwd_ks(int ks, const CUtensorMap& x1, const CUtensorMap& x2, const CUtensorMap& y1,
                              const CUtensorMap& y2, const AttnBwdParams& p, dim3 grid, cudaStream_t st) {
    switch (ks) {
        case 1: return launch_attn_bwd<1, MODE>(x1, x2, y1, y2, p, grid, st);
        case 2: return launch_attn_bwd<2, MODE>(x1, x2, y1, y2, p, grid, st);
        case 3: return launch_attn_bwd<3, MODE>(x1, x2, y1, y2, p, grid, st);
        case 4: return launch_attn_bwd<4, MODE>(x1, x2, y1, y2, p, grid, st);
        case 5: return launch_attn_bwd<5, MODE>(x1, x2, y1, y2, p, grid, st);
        case 6: return launch_attn_bwd<6, MODE>(x1, x2, y1, y2, p, grid, st);
        case 7: return launch_attn_bwd<7, MODE>(x1, x2, y1, y2, p, grid, st);
        default: return launch_attn_bwd<8, MODE>(x1, x2, y1, y2, p, grid, st);
    }
}

static int attn_tmap(CUtensorMap* out, int dtype, const void* ptr, long long ld, int rows, int d, int heads, int images, int box_rows) {
    uint64_t dims[4] = {(uint64_t)d, (uint64_t)rows, (uint64_t)heads, (uint64_t)images};
    uint64_t str[3] = {(uint64_t)ld * 2, (uint64_t)d * 2, (uint64_t)rows * ld * 2};
    uint32_t box[4] = {64, (uint32_t)box_rows, 1, 1};
    uint32_t estr[4] = {1, 1, 1, 1};
    return make_tmap(out, dtype, 4, ptr, dims, str, box, estr);
}

}  // namespace cb

using namespace cb;


extern "C" int cb_attention_fwd(const void* Q, long long ldq, const void* K, long long ldk, const void* V, long long ldv,
                                void* O, long long ldo, float* lse, void* P, long long ldp, int dtype, int images,
                                int heads, int nq, int nk, int d, float scale, int causal, void* stream) {
    CB_REQUIRE(dtype == CB_F16 || dtype == CB_BF16, CB_ERR_ARG, "attention_fwd: dtype must be f16/bf16");
    CB_REQUIRE(Q && K && V && O && images > 0 && heads > 0 && nq > 0 && nk > 0 && scale > 0.f, CB_ERR_ARG, "attention_fwd: bad args");
    CB_REQUIRE(d >= 8 && d <= 128 && d % 8 == 0, CB_ERR_ARG, "attention_fwd: head dim %d unsupported (8..128, multiple of 8)", d);
    CB_REQUIRE((ldo * 2) % 16 == 0 && ((long long)d * 2) % 16 == 0 && (reinterpret_cast<uintptr_t>(O) & 15u) == 0,
               CB_ERR_ALIGN, "attention_fwd: O alignment");
    const int es = 2;
    AttnParams p;
    memset(&p, 0, sizeof(p));
    p.nq = nq; p.nk = nk; p.heads = heads; p.images = images;
    p.d = d;
    p.causal = causal;
    p.scale_log2e = scale * 1.4426950408889634f;
    p.O = O; p.ldo = ldo; p.lse = lse;
    p.P = P; p.ldp = ldp; p.is_bf16 = dtype == CB_BF16;
    p.two_pass = P != nullptr ? 1 : 0;
    if (P) CB_REQUIRE(ldp >= nk && ldp % 8 == 0 && (reinterpret_cast<uintptr_t>(P) & 15u) == 0, CB_ERR_ALIGN, "attention_fwd: P row pitch must be a multiple of 8 elements >= nk");
    CUtensorMap tq, tk, tv;
    uint32_t estr[4] = {1, 1, 1, 1};
    uint32_t box[4] = {64, kBQ, 1, 1};
    uint32_t boxkv[4] = {64, kBKV, 1, 1};
    {
        uint64_t dims[4] = {(uint64_t)d, (uint64_t)nq, (uint64_t)heads, (uint64_t)images};
        uint64_t str[3] = {(uint64_t)ldq * es, (uint64_t)d * es, (uint64_t)nq * ldq * es};
        int rc = make_tmap(&tq, dtype, 4, Q, dims, str, box, estr);
        if (rc) return rc;
    }
    {
        uint64_t dims[4] = {(uint64_t)d, (uint64_t)nk, (uint64_t)heads, (uint64_t)images};
        uint64_t str[3] = {(uint64_t)ldk * es, (uint64_t)d * es, (uint64_t)nk * ldk * es};
        int rc = make_tmap(&tk, dtype, 4, K, dims, str, boxkv, estr);
        if (rc) return rc;
        uint64_t strv[3] = {(uint64_t)ldv * es, (uint64_t)d * es, (uint64_t)nk * ldv * es};
        rc = make_tmap(&tv, dtype, 4, V, dims, strv, boxkv, estr);
        if (rc) return rc;
    }
    dim3 grid((unsigned)ceil_div(nq, kBQ), (unsigned)heads, (unsigned)images);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    int rc;
    switch ((d + 15) / 16) {      // k16 steps of the head dim (d is a multiple of 8 up to 128)
        case 1: rc = launch_attn<1>(tq, tk, tv, p, grid, st); break;
        case 2: rc = launch_attn<2>(tq, tk, tv, p, grid, st); break;
        case 3: rc = launch_attn<3>(tq, tk, tv, p, grid, st); break;
        case 4: rc = launch_attn<4>(tq, tk, tv, p, grid, st); break;
        case 5: rc = launch_attn<5>(tq, tk, tv, p, grid, st); break;
        case 6: rc = launch_attn<6>(tq, tk, tv, p, grid, st); break;
        case 7: rc = launch_attn<7>(tq, tk, tv, p, grid, st); break;
        default: rc = launch_attn<8>(tq, tk, tv, p, grid, st); break;
    }
    // causal P: zero the key blocks a query tile never visits (none when the first tile already visits every block)
    if (rc || !P || !causal || ceil_div(min(nq, kBQ), kBKV) >= ceil_div(nk, kBKV)) return rc;
    CB_LAUNCH((cb_attention_p_tail_kernel), grid, 128, 0, st, p);
    CB_CUDA(cudaGetLastError());
    count_launches(1);
    return 0;
}

static int attention_bwd_impl(const void* Q, long long ldq, const void* K, long long ldk, const void* V, long long ldv,
                              const void* O, long long ldo, const void* dO, long long lddo, const float* lse, float* delta,
                              void* dQ, long long lddq, void* dK, long long lddk, void* dV, long long lddv, void* dS,
                              long long ldds, bool run_dq, bool run_dkdv, int dtype, int images, int heads, int nq, int nk,
                              int d, float scale, int causal, void* stream) {
    CB_REQUIRE(dtype == CB_F16 || dtype == CB_BF16, CB_ERR_ARG, "attention_bwd: dtype must be f16/bf16");
    CB_REQUIRE(Q && K && V && O && dO && lse && delta && images > 0 && heads > 0 && nq > 0 && nk > 0 && scale > 0.f,
               CB_ERR_ARG, "attention_bwd: bad args");
    CB_REQUIRE(!run_dkdv || (dK && dV), CB_ERR_ARG, "attention_bwd: dK/dV required");
    CB_REQUIRE(d >= 8 && d <= 128 && d % 8 == 0, CB_ERR_ARG, "attention_bwd: head dim %d unsupported (8..128, multiple of 8)", d);
    const void* ptrs[8] = {Q, K, V, O, dO, dQ, dK, dV};
    const long long lds[8] = {ldq, ldk, ldv, ldo, lddo, lddq, lddk, lddv};
    for (int i = 0; i < 8; ++i)
        CB_REQUIRE(ptrs[i] == nullptr || ((lds[i] * 2) % 16 == 0 && (reinterpret_cast<uintptr_t>(ptrs[i]) & 15u) == 0), CB_ERR_ALIGN,
                   "attention_bwd: operand %d must be 16-byte aligned with a 16-byte multiple row pitch", i);
    if (dS) CB_REQUIRE(ldds >= nk && ldds % 8 == 0 && (reinterpret_cast<uintptr_t>(dS) & 15u) == 0, CB_ERR_ALIGN, "attention_bwd: dS row pitch must be a multiple of 8 elements >= nk");
    AttnBwdParams p;
    memset(&p, 0, sizeof(p));
    p.heads = heads; p.images = images; p.d = d;
    const int ks = (d + 15) / 16;
    p.causal = causal; p.scale = scale; p.scale_log2e = scale * 1.4426950408889634f;
    p.lse = lse; p.delta = delta; p.O = O; p.dO = dO; p.ldo = ldo; p.lddo = lddo;
    p.is_bf16 = dtype == CB_BF16; p.nq = nq;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    CUtensorMap x1, x2, y1, y2;
    int rc = 0;
    if (run_dq) {
        // ---- MODE 0: dQ (+ delta, + optional dS export) ----
        if ((rc = attn_tmap(&x1, dtype, Q, ldq, nq, d, heads, images, kBQ))) return rc;
        if ((rc = attn_tmap(&x2, dtype, dO, lddo, nq, d, heads, images, kBQ))) return rc;
        if ((rc = attn_tmap(&y1, dtype, K, ldk, nk, d, heads, images, kBKV))) return rc;
        if ((rc = attn_tmap(&y2, dtype, V, ldv, nk, d, heads, images, kBKV))) return rc;
        p.n_stat = nq; p.n_stream = nk; p.out1 = dQ; p.ld1 = lddq; p.out2 = nullptr; p.ld2 = 0; p.dS = dS; p.ldds = ldds;
        dim3 grid((unsigned)ceil_div(nq, kBQ), (unsigned)heads, (unsigned)images);
        rc = launch_attn_bwd_ks<0>(ks, x1, x2, y1, y2, p, grid, st);
        if (rc) return rc;
    }
    if (run_dkdv) {
        // ---- MODE 1: dK, dV ----
        if ((rc = attn_tmap(&x1, dtype, K, ldk, nk, d, heads, images, kBQ))) return rc;
        if ((rc = attn_tmap(&x2, dtype, V, ldv, nk, d, heads, images, kBQ))) return rc;
        if ((rc = attn_tmap(&y1, dtype, Q, ldq, nq, d, heads, images, kBKV))) return rc;
        if ((rc = attn_tmap(&y2, dtype, dO, lddo, nq, d, heads, images, kBKV))) return rc;
        p.n_stat = nk; p.n_stream = nq; p.out1 = dV; p.ld1 = lddv; p.out2 = dK; p.ld2 = lddk; p.dS = nullptr; p.ldds = 0;
        dim3 grid((unsigned)ceil_div(nk, kBQ), (unsigned)heads, (unsigned)images);
        rc = launch_attn_bwd_ks<1>(ks, x1, x2, y1, y2, p, grid, st);
    }
    return rc;
}

extern "C" int cb_attention_bwd(const void* Q, long long ldq, const void* K, long long ldk, const void* V, long long ldv,
                                const void* O, long long ldo, const void* dO, long long lddo, const float* lse, float* delta,
                                void* dQ, long long lddq, void* dK, long long lddk, void* dV, long long lddv, int dtype,
                                int images, int heads, int nq, int nk, int d, float scale, int causal, void* stream) {
    CB_REQUIRE(dQ != nullptr, CB_ERR_ARG, "attention_bwd: dQ required");
    return attention_bwd_impl(Q, ldq, K, ldk, V, ldv, O, ldo, dO, lddo, lse, delta, dQ, lddq, dK, lddk, dV, lddv, nullptr, 0,
                              true, true, dtype, images, heads, nq, nk, d, scale, causal, stream);
}

extern "C" int cb_attention_bwd_dq(const void* Q, long long ldq, const void* K, long long ldk, const void* V, long long ldv,
                                   const void* O, long long ldo, const void* dO, long long lddo, const float* lse,
                                   float* delta, void* dQ, long long lddq, void* dS, long long ldds, int dtype, int images,
                                   int heads, int nq, int nk, int d, float scale, int causal, void* stream) {
    CB_REQUIRE(dQ != nullptr || dS != nullptr, CB_ERR_ARG, "attention_bwd_dq: nothing to compute");
    return attention_bwd_impl(Q, ldq, K, ldk, V, ldv, O, ldo, dO, lddo, lse, delta, dQ, lddq, nullptr, 0, nullptr, 0, dS, ldds,
                              true, false, dtype, images, heads, nq, nk, d, scale, causal, stream);
}
