// celebbasis_b200 — shared device/host helpers for the sm_90a kernels.
//
// Everything here is hand-written PTX wrappers for the Hopper execution model
// (mbarrier, TMA bulk-tensor loads, wgmma, thread-block clusters) plus the error plumbing of the
// C-ABI.  No CUTLASS/CuTe types are used; bit layouts of the wgmma descriptors follow the
// PTX ISA tables.
#pragma once

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/celebbasis_b200.h"
#include "cb_wgmma.cuh"

namespace cb {

// ---------------------------------------------------------------------------------------------
// error plumbing (thread-local message; C-ABI returns int codes, never throws)
// ---------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int  check_cuda(cudaError_t e, const char* what);

#define CB_REQUIRE(cond, code, ...)                      \
    do {                                                 \
        if (!(cond)) {                                   \
            ::cb::set_error(__VA_ARGS__);                \
            return (code);                               \
        }                                                \
    } while (0)

#define CB_CUDA(call)                                                 \
    do {                                                              \
        int _cb_rc = ::cb::check_cuda((call), #call);                 \
        if (_cb_rc != 0) return _cb_rc;                               \
    } while (0)

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

int device_sm_count();
// one-warp-per-row LayerNorm (cb_norm.cu): fallback of the vectorised kernels in cb_layernorm.cu
int layernorm_fwd_legacy(const void* x, int x_dtype, void* y, int y_dtype, const float* gamma, const float* beta, int M,
                         int C, float eps, float* mean_out, float* rstd_out, void* stream);
int layernorm_bwd_legacy(const void* dy, int dy_dtype, const void* x, int x_dtype, const float* gamma, const float* mean,
                         const float* rstd, void* dx, int dx_dtype, void* dx_lp, int M, int C, int accumulate,
                         void* stream);
void count_launches(int n);  // bookkeeping for cb_launch_count()
bool pdl_enabled();          // programmatic dependent launch on (default) unless CB_PDL=0

#if defined(__CUDACC__)
// Every kernel is launched with the programmatic-stream-serialization attribute: its CTAs may be scheduled while the
// previous kernel in the stream drains (prologue overlap); the kernel itself calls pdl_sync() before touching memory
// the predecessor may still be writing.  Also valid under stream capture (programmatic graph edges).
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                        Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
// same, as thread-block clusters of `cluster` CTAs (runtime cluster shape)
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_kernel_cluster(void (*kern)(KArgs...), dim3 grid, dim3 block, dim3 cluster, size_t smem,
                                                cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[2];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = cluster.x;
    at[0].val.clusterDim.y = cluster.y;
    at[0].val.clusterDim.z = cluster.z;
    at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = pdl_enabled() ? 2 : 1;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
#define CB_LAUNCH(kern, grid, block, smem, st, ...) \
    ::cb::launch_kernel(kern, dim3(grid), dim3(block), (size_t)(smem), (st), ##__VA_ARGS__)
#endif

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
#if defined(__CUDACC__)

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }

// Programmatic dependent launch: let the next kernel's CTAs be scheduled, then wait until the previous kernel in the
// stream has completed and its writes are visible.  No-ops when the kernel was launched without the attribute.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_sync() {
    pdl_launch_dependents();
    pdl_wait();
}

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n"
        ".reg .pred P;\n"
        "elect.sync _|P, 0xffffffff;\n"
        "selp.u32 %0, 1, 0, P;\n"
        "}\n"
        : "=r"(pred));
    return pred != 0;
}

// ---- mbarrier ---------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred P;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n"
        "selp.u32 %0, 1, 0, P;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug must trap (context error -> host sees it) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    // the poll loop shares issue slots with the compute warps: keep it to try_wait + branch (no clock reads)
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > (1u << 26)) __trap();     // seconds of polling: protocol bug
    }
}

// ---- TMA ----------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0,
                                            int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], "
        "[%2];" ::"r"(dst),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0,
                                            int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, "
        "%5}], [%2];" ::"r"(dst),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0,
                                            int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, "
        "%5, %6}], [%2];" ::"r"(dst),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// 1-D bulk copy global -> shared (TMA engine, no tensor map): one instruction moves up to ~1 MiB and completes on an mbarrier
__device__ __forceinline__ void tma_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar)
                 : "memory");
}

// ---- wgmma (warpgroup MMA, fp32 accumulators in registers) -----------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keep the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// named barrier over `n` threads (n a multiple of 32); ids 0..15
__device__ __forceinline__ void named_bar(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// 32 bytes (8 floats) into the shared memory of CTA `cta` of the cluster at the offset `addr` has in this CTA
__device__ __forceinline__ void st_cluster_f32x8(uint32_t addr, uint32_t cta, const uint32_t* v) {
    asm volatile(
        "{\n"
        ".reg .b32 ra;\n"
        "mapa.shared::cluster.u32 ra, %0, %1;\n"
        "st.shared::cluster.v4.b32 [ra], {%2, %3, %4, %5};\n"
        "st.shared::cluster.v4.b32 [ra + 16], {%6, %7, %8, %9};\n"
        "}\n" ::"r"(addr),
        "r"(cta), "r"(v[0]), "r"(v[1]), "r"(v[2]), "r"(v[3]), "r"(v[4]), "r"(v[5]), "r"(v[6]), "r"(v[7])
        : "memory");
}
__device__ __forceinline__ void st_cluster_f32x2(uint32_t addr, uint32_t cta, float a, float b) {
    asm volatile(
        "{\n"
        ".reg .b32 ra;\n"
        "mapa.shared::cluster.u32 ra, %0, %1;\n"
        "st.shared::cluster.v2.f32 [ra], {%2, %3};\n"
        "}\n" ::"r"(addr),
        "r"(cta), "f"(a), "f"(b)
        : "memory");
}
// split cluster barrier: arrive early (all CTAs of the cluster have started once everyone's wait returns), wait late
__device__ __forceinline__ void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ float4 ld_shared_f32x4(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
    return v;
}

// ---- wgmma shared-memory matrix descriptor (SWIZZLE_128B) ---------------------------------------------------
// [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [49,52) base offset (0: 1 KiB aligned atoms) | [62,64) layout (1 = 128B
// swizzle).  K-major: SBO = 1024 (8-row groups), LBO unused; a 16-element k step adds 32 bytes to the start address.
// MN-major: LBO = bytes between 64-element MN blocks, SBO = 1024 (8 k rows); a 16-row k step adds 2048 bytes.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
    d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
    d |= static_cast<uint64_t>(1) << 62;
    return d;
}

// ---- small math ---------------------------------------------------------------------------------------
__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
__device__ __forceinline__ float quick_gelu_f(float x) { return x / (1.0f + __expf(-1.702f * x)); }
__device__ __forceinline__ float gelu_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

template <typename T> struct cvt;
template <> struct cvt<__half> {
    static __device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
    static __device__ __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
};
template <> struct cvt<__nv_bfloat16> {
    static __device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
    static __device__ __forceinline__ __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};
template <> struct cvt<float> {
    static __device__ __forceinline__ float to_f(float v) { return v; }
    static __device__ __forceinline__ float from_f(float v) { return v; }
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

#endif  // __CUDACC__

}  // namespace cb
