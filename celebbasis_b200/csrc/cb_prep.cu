// Checkpoint-load-time kernels: fp32 checkpoint tensors -> the 16-bit operand layouts the GEMM kernels read.
// (The reference keeps fp32 nn.Parameters and lets cuDNN pick layouts; here the packs are made once per load.)
#include "cb_common.cuh"

namespace cb {

__device__ __forceinline__ void st16(void* p, int dt, size_t i, float v) {
    if (dt == CB_F32) reinterpret_cast<float*>(p)[i] = v;
    else if (dt == CB_F16) reinterpret_cast<__half*>(p)[i] = __float2half_rn(v);
    else reinterpret_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(v);
}

// [Cout][Cin][kh][kw] fp32 -> [kh*kw][Cout_pad][Cin_pad] (tap-major, Cin contiguous), zero padded, optionally with a
// per-output-channel scale folded in (eval BatchNorm after the conv: iresnet.py:41-58)
__global__ void pack_conv_weight_kernel(const float* __restrict__ w, void* __restrict__ out, int o_dtype, int cout, int cin,
                                        int taps, int cout_pad, int cin_pad, const float* __restrict__ oscale) {
    const size_t total = (size_t)taps * cout_pad * cin_pad;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int ci = (int)(i % cin_pad);
        const size_t r = i / cin_pad;
        const int co = (int)(r % cout_pad);
        const int tap = (int)(r / cout_pad);
        float v = 0.f;
        if (co < cout && ci < cin) {
            v = w[((size_t)co * cin + ci) * taps + tap];
            if (oscale) v *= oscale[co];
        }
        st16(out, o_dtype, i, v);
    }
}

// plain element-wise convert of n fp32 values (any n; the 2-D cast kernel needs cols % 4 == 0)
__global__ void convert_f32_kernel(const float* __restrict__ x, void* __restrict__ out, int o_dtype, size_t n, float scale) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        st16(out, o_dtype, i, x[i] * scale);
}

static inline int grid_for(size_t n, int threads) {
    size_t g = (n + threads - 1) / threads;
    const size_t cap = (size_t)device_sm_count() * 16;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace cb

using namespace cb;

extern "C" int cb_pack_conv_weight(const float* w, void* out, int o_dtype, int cout, int cin, int kh, int kw, int cout_pad,
                                   int cin_pad, const float* out_scale, void* stream) {
    CB_REQUIRE(w && out && cout > 0 && cin > 0 && kh > 0 && kw > 0 && cout_pad >= cout && cin_pad >= cin, CB_ERR_ARG,
               "pack_conv_weight: bad args");
    CB_REQUIRE(o_dtype == CB_F16 || o_dtype == CB_BF16 || o_dtype == CB_F32, CB_ERR_ARG,
               "pack_conv_weight: unsupported dtype %d", o_dtype);
    const size_t total = (size_t)kh * kw * cout_pad * cin_pad;
    pack_conv_weight_kernel<<<grid_for(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        w, out, o_dtype, cout, cin, kh * kw, cout_pad, cin_pad, out_scale);
    CB_CUDA(cudaGetLastError());
    count_launches(1);
    return 0;
}

extern "C" int cb_convert_f32(const float* x, void* out, int o_dtype, long long n, float scale, void* stream) {
    CB_REQUIRE(x && out && n > 0, CB_ERR_ARG, "convert_f32: bad args");
    CB_REQUIRE(o_dtype == CB_F16 || o_dtype == CB_BF16 || o_dtype == CB_F32, CB_ERR_ARG,
               "convert_f32: unsupported dtype %d", o_dtype);
    convert_f32_kernel<<<grid_for((size_t)n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, out, o_dtype,
                                                                                                    (size_t)n, scale);
    CB_CUDA(cudaGetLastError());
    count_launches(1);
    return 0;
}
