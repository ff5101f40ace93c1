// HBM-bound pointwise / row-wise kernels of the hot path (channels-last, vectorised where the
// layout allows it).  Each entry point cites the reference arithmetic it replaces.
#include "cb_common.cuh"

namespace cb {

__device__ __forceinline__ float ld_any(const void* p, int dt, size_t i) {
    if (dt == CB_F32) return reinterpret_cast<const float*>(p)[i];
    if (dt == CB_F16) return __half2float(reinterpret_cast<const __half*>(p)[i]);
    return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
}
__device__ __forceinline__ void st_any(void* p, int dt, size_t i, float v) {
    if (dt == CB_F32) reinterpret_cast<float*>(p)[i] = v;
    else if (dt == CB_F16) reinterpret_cast<__half*>(p)[i] = __float2half_rn(v);
    else reinterpret_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(v);
}

// 4-wide typed access (16 B for f32, 8 B for 16-bit types)
template <typename T> struct V4;
template <> struct V4<float> {
    static __device__ __forceinline__ void ld(const float* p, float (&f)[4]) {
        const float4 v = *reinterpret_cast<const float4*>(p);
        f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
    }
    static __device__ __forceinline__ void st(float* p, const float (&f)[4]) {
        *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
    }
};
template <> struct V4<__half> {
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
template <> struct V4<__nv_bfloat16> {
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

// ---- out = a*x + b*y (y optional); 2-D strided so it also serves as cast / concat / split copy ---------
template <typename TX, typename TY, typename TO>
__global__ void axpby2d_kernel(const TX* __restrict__ x, long long ldx, float a, const TY* __restrict__ y,
                               long long ldy, float b, TO* __restrict__ o, long long ldo, long long rows, int cols4) {
    pdl_sync();
    const long long total = rows * cols4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / cols4;
        const int c = (int)(i - r * cols4) * 4;
        float fx[4], fo[4];
        V4<TX>::ld(x + r * ldx + c, fx);
        if (y) {
            float fy[4];
            V4<TY>::ld(y + r * ldy + c, fy);
#pragma unroll
            for (int k = 0; k < 4; ++k) fo[k] = a * fx[k] + b * fy[k];
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) fo[k] = a * fx[k];
        }
        V4<TO>::st(o + r * ldo + c, fo);
    }
}

// ---- unary activations -----------------------------------------------------------------------------------
__device__ __forceinline__ float act_fwd(float x, int act) {
    if (act == CB_ACT_SILU) return silu_f(x);
    if (act == CB_ACT_QUICK_GELU) return quick_gelu_f(x);
    if (act == CB_ACT_GELU) return gelu_f(x);
    return x;
}
__device__ __forceinline__ float act_grad(float x, int act) {
    if (act == CB_ACT_SILU) {
        const float s = 1.f / (1.f + __expf(-x));
        return s * (1.f + x * (1.f - s));
    }
    if (act == CB_ACT_QUICK_GELU) {
        const float s = 1.f / (1.f + __expf(-1.702f * x));
        return s * (1.f + 1.702f * x * (1.f - s));
    }
    if (act == CB_ACT_GELU) {
        const float cdf = 0.5f * (1.f + erff(x * 0.70710678118654752f));
        const float pdf = 0.3989422804014327f * __expf(-0.5f * x * x);
        return cdf + x * pdf;
    }
    return 1.f;
}

__global__ void act_fwd_kernel(const void* x, int xdt, void* y, int ydt, size_t n, int act) {
    pdl_sync();
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        st_any(y, ydt, i, act_fwd(ld_any(x, xdt, i), act));
}
__global__ void act_bwd_kernel(const void* dy, int gdt, const void* x, int xdt, void* dx, int ddt, size_t n, int act) {
    pdl_sync();
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        st_any(dx, ddt, i, ld_any(dy, gdt, i) * act_grad(ld_any(x, xdt, i), act));
}

// ---- GEGLU: out[m][f] = in[m][f] * gelu(in[m][F+f])  (ldm/modules/attention.py:37-45) ------------------------
template <typename T>
__global__ void geglu_fwd_kernel(const T* __restrict__ in, T* __restrict__ out, long long M, int F, int il) {
    pdl_sync();
    const int f4 = F >> 2;
    const long long total = M * f4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long m = i / f4;
        const int c = (int)(i - m * f4) * 4;
        float a[4], g[4], o[4];
        const int ao = il ? ((c >> 5) << 6) + (c & 31) : c;       // interleaved: 64-column groups of 32 values + 32 gates
        const int go = il ? ao + 32 : F + c;
        V4<T>::ld(in + m * 2 * F + ao, a);
        V4<T>::ld(in + m * 2 * F + go, g);
#pragma unroll
        for (int k = 0; k < 4; ++k) o[k] = a[k] * gelu_f(g[k]);
        V4<T>::st(out + m * F + c, o);
    }
}
template <typename T, typename TG>
__global__ void geglu_bwd_kernel(const TG* __restrict__ dout, const T* __restrict__ in, TG* __restrict__ din,
                                 long long M, int F, int il) {
    pdl_sync();
    const int f4 = F >> 2;
    const long long total = M * f4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long m = i / f4;
        const int c = (int)(i - m * f4) * 4;
        float a[4], g[4], d[4], da[4], dg[4];
        const int ao = il ? ((c >> 5) << 6) + (c & 31) : c;
        const int go = il ? ao + 32 : F + c;
        V4<T>::ld(in + m * 2 * F + ao, a);
        V4<T>::ld(in + m * 2 * F + go, g);
        V4<TG>::ld(dout + m * F + c, d);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            da[k] = d[k] * gelu_f(g[k]);
            dg[k] = d[k] * a[k] * act_grad(g[k], CB_ACT_GELU);
        }
        V4<TG>::st(din + m * 2 * F + ao, da);
        V4<TG>::st(din + m * 2 * F + go, dg);
    }
}

// ---- row softmax (attention.py:185 `sim.softmax(dim=-1)`; CLIP causal variant) -----------------------------
// One block per row.  Input scores already carry the d^-0.5 scale (GEMM alpha).  Columns >= ncols (row
// padding up to ld) are written as 0 so the P.V GEMM can read the padded row.
template <typename T>
__global__ void __launch_bounds__(128)
softmax_fwd_kernel(const T* __restrict__ s, T* __restrict__ p, int ncols, int ld, int causal_period) {
    pdl_sync();
    __shared__ float red[4];
    const long long row = blockIdx.x;
    const T* sr = s + row * ld;
    T* pr = p + row * ld;
    int limit = ncols;
    if (causal_period > 0) limit = min(ncols, (int)(row % causal_period) + 1);
    float mx = -INFINITY;
    for (int c = threadIdx.x; c < limit; c += 128) mx = fmaxf(mx, cvt<T>::to_f(sr[c]));
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
    __syncthreads();
    float sum = 0.f;
    for (int c = threadIdx.x; c < limit; c += 128) sum += __expf(cvt<T>::to_f(sr[c]) - mx);
    sum = warp_sum(sum);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
    __syncthreads();
    sum = red[0] + red[1] + red[2] + red[3];
    const float inv = 1.f / sum;
    for (int c = threadIdx.x; c < ld; c += 128) {
        const float v = c < limit ? __expf(cvt<T>::to_f(sr[c]) - mx) * inv : 0.f;
        pr[c] = cvt<T>::from_f(v);
    }
}
// dS = P * (dP - sum_j dP_j P_j)
template <typename T, typename TG>
__global__ void __launch_bounds__(128)
softmax_bwd_kernel(const TG* __restrict__ dp, const T* __restrict__ p, TG* __restrict__ ds, int ncols, int ld) {
    pdl_sync();
    __shared__ float red[4];
    const long long row = blockIdx.x;
    const TG* dr = dp + row * ld;
    const T* pr = p + row * ld;
    TG* or_ = ds + row * ld;
    float dot = 0.f;
    for (int c = threadIdx.x; c < ncols; c += 128) dot += cvt<TG>::to_f(dr[c]) * cvt<T>::to_f(pr[c]);
    dot = warp_sum(dot);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = dot;
    __syncthreads();
    dot = red[0] + red[1] + red[2] + red[3];
    for (int c = threadIdx.x; c < ld; c += 128) {
        const float v = c < ncols ? cvt<T>::to_f(pr[c]) * (cvt<TG>::to_f(dr[c]) - dot) : 0.f;
        or_[c] = cvt<TG>::from_f(v);
    }
}

// ---- nearest 2x upsample (openaimodel.py:112-117 F.interpolate(scale_factor=2, mode="nearest")) ------------
template <typename T>
__global__ void upsample2x_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, int N, int H, int W, int C4) {
    pdl_sync();
    const long long total = (long long)N * (2 * H) * (2 * W) * C4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C4);
        long long t = i / C4;
        const int ow = (int)(t % (2 * W)); t /= (2 * W);
        const int oh = (int)(t % (2 * H));
        const int n = (int)(t / (2 * H));
        const size_t src = ((((size_t)n * H + (oh >> 1)) * W + (ow >> 1)) * C4 + c) * 4;
        float f[4];
        V4<T>::ld(x + src, f);
        V4<T>::st(y + (size_t)i * 4, f);
    }
}
// dx[n][h][w] (+)= sum of the 2x2 block of dy
template <typename TG, typename TD>
__global__ void upsample2x_bwd_kernel(const TG* __restrict__ dy, TD* __restrict__ dx, int N, int H, int W, int C4,
                                      int accumulate) {
    pdl_sync();
    const long long total = (long long)N * H * W * C4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C4);
        long long t = i / C4;
        const int w = (int)(t % W); t /= W;
        const int h = (int)(t % H);
        const int n = (int)(t / H);
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int dh = 0; dh < 2; ++dh)
#pragma unroll
            for (int dw = 0; dw < 2; ++dw) {
                float f[4];
                V4<TG>::ld(dy + ((((size_t)n * 2 * H + 2 * h + dh) * 2 * W + 2 * w + dw) * C4 + c) * 4, f);
#pragma unroll
                for (int k = 0; k < 4; ++k) acc[k] += f[k];
            }
        if (accumulate) {
            float p[4];
            V4<TD>::ld(dx + (size_t)i * 4, p);
#pragma unroll
            for (int k = 0; k < 4; ++k) acc[k] += p[k];
        }
        V4<TD>::st(dx + (size_t)i * 4, acc);
    }
}
// zero-insertion (input of the stride-2 conv dgrad): z[n][2h][2w] = dy[n][h][w], other positions 0
template <typename T>
__global__ void zero_insert2x_kernel(const T* __restrict__ dy, T* __restrict__ z, int N, int H, int W, int C4) {
    pdl_sync();
    const long long total = (long long)N * (2 * H) * (2 * W) * C4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C4);
        long long t = i / C4;
        const int ow = (int)(t % (2 * W)); t /= (2 * W);
        const int oh = (int)(t % (2 * H));
        const int n = (int)(t / (2 * H));
        float f[4] = {0.f, 0.f, 0.f, 0.f};
        if (((oh | ow) & 1) == 0) V4<T>::ld(dy + ((((size_t)n * H + (oh >> 1)) * W + (ow >> 1)) * C4 + c) * 4, f);
        V4<T>::st(z + (size_t)i * 4, f);
    }
}

// ---- layout: NCHW fp32 <-> NHWC (channel-padded) (ddpm.py:344-350 rearrange 'b h w c -> b c h w') ------------
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, void* __restrict__ y, int ydt, int N, int C, int HW,
                                    int Cpad) {
    pdl_sync();
    const long long total = (long long)N * HW * Cpad;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % Cpad);
        const long long t = i / Cpad;
        const int p = (int)(t % HW);
        const int n = (int)(t / HW);
        const float v = c < C ? x[((size_t)n * C + c) * HW + p] : 0.f;
        st_any(y, ydt, (size_t)i, v);
    }
}
__global__ void nhwc_to_nchw_kernel(const void* __restrict__ x, int xdt, float* __restrict__ y, int N, int C, int HW,
                                    int Cpad) {
    pdl_sync();
    const long long total = (long long)N * C * HW;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int p = (int)(i % HW);
        const long long t = i / HW;
        const int c = (int)(t % C);
        const int n = (int)(t / C);
        y[i] = ld_any(x, xdt, ((size_t)n * HW + p) * Cpad + c);
    }
}

// ---- eps-MSE loss + its gradient (ddpm.py:294-307 get_loss 'l2', :1084-1096) -------------------------------
// loss[b] = mean_i (pred[b,i]-target[b,i])^2  (loss_simple, one value per sample; one CTA per sample, so the sum is
// taken in a fixed order);
// grad = d(mean_b loss[b]) / d pred * gscale = 2*(pred-target)/(B*per_sample) * gscale.
__global__ void mse_fwd_bwd_kernel(const float* __restrict__ pred, const float* __restrict__ target,
                                   float* __restrict__ loss, float* __restrict__ grad, int per_sample, float ginv,
                                   float gscale) {
    pdl_sync();
    __shared__ float red[32];
    const int b = blockIdx.y;
    const size_t base = (size_t)b * per_sample;
    float acc = 0.f;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < per_sample; i += gridDim.x * blockDim.x) {
        const float d = pred[base + i] - target[base + i];
        acc += d * d;
        if (grad) grad[base + i] = 2.f * d * ginv * gscale;
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
        loss[b] = s / (float)per_sample;
    }
}

// ---- sinusoidal timestep embedding (diffusionmodules/util.py:151-171) ----------------------------------------
__global__ void timestep_embedding_kernel(const long long* __restrict__ t, void* __restrict__ out, int odt, int B,
                                          int dim, float max_period) {
    pdl_sync();
    const int half = dim / 2;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * half) return;
    const int b = i / half, k = i - b * half;
    const float freq = expf(-logf(max_period) * (float)k / (float)half);
    const float arg = (float)t[b] * freq;
    st_any(out, odt, (size_t)b * dim + k, cosf(arg));
    st_any(out, odt, (size_t)b * dim + half + k, sinf(arg));
    if ((dim & 1) && k == 0) st_any(out, odt, (size_t)b * dim + dim - 1, 0.f);
}

// ---- per-channel affine (+ optional PReLU): eval-mode BatchNorm2d / nn.PReLU of iresnet.py:26-64 -------------
template <typename T, typename TY>
__global__ void channel_affine_act_kernel(const T* __restrict__ x, TY* __restrict__ y, const float* __restrict__ scale,
                                          const float* __restrict__ shift, const float* __restrict__ slope,
                                          long long rows, int C4) {
    pdl_sync();
    const long long total = rows * C4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C4) * 4;
        float f[4];
        V4<T>::ld(x + i * 4, f);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            float v = f[k];
            if (scale) v = v * scale[c + k] + shift[c + k];
            if (slope) v = v > 0.f ? v : v * slope[c + k];
            f[k] = v;
        }
        V4<TY>::st(y + i * 4, f);
    }
}

// ---- face crop for the CosFace backbone: affine_grid + grid_sample(bilinear, zeros, align_corners) then
//      bilinear resize to out_hw x out_hw (align_corners) -- meta_net.py:253-262.  faces is [B][H][W][6]
//      (two stacked RGB crops, face_id.py:598-644); output image f = chunk*B + b, NHWC with Cpad channels.
__device__ __forceinline__ float warp_src(const float* __restrict__ img, int H, int W, int cstride, float gy, float gx) {
    // grid_sample with align_corners=True: normalised (gx,gy) -> pixel coordinates, zero padding
    const float ix = (gx + 1.f) * 0.5f * (W - 1), iy = (gy + 1.f) * 0.5f * (H - 1);
    const float x0f = floorf(ix), y0f = floorf(iy);
    const int x0 = (int)x0f, y0 = (int)y0f, x1 = x0 + 1, y1 = y0 + 1;
    const float wx1 = ix - x0f, wy1 = iy - y0f, wx0 = 1.f - wx1, wy0 = 1.f - wy1;
    float acc = 0.f;
    if (y0 >= 0 && y0 < H) {
        if (x0 >= 0 && x0 < W) acc += img[((size_t)y0 * W + x0) * cstride] * wy0 * wx0;
        if (x1 >= 0 && x1 < W) acc += img[((size_t)y0 * W + x1) * cstride] * wy0 * wx1;
    }
    if (y1 >= 0 && y1 < H) {
        if (x0 >= 0 && x0 < W) acc += img[((size_t)y1 * W + x0) * cstride] * wy1 * wx0;
        if (x1 >= 0 && x1 < W) acc += img[((size_t)y1 * W + x1) * cstride] * wy1 * wx1;
    }
    return acc;
}
__global__ void face_warp_resize_kernel(const float* __restrict__ faces, void* __restrict__ out, int odt, int B, int H,
                                        int W, int n_chunks, int out_hw, int Cpad, float m00, float m01, float m02,
                                        float m10, float m11, float m12) {
    pdl_sync();
    const int total = n_chunks * B * out_hw * out_hw * Cpad;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int c = idx % Cpad;
    int t = idx / Cpad;
    const int j = t % out_hw; t /= out_hw;
    const int i = t % out_hw;
    const int f = t / out_hw;
    float v = 0.f;
    if (c < 3) {
        const int chunk = f / B, b = f - chunk * B;
        const int cs = 3 * n_chunks;
        const float* img = faces + (size_t)b * H * W * cs + chunk * 3 + c;
        const float sy = (float)i * (float)(H - 1) / (float)(out_hw - 1);
        const float sx = (float)j * (float)(W - 1) / (float)(out_hw - 1);
        const int y0 = (int)floorf(sy), x0 = (int)floorf(sx);
        const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
        const float ly = sy - y0, lx = sx - x0;
        const int ys[2] = {y0, y1}, xs[2] = {x0, x1};
        const float wy[2] = {1.f - ly, ly}, wx[2] = {1.f - lx, lx};
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int bb = 0; bb < 2; ++bb) {
                // warped pixel (ys[a], xs[bb]) = grid_sample(img, affine_grid)
                const float gx0 = -1.f + 2.f * xs[bb] / (float)(W - 1);
                const float gy0 = -1.f + 2.f * ys[a] / (float)(H - 1);
                const float gx = m00 * gx0 + m01 * gy0 + m02;
                const float gy = m10 * gx0 + m11 * gy0 + m12;
                v += wy[a] * wx[bb] * warp_src(img, H, W, cs, gy, gx);
            }
    }
    st_any(out, odt, (size_t)idx, v);
}

// ---- row L2 normalise: F.normalize(x, dim=-1, p=2) (meta_net.py:264) ------------------------------------------
__global__ void l2norm_rows_kernel(const float* __restrict__ x, float* __restrict__ y, int D) {
    pdl_sync();
    __shared__ float red[8];
    const float* xr = x + (size_t)blockIdx.x * D;
    float q = 0.f;
    for (int i = threadIdx.x; i < D; i += blockDim.x) q += xr[i] * xr[i];
    q = warp_sum(q);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = q;
    __syncthreads();
    float s = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
    const float inv = 1.f / fmaxf(sqrtf(s), 1e-12f);
    for (int i = threadIdx.x; i < D; i += blockDim.x) y[(size_t)blockIdx.x * D + i] = xr[i] * inv;
}

static inline int grid_for(long long n, int threads) {
    long long b = (n + threads - 1) / threads;
    const long long cap = 32LL * device_sm_count();
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return (int)b;
}

}  // namespace cb

using namespace cb;

#define CB_DISPATCH(dtype, T, ...)                                               \
    if ((dtype) == CB_F32) { using T = float; __VA_ARGS__; }                     \
    else if ((dtype) == CB_F16) { using T = __half; __VA_ARGS__; }               \
    else if ((dtype) == CB_BF16) { using T = __nv_bfloat16; __VA_ARGS__; }       \
    else { cb::set_error("unsupported dtype %d", (int)(dtype)); return CB_ERR_ARG; }
#define CB_DISPATCH16(dtype, T, ...)                                             \
    if ((dtype) == CB_F16) { using T = __half; __VA_ARGS__; }                    \
    else if ((dtype) == CB_BF16) { using T = __nv_bfloat16; __VA_ARGS__; }       \
    else { cb::set_error("dtype %d must be f16/bf16", (int)(dtype)); return CB_ERR_ARG; }

// element size of a CB_F16 / CB_BF16 / CB_F32 code, 0 for any other code
static inline int dt_size(int dt) { return dt == CB_F32 ? 4 : (dt == CB_F16 || dt == CB_BF16) ? 2 : 0; }
static inline bool act_ok(int act) {
    return act == CB_ACT_NONE || act == CB_ACT_SILU || act == CB_ACT_GELU || act == CB_ACT_QUICK_GELU;
}
// the V4 accesses move 4 elements at once: 16 B for fp32, 8 B for the 16-bit types
static inline bool vec4_aligned(const void* p, int dt) {
    return (reinterpret_cast<uintptr_t>(p) & (uintptr_t)(4 * dt_size(dt) - 1)) == 0;
}

extern "C" int cb_axpby2d(const void* x, int x_dtype, long long ldx, float a, const void* y, int y_dtype,
                          long long ldy, float b, void* out, int o_dtype, long long ldo, long long rows, int cols,
                          void* stream) {
    CB_REQUIRE(rows > 0 && cols > 0 && cols % 4 == 0 && ldx % 4 == 0 && ldo % 4 == 0 && (y == nullptr || ldy % 4 == 0),
               CB_ERR_ARG, "axpby2d: cols/ld must be multiples of 4 (rows=%lld cols=%d)", rows, cols);
    if (y == nullptr) y_dtype = x_dtype;
    CB_REQUIRE(dt_size(x_dtype) && dt_size(y_dtype) && dt_size(o_dtype), CB_ERR_ARG, "axpby2d: unsupported dtype");
    CB_REQUIRE(vec4_aligned(x, x_dtype) && (y == nullptr || vec4_aligned(y, y_dtype)) && vec4_aligned(out, o_dtype),
               CB_ERR_ALIGN, "axpby2d: x, y and out must be aligned to 4 elements");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int c4 = cols / 4;
    const int grid = grid_for(rows * c4, 256);
    CB_DISPATCH(x_dtype, TX, CB_DISPATCH(y_dtype, TY, CB_DISPATCH(o_dtype, TO,
CB_LAUNCH((axpby2d_kernel<TX, TY, TO>), grid, 256, 0, st, (const TX*)x, ldx, a, (const TY*)y, ldy, b, (TO*)out, ldo, rows, c4))));
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_act_fwd(const void* x, int x_dtype, void* y, int y_dtype, long long n, int act, void* stream) {
    CB_REQUIRE(n > 0, CB_ERR_ARG, "act_fwd: n<=0");
    CB_REQUIRE(dt_size(x_dtype) && dt_size(y_dtype) && act_ok(act), CB_ERR_ARG, "act_fwd: unsupported dtype or act %d", act);
CB_LAUNCH((act_fwd_kernel), grid_for(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream), x, x_dtype, y, y_dtype, (size_t)n, act);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}
extern "C" int cb_act_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, void* dx, int dx_dtype,
                          long long n, int act, void* stream) {
    CB_REQUIRE(n > 0, CB_ERR_ARG, "act_bwd: n<=0");
    CB_REQUIRE(dt_size(dy_dtype) && dt_size(x_dtype) && dt_size(dx_dtype) && act_ok(act), CB_ERR_ARG,
               "act_bwd: unsupported dtype or act %d", act);
CB_LAUNCH((act_bwd_kernel), grid_for(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream), dy, dy_dtype, x, x_dtype, dx, dx_dtype, (size_t)n, act);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_geglu_fwd(const void* in, void* out, int dtype, long long M, int F, int interleave, void* stream) {
    CB_REQUIRE(M > 0 && F > 0 && F % (interleave ? 32 : 4) == 0, CB_ERR_ARG, "geglu_fwd: bad shape");
    CB_REQUIRE(dt_size(dtype) == 2, CB_ERR_ARG, "geglu_fwd: dtype %d must be f16/bf16", dtype);
    CB_REQUIRE(vec4_aligned(in, dtype) && vec4_aligned(out, dtype), CB_ERR_ALIGN,
               "geglu_fwd: in and out must be 8-byte aligned");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    CB_DISPATCH16(dtype, T,CB_LAUNCH((geglu_fwd_kernel<T>), grid_for(M * (F / 4), 256), 256, 0, st, (const T*)in, (T*)out, M, F, interleave));
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}
extern "C" int cb_geglu_bwd(const void* dout, const void* in, void* din, int dtype, int g_dtype, long long M, int F,
                            int interleave, void* stream) {
    CB_REQUIRE(M > 0 && F > 0 && F % (interleave ? 32 : 4) == 0, CB_ERR_ARG, "geglu_bwd: bad shape");
    CB_REQUIRE(dt_size(dtype) == 2 && dt_size(g_dtype) == 2, CB_ERR_ARG, "geglu_bwd: dtypes must be f16/bf16");
    CB_REQUIRE(vec4_aligned(dout, g_dtype) && vec4_aligned(in, dtype) && vec4_aligned(din, g_dtype), CB_ERR_ALIGN,
               "geglu_bwd: dout, in and din must be 8-byte aligned");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    CB_DISPATCH16(dtype, T, CB_DISPATCH16(g_dtype, TG,
CB_LAUNCH((geglu_bwd_kernel<T, TG>), grid_for(M * (F / 4), 256), 256, 0, st, (const TG*)dout, (const T*)in, (TG*)din, M, F, interleave)));
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_softmax_fwd(const void* s, void* p, int dtype, long long rows, int ncols, int ld, int causal_period,
                              void* stream) {
    CB_REQUIRE(rows > 0 && ncols > 0 && ld >= ncols, CB_ERR_ARG, "softmax_fwd: bad shape");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    CB_DISPATCH16(dtype, T,CB_LAUNCH((softmax_fwd_kernel<T>), (unsigned)rows, 128, 0, st, (const T*)s, (T*)p, ncols, ld, causal_period));
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}
extern "C" int cb_softmax_bwd(const void* dp, const void* p, void* ds, int p_dtype, int g_dtype, long long rows,
                              int ncols, int ld, void* stream) {
    CB_REQUIRE(rows > 0 && ncols > 0 && ld >= ncols, CB_ERR_ARG, "softmax_bwd: bad shape");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    CB_DISPATCH16(p_dtype, T, CB_DISPATCH16(g_dtype, TG,
CB_LAUNCH((softmax_bwd_kernel<T, TG>), (unsigned)rows, 128, 0, st, (const TG*)dp, (const T*)p, (TG*)ds, ncols, ld)));
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_upsample2x_fwd(const void* x, void* y, int dtype, int N, int H, int W, int C, void* stream) {
    CB_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0, CB_ERR_ARG, "upsample2x_fwd: bad shape");
    CB_REQUIRE(dt_size(dtype), CB_ERR_ARG, "upsample2x_fwd: unsupported dtype %d", dtype);
    CB_REQUIRE(vec4_aligned(x, dtype) && vec4_aligned(y, dtype), CB_ERR_ALIGN,
               "upsample2x_fwd: x and y must be aligned to 4 elements");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long total = (long long)N * 4 * H * W * (C / 4);
    CB_DISPATCH(dtype, T,CB_LAUNCH((upsample2x_fwd_kernel<T>), grid_for(total, 256), 256, 0, st, (const T*)x, (T*)y, N, H, W, C / 4));
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}
extern "C" int cb_upsample2x_bwd(const void* dy, int dy_dtype, void* dx, int dx_dtype, int N, int H, int W, int C,
                                 int accumulate, void* stream) {
    CB_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0, CB_ERR_ARG, "upsample2x_bwd: bad shape");
    CB_REQUIRE(dt_size(dy_dtype) && dt_size(dx_dtype), CB_ERR_ARG, "upsample2x_bwd: unsupported dtype");
    CB_REQUIRE(vec4_aligned(dy, dy_dtype) && vec4_aligned(dx, dx_dtype), CB_ERR_ALIGN,
               "upsample2x_bwd: dy and dx must be aligned to 4 elements");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long total = (long long)N * H * W * (C / 4);
    CB_DISPATCH(dy_dtype, TG, CB_DISPATCH(dx_dtype, TD,
CB_LAUNCH((upsample2x_bwd_kernel<TG, TD>), grid_for(total, 256), 256, 0, st, (const TG*)dy, (TD*)dx, N, H, W, C / 4, accumulate)));
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}
extern "C" int cb_zero_insert2x(const void* dy, void* z, int dtype, int N, int H, int W, int C, void* stream) {
    CB_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0, CB_ERR_ARG, "zero_insert2x: bad shape");
    CB_REQUIRE(dt_size(dtype), CB_ERR_ARG, "zero_insert2x: unsupported dtype %d", dtype);
    CB_REQUIRE(vec4_aligned(dy, dtype) && vec4_aligned(z, dtype), CB_ERR_ALIGN,
               "zero_insert2x: dy and z must be aligned to 4 elements");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long total = (long long)N * 4 * H * W * (C / 4);
    CB_DISPATCH(dtype, T,CB_LAUNCH((zero_insert2x_kernel<T>), grid_for(total, 256), 256, 0, st, (const T*)dy, (T*)z, N, H, W, C / 4));
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_nchw_to_nhwc(const float* x, void* y, int y_dtype, int N, int C, int HW, int Cpad, void* stream) {
    CB_REQUIRE(N > 0 && C > 0 && HW > 0 && Cpad >= C, CB_ERR_ARG, "nchw_to_nhwc: bad shape");
    CB_REQUIRE(dt_size(y_dtype), CB_ERR_ARG, "nchw_to_nhwc: unsupported dtype %d", y_dtype);
CB_LAUNCH((nchw_to_nhwc_kernel), grid_for((long long)N * HW * Cpad, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream), x, y, y_dtype, N, C, HW, Cpad);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}
extern "C" int cb_nhwc_to_nchw(const void* x, int x_dtype, float* y, int N, int C, int HW, int Cpad, void* stream) {
    CB_REQUIRE(N > 0 && C > 0 && HW > 0 && Cpad >= C, CB_ERR_ARG, "nhwc_to_nchw: bad shape");
    CB_REQUIRE(dt_size(x_dtype), CB_ERR_ARG, "nhwc_to_nchw: unsupported dtype %d", x_dtype);
CB_LAUNCH((nhwc_to_nchw_kernel), grid_for((long long)N * HW * C, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream), x, x_dtype, y, N, C, HW, Cpad);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_mse_fwd_bwd(const float* pred, const float* target, float* loss, float* grad, int B,
                              int per_sample, float gscale, void* stream) {
    CB_REQUIRE(B > 0 && per_sample > 0 && pred && target && loss, CB_ERR_ARG, "mse: bad args");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    CB_LAUNCH((mse_fwd_bwd_kernel), dim3(1, B), 1024, 0, st, pred, target, loss, grad, per_sample,
                                                    1.f / ((float)B * (float)per_sample), gscale);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_timestep_embedding(const long long* t, void* out, int o_dtype, int B, int dim, float max_period,
                                     void* stream) {
    CB_REQUIRE(B > 0 && dim >= 2, CB_ERR_ARG, "timestep_embedding: bad shape");
    CB_REQUIRE(dt_size(o_dtype), CB_ERR_ARG, "timestep_embedding: unsupported dtype %d", o_dtype);
    const int n = B * (dim / 2);
CB_LAUNCH((timestep_embedding_kernel), ceil_div(n, 128), 128, 0, reinterpret_cast<cudaStream_t>(stream), t, out, o_dtype, B, dim, max_period);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_channel_affine_act(const void* x, int x_dtype, void* y, int y_dtype, const float* scale,
                                     const float* shift, const float* slope, long long rows, int C, void* stream) {
    CB_REQUIRE(rows > 0 && C > 0 && C % 4 == 0, CB_ERR_ARG, "channel_affine_act: bad shape");
    CB_REQUIRE((scale == nullptr) == (shift == nullptr), CB_ERR_ARG, "channel_affine_act: scale and shift go together");
    CB_REQUIRE(dt_size(x_dtype) && dt_size(y_dtype), CB_ERR_ARG, "channel_affine_act: unsupported dtype");
    CB_REQUIRE(vec4_aligned(x, x_dtype) && vec4_aligned(y, y_dtype), CB_ERR_ALIGN,
               "channel_affine_act: x and y must be aligned to 4 elements");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    CB_DISPATCH(x_dtype, T, CB_DISPATCH(y_dtype, TY,
CB_LAUNCH((channel_affine_act_kernel<T, TY>), grid_for(rows * (C / 4), 256), 256, 0, st, (const T*)x, (TY*)y, scale, shift, slope, rows, C / 4)));
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_face_warp_resize(const float* faces, void* out, int o_dtype, int B, int H, int W, int n_chunks,
                                   int out_hw, int Cpad, const float* host_affine6, void* stream) {
    CB_REQUIRE(B > 0 && H > 1 && W > 1 && n_chunks > 0 && out_hw > 1 && Cpad >= 3 && host_affine6, CB_ERR_ARG, "face_warp_resize: bad args");
    CB_REQUIRE(dt_size(o_dtype), CB_ERR_ARG, "face_warp_resize: unsupported dtype %d", o_dtype);
    const int total = n_chunks * B * out_hw * out_hw * Cpad;
CB_LAUNCH((face_warp_resize_kernel), ceil_div(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream), 
        faces, out, o_dtype, B, H, W, n_chunks, out_hw, Cpad, host_affine6[0], host_affine6[1], host_affine6[2],
        host_affine6[3], host_affine6[4], host_affine6[5]);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_l2norm_rows(const float* x, float* y, int rows, int D, void* stream) {
    CB_REQUIRE(rows > 0 && D > 0, CB_ERR_ARG, "l2norm_rows: bad shape");
CB_LAUNCH((l2norm_rows_kernel), rows, 256, 0, reinterpret_cast<cudaStream_t>(stream), x, y, D);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}
