// Device-side data path of FaceIdDatasetStyleGAN3.__getitem__ (ldm/data/face_id.py:526-532 transform chain, :451-470
// _add_bg, :598-644): horizontal flip, ColorJitter (brightness / contrast / saturation / hue in the drawn order), ToTensor,
// Normalize(0.5, 0.5) and the random rescale + paste onto a -1 background.  The random DRAWS stay on the host (a handful
// of scalars per sample, drawn with the same torch / numpy calls in the same order as the reference); the pixel work -- 8
// PIL workers in the reference -- runs here.  Colour arithmetic follows torchvision's tensor kernels
// (transforms/_functional_tensor.py: _blend, rgb_to_grayscale, _rgb2hsv, _hsv2rgb); geometry follows
// F.interpolate(mode='bilinear', align_corners=True) (ATen UpSampleBilinear2d index math).
#include <algorithm>

#include "cb_common.cuh"

namespace cb {

__device__ __forceinline__ float clamp01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }
__device__ __forceinline__ float gray_of(float r, float g, float b) { return 0.2989f * r + 0.587f * g + 0.114f * b; }

__device__ __forceinline__ void hue_shift(float& r, float& g, float& b, float hf) {
    const float maxc = fmaxf(r, fmaxf(g, b)), minc = fminf(r, fminf(g, b));
    const bool eqc = maxc == minc;
    const float cr = maxc - minc;
    const float s = cr / (eqc ? 1.f : maxc);
    const float div = eqc ? 1.f : cr;
    const float rc = (maxc - r) / div, gc = (maxc - g) / div, bc = (maxc - b) / div;
    float h = 0.f;
    if (maxc == r) h = bc - gc;
    else if (maxc == g) h = 2.f + rc - bc;
    else h = 4.f + gc - rc;
    h = fmodf(h / 6.f + 1.f, 1.f);
    h = h + hf;
    h = h - floorf(h);                         // python (h + hue_factor) % 1.0
    const float v = maxc;
    const float i_f = floorf(h * 6.f);
    const float f = h * 6.f - i_f;
    int i = (int)i_f;
    i = ((i % 6) + 6) % 6;
    const float p = clamp01(v * (1.f - s));
    const float q = clamp01(v * (1.f - s * f));
    const float t = clamp01(v * (1.f - s * (1.f - f)));
    switch (i) {
        case 0: r = v; g = t; b = p; break;
        case 1: r = q; g = v; b = p; break;
        case 2: r = p; g = v; b = t; break;
        case 3: r = p; g = q; b = v; break;
        case 4: r = t; g = p; b = v; break;
        default: r = v; g = p; b = q; break;
    }
}

// applies the ops order[0..n_ops) (0 brightness, 1 contrast, 2 saturation, 3 hue; < 0 = skip) to one pixel
__device__ __forceinline__ void jitter_pixel(float& r, float& g, float& b, const int* order, const float* fac, int n_ops,
                                             float cmean) {
    for (int k = 0; k < n_ops; ++k) {
        const int op = order[k];
        if (op == 0) {
            const float f = fac[0];
            r = clamp01(f * r); g = clamp01(f * g); b = clamp01(f * b);
        } else if (op == 1) {
            const float f = fac[1], m = (1.f - f) * cmean;
            r = clamp01(f * r + m); g = clamp01(f * g + m); b = clamp01(f * b + m);
        } else if (op == 2) {
            const float f = fac[2], gy = (1.f - f) * gray_of(r, g, b);
            r = clamp01(f * r + gy); g = clamp01(f * g + gy); b = clamp01(f * b + gy);
        } else if (op == 3) {
            hue_shift(r, g, b, fac[3]);
        }
    }
}

// iparams [B][5] = {flip, order0..3}; fparams [B][4] = {brightness, contrast, saturation, hue}
// pass 1: sum over the image of gray(ops before the contrast op) -> gsum[b] (double); one CTA per image, so the sum is
// taken in a fixed order
__global__ void jitter_mean_kernel(const uint8_t* __restrict__ src, const int* __restrict__ iparams,
                                   const float* __restrict__ fparams, double* __restrict__ gsum, int HW) {
    const int b = blockIdx.y;
    const int* ip = iparams + b * 5;
    const float* fp = fparams + b * 4;
    int n_before = -1;
    for (int k = 0; k < 4; ++k)
        if (ip[1 + k] == 1) { n_before = k; break; }
    float acc = 0.f;
    if (n_before >= 0) {
        const uint8_t* s = src + (size_t)b * HW * 3;
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
            float r = s[3 * i] * (1.f / 255.f), g = s[3 * i + 1] * (1.f / 255.f), bl = s[3 * i + 2] * (1.f / 255.f);
            jitter_pixel(r, g, bl, ip + 1, fp, n_before, 0.f);
            acc += gray_of(r, g, bl);
        }
    }
    acc = warp_sum(acc);
    __shared__ float s_part[32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) s_part[warp] = acc;
    __syncthreads();
    if (warp == 0) {
        float v = lane < (blockDim.x >> 5) ? s_part[lane] : 0.f;
        v = warp_sum(v);
        if (lane == 0 && n_before >= 0) gsum[b] = (double)v;
    }
}

// pass 2: flip + all ops + ToTensor + Normalize -> fp32 HWC in [-1, 1], written at channel offset c_off of a [.][c_total] row
__global__ void face_augment_kernel(const uint8_t* __restrict__ src, const int* __restrict__ iparams,
                                    const float* __restrict__ fparams, const double* __restrict__ gsum,
                                    float* __restrict__ out, int H, int W, int c_total, int c_off) {
    const int b = blockIdx.y;
    const int* ip = iparams + b * 5;
    const float* fp = fparams + b * 4;
    const int HW = H * W;
    const float cmean = (float)(gsum[b] / (double)HW);
    const bool flip = ip[0] != 0;
    const uint8_t* s = src + (size_t)b * HW * 3;
    float* o = out + (size_t)b * HW * c_total + c_off;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
        const int y = i / W, x = i - y * W;
        const int sx = flip ? (W - 1 - x) : x;
        const uint8_t* px = s + ((size_t)y * W + sx) * 3;
        float r = px[0] * (1.f / 255.f), g = px[1] * (1.f / 255.f), bl = px[2] * (1.f / 255.f);
        jitter_pixel(r, g, bl, ip + 1, fp, 4, cmean);
        float* po = o + (size_t)i * c_total;
        po[0] = (r - 0.5f) / 0.5f;
        po[1] = (g - 0.5f) / 0.5f;
        po[2] = (bl - 0.5f) / 0.5f;
    }
}

// _add_bg: out = -1 everywhere, the face (channels [c_off, c_off+3) of `faces`) bilinearly resized (align_corners) to
// (rh, rw) pasted at (pos_h, pos_w).  geo [B][4] = {rh, rw, pos_h, pos_w}
__global__ void paste_resized_kernel(const float* __restrict__ faces, int c_total, int c_off, const int* __restrict__ geo,
                                     float* __restrict__ out, int H, int W) {
    const int b = blockIdx.y;
    const int rh = geo[b * 4], rw = geo[b * 4 + 1], ph = geo[b * 4 + 2], pw = geo[b * 4 + 3];
    const float sh = rh > 1 ? (float)(H - 1) / (float)(rh - 1) : 0.f;
    const float sw = rw > 1 ? (float)(W - 1) / (float)(rw - 1) : 0.f;
    const float* f = faces + (size_t)b * H * W * c_total + c_off;
    float* o = out + (size_t)b * H * W * 3;
    const int HW = H * W;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
        const int y = i / W, x = i - y * W;
        const int yy = y - ph, xx = x - pw;
        float v0 = -1.f, v1 = -1.f, v2 = -1.f;
        if (yy >= 0 && yy < rh && xx >= 0 && xx < rw) {
            const float h1r = sh * yy, w1r = sw * xx;
            const int h1 = (int)h1r, w1 = (int)w1r;
            const int h1p = h1 < H - 1 ? 1 : 0, w1p = w1 < W - 1 ? 1 : 0;
            const float hl1 = h1r - h1, hl0 = 1.f - hl1, wl1 = w1r - w1, wl0 = 1.f - wl1;
            const float* p00 = f + ((size_t)h1 * W + w1) * c_total;
            const float* p01 = p00 + (size_t)w1p * c_total;
            const float* p10 = p00 + (size_t)h1p * W * c_total;
            const float* p11 = p10 + (size_t)w1p * c_total;
            v0 = hl0 * (wl0 * p00[0] + wl1 * p01[0]) + hl1 * (wl0 * p10[0] + wl1 * p11[0]);
            v1 = hl0 * (wl0 * p00[1] + wl1 * p01[1]) + hl1 * (wl0 * p10[1] + wl1 * p11[1]);
            v2 = hl0 * (wl0 * p00[2] + wl1 * p01[2]) + hl1 * (wl0 * p10[2] + wl1 * p11[2]);
        }
        o[3 * (size_t)i] = v0;
        o[3 * (size_t)i + 1] = v1;
        o[3 * (size_t)i + 2] = v2;
    }
}

}  // namespace cb

using namespace cb;

extern "C" int cb_face_augment(const unsigned char* src_u8, const int* iparams, const float* fparams, double* ws, float* out,
                               int B, int H, int W, int c_total, int c_off, void* stream) {
    CB_REQUIRE(src_u8 && iparams && fparams && ws && out && B > 0 && H > 0 && W > 0 && c_off >= 0 && c_off + 3 <= c_total,
               CB_ERR_ARG, "face_augment: bad args");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    CB_CUDA(cudaMemsetAsync(ws, 0, sizeof(double) * B, st));
    const int HW = H * W;
    dim3 grid((unsigned)std::min(ceil_div(HW, 256 * 4), 4 * device_sm_count()), (unsigned)B);
    jitter_mean_kernel<<<dim3(1, (unsigned)B), 1024, 0, st>>>(src_u8, iparams, fparams, ws, HW);
    face_augment_kernel<<<grid, 256, 0, st>>>(src_u8, iparams, fparams, ws, out, H, W, c_total, c_off);
    CB_CUDA(cudaGetLastError());
    count_launches(2);
    return 0;
}

extern "C" int cb_paste_resized(const float* faces, int c_total, int c_off, const int* geo, float* out, int B, int H, int W,
                                void* stream) {
    CB_REQUIRE(faces && geo && out && B > 0 && H > 1 && W > 1 && c_off >= 0 && c_off + 3 <= c_total, CB_ERR_ARG,
               "paste_resized: bad args");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    dim3 grid((unsigned)std::min(ceil_div(H * W, 256 * 4), 4 * device_sm_count()), (unsigned)B);
    paste_resized_kernel<<<grid, 256, 0, st>>>(faces, c_total, c_off, geo, out, H, W);
    CB_CUDA(cudaGetLastError());
    count_launches(1);
    return 0;
}
