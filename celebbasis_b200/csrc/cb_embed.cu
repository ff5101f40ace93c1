// The trainable corner of CelebBasis, kept in fp32 on CUDA cores (it is ~5 MFLOP per step):
//   face feature v (F,512) -> EqualLinear(512->1024)+LeakyReLU(0.2) -> (F,2,512) -> L2-normalise ->
//   contraction with the PCA celeb basis (2,513,768) + mean -> 2 token embeddings -> scatter into the
//   prompt's token-embedding rows -> + position embedding; and the exact reverse for the gradient of the
//   1024x512 weight / 1024 bias, plus AdamW.
// Reference: ldm/modules/id_embedding/meta_net.py:27-48,61-87,250-302; ldm/modules/embedding_manager.py:279-394;
// ldm/modules/encoders/modules.py:232-298; ldm/models/diffusion/ddpm.py:1442-1454 (AdamW).
#include "cb_common.cuh"

namespace cb {

__device__ __forceinline__ float block_sum_256(float v, float* red) {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w];
    __syncthreads();
    return s;
}

__global__ void embedding_gather_kernel(const long long* __restrict__ ids, const float* __restrict__ table,
                                        float* __restrict__ out, int n, int D, int V) {
    pdl_sync();
    const int row = blockIdx.x;
    long long id = ids[row];
    if (id < 0) id = 0;
    if (id >= V) id = V - 1;
    const float4* src = reinterpret_cast<const float4*>(table + (size_t)id * D);
    float4* dst = reinterpret_cast<float4*>(out + (size_t)row * D);
    for (int c = threadIdx.x; c < D / 4; c += blockDim.x) dst[c] = src[c];
}

// pre[f][o] = v[f] . W[o] + b[o]: one warp per output row o (all faces at once), 8 outputs per block => out_dim/8 blocks
constexpr int kMaxFaces = 16;
__global__ void __launch_bounds__(256)
celeb_mlp_pre_kernel(const float* __restrict__ v, const float* __restrict__ W, const float* __restrict__ b,
                     float* __restrict__ pre, int F, int in_dim, int out_dim) {
    pdl_sync();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int o = blockIdx.x * 8 + warp;
    if (o >= out_dim) return;
    float acc[kMaxFaces];
#pragma unroll
    for (int f = 0; f < kMaxFaces; ++f) acc[f] = 0.f;
    const float* wr = W + (size_t)o * in_dim;
    for (int i = lane; i < in_dim; i += 32) {
        const float w = wr[i];
#pragma unroll
        for (int f = 0; f < kMaxFaces; ++f)
            if (f < F) acc[f] += w * v[(size_t)f * in_dim + i];
    }
#pragma unroll
    for (int f = 0; f < kMaxFaces; ++f) {
        if (f < F) {
            const float t = warp_sum(acc[f]);
            if (lane == 0) pre[(size_t)f * out_dim + o] = t + b[o];
        }
    }
}

// block per (face f, token e): act = leaky(pre) ; coef = act / max(||act||, 1e-12)
__global__ void __launch_bounds__(256)
celeb_mlp_norm_kernel(const float* __restrict__ pre, float* __restrict__ coef, float* __restrict__ nrm, int K, float slope) {
    pdl_sync();
    __shared__ float red[8];
    float q = 0.f;
    for (int j = threadIdx.x; j < K; j += 256) {
        const float pv = pre[(size_t)blockIdx.x * K + j];
        const float a = pv > 0.f ? pv : slope * pv;
        q += a * a;
    }
    q = block_sum_256(q, red);
    const float n = fmaxf(sqrtf(q), 1e-12f);
    if (threadIdx.x == 0) nrm[blockIdx.x] = n;
    for (int j = threadIdx.x; j < K; j += 256) {
        const float pv = pre[(size_t)blockIdx.x * K + j];
        coef[(size_t)blockIdx.x * K + j] = (pv > 0.f ? pv : slope * pv) / n;
    }
}

// z[f][e][c] = sum_k coef[f][e][k] * basis[e][1+k][c] + basis[e][0][c]; grid (F*es, D/128)
__global__ void __launch_bounds__(128)
celeb_basis_fwd_kernel(const float* __restrict__ coef, const float* __restrict__ basis, float* __restrict__ z, int K,
                       int D, int es) {
    pdl_sync();
    extern __shared__ float sc[];  // [K]
    const int e = blockIdx.x % es;
    for (int k = threadIdx.x; k < K; k += 128) sc[k] = coef[(size_t)blockIdx.x * K + k];
    __syncthreads();
    const float* be = basis + (size_t)e * (K + 1) * D;
    const int c = blockIdx.y * 128 + threadIdx.x;
    if (c >= D) return;
    float a0 = be[c], a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int k = 0;
    for (; k + 3 < K; k += 4) {
        a0 += sc[k] * be[(size_t)(k + 1) * D + c];
        a1 += sc[k + 1] * be[(size_t)(k + 2) * D + c];
        a2 += sc[k + 2] * be[(size_t)(k + 3) * D + c];
        a3 += sc[k + 3] * be[(size_t)(k + 4) * D + c];
    }
    for (; k < K; ++k) a0 += sc[k] * be[(size_t)(k + 1) * D + c];
    z[(size_t)blockIdx.x * D + c] = (a0 + a1) + (a2 + a3);
}

// dcoef[f][e][k] = sum_c dz[f][e][c] * basis[e][1+k][c]   (warp per k; grid (F*es, 16))
__global__ void __launch_bounds__(256)
celeb_basis_bwd_kernel(const float* __restrict__ dz, const float* __restrict__ basis, float* __restrict__ dcoef, int K,
                       int D, int es) {
    pdl_sync();
    extern __shared__ float sd[];  // [D]
    const int e = blockIdx.x % es;
    for (int c = threadIdx.x; c < D; c += 256) sd[c] = dz[(size_t)blockIdx.x * D + c];
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float* be = basis + (size_t)e * (K + 1) * D;
    const int kper = (K + gridDim.y - 1) / gridDim.y;
    const int k0 = blockIdx.y * kper, k1 = min(K, k0 + kper);
    for (int k = k0 + warp; k < k1; k += 8) {
        const float* br = be + (size_t)(k + 1) * D;
        float acc = 0.f;
        for (int c = lane; c < D; c += 32) acc += sd[c] * br[c];
        acc = warp_sum(acc);
        if (lane == 0) dcoef[(size_t)blockIdx.x * K + k] = acc;
    }
}

// dpre[f][e*K+j] = leaky'(pre) * ((dcoef - coef*(coef.dcoef)) / nrm) * gscale
__global__ void __launch_bounds__(256)
celeb_mlp_bwd_pre_kernel(const float* __restrict__ dcoef, const float* __restrict__ coef, const float* __restrict__ nrm,
                         const float* __restrict__ pre, float* __restrict__ dpre, int K, float slope, float gscale) {
    pdl_sync();
    __shared__ float red[8];
    float dot = 0.f;
    for (int j = threadIdx.x; j < K; j += 256)
        dot += coef[(size_t)blockIdx.x * K + j] * dcoef[(size_t)blockIdx.x * K + j];
    dot = block_sum_256(dot, red);
    const float inv = gscale / nrm[blockIdx.x];
    for (int j = threadIdx.x; j < K; j += 256) {
        const size_t i = (size_t)blockIdx.x * K + j;
        const float dx = (dcoef[i] - coef[i] * dot) * inv;
        dpre[i] = pre[i] > 0.f ? dx : slope * dx;
    }
}

// dW[o][i] = sum_f dpre[f][o] * v[f][i] ; db[o] = sum_f dpre[f][o]
__global__ void celeb_mlp_bwd_w_kernel(const float* __restrict__ dpre, const float* __restrict__ v,
                                       float* __restrict__ dW, float* __restrict__ db, int F, int out_dim, int in_dim) {
    pdl_sync();
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= out_dim * in_dim) return;
    const int o = idx / in_dim, i = idx - o * in_dim;
    float acc = 0.f, accb = 0.f;
    for (int f = 0; f < F; ++f) {
        const float d = dpre[(size_t)f * out_dim + o];
        acc += d * v[(size_t)f * in_dim + i];
        accb += d;
    }
    dW[idx] = acc;
    if (i == 0) db[o] = accb;
}

// out[b][i] = (map>=0 ? tok[b][map] : z[-(map+1)]) + pos[i]
__global__ void embed_inject_fwd_kernel(const float* __restrict__ tok, const float* __restrict__ z,
                                        const int* __restrict__ map, const float* __restrict__ pos,
                                        float* __restrict__ out, int T, int D) {
    pdl_sync();
    const int row = blockIdx.x;  // b*T + i
    const int b = row / T, i = row - b * T;
    const int m = map[row];
    const float* src = m >= 0 ? tok + ((size_t)b * T + m) * D : z + (size_t)(-(m + 1)) * D;
    for (int c = threadIdx.x; c < D; c += blockDim.x) out[(size_t)row * D + c] = src[c] + pos[(size_t)i * D + c];
}
// one CTA per z row: the token rows that received it are summed in row order (bit-identical from run to run)
__global__ void embed_inject_bwd_kernel(const float* __restrict__ dout, const int* __restrict__ map,
                                        float* __restrict__ dz, int rows, int D) {
    pdl_sync();
    const int zr = blockIdx.x;
    for (int c = threadIdx.x; c < D; c += blockDim.x) {
        float acc = 0.f;
        for (int row = 0; row < rows; ++row)
            if (map[row] == -(zr + 1)) acc += dout[(size_t)row * D + c];
        dz[(size_t)zr * D + c] = acc;
    }
}

__global__ void adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                             float* __restrict__ v, long long n, float lr, float b1, float b2, float eps, float wd,
                             int step, const int* __restrict__ step_dev) {
    pdl_sync();
    // graph-replay friendly: with step_dev the step counter lives on the device.  The bias corrections are formed here
    // for both paths, so a host-counted and a device-counted run produce the same bits.
    const float t = (float)(step_dev ? *step_dev + 1 : step);
    const float bc1 = 1.f - powf(b1, t);
    const float bc2_sqrt = sqrtf(1.f - powf(b2, t));
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float gi = g[i];
        float pi = p[i] * (1.f - lr * wd);
        const float mi = b1 * m[i] + (1.f - b1) * gi;
        const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
        m[i] = mi;
        v[i] = vi;
        const float denom = sqrtf(vi) / bc2_sqrt + eps;
        pi -= (lr / bc1) * (mi / denom);
        p[i] = pi;
    }
}

__global__ void bump_step_kernel(int* step_dev) {
    pdl_sync(); *step_dev += 1; }

// z = scale * (mean + exp(0.5*clamp(logvar,-30,20)) * eps); moments NCHW [N][2*Cz][HW]
__global__ void posterior_sample_kernel(const float* __restrict__ moments, const float* __restrict__ eps,
                                        float* __restrict__ z, int N, int Cz, int HW, float scale) {
    pdl_sync();
    const long long total = (long long)N * Cz * HW;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int p = (int)(i % HW);
        const long long t = i / HW;
        const int c = (int)(t % Cz);
        const int n = (int)(t / Cz);
        const float mean = moments[((size_t)n * 2 * Cz + c) * HW + p];
        float lv = moments[((size_t)n * 2 * Cz + Cz + c) * HW + p];
        lv = fminf(fmaxf(lv, -30.f), 20.f);
        z[i] = scale * (mean + expf(0.5f * lv) * eps[i]);
    }
}

// x_t = sqrt(acp[t]) * x0 + sqrt(1-acp[t]) * noise, t read on the device (ddpm.py:289-292, util.py:96-99)
__global__ void q_sample_kernel(const float* __restrict__ x0, const float* __restrict__ noise,
                                const long long* __restrict__ t, const float* __restrict__ sqrt_ac,
                                const float* __restrict__ sqrt_1mac, float* __restrict__ out, int per_sample) {
    pdl_sync();
    const int b = blockIdx.y;
    const float a = sqrt_ac[t[b]], s = sqrt_1mac[t[b]];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < per_sample; i += gridDim.x * blockDim.x) {
        const size_t k = (size_t)b * per_sample + i;
        out[k] = a * x0[k] + s * noise[k];
    }
}

// Masked DDIM blend before a step (ddim.py:144-147 around ddpm.py:289-292), one (b, c) row of HW pixels per blockIdx.y:
//   img_orig = sqrt_ac[t_b]*x0 + sqrt_1mac[t_b]*noise;  out = img_orig*m + (1-m)*img
// every operation is an explicitly rounded fp32 op in the reference's evaluation order (no FMA contraction), so the
// result is bit-identical to the eager fp32 expression.  The mask row is mask + b*mask_sb + c*mask_sc (a stride of 0
// broadcasts); `out` may alias `img` (each element is read before it is written, by the same thread).
__device__ __forceinline__ float masked_blend(float a, float s, float x0, float nz, float m, float im) {
    const float orig = __fadd_rn(__fmul_rn(a, x0), __fmul_rn(s, nz));
    return __fadd_rn(__fmul_rn(orig, m), __fmul_rn(__fsub_rn(1.f, m), im));
}

template <bool kVec>
__global__ void q_sample_masked_kernel(const float* __restrict__ x0, const float* __restrict__ noise,
                                       const long long* __restrict__ t, const float* __restrict__ sqrt_ac,
                                       const float* __restrict__ sqrt_1mac, const float* __restrict__ mask,
                                       long long mask_sb, long long mask_sc, const float* img, float* out, int C,
                                       int HW) {
    pdl_sync();
    const int b = blockIdx.y / C, c = blockIdx.y % C;
    const float a = sqrt_ac[t[b]], s = sqrt_1mac[t[b]];
    const size_t row = (size_t)blockIdx.y * HW;
    const float* mrow = mask + b * mask_sb + c * mask_sc;
    if (kVec) {
        const int n4 = HW >> 2;
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x) {
            const float4 xv = reinterpret_cast<const float4*>(x0 + row)[i];
            const float4 nv = reinterpret_cast<const float4*>(noise + row)[i];
            const float4 mv = reinterpret_cast<const float4*>(mrow)[i];
            const float4 iv = reinterpret_cast<const float4*>(img + row)[i];
            float4 o;
            o.x = masked_blend(a, s, xv.x, nv.x, mv.x, iv.x);
            o.y = masked_blend(a, s, xv.y, nv.y, mv.y, iv.y);
            o.z = masked_blend(a, s, xv.z, nv.z, mv.z, iv.z);
            o.w = masked_blend(a, s, xv.w, nv.w, mv.w, iv.w);
            reinterpret_cast<float4*>(out + row)[i] = o;
        }
    } else {
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x)
            out[row + i] = masked_blend(a, s, x0[row + i], noise[row + i], mrow[i], img[row + i]);
    }
}

// One DDPM ancestral step for eps-prediction (LatentDiffusion.p_sample -> p_mean_variance -> predict_start_from_noise ->
// q_posterior, ddpm.py:231-244,1118-1179), one sample of n values per blockIdx.y, t read on the device:
//   x_recon = sr[t]*x - srm1[t]*eps  (clamped to [-1, 1] with clip);  mean = c1[t]*x_recon + c2[t]*x
//   x_prev  = mean + ((1 - (t == 0)) * exp(0.5*lv[t])) * (noise*temperature)
// every operation is an explicitly rounded fp32 op in the reference's evaluation order (no FMA contraction; clamp keeps
// NaN as torch's does), so the result is bit-identical to the eager fp32 expression.  `x_prev` may alias `x` (each
// element is read before it is written, by the same thread).
__device__ __forceinline__ void ddpm_step(float x, float e, float nz, float sr, float srm1, float c1, float c2, float sd,
                                          float temp, bool clip, float& xp, float& x0) {
    float r = __fsub_rn(__fmul_rn(sr, x), __fmul_rn(srm1, e));
    if (clip && !isnan(r)) r = fminf(fmaxf(r, -1.f), 1.f);
    x0 = r;
    const float mean = __fadd_rn(__fmul_rn(c1, r), __fmul_rn(c2, x));
    xp = __fadd_rn(mean, __fmul_rn(sd, __fmul_rn(nz, temp)));
}

template <bool kVec>
__global__ void p_sample_kernel(const float* x, const float* __restrict__ eps, const float* __restrict__ noise,
                                const long long* __restrict__ t, const float* __restrict__ sqrt_recip_ac,
                                const float* __restrict__ sqrt_recipm1_ac, const float* __restrict__ coef1,
                                const float* __restrict__ coef2, const float* __restrict__ log_var, float temp,
                                int clip, float* x_prev, float* x0_out, int n) {
    pdl_sync();
    const int b = blockIdx.y;
    const long long tb = t[b];
    const float sr = sqrt_recip_ac[tb], srm1 = sqrt_recipm1_ac[tb], c1 = coef1[tb], c2 = coef2[tb];
    // nonzero_mask * exp(0.5 * log_variance): both (B,1,1,1) in the reference, multiplied before the noise
    const float sd = __fmul_rn(tb == 0 ? 0.f : 1.f, expf(__fmul_rn(0.5f, log_var[tb])));
    const bool cl = clip != 0;
    const size_t row = (size_t)b * n;
    if (kVec) {
        const int n4 = n >> 2;
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x) {
            const float4 xv = reinterpret_cast<const float4*>(x + row)[i];
            const float4 ev = reinterpret_cast<const float4*>(eps + row)[i];
            const float4 nv = reinterpret_cast<const float4*>(noise + row)[i];
            float4 o, r;
            ddpm_step(xv.x, ev.x, nv.x, sr, srm1, c1, c2, sd, temp, cl, o.x, r.x);
            ddpm_step(xv.y, ev.y, nv.y, sr, srm1, c1, c2, sd, temp, cl, o.y, r.y);
            ddpm_step(xv.z, ev.z, nv.z, sr, srm1, c1, c2, sd, temp, cl, o.z, r.z);
            ddpm_step(xv.w, ev.w, nv.w, sr, srm1, c1, c2, sd, temp, cl, o.w, r.w);
            reinterpret_cast<float4*>(x_prev + row)[i] = o;
            if (x0_out) reinterpret_cast<float4*>(x0_out + row)[i] = r;
        }
    } else {
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
            float o, r;
            ddpm_step(x[row + i], eps[row + i], noise[row + i], sr, srm1, c1, c2, sd, temp, cl, o, r);
            x_prev[row + i] = o;
            if (x0_out) x0_out[row + i] = r;
        }
    }
}

// DDIM update with classifier-free guidance (ldm/models/diffusion/ddim.py:166-204)
__global__ void ddim_step_kernel(const float* __restrict__ x, const float* __restrict__ e_u, const float* __restrict__ e_c,
                                 const float* __restrict__ noise, float* __restrict__ x_prev, float* __restrict__ pred_x0,
                                 long long n, float scale, float sqrt_at, float sqrt_aprev, float sigma, float sqrt_1m_at,
                                 float dir_coef) {
    pdl_sync();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        float e = e_u[i];
        if (e_c) e = e + scale * (e_c[i] - e);
        const float p0 = (x[i] - sqrt_1m_at * e) / sqrt_at;
        float xp = sqrt_aprev * p0 + dir_coef * e;
        if (noise) xp += sigma * noise[i];
        x_prev[i] = xp;
        if (pred_x0) pred_x0[i] = p0;
    }
}


__global__ void ema_rows_kernel(float* __restrict__ table, const long long* __restrict__ idx, int idx_stride,
                                const float* __restrict__ src, int B, int row, int n_rows, float m) {
    pdl_sync();
    const int b = blockIdx.y;
    const long long id = idx[(size_t)b * idx_stride];
    if (id < 0 || id >= n_rows) return;
    // samples of one batch that share an identity must update in batch order (the reference loops b = 0..B-1): only the
    // block of the LAST sample with this identity folds all of them, in order
    for (int b2 = b + 1; b2 < B; ++b2)
        if (idx[(size_t)b2 * idx_stride] == id) return;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < row; i += gridDim.x * blockDim.x) {
        float v = table[(size_t)id * row + i];
        for (int b1 = 0; b1 <= b; ++b1)
            if (idx[(size_t)b1 * idx_stride] == id) v = m * v + (1.f - m) * src[(size_t)b1 * row + i];
        table[(size_t)id * row + i] = v;
    }
}

// mean over the batch of the per-sample losses, summed in sample order (torch's mean of a (B,) fp32 tensor for the
// batch sizes a training step uses): one thread, B values
__global__ void loss_mean_kernel(const float* __restrict__ loss, float* __restrict__ out, int B) {
    pdl_sync();
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += loss[b];
    out[0] = s / (float)B;
}

// EMA over a fixed-capacity list of n (identity slot, source row) pairs, folded in list order: entry k updates
// table[ids[slot[k]]] with src[src_row[k]]; slot[k] < 0 is an unused entry.  One CTA per entry; as in ema_rows_kernel,
// only the CTA of the LAST entry of an identity writes, folding every entry of that identity in order.
__global__ void ema_rows_sel_kernel(float* __restrict__ table, const long long* __restrict__ ids,
                                    const int* __restrict__ slot, const int* __restrict__ src_row,
                                    const float* __restrict__ src, int n, int row, int n_rows, float m) {
    pdl_sync();
    const int k = blockIdx.y;
    if (slot[k] < 0) return;
    const long long id = ids[slot[k]];
    if (id < 0 || id >= n_rows) return;
    for (int k2 = k + 1; k2 < n; ++k2)
        if (slot[k2] >= 0 && ids[slot[k2]] == id) return;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < row; i += gridDim.x * blockDim.x) {
        float v = table[(size_t)id * row + i];
        for (int k1 = 0; k1 <= k; ++k1)
            if (slot[k1] >= 0 && ids[slot[k1]] == id) v = m * v + (1.f - m) * src[(size_t)src_row[k1] * row + i];
        table[(size_t)id * row + i] = v;
    }
}

// ---- weighted diffusion loss (ddpm.py:1084-1099), the timestep read on the device --------------------------------
// pass 1, one CTA per sample: loss_simple[b] = mean_i (pred-target)^2 (the sum in a fixed order, as mse_fwd_bwd_kernel)
// and d loss / d pred = 2*(pred-target)/per_sample * f_b * gscale, f_b = (lsw/exp(logvar[t_b]) + ew*lvlb[t_b]) / B
__global__ void diffusion_loss_sample_kernel(const float* __restrict__ pred, const float* __restrict__ target,
                                             const long long* __restrict__ t, const float* __restrict__ logvar,
                                             const float* __restrict__ lvlb, float* __restrict__ loss_simple,
                                             float* __restrict__ grad, int per_sample, int B, float lsw, float ew,
                                             float gscale) {
    pdl_sync();
    __shared__ float red[32];
    const int b = blockIdx.y;
    const size_t base = (size_t)b * per_sample;
    const long long tb = t[b];
    const float f = (lsw / expf(logvar[tb]) + ew * lvlb[tb]) / (float)B;
    const float gcoef = 2.f * (f / (float)per_sample) * gscale;
    float acc = 0.f;
    for (int i = threadIdx.x; i < per_sample; i += blockDim.x) {
        const float d = pred[base + i] - target[base + i];
        acc += d * d;
        if (grad) grad[base + i] = d * gcoef;
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
        loss_simple[b] = s / (float)per_sample;
    }
}

// pass 2, one thread: the batch means in sample order, in the reference's order of operations
//   loss = lsw * mean_b(loss_simple[b]/exp(logvar[t_b]) + logvar[t_b]) + ew * loss_vlb,
//   loss_vlb = mean_b(lvlb[t_b] * loss_simple[b])
__global__ void diffusion_loss_batch_kernel(const float* __restrict__ loss_simple, const long long* __restrict__ t,
                                            const float* __restrict__ logvar, const float* __restrict__ lvlb,
                                            float* __restrict__ loss, float* __restrict__ loss_vlb, int B, float lsw,
                                            float ew) {
    pdl_sync();
    float s = 0.f, v = 0.f;
    for (int b = 0; b < B; ++b) {
        const float lv = logvar[t[b]];
        s += loss_simple[b] / expf(lv) + lv;
        v += lvlb[t[b]] * loss_simple[b];
    }
    const float vlb = v / (float)B;
    loss_vlb[0] = vlb;
    loss[0] = lsw * (s / (float)B) + ew * vlb;
}

// ---- Textual Inversion coarse regulariser of one placeholder (embedding_manager.py:170-180, ddpm.py:1101-1107) -----
// mean((P-P0)(P-P0)^T / n) over its nv rows = |S|^2 / (nv^2 n) with S = sum_i (p_i - p0_i):
//   loss[0] += w * |S|^2 * inv;  grad_i += 2 w S inv for every row i;  inv = 1 / (nv^2 n).  One CTA of 256 threads.
__global__ void __launch_bounds__(256)
ti_coarse_reg_kernel(const float* __restrict__ p, const float* __restrict__ p0, float* __restrict__ grad,
                     float* __restrict__ loss, int nv, int D, float inv, float w) {
    pdl_sync();
    __shared__ float red[8];
    float acc = 0.f;
    for (int c = threadIdx.x; c < D; c += blockDim.x) {
        float s = 0.f;
        for (int i = 0; i < nv; ++i) s += p[(size_t)i * D + c] - p0[(size_t)i * D + c];
        acc += s * s;
        const float g = 2.f * w * s * inv;
        for (int i = 0; i < nv; ++i) grad[(size_t)i * D + c] += g;
    }
    const float tot = block_sum_256(acc, red);
    if (threadIdx.x == 0) loss[0] += w * (tot * inv);
}
}  // namespace cb

using namespace cb;

extern "C" int cb_ddim_step(const float* x, const float* e_uncond, const float* e_cond, const float* noise,
                            float* x_prev, float* pred_x0, long long n, float guidance_scale, float a_t, float a_prev,
                            float sigma_t, float sqrt_one_minus_at, void* stream) {
    CB_REQUIRE(n > 0 && x && e_uncond && x_prev, CB_ERR_ARG, "ddim_step: bad args");
    const float dir = sqrtf(fmaxf(1.f - a_prev - sigma_t * sigma_t, 0.f));
    long long blocks = (n + 255) / 256;
    if (blocks > 1184) blocks = 1184;
CB_LAUNCH((ddim_step_kernel), (unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream), 
        x, e_uncond, e_cond, noise, x_prev, pred_x0, n, guidance_scale, sqrtf(a_t), sqrtf(a_prev), sigma_t,
        sqrt_one_minus_at, dir);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_q_sample(const float* x0, const float* noise, const long long* t, const float* sqrt_ac,
                           const float* sqrt_1mac, float* out, int B, int per_sample, void* stream) {
    CB_REQUIRE(B > 0 && per_sample > 0, CB_ERR_ARG, "q_sample: bad shape");
    dim3 grid((unsigned)((per_sample + 255) / 256 > 64 ? 64 : (per_sample + 255) / 256), (unsigned)B);
CB_LAUNCH((q_sample_kernel), grid, 256, 0, reinterpret_cast<cudaStream_t>(stream), x0, noise, t, sqrt_ac, sqrt_1mac, out, per_sample);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_q_sample_masked(const float* x0, const float* noise, const long long* t, const float* sqrt_ac,
                                  const float* sqrt_1mac, const float* mask, long long mask_bstride,
                                  long long mask_cstride, const float* img, float* out, int B, int C, int HW,
                                  void* stream) {
    CB_REQUIRE(x0 && noise && t && sqrt_ac && sqrt_1mac && mask && img && out, CB_ERR_ARG,
               "q_sample_masked: NULL pointer");
    CB_REQUIRE(B > 0 && C > 0 && HW > 0 && (long long)B * C <= 65535, CB_ERR_ARG, "q_sample_masked: bad shape");
    CB_REQUIRE(mask_bstride >= 0 && mask_cstride >= 0, CB_ERR_ARG,
               "q_sample_masked: mask strides must be >= 0 (0 = broadcast)");
    auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
    const bool vec = HW % 4 == 0 && mask_bstride % 4 == 0 && mask_cstride % 4 == 0 && al16(x0) && al16(noise) &&
                     al16(mask) && al16(img) && al16(out);
    const int per_block = 256 * (vec ? 4 : 1);
    int bx = (HW + per_block - 1) / per_block;
    if (bx > 64) bx = 64;
    dim3 grid((unsigned)bx, (unsigned)(B * C));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (vec)
        CB_LAUNCH((q_sample_masked_kernel<true>), grid, 256, 0, st, x0, noise, t, sqrt_ac, sqrt_1mac, mask,
                  mask_bstride, mask_cstride, img, out, C, HW);
    else
        CB_LAUNCH((q_sample_masked_kernel<false>), grid, 256, 0, st, x0, noise, t, sqrt_ac, sqrt_1mac, mask,
                  mask_bstride, mask_cstride, img, out, C, HW);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_p_sample(const float* x, const float* eps, const float* noise, const long long* t,
                           const float* sqrt_recip_ac, const float* sqrt_recipm1_ac, const float* coef1,
                           const float* coef2, const float* log_var, float temperature, int clip_denoised,
                           float* x_prev, float* x0, int B, int n, void* stream) {
    CB_REQUIRE(x && eps && noise && t && sqrt_recip_ac && sqrt_recipm1_ac && coef1 && coef2 && log_var && x_prev,
               CB_ERR_ARG, "p_sample: NULL pointer");
    CB_REQUIRE(B > 0 && B <= 65535 && n > 0, CB_ERR_ARG, "p_sample: bad shape");
    auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
    const bool vec = n % 4 == 0 && al16(x) && al16(eps) && al16(noise) && al16(x_prev) && (!x0 || al16(x0));
    const int per_block = 256 * (vec ? 4 : 1);
    int bx = (n + per_block - 1) / per_block;
    if (bx > 64) bx = 64;
    dim3 grid((unsigned)bx, (unsigned)B);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (vec)
        CB_LAUNCH((p_sample_kernel<true>), grid, 256, 0, st, x, eps, noise, t, sqrt_recip_ac, sqrt_recipm1_ac, coef1,
                  coef2, log_var, temperature, clip_denoised, x_prev, x0, n);
    else
        CB_LAUNCH((p_sample_kernel<false>), grid, 256, 0, st, x, eps, noise, t, sqrt_recip_ac, sqrt_recipm1_ac, coef1,
                  coef2, log_var, temperature, clip_denoised, x_prev, x0, n);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_embedding_gather(const long long* ids, const float* table, float* out, int n, int D, int V,
                                   void* stream) {
    CB_REQUIRE(n > 0 && D > 0 && D % 4 == 0 && V > 0, CB_ERR_ARG, "embedding_gather: bad shape");
    CB_REQUIRE(((reinterpret_cast<uintptr_t>(table) | reinterpret_cast<uintptr_t>(out)) & 15) == 0, CB_ERR_ALIGN,
               "embedding_gather: table and out must be 16-byte aligned");
CB_LAUNCH((embedding_gather_kernel), n, 192, 0, reinterpret_cast<cudaStream_t>(stream), ids, table, out, n, D, V);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_celeb_mlp_fwd(const float* v, const float* W, const float* b, float* pre, float* coef, float* nrm,
                                int F, int in_dim, int K, int es, float slope, void* stream) {
    CB_REQUIRE(F > 0 && F <= kMaxFaces && in_dim > 0 && K > 0 && es > 0, CB_ERR_ARG, "celeb_mlp_fwd: bad shape (F <= %d)", kMaxFaces);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int out_dim = es * K;
    CB_LAUNCH((celeb_mlp_pre_kernel), ceil_div(out_dim, 8), 256, 0, st, v, W, b, pre, F, in_dim, out_dim);
    CB_LAUNCH((celeb_mlp_norm_kernel), F * es, 256, 0, st, (const float*)pre, coef, nrm, K, slope);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(2);
    return 0;
}

extern "C" int cb_celeb_basis_fwd(const float* coef, const float* basis, float* z, int F, int es, int K, int D,
                                  void* stream) {
    CB_REQUIRE(F > 0 && es > 0 && K > 0 && D > 0 && K * 4 <= 48 * 1024, CB_ERR_ARG, "celeb_basis_fwd: bad shape");
    CB_LAUNCH((celeb_basis_fwd_kernel), dim3(F * es, ceil_div(D, 128)), 128, K * sizeof(float), reinterpret_cast<cudaStream_t>(stream), coef, basis, z, K, D, es);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_celeb_basis_bwd(const float* dz, const float* basis, float* dcoef, int F, int es, int K, int D,
                                  void* stream) {
    CB_REQUIRE(F > 0 && es > 0 && K > 0 && D > 0 && D * 4 <= 48 * 1024, CB_ERR_ARG, "celeb_basis_bwd: bad shape");
    CB_LAUNCH((celeb_basis_bwd_kernel), dim3(F * es, 16), 256, D * sizeof(float), reinterpret_cast<cudaStream_t>(stream), dz, basis, dcoef, K, D, es);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_celeb_mlp_bwd(const float* dcoef, const float* coef, const float* nrm, const float* pre,
                                const float* v, float* dpre_ws, float* dW, float* db, int F, int in_dim, int K, int es,
                                float slope, float gscale, void* stream) {
    CB_REQUIRE(F > 0 && in_dim > 0 && K > 0 && es > 0, CB_ERR_ARG, "celeb_mlp_bwd: bad shape");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
CB_LAUNCH((celeb_mlp_bwd_pre_kernel), F * es, 256, 0, st, dcoef, coef, nrm, pre, dpre_ws, K, slope, gscale);
    const int out_dim = es * K;
CB_LAUNCH((celeb_mlp_bwd_w_kernel), ceil_div(out_dim * in_dim, 256), 256, 0, st, dpre_ws, v, dW, db, F, out_dim, in_dim);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(2);
    return 0;
}

extern "C" int cb_embed_inject_fwd(const float* tok, const float* z, const int* map, const float* pos, float* out,
                                   int B, int T, int D, void* stream) {
    CB_REQUIRE(B > 0 && T > 0 && D > 0, CB_ERR_ARG, "embed_inject_fwd: bad shape");
CB_LAUNCH((embed_inject_fwd_kernel), B * T, 256, 0, reinterpret_cast<cudaStream_t>(stream), tok, z, map, pos, out, T, D);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_embed_inject_bwd(const float* dout, const int* map, float* dz, int n_z_rows, int B, int T, int D,
                                   void* stream) {
    CB_REQUIRE(B > 0 && T > 0 && D > 0 && n_z_rows > 0, CB_ERR_ARG, "embed_inject_bwd: bad shape");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    CB_LAUNCH((embed_inject_bwd_kernel), n_z_rows, 256, 0, st, dout, map, dz, B * T, D);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_adamw_step(float* p, const float* g, float* m, float* v, long long n, float lr, float beta1,
                             float beta2, float eps, float weight_decay, int step, int* step_dev, void* stream) {
    CB_REQUIRE(n > 0 && (step >= 1 || step_dev != nullptr), CB_ERR_ARG, "adamw: bad args");
    long long blocks = (n + 255) / 256;
    if (blocks > 1184) blocks = 1184;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
CB_LAUNCH((adamw_kernel), (unsigned)blocks, 256, 0, st, p, g, m, v, n, lr, beta1, beta2, eps, weight_decay, step, step_dev);
    if (step_dev)CB_LAUNCH((bump_step_kernel), 1, 1, 0, st, step_dev);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(2);
    return 0;
}

extern "C" int cb_posterior_sample(const float* moments, const float* eps, float* z, int N, int Cz, int HW,
                                   float scale, void* stream) {
    CB_REQUIRE(N > 0 && Cz > 0 && HW > 0, CB_ERR_ARG, "posterior_sample: bad shape");
    const long long total = (long long)N * Cz * HW;
CB_LAUNCH((posterior_sample_kernel), (unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream), moments, eps, z, N, Cz, HW, scale);
    CB_CUDA(cudaGetLastError());
    cb::count_launches(1);
    return 0;
}

extern "C" int cb_ema_rows(float* table, const long long* idx, int idx_stride, const float* src, int B, int row, int n_rows,
                           float momentum, void* stream) {
    CB_REQUIRE(table && idx && src && B > 0 && row > 0 && n_rows > 0 && idx_stride > 0, CB_ERR_ARG, "ema_rows: bad args");
    const int gx = ceil_div(row, 256);
    dim3 grid((unsigned)(gx < 8 ? gx : 8), (unsigned)B);
    CB_LAUNCH((ema_rows_kernel), grid, 256, 0, reinterpret_cast<cudaStream_t>(stream), table, idx, idx_stride, src, B, row,
              n_rows, momentum);
    CB_CUDA(cudaGetLastError());
    count_launches(1);
    return 0;
}

extern "C" int cb_loss_mean(const float* loss, float* out, int B, void* stream) {
    CB_REQUIRE(loss && out && B > 0, CB_ERR_ARG, "loss_mean: bad args");
    CB_LAUNCH((loss_mean_kernel), 1, 1, 0, reinterpret_cast<cudaStream_t>(stream), loss, out, B);
    CB_CUDA(cudaGetLastError());
    count_launches(1);
    return 0;
}

extern "C" int cb_ema_rows_sel(float* table, const long long* ids, const int* slot, const int* src_row, const float* src,
                               int n, int row, int n_rows, float momentum, void* stream) {
    CB_REQUIRE(table && ids && slot && src_row && src && n > 0 && n <= 65535 && row > 0 && n_rows > 0, CB_ERR_ARG,
               "ema_rows_sel: bad args");
    const int gx = ceil_div(row, 256);
    dim3 grid((unsigned)(gx < 8 ? gx : 8), (unsigned)n);
    CB_LAUNCH((ema_rows_sel_kernel), grid, 256, 0, reinterpret_cast<cudaStream_t>(stream), table, ids, slot, src_row,
              src, n, row, n_rows, momentum);
    CB_CUDA(cudaGetLastError());
    count_launches(1);
    return 0;
}

extern "C" int cb_diffusion_loss_fwd_bwd(const float* pred, const float* target, const long long* t, const float* logvar,
                                         const float* lvlb_weights, float l_simple_weight, float original_elbo_weight,
                                         float* loss_simple, float* loss, float* loss_vlb, float* grad, int B,
                                         int per_sample, float gscale, void* stream) {
    CB_REQUIRE(pred && target && t && logvar && lvlb_weights && loss_simple && loss && loss_vlb, CB_ERR_ARG,
               "diffusion_loss: NULL pointer");
    CB_REQUIRE(B > 0 && B <= 65535 && per_sample > 0, CB_ERR_ARG, "diffusion_loss: bad shape");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    CB_LAUNCH((diffusion_loss_sample_kernel), dim3(1, B), 1024, 0, st, pred, target, t, logvar, lvlb_weights,
              loss_simple, grad, per_sample, B, l_simple_weight, original_elbo_weight, gscale);
    CB_LAUNCH((diffusion_loss_batch_kernel), 1, 1, 0, st, (const float*)loss_simple, t, logvar, lvlb_weights, loss,
              loss_vlb, B, l_simple_weight, original_elbo_weight);
    CB_CUDA(cudaGetLastError());
    count_launches(2);
    return 0;
}

extern "C" int cb_ti_coarse_reg(const float* rows, const float* init_rows, float* grad, float* loss, int nv, int D,
                                int n_init, float weight, void* stream) {
    CB_REQUIRE(rows && init_rows && grad && loss && nv > 0 && D > 0 && n_init > 0, CB_ERR_ARG, "ti_coarse_reg: bad args");
    const float inv = 1.f / ((float)nv * (float)nv * (float)n_init);
    CB_LAUNCH((ti_coarse_reg_kernel), 1, 256, 0, reinterpret_cast<cudaStream_t>(stream), rows, init_rows, grad, loss, nv,
              D, inv, weight);
    CB_CUDA(cudaGetLastError());
    count_launches(1);
    return 0;
}
