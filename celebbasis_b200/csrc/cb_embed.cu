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
                             float bc1, float bc2_sqrt, const int* __restrict__ step_dev) {
    pdl_sync();
    if (step_dev) {  // graph-replay friendly: the step counter lives on the device
        const float t = (float)(*step_dev + 1);
        bc1 = 1.f - powf(b1, t);
        bc2_sqrt = sqrtf(1.f - powf(b2, t));
    }
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

extern "C" int cb_embedding_gather(const long long* ids, const float* table, float* out, int n, int D, int V,
                                   void* stream) {
    CB_REQUIRE(n > 0 && D > 0 && D % 4 == 0 && V > 0, CB_ERR_ARG, "embedding_gather: bad shape");
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
    const float bc1 = 1.f - powf(beta1, (float)(step >= 1 ? step : 1));
    const float bc2s = sqrtf(1.f - powf(beta2, (float)(step >= 1 ? step : 1)));
    long long blocks = (n + 255) / 256;
    if (blocks > 1184) blocks = 1184;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
CB_LAUNCH((adamw_kernel), (unsigned)blocks, 256, 0, st, p, g, m, v, n, lr, beta1, beta2, eps, weight_decay, bc1, bc2s, step_dev);
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
