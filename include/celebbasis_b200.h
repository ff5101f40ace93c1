/*
 * celebbasis_b200 — C-ABI of the H100-native (sm_90a) hot path of CelebBasis.
 *
 * The reference (ygtxr1997/CelebBasis) has no FFI: its hot path is a chain of stock ATen calls
 * made from Python (SURVEY.md §8b).  This header is therefore the boundary a maintainer would
 * bind with ctypes from the reference's own modules; every entry point names the reference
 * code whose arithmetic it replaces (file:line relative to the reference tree).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name says `host`; the caller (PyTorch's caching
 *     allocator in our host mirror) owns all buffers including workspaces; nothing here allocates.
 *   - all work is enqueued on the cudaStream_t passed in (as void*); no hidden synchronisation;
 *     every entry point is CUDA-graph capturable and re-entrant.
 *   - return value: 0 = ok, negative = argument check failed, positive = cudaError_t.
 *     cb_last_error() returns a thread-local message for the last non-zero return.
 *   - activations are channels-last: images are NHWC ([N][H][W][C], C contiguous), token
 *     matrices are [rows][channels].  Module inputs/outputs in the Python mirror stay NCHW fp32
 *     exactly like the reference (ldm/models/diffusion/ddpm.py:344-350).
 */
#ifndef CELEBBASIS_B200_H_
#define CELEBBASIS_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CB_ABI_VERSION 6
#define CB_GN_WS_BYTES 131072

/* element types */
enum { CB_F16 = 0, CB_BF16 = 1, CB_F32 = 2 };
/* activation fused into the GEMM epilogue */
enum { CB_ACT_NONE = 0, CB_ACT_SILU = 1, CB_ACT_GELU = 2, CB_ACT_QUICK_GELU = 3, CB_ACT_PRELU = 4 };
/* operand majorness: K-major = reduction dim contiguous; MN-major = M (or N) contiguous */
enum { CB_MAJOR_K = 0, CB_MAJOR_MN = 1 };

/* error codes (negative) */
enum {
    CB_OK = 0,
    CB_ERR_ARG = -1,       /* invalid argument / unsupported shape */
    CB_ERR_ALIGN = -2,     /* pointer or stride alignment */
    CB_ERR_DRIVER = -3,    /* CUDA driver entry point unavailable / tensor-map encode failed */
    CB_ERR_NO_DEVICE = -4, /* no sm_90 device */
};

int cb_abi_version(void);
const char* cb_last_error(void);
/* 1 if the current device is compute capability 10.x, else 0 (never throws). */
int cb_device_ok(void);
/* number of kernels this library has launched (or captured into a CUDA graph) in this process. */
unsigned long long cb_launch_count(void);

/* ---------------------------------------------------------------------------------------------
 * cb_gemm — wgmma tensor-core GEMM / implicit-GEMM convolution with TMA-staged operands.
 *
 *   D[b][m][n] = act(alpha * sum_{tap,k} A_tap[b][m][k] * B[b][tap][n][k] + bias[...]) + R[b][m][n]
 *
 * Replaces every torch.nn.Linear / Conv2d / einsum contraction on the path:
 *   ldm/modules/attention.py:170-193 (to_q/k/v/out, q.k^T, p.v), :37-64 (GEGLU / FF),
 *   ldm/modules/diffusionmodules/openaimodel.py:255-275 (ResBlock convs), :91-160 (up/down convs),
 *   ldm/modules/diffusionmodules/model.py:82-202 (VAE ResnetBlock/AttnBlock),
 *   ldm/modules/id_embedding/iresnet.py:26-64 (IBasicBlock convs),
 *   transformers CLIPAttention/CLIPMLP called from ldm/modules/encoders/modules.py:320-340.
 * and, with operand majors swapped, their activation-gradient (dgrad) counterparts that autograd
 * runs in the reference (SURVEY.md §8 a29).
 *
 * Plain mode (conv == 0): A is [batch][M][K] (K-major, row stride lda) or, with
 * a_major == CB_MAJOR_MN, stored transposed as [batch][K][M] (row stride lda).  B likewise is
 * [batch][N][K] (K-major) or [batch][K][N] (MN-major).  Strides are in ELEMENTS.
 *
 * Conv mode (conv == 1): A is an NHWC image [img_n][img_h][img_w][K] (K = input channels, K-major)
 * and row m of the GEMM is output pixel (img, oh, ow) in raster order; tap (r,s) reads input pixel
 * (oh*stride + r - pad_top, ow*stride + s - pad_left); out-of-image taps read zeros (TMA OOB fill).
 * B rows for tap t start at row t*b_tap_rows: K-major B is [taps*b_tap_rows][K]; MN-major B is
 * [taps*b_tap_rows (k index)][N] (used for dgrad with the forward weight pack).  M is implied:
 * M = img_n*out_h*out_w.  tap order is r-major (t = r*kw + s); flip_taps reverses it (dgrad).
 * ------------------------------------------------------------------------------------------- */
typedef struct cb_gemm_desc {
    int32_t M, N, K;
    int32_t batch;
    int32_t ab_dtype; /* CB_F16 or CB_BF16 (both operands) */

    const void* A;
    int64_t lda;
    int64_t a_batch_stride;
    int32_t a_major;

    const void* B;
    int64_t ldb;
    int64_t b_batch_stride;
    int32_t b_major;

    /* conv mode */
    int32_t conv;
    int32_t img_n, img_h, img_w;
    int32_t out_h, out_w;
    int32_t kh, kw;
    int32_t stride;
    int32_t pad_top, pad_left;
    int32_t b_tap_rows;
    int32_t flip_taps;

    /* epilogue */
    void* D;
    int32_t d_dtype; /* CB_F16 / CB_BF16 / CB_F32 */
    int64_t ldd;
    int64_t d_batch_stride;
    int32_t d_transposed; /* write D[b][n][m] (row stride ldd) instead of D[b][m][n] */

    const float* bias;     /* fp32 [bias_rows][N] or NULL */
    int32_t bias_row_div;  /* bias row = (global row m) / bias_row_div; 0 => single row */
    int64_t ldbias;

    const void* R; /* residual added after the activation, same logical shape as D, or NULL */
    int32_t r_dtype;
    int64_t ldr;
    int64_t r_batch_stride;

    float alpha;
    int32_t act;

    /* two-level batch: batch index z = zo*batch_inner + zi uses offset zi*stride + zo*stride2
     * (e.g. zi = attention head, zo = image).  batch_inner == 0 means a single level. */
    int32_t batch_inner;
    int64_t a_batch_stride2, b_batch_stride2, d_batch_stride2, r_batch_stride2;

    /* optional split-K workspace (caller-owned, 64 KiB of counters + one fp32 partial tile per k-slice and output
     * tile; the counters must be ALL ZERO before its first use and every launch leaves them zero).  With it, shapes
     * whose tile grid cannot fill the SMs (bs=1 low-resolution layers: M <= 256 rows against 1280-2560 channel
     * weights) spread their k-loop over several CTAs that store their fp32 partial tiles into their own slices; the
     * last CTA of a tile adds them in slice order (bit-reproducible) and runs the epilogue.  NULL disables split-K.
     * Launches sharing a workspace must be stream-ordered. */
    void* splitk_ws;
    int64_t splitk_ws_bytes;

    /* profiling aid, NULL in production: device buffer of 8 x uint64 per CTA receiving %globaltimer stamps
     * {start, setup done, first stage full, last MMA issued, accumulator ready, exit, 4th stage full, -}. */
    void* debug_timeline;

    /* tuning overrides, 0 = the library's cost model: tile width (64 / 128 / 160 / 256; 160 only with K-major B, 256 only
     * with K-major A and N >= 256; a width the operand majors do not allow is ignored) and the
     * number of split-K slices (1 = no split; ignored when the workspace cannot hold it).  Without a splits request
     * the split count depends on the shape only, never on tile_n / stages / cta_pair / splitk_cluster, so those knobs
     * do not change the results.  The host autotuner (celebbasis_b200/ops.py) times them once per shape and passes the
     * winner here. */
    int32_t tile_n;
    int32_t splits;
    int32_t stages;      /* 0 = auto, 3 = 3-stage ring / 2 CTAs per SM, 6 = 6-stage ring / 1 CTA per SM */
    int32_t cta_pair;    /* tile request of the host autotuner: >= 1 = large-M tiles (128 x 128 or 128 x 256 by tile_n;
                          * sm_90 has no two-CTA MMA, so every tile is one CTA); 0 = the library's choice */

    /* second destination (optional, batch == 1, not transposed): the same epilogue value is also written to
     * D2[row][col] (row pitch ldd2 elements, dtype d2_dtype).  Used to place a UNet skip activation straight into the
     * concat buffer of the output block that will consume it (torch.cat([h, hs.pop()], dim=1), openaimodel.py:737-739)
     * and for 16-bit copies of fp32 results. */
    void* D2;
    int64_t ldd2;
    int32_t d2_dtype;
    int32_t glu;         /* 1 = GEGLU epilogue (attention.py:37-45): the N output columns are 64-column groups of 32 value
                          * columns followed by their 32 gate columns (weight rows interleaved by the caller);
                          * D2[row][32*group + j] = (value + bias) * gelu(gate + bias); D (may be NULL) keeps the
                          * pre-activations in that interleaved layout for cb_geglu_bwd(interleave = 1) */
    /* CB_ACT_PRELU: per-column negative slopes [N] (iresnet.py:41-58 PReLU after conv1 + bn2);
     * d2_scale / d2_shift (optional, [N] each): the D2 copy is v * scale[col] + shift[col] -- the eval BatchNorm that the
     * NEXT layer applies to its input (IBasicBlock.bn1, iresnet.py:47) folded into this layer's epilogue. */
    const float* act_param;
    const float* d2_scale;
    const float* d2_shift;
    /* 1 = the `splits` k-slices of a tile form a thread-block cluster (1,1,splits; 2..16 slices) and reduce through
     * distributed shared memory: every CTA sends the 8-column groups of its partial accumulator to the group's owner CTA
     * (round-robin) and each owner runs the epilogue for its groups -- two cluster barriers instead of L2 reductions,
     * fence, arrival counter and read-back.  Needs `splits` > 1 (caller-tuned) and an exchange buffer that fits the TMA
     * ring (CB_ERR_ARG otherwise); ignored by the CTA-pair variant. */
    int32_t splitk_cluster;
} cb_gemm_desc;

int cb_gemm(const cb_gemm_desc* desc, void* stream);


/* ---------------------------------------------------------------------------------------------
 * Normalisation (channels-last).  ws = caller workspace of CB_GN_WS_BYTES bytes (per-CTA partial sums, added up in
 * CTA order); it needs no initialisation, and calls sharing it must be stream-ordered.
 * cb_groupnorm_*: ldm/modules/diffusionmodules/util.py:199-216 (GroupNorm32, eps 1e-5),
 *   ldm/modules/attention.py:76-77 and ldm/modules/diffusionmodules/model.py:38-39 (Normalize, eps 1e-6),
 *   optionally fused with the nn.SiLU that follows (openaimodel.py:201-241, model.py:33-35 nonlinearity).
 * cb_layernorm_*: nn.LayerNorm in BasicTransformerBlock (attention.py:196-215) and the CLIP layers.
 * The *_bwd entry points are the activation gradients torch.autograd computes in the reference
 * (SURVEY.md §8 a29); accumulate != 0 adds into dx (residual-branch join).
 * ------------------------------------------------------------------------------------------- */
/* cb_groupnorm_fwd: rows of x must be multiples of 16 bytes (C * sizeof(x) % 16 == 0; CB_ERR_ARG otherwise).
 *   Statistics: fp32 partial sums of x and x^2 per group, added in fp64; variance = E[x^2] - mean^2 (one pass).  With
 *   u = 2^-24 and a group's mean mu, variance s2: |mean_out - mu| <= K u mean|x| and |rstd_out - r| / r <=
 *   K u (1 + mu^2 / (s2 + eps)), r = 1 / sqrt(s2 + eps): the mu^2 term is the cancellation of the one-pass variance, so
 *   groups whose mean is large against their spread get proportionally less accurate statistics.  LayerNorm forms its
 *   variance in two passes and has no such term.  tests/test_gpu_norm_sweep.py holds the measured K.
 * cb_groupnorm_bwd: dx_lp (optional, dtype of dy): the result is also written as a 16-bit copy -- the operand of the
 * dgrad GEMM that consumes dx next (saves a cast launch per ResBlock / transformer block of the backward pass).
 * act_silu: bit 0 = fuse SiLU; bits 8..23 = CB_GN_CTA_CAP(n); other bits are ignored. */
#define CB_GN_CTA_CAP(n) (((n) & 0xFFFF) << 8) /* OR into act_silu (cb_groupnorm_fwd): at most n CTAs on the streaming kernel pair */
/* How cb_groupnorm_fwd / _bwd would run a (N, HW, C, G) problem whose staged element costs `bytes_per_elem` bytes
 * (fwd: sizeof(x); bwd: sizeof(x) + sizeof(dy)): returns 1 and fills plan[4] = {CTAs per cluster, groups per cluster slab,
 * rows per CTA, dynamic shared memory bytes} when the thread-block-cluster variant applies (slabs of groups, statistics
 * through distributed shared memory), 0 when the rows do not fit and a statistics + apply kernel pair takes over
 * (forward: rows streamed through shared memory by TMA; backward: plain loads).
 * Host-only (no launch): lets integrators and the CPU tests see the launch geometry. */
int cb_groupnorm_cluster_plan(int N, int HW, int C, int G, int bytes_per_elem, int* plan);
int cb_groupnorm_fwd(const void* x, int x_dtype, void* y, int y_dtype, const float* gamma, const float* beta,
                     int N, int HW, int C, int G, float eps, int act_silu, float* mean_out, float* rstd_out,
                     double* ws, void* stream);
int cb_groupnorm_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, const float* gamma,
                     const float* beta, const float* mean, const float* rstd, void* dx, int dx_dtype, void* dx_lp, int N,
                     int HW, int C, int G, int act_silu, int accumulate, double* ws, void* stream);
int cb_layernorm_fwd(const void* x, int x_dtype, void* y, int y_dtype, const float* gamma, const float* beta, int M,
                     int C, float eps, float* mean_out, float* rstd_out, void* stream);
/* dx_lp (optional): a second copy of the final dx in dy's 16-bit dtype, for the GEMM that consumes it next */
int cb_layernorm_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, const float* gamma, const float* mean,
                     const float* rstd, void* dx, int dx_dtype, void* dx_lp, int M, int C, int accumulate,
                     void* stream);

/* ---------------------------------------------------------------------------------------------
 * Pointwise / row-wise kernels.
 * cb_axpby2d: out = a*x + b*y over a [rows][cols] view with independent row strides (elements) and
 *   dtypes; y may be NULL.  Serves residual adds, casts, torch.cat / chunk along channels
 *   (openaimodel.py:736-739 skip concat), q_sample (ddpm.py:289-292) and the EMA update
 *   (embedding_manager.py:484-489).
 * cb_act_fwd/bwd: SiLU (openaimodel.py:208,222 emb_layers), quick-GELU (CLIP MLP), GELU.
 * cb_geglu_*: ldm/modules/attention.py:37-45.      cb_softmax_*: attention.py:185 (+ CLIP causal mask,
 *   modules.py:24-31: row r may attend columns <= r % causal_period).
 * cb_upsample2x_*: openaimodel.py:112-117 nearest x2.   cb_zero_insert2x: input of the stride-2 conv dgrad.
 * cb_nchw_to_nhwc / cb_nhwc_to_nchw: ddpm.py:344-350 layout glue (+ channel padding to a multiple of 8).
 * cb_mse_fwd_bwd: ddpm.py:294-307 + :1084-1096: loss_simple[b] = mean over (C,H,W) of the squared error, and
 *   d(mean_b loss_simple[b])/dpred * gscale.
 * cb_timestep_embedding: diffusionmodules/util.py:151-171.
 * Every dtype argument is CB_F16, CB_BF16 or CB_F32 (CB_ERR_ARG otherwise; cb_geglu_* and cb_softmax_* take the
 * 16-bit types only); cb_act_* take CB_ACT_NONE, _SILU, _GELU or _QUICK_GELU (CB_ERR_ARG otherwise).
 * cb_axpby2d, cb_geglu_*, cb_upsample2x_* and cb_zero_insert2x move 4 elements per access: every tensor pointer they
 *   take must be aligned to 4 elements of its dtype (16 B for fp32, 8 B for fp16 / bf16), CB_ERR_ALIGN otherwise.
 *   cb_geglu_* with interleave = 1 need F % 32 == 0 (whole 64-column groups), CB_ERR_ARG otherwise.
 * ------------------------------------------------------------------------------------------- */
int cb_axpby2d(const void* x, int x_dtype, long long ldx, float a, const void* y, int y_dtype, long long ldy, float b,
               void* out, int o_dtype, long long ldo, long long rows, int cols, void* stream);
int cb_act_fwd(const void* x, int x_dtype, void* y, int y_dtype, long long n, int act, void* stream);
int cb_act_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, void* dx, int dx_dtype, long long n, int act,
               void* stream);
/* interleave = 1: `in` / `din` rows are 64-column groups of 32 values followed by their 32 gates (the layout the GEGLU
 * epilogue of cb_gemm keeps), instead of [all values | all gates] */
int cb_geglu_fwd(const void* in, void* out, int dtype, long long M, int F, int interleave, void* stream);
int cb_geglu_bwd(const void* dout, const void* in, void* din, int dtype, int g_dtype, long long M, int F,
                 int interleave, void* stream);
int cb_softmax_fwd(const void* s, void* p, int dtype, long long rows, int ncols, int ld, int causal_period,
                   void* stream);
int cb_softmax_bwd(const void* dp, const void* p, void* ds, int p_dtype, int g_dtype, long long rows, int ncols,
                   int ld, void* stream);
int cb_upsample2x_fwd(const void* x, void* y, int dtype, int N, int H, int W, int C, void* stream);
int cb_upsample2x_bwd(const void* dy, int dy_dtype, void* dx, int dx_dtype, int N, int H, int W, int C,
                      int accumulate, void* stream);
int cb_zero_insert2x(const void* dy, void* z, int dtype, int N, int H, int W, int C, void* stream);
int cb_nchw_to_nhwc(const float* x, void* y, int y_dtype, int N, int C, int HW, int Cpad, void* stream);
int cb_nhwc_to_nchw(const void* x, int x_dtype, float* y, int N, int C, int HW, int Cpad, void* stream);
int cb_mse_fwd_bwd(const float* pred, const float* target, float* loss /* [B] */, float* grad, int B, int per_sample,
                   float gscale, void* stream);
int cb_timestep_embedding(const long long* t, void* out, int o_dtype, int B, int dim, float max_period,
                          void* stream);

/* ---------------------------------------------------------------------------------------------
 * Celeb-basis embedding path (fp32): the only trainable tensors of the method live here.
 * cb_embedding_gather: token_embedding(input_ids), ldm/modules/encoders/modules.py:237.  table and out must be
 *   16-byte aligned (CB_ERR_ALIGN otherwise); an id outside [0, V) takes the nearest valid row.
 * cb_celeb_mlp_fwd: EqualLinear(512->es*K, lr_mul=1)+LeakyReLU(0.2) -> 'b (e h d) -> b e h d' -> L2 normalise,
 *   ldm/modules/id_embedding/meta_net.py:27-48,61-87,266-273.  pre/coef/nrm are saved for backward.
 * cb_celeb_basis_fwd/bwd: einsum('b e h k, e k c -> b e h c', x, basis[:,1:]) + basis[:,0], meta_net.py:275-289
 *   (also embedding_manager.py:464-475 at inference and scripts/extract_pt.py:113-118).
 * cb_celeb_mlp_bwd: gradient of W (es*K x in_dim) and b; gscale un-does the fp16 loss scale.
 * cb_embed_inject_fwd/bwd: the row rewrite of EmbeddingManagerId.forward (embedding_manager.py:322-360) as one
 *   gather: map[b][i] >= 0 takes token row map[b][i] of the same prompt, map < 0 takes z row -(map+1);
 *   then + position_embedding (modules.py:295-296).  The integer map is produced on the host by the
 *   bit-exact mirror of ldm/modules/id_embedding/helpers.py:6-41.
 * cb_adamw_step: torch.optim.AdamW step on the flat trainable buffer (ddpm.py:1442-1454); if step_dev is
 *   not NULL the 1-based step counter is read from (and bumped on) the device so the launch is graph-replayable.
 *   The bias corrections are formed on the device either way: a host-counted and a device-counted run give the same bits.
 * cb_posterior_sample: DiagonalGaussianDistribution.sample * scale_factor (distributions.py:25-37, ddpm.py:590-597)
 *   with the normal draw eps supplied by the caller (the reference draws it on the CPU).
 * ------------------------------------------------------------------------------------------- */
int cb_embedding_gather(const long long* ids, const float* table, float* out, int n, int D, int V, void* stream);
int cb_celeb_mlp_fwd(const float* v, const float* W, const float* b, float* pre, float* coef, float* nrm, int F,
                     int in_dim, int K, int es, float slope, void* stream);
int cb_celeb_basis_fwd(const float* coef, const float* basis, float* z, int F, int es, int K, int D, void* stream);
int cb_celeb_basis_bwd(const float* dz, const float* basis, float* dcoef, int F, int es, int K, int D, void* stream);
int cb_celeb_mlp_bwd(const float* dcoef, const float* coef, const float* nrm, const float* pre, const float* v,
                     float* dpre_ws, float* dW, float* db, int F, int in_dim, int K, int es, float slope,
                     float gscale, void* stream);
int cb_embed_inject_fwd(const float* tok, const float* z, const int* map, const float* pos, float* out, int B, int T,
                        int D, void* stream);
int cb_embed_inject_bwd(const float* dout, const int* map, float* dz, int n_z_rows, int B, int T, int D,
                        void* stream);
int cb_adamw_step(float* p, const float* g, float* m, float* v, long long n, float lr, float beta1, float beta2,
                  float eps, float weight_decay, int step, int* step_dev, void* stream);
int cb_posterior_sample(const float* moments, const float* eps, float* z, int N, int Cz, int HW, float scale,
                        void* stream);
/* cb_loss_mean: out[0] = (loss[0] + ... + loss[B-1]) / B, added in sample order: the batch mean of the per-sample
 *   losses (ddpm.py:1084-1096) inside a captured training step. */
int cb_loss_mean(const float* loss, float* out, int B, void* stream);
/* cb_diffusion_loss_fwd_bwd: LatentDiffusion.p_losses with its loss weights (ddpm.py:1084-1099), replacing
 *   loss_simple = get_loss(...).mean([1,2,3]); loss = loss_simple/exp(logvar[t]) + logvar[t];
 *   loss = l_simple_weight * loss.mean(); loss_vlb = (lvlb_weights[t] * loss_simple).mean();
 *   loss += original_elbo_weight * loss_vlb
 * with t read on the device (int64, B entries; logvar and lvlb_weights are fp32 tables indexed by it), so a captured
 * step replays with a new t.  pred / target / grad are [B][per_sample] fp32; loss_simple is [B], loss and loss_vlb one
 * float each.  grad (may be NULL) = d loss / d pred * gscale: sample b's factor
 * (l_simple_weight/exp(logvar[t_b]) + original_elbo_weight*lvlb_weights[t_b]) / B is folded into 2*(pred-target)/per_sample.
 * Every sum is taken in a fixed order (the batch means in sample order): bit-reproducible.  Two launches. */
int cb_diffusion_loss_fwd_bwd(const float* pred, const float* target, const long long* t, const float* logvar,
                              const float* lvlb_weights, float l_simple_weight, float original_elbo_weight,
                              float* loss_simple, float* loss, float* loss_vlb, float* grad, int B, int per_sample,
                              float gscale, void* stream);
/* cb_ti_coarse_reg: the Textual Inversion coarse regulariser of ONE placeholder, weighted (embedding_manager.py:170-180
 *   embedding_to_coarse_loss, ddpm.py:1101-1107 `loss += embedding_reg_weight * loss_embedding_reg.mean()`).  rows and
 *   init_rows are the placeholder's nv trained and initial rows of D floats; n_init = len(initial_embeddings).  With
 *   S = sum_i (rows_i - init_rows_i), mean((P-P0)(P-P0)^T / n_init) = |S|^2 / (nv^2 n_init), so
 *     loss[0] += weight * |S|^2 / (nv^2 n_init);   grad_i += 2 weight S / (nv^2 n_init) for each of the nv rows.
 *   One launch per placeholder with an initializer word, after the step's other gradient writes. */
int cb_ti_coarse_reg(const float* rows, const float* init_rows, float* grad, float* loss, int nv, int D, int n_init,
                     float weight, void* stream);
/* cb_ddim_step: one DDIM update with classifier-free guidance, ldm/models/diffusion/ddim.py:166-204:
 *   e = e_u + s*(e_c - e_u) (e_c may be NULL); pred_x0 = (x - sqrt(1-a_t) e)/sqrt(a_t);
 *   x_prev = sqrt(a_prev) pred_x0 + sqrt(1 - a_prev - sigma^2) e + sigma * noise (noise may be NULL). */
int cb_ddim_step(const float* x, const float* e_uncond, const float* e_cond, const float* noise, float* x_prev,
                 float* pred_x0, long long n, float guidance_scale, float a_t, float a_prev, float sigma_t,
                 float sqrt_one_minus_at, void* stream);
/* cb_q_sample: DDPM.q_sample (ddpm.py:289-292) with the timestep read on the device: out = sqrt_ac[t]*x0 + sqrt_1mac[t]*noise */
int cb_q_sample(const float* x0, const float* noise, const long long* t, const float* sqrt_ac, const float* sqrt_1mac,
                float* out, int B, int per_sample, void* stream);
/* cb_q_sample_masked: the inpainting / outpainting blend DDIMSampler.ddim_sampling applies before every step when a mask
 *   is given (ddim.py:144-147), with DDPM.q_sample (ddpm.py:289-292) fused in; x0, noise, img, out are [B][C][HW] fp32:
 *     out = (sqrt_ac[t_b]*x0 + sqrt_1mac[t_b]*noise) * m + (1 - m) * img,   m = mask[b*mask_bstride + c*mask_cstride + p]
 *   t is read on the device (int64, B entries).  The fp32 mask's spatial dimensions are dense; a batch or channel stride
 *   of 0 broadcasts that dimension ((B,1,h,w), (1,1,h,w) and (B,C,h,w) masks; soft values allowed).  out may alias img.
 *   Each operation is rounded separately, in the reference's order: bit-identical to the eager fp32 expression. */
int cb_q_sample_masked(const float* x0, const float* noise, const long long* t, const float* sqrt_ac,
                       const float* sqrt_1mac, const float* mask, long long mask_bstride, long long mask_cstride,
                       const float* img, float* out, int B, int C, int HW, void* stream);
/* cb_p_sample: one DDPM ancestral step of LatentDiffusion.p_sample for eps-prediction (ddpm.py:1149-1178, through
 *   p_mean_variance :1118-1147, predict_start_from_noise :231-235 and q_posterior :237-244); x, eps, noise, x_prev, x0
 *   are [B][n] fp32, t is read on the device (int64, B entries), the five tables are the model's fp32 schedule buffers:
 *     x_recon = sqrt_recip_ac[t]*x - sqrt_recipm1_ac[t]*eps, clamped to [-1, 1] when clip_denoised != 0
 *     mean    = coef1[t]*x_recon + coef2[t]*x
 *     x_prev  = mean + ((1 - (t == 0)) * exp(0.5*log_var[t])) * (noise*temperature)
 *   x0 (may be NULL) receives x_recon.  x_prev may alias x.  Each operation is rounded separately, in the reference's
 *   order: bit-identical to the eager fp32 expression.  A NULL required pointer or a non-positive size launches
 *   nothing and returns CB_ERR_ARG. */
int cb_p_sample(const float* x, const float* eps, const float* noise, const long long* t, const float* sqrt_recip_ac,
                const float* sqrt_recipm1_ac, const float* coef1, const float* coef2, const float* log_var,
                float temperature, int clip_denoised, float* x_prev, float* x0, int B, int n, void* stream);

/* ---------------------------------------------------------------------------------------------
 * CosFace-R100 front end (no-grad): meta_net.py:253-264, iresnet.py:26-64.
 * cb_face_warp_resize: fixed 2x3 affine warp (affine_grid + grid_sample bilinear/zeros/align_corners) of the
 *   [B][H][W][3*n_chunks] face stack followed by bilinear resize to out_hw (align_corners), NHWC output with
 *   Cpad channels, image f = chunk*B + b (torch.cat(chunk(...), 0) order, meta_net.py:336-337).
 *   host_affine6 is a HOST pointer to the 6 matrix entries (trans_matrix, meta_net.py:131-142).
 * cb_channel_affine_act: eval BatchNorm2d as y = x*scale[c]+shift[c] and/or PReLU slope[c] (the scale / shift pair or
 *   slope may be NULL; scale and shift are given together, CB_ERR_ARG otherwise).  x and y must be aligned to 4
 *   elements of their dtypes (CB_ERR_ALIGN otherwise); y may be x.
 * cb_l2norm_rows: F.normalize(v, dim=-1).
 * ------------------------------------------------------------------------------------------- */
int cb_channel_affine_act(const void* x, int x_dtype, void* y, int y_dtype, const float* scale, const float* shift,
                          const float* slope, long long rows, int C, void* stream);
int cb_face_warp_resize(const float* faces, void* out, int o_dtype, int B, int H, int W, int n_chunks, int out_hw,
                        int Cpad, const float* host_affine6, void* stream);
int cb_l2norm_rows(const float* x, float* y, int rows, int D, void* stream);
/* cb_ema_rows: EmbeddingManagerId._momentum_update, training branch (embedding_manager.py:484-489), with the identity
 * index read on the device: table[idx[b*idx_stride]] = m*table[...] + (1-m)*src[b] for b < B, rows of `row` floats;
 * indices outside [0, n_rows) are skipped (the reference's `if id_idx < len(self.id_embeddings)`). */
int cb_ema_rows(float* table, const long long* idx, int idx_stride, const float* src, int B, int row, int n_rows,
                float momentum, void* stream);
/* cb_ema_rows_sel: the same update over a fixed-capacity list of n entries, for two- and three-person prompts
 * (embedding_manager.py:321-392: per sample, then its first, second and third identity).  Entry k folds
 * src[src_row[k]] into table[ids[slot[k]]]; slot[k] < 0 marks an unused entry, identities outside [0, n_rows) are
 * skipped, and entries of one identity fold in list order.  ids is the device (B, n_chunks) int64 identity tensor, so
 * a captured step replays with new identities and a new slot list. */
int cb_ema_rows_sel(float* table, const long long* ids, const int* slot, const int* src_row, const float* src, int n,
                    int row, int n_rows, float momentum, void* stream);

/* ---------------------------------------------------------------------------------------------
 * cb_attention_fwd -- fused softmax(Q K^T * scale [+ causal mask]) V with wgmma (flash style): the scores live in
 * registers, K/V blocks of 64 keys are TMA-staged in shared memory, the softmax runs on the accumulator fragments.
 * Replaces ldm/modules/attention.py:178-191 (CrossAttention: self and cross) and the masked CLIP attention driven
 * from ldm/modules/encoders/modules.py:24-31,320-340.
 *   Q [images*nq][ldq], K/V [images*nk][ldk/ldv], O [images*nq][ldo]: head h occupies columns [h*d, (h+1)*d);
 *   16-bit operands (dtype), d a multiple of 8 up to 128; strides in elements.
 *   lse (optional) [images][heads][nq] fp32: log-sum-exp of the scaled scores.
 *   P (optional) [images*heads][nq][ldp] 16-bit: the normalised probabilities, written for a backward pass that
 *   wants them (two-pass mode: pass 1 row max/sum, pass 2 probabilities + P.V); ldp multiple of 8, >= nk,
 *   columns nk..ldp-1 are written as 0.
 * ------------------------------------------------------------------------------------------- */
int cb_attention_fwd(const void* Q, long long ldq, const void* K, long long ldk, const void* V, long long ldv, void* O,
                     long long ldo, float* lse, void* P, long long ldp, int dtype, int images, int heads, int nq,
                     int nk, int d, float scale, int causal, void* stream);

/* ---------------------------------------------------------------------------------------------
 * cb_attention_bwd -- flash-style backward of the same attention (the gradient torch.autograd derives for
 * ldm/modules/attention.py:178-191): dQ, dK, dV from Q, K, V, O, dO and the forward's lse, recomputing the
 * probabilities tile by tile in registers; no (heads x N x N) tensor and no atomics.  Two launches: query-stationary
 * (dQ, also writes delta = rowsum(dO o O)) then key-stationary (dK, dV).
 *   layouts as cb_attention_fwd; dQ/dK/dV use the layouts of Q/K/V with their own row pitches;
 *   delta: caller workspace [images][heads][nq] fp32.
 * ------------------------------------------------------------------------------------------- */
int cb_attention_bwd(const void* Q, long long ldq, const void* K, long long ldk, const void* V, long long ldv,
                     const void* O, long long ldo, const void* dO, long long lddo, const float* lse, float* delta,
                     void* dQ, long long lddq, void* dK, long long lddk, void* dV, long long lddv, int dtype, int images,
                     int heads, int nq, int nk, int d, float scale, int causal, void* stream);

/* Query-stationary half only: dQ (optional) and, optionally, dS = P o (dP - delta) * scale exported as
 * [images*heads][nq][ldds] (16-bit, ldds a multiple of 8 >= nk) -- for short key sequences (cross attention on the 77
 * prompt tokens, attention.py:170-193 with context=cond), where dK = dS^T Q and dV = P^T dO are better done as two small
 * cb_gemm launches over the exported dS and the forward's P than by 8 key-stationary CTAs. */
int cb_attention_bwd_dq(const void* Q, long long ldq, const void* K, long long ldk, const void* V, long long ldv,
                        const void* O, long long ldo, const void* dO, long long lddo, const float* lse, float* delta,
                        void* dQ, long long lddq, void* dS, long long ldds, int dtype, int images, int heads, int nq,
                        int nk, int d, float scale, int causal, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Checkpoint-load-time packing (once per load_state_dict; the reference keeps fp32 nn.Parameters,
 * ldm/modules/diffusionmodules/openaimodel.py:201-241, and lets cuDNN choose layouts per call).
 * cb_pack_conv_weight: [Cout][Cin][kh][kw] fp32 -> [kh*kw][Cout_pad][Cin_pad] 16-bit (tap-major, Cin contiguous, zero
 *   padded) -- the B operand of the implicit-GEMM convolution; out_scale (optional, [Cout]) folds an eval BatchNorm
 *   that follows the convolution (ldm/modules/id_embedding/iresnet.py:41-58) into the weights.
 * cb_convert_f32: out[i] = (o_dtype) (scale * x[i]) for any n.
 * o_dtype is CB_F16, CB_BF16 or CB_F32 for both (CB_ERR_ARG otherwise).
 * ------------------------------------------------------------------------------------------- */
int cb_pack_conv_weight(const float* w, void* out, int o_dtype, int cout, int cin, int kh, int kw, int cout_pad,
                        int cin_pad, const float* out_scale, void* stream);
int cb_convert_f32(const float* x, void* out, int o_dtype, long long n, float scale, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Parameter gradients for fine-tuning the UNet and the CLIP text encoder (`unfreeze_model`, ddpm.py:1450-1452): the
 * weight, bias and affine gradients torch.autograd computes for the reference's nn.Conv2d / nn.Linear / GroupNorm32 /
 * nn.LayerNorm / nn.Embedding.  Outputs are fp32; alpha scales every result (e.g. 1 / the static loss scale).  Every sum
 * is taken in a fixed order: bit-reproducible from run to run.
 * cb_conv_wgrad: dW[co][ci][ky][kx] = alpha * sum_{n,oh,ow} dy[n][oh][ow][co] * x[n][oh*s+ky-pad][ow*s+kx-pad][ci]
 *   (zero outside the image) for k x k kernels, k = 1 or 3, stride s, symmetric padding; x is NHWC [N*H*W][ldx], dy
 *   [N*OH*OW][lddy], both of `dtype` (CB_F16 / CB_BF16); dW is written in the nn.Parameter layout [cout][cin][k][k].
 *   cin, cout, ldx and lddy must be multiples of 8 and the pointers 16-byte aligned (CB_ERR_ALIGN otherwise): pad the
 *   channels with zeros and slice the result.  One cb_gemm launch (M = cout, N = cin*k*k, K = N*OH*OW, both operands
 *   MN-major) over `col`, the taps of x gathered in the parameter's column order by one more launch; a 1x1 stride-1
 *   unpadded convolution (and so a linear layer, x = [rows][in]) reads x directly and needs no col.  The k-loop is split
 *   into a number of slices that depends on the shape and the device's SM count only, reduced in slice order through
 *   splitk_ws (the cb_gemm split-K workspace: zero-filled before its first use, every call leaves its counters zero).
 * cb_conv_wgrad_ws_bytes: host-only; the bytes of `col` (0: not used) and of splitk_ws (0: not used) that cb_conv_wgrad
 *   needs for a geometry (CB_ERR_ARG if cb_conv_wgrad would refuse the geometry).
 * cb_colsum: out[g][c] = alpha * sum of rows [g*rows/groups, (g+1)*rows/groups) of x[rows][ldx], column c < C (x of
 *   any dtype).  groups = 1: a bias gradient; groups = images: the per-image sum of a pixel gradient (the gradient of a
 *   ResBlock's emb_layers output, openaimodel.py:262-266 `h = h + emb_out`); a [B][T*D] view of the CLIP embedding
 *   gradient: the position-embedding gradient (modules.py:295-296).
 * cb_groupnorm_affine_bwd / cb_layernorm_affine_bwd: dgamma[c] = alpha * sum dz*xh, dbeta[c] = alpha * sum dz over all
 *   rows, xh = (x - mean) * rstd from the forward's saved statistics ([N][G] / one per row), dz = dy, or
 *   dy * silu'(xh*gamma + beta) with act_silu bit 0 (GroupNorm fused with SiLU).  Either output may be NULL.
 * cb_embedding_bwd: dtable[v] = alpha * sum of the rows dout[i] (row pitch ld) of the tokens i with ids[i] == v, added in
 *   token order; ids are clamped to [0, V) like cb_embedding_gather; rows of ids that do not occur are not written.
 * ------------------------------------------------------------------------------------------- */
int cb_conv_wgrad_ws_bytes(int N, int H, int W, int cin, int cout, int k, int stride, int pad, long long* col_bytes,
                           long long* splitk_bytes);
int cb_conv_wgrad(const void* x, long long ldx, const void* dy, long long lddy, int dtype, int N, int H, int W, int cin,
                  int cout, int k, int stride, int pad, float alpha, float* dW, void* col, void* splitk_ws,
                  long long splitk_ws_bytes, void* stream);
int cb_colsum(const void* x, int x_dtype, long long ldx, float* out, long long rows, int C, int groups, float alpha,
              void* stream);
int cb_groupnorm_affine_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, const float* gamma,
                            const float* beta, const float* mean, const float* rstd, float* dgamma, float* dbeta, int N,
                            int HW, int C, int G, int act_silu, float alpha, void* stream);
int cb_layernorm_affine_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, const float* mean,
                            const float* rstd, float* dgamma, float* dbeta, int M, int C, float alpha, void* stream);
int cb_embedding_bwd(const long long* ids, const float* dout, long long ld, float* dtable, int n, int D, int V,
                     float alpha, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Device-side data path (SURVEY 8f-2): the pixel work of FaceIdDatasetStyleGAN3.__getitem__
 * (ldm/data/face_id.py:526-532 transform chain, :451-470 _add_bg, :598-644).  Random draws stay on the host.
 * cb_face_augment: uint8 [B][H][W][3] -> RandomHorizontalFlip, ColorJitter (ops in the drawn order, torchvision tensor
 *   arithmetic), ToTensor, Normalize(0.5,0.5): fp32 in [-1,1] written into channels [c_off, c_off+3) of an
 *   [B][H][W][c_total] tensor (the `faces` stack).  iparams [B][5] = {flip, op order x4 (0 brightness, 1 contrast,
 *   2 saturation, 3 hue, <0 skip)}, fparams [B][4] = {brightness, contrast, saturation, hue factor}; ws: B doubles.
 * cb_paste_resized: _add_bg -- out [B][H][W][3] = -1 with the face (channels [c_off, c_off+3) of faces) resized
 *   bilinearly (align_corners=True, ATen index math) to (rh, rw) and pasted at (pos_h, pos_w); geo [B][4].
 * ------------------------------------------------------------------------------------------- */
int cb_face_augment(const unsigned char* src_u8, const int* iparams, const float* fparams, double* ws, float* out, int B,
                    int H, int W, int c_total, int c_off, void* stream);
int cb_paste_resized(const float* faces, int c_total, int c_off, const int* geo, float* out, int B, int H, int W,
                     void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CELEBBASIS_B200_H_ */
