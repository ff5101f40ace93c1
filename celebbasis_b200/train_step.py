"""One CelebBasis training step (SURVEY.md §8 rows a1-a31) on the sm_90a kernels.

    image --VAE encode--> z --q_sample(t, noise)--> x_t --\
    faces --warp/resize--> CosFace R100 --> v -- MLP(W,b) --> coef --basis--> 2 token embeddings      UNet --> eps
    caption --tokenise--> ids --gather--> token rows --inject @placeholder--> +pos --> CLIP text --> context --/
    loss = MSE(eps, noise);  backward: UNet -> d(context) -> CLIP -> d(embeddings) -> d(W), d(b);  AdamW.

This is the function LatentDiffusion.shared_step + loss.backward() + optimizer.step() of the reference performs
(ldm/models/diffusion/ddpm.py:921-936,1069-1116,1442-1454).  Forward and backward are launched back to back so the
whole step can be captured in one CUDA graph; torch is used for buffers, streams and the graph only.
"""
import contextlib

import numpy as np
import torch

from . import ops
from .clip_engine import CLIPTextEngine
from .iresnet_engine import IResNetEngine
from .unet_engine import UNetEngine
from .vae_engine import VAEEncoderEngine

TRANS_MATRIX = (1.07695457, -0.03625215, -1.56352194 / 512, 0.03625215, 1.07695457, -5.32134629 / 512)


def get_rep_pos(tokenized, rep_tokens):
    """ldm/modules/id_embedding/helpers.py:6-10 on a host int array."""
    tok = np.asarray(tokenized)
    return [np.where(tok == int(t))[0] for t in rep_tokens]


def placeholder_row_map(n_rows, r_pos, reps):
    """Host mirror of shift_tensor_dim0 (helpers.py:13-41) expressed as a gather map.

    Returns (src, final_pos): src[i] = index of the ORIGINAL row that sits in row i after the reference's two
    in-place advanced-index writes; final_pos[k] = (occurrences, reps) array of rows that then receive the learned
    embeddings for placeholder k.  Pure integer arithmetic, bit-exact with the reference."""
    offset = np.zeros(n_rows, dtype=np.int64)
    cat = np.concatenate(r_pos) if len(r_pos) else np.zeros(0, dtype=np.int64)
    for p in cat:
        offset[p + 1:] += reps - 1
    n_occ = cat.shape[0]
    target = (np.arange(n_rows) + offset)[: n_rows - n_occ * (reps - 1)]
    src = np.arange(n_rows)
    src[target] = np.arange(target.shape[0])                     # "shift words"
    final = target[cat].repeat(reps) + np.tile(np.arange(reps), n_occ)
    before = src.copy()
    src[final] = before[target[cat].repeat(reps)]                # "fill blanks with repeat words"
    out, lo = [], 0
    for p in r_pos:
        k = p.shape[0]
        out.append(final[lo: lo + k * reps].reshape(k, reps))
        lo += k * reps
    return src, out


def build_inject_map_multi(ids, per_sample, reps):
    """ids: (B,T) host int64.  per_sample[b] = (placeholder_tokens, z_row_bases): the k-th placeholder of prompt b is
    replaced by z rows z_row_bases[k] .. +reps-1.  map[b][i] >= 0: take token row map[b][i] of prompt b; < 0: take
    z row -(map+1).  (EmbeddingManagerId.forward, embedding_manager.py:322-392: one/two/three persons.)"""
    ids = np.asarray(ids)
    B, T = ids.shape
    m = np.zeros((B, T), dtype=np.int32)
    positions = []
    for b in range(B):
        toks, bases = per_sample[b]
        pos = get_rep_pos(ids[b], toks)
        src, fin = placeholder_row_map(T, pos, reps)
        row = src.astype(np.int32)
        for k, base in enumerate(bases):
            for one_pos in fin[k]:
                for j, p in enumerate(one_pos):
                    row[int(p)] = -(int(base) + j + 1)
        m[b] = row
        positions.append(fin)
    return m, positions


def build_inject_map(ids, placeholder_token, reps, z_row_of_sample):
    """Single-person prompts (num_ids == 1 branch, embedding_manager.py:347-360)."""
    B = np.asarray(ids).shape[0]
    return build_inject_map_multi(ids, [([placeholder_token], [z_row_of_sample(b) * reps]) for b in range(B)], reps)


class CelebBasisStep:
    def __init__(self, params, state_dict, basis, device, *, tokenizer, placeholder="sks", clip_layers=None,
                 dtype=torch.float16, loss_scale=1024.0, vae_res_dtype=torch.float32, lr=5e-3, id_coefficients=None,
                 id_embeddings=None):
        self.dev = torch.device(device)
        self.dt = dtype
        sd = state_dict
        sub = lambda pre: {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}
        self.unet = UNetEngine(params["unet_config"]["params"], sub("model.diffusion_model."), self.dev, dtype=dtype,
                               loss_scale=loss_scale)
        self.clip = CLIPTextEngine(sub("cond_stage_model.transformer."), self.dev, dtype=dtype, loss_scale=loss_scale)
        fs = params["first_stage_config"]["params"]
        self.vae = VAEEncoderEngine(fs["ddconfig"], fs["embed_dim"], sub("first_stage_model."), self.dev, dtype=dtype,
                                    res_dtype=vae_res_dtype)
        self.face = IResNetEngine(sub("embedding_manager.meta_id_net.id_model."), self.dev, dtype=dtype)
        pc = params["personalization_config"]["params"]
        self.es = pc["num_embeds_per_token"]
        self.K = pc["meta_inner_dim"]
        self.momentum = pc.get("momentum", 0.9)
        self.max_ids = pc.get("max_ids", 10)
        self.W = sd["embedding_manager.meta_id_net.stylegan_mlp.net.0.weight"].detach().to(self.dev, torch.float32).contiguous()
        self.b = sd["embedding_manager.meta_id_net.stylegan_mlp.net.0.bias"].detach().to(self.dev, torch.float32).contiguous()
        # trainable tensors live in ONE flat fp32 buffer (what the data-parallel all-reduce and AdamW operate on)
        self.flat = torch.cat([self.W.flatten(), self.b.flatten()]).contiguous()
        self.W = self.flat[: self.W.numel()].view_as(self.W)
        self.b = self.flat[self.W.numel():]
        self.grad = torch.zeros_like(self.flat)
        self.gW = self.grad[: self.W.numel()].view_as(self.W)
        self.gb = self.grad[self.W.numel():]
        self.adam_m = torch.zeros_like(self.flat)
        self.adam_v = torch.zeros_like(self.flat)
        self.step_dev = torch.zeros(1, dtype=torch.int32, device=self.dev)
        self.lr = lr
        self.overlap_branches = True     # VAE encode || face net + CLIP text on two streams (see run())
        self._side = None
        self._warm = False
        self.basis = basis.detach().to(self.dev, torch.float32).contiguous()
        self.tokenizer = tokenizer
        self.placeholder_token = int(tokenizer(placeholder)["input_ids"][0, 1])
        self.scale_factor = float(params["scale_factor"])
        # schedule (ddpm.py:126-178; util.py:21-25: float64 linspace of sqrt(beta), squared)
        T = params["timesteps"]
        betas = torch.linspace(params["linear_start"] ** 0.5, params["linear_end"] ** 0.5, T, dtype=torch.float64) ** 2
        ac = np.cumprod(1.0 - betas.numpy(), axis=0)
        self.sqrt_ac = torch.tensor(np.sqrt(ac), dtype=torch.float32, device=self.dev)
        self.sqrt_1mac = torch.tensor(np.sqrt(1.0 - ac), dtype=torch.float32, device=self.dev)
        self.num_timesteps = T
        # per-identity EMA side state, initialised as EmbeddingManagerId does (embedding_manager.py:229-252): ONE randn
        # coefficient tensor shared by every identity, embeddings = the initializer word's token embedding
        self.test_mode = pc.get("test_mode", "coefficient")
        self.save_fp16 = bool(pc.get("save_fp16", True))
        if id_coefficients is None:
            id_coefficients = [torch.randn(self.es, 1, self.K)] * self.max_ids
        if id_embeddings is None:
            words = pc.get("initializer_words") or []
            if words:
                wid = int(tokenizer(words[0])["input_ids"][0, 1])
                init = self.clip.tok_table[wid].detach().float().cpu()
                id_embeddings = [init.unsqueeze(0).repeat(self.es, 1)] * self.max_ids
            else:
                id_embeddings = [torch.rand(self.es, self.clip.hidden) for _ in range(self.max_ids)]
        self.id_coefficients = torch.stack([c.detach().float().reshape(self.es, 1, self.K) for c in id_coefficients]) \
            .to(self.dev).contiguous()
        self.id_embeddings = torch.stack([e.detach().float().reshape(self.es, -1) for e in id_embeddings]) \
            .to(self.dev).contiguous()
        self._prio = None
        self.last = {}

    # ------------------------------------------------------------------------------------------
    def tokenize(self, captions):
        return self.tokenizer(captions, truncation=True, max_length=77, return_length=True,
                              return_overflowing_tokens=False, padding="max_length", return_tensors="pt")["input_ids"]

    def encode_first_stage(self, image_nhwc, posterior_eps):
        """get_input (ddpm.py:344-350,702-759): HWC->CHW, VAE encode, posterior sample * scale_factor."""
        x = image_nhwc.permute(0, 3, 1, 2).contiguous().float()   # layout glue exactly as ddpm.py:348-349
        moments = self.vae.encode_moments(x)
        z = ops.posterior_sample(moments, posterior_eps.contiguous(), self.scale_factor)
        return z, moments

    def face_features(self, faces, n_chunks):
        x, geo = ops.face_warp_resize(faces.contiguous(), n_chunks, TRANS_MATRIX, out_hw=112, cpad=8, dtype=self.dt)
        feat = self.face.forward(x, geo)
        return ops.l2norm_rows(feat)

    def q_sample(self, z, t, noise):
        """ddpm.py:289-292 per sample (the two coefficients are device scalars gathered by t)."""
        return ops.q_sample(z.contiguous(), noise.contiguous(), t.contiguous(), self.sqrt_ac, self.sqrt_1mac)

    # ------------------------------------------------------------------------------------------
    def prepare(self, captions):
        """Host side of the step: tokenise, locate the placeholder, build the row map (bit-exact integer path)."""
        ids = self.tokenize(captions)
        map_np, positions = build_inject_map(ids.numpy(), self.placeholder_token, self.es, lambda b: b)
        return ids, map_np, positions

    def forward_backward(self, batch, draws, need_grad=True, ema_update=True):
        """batch: dict as face_id.py:598-644 yields (tensors on self.dev); draws: t (B,), noise, posterior_eps.
        Returns the loss (1-element device tensor).  Gradients of (W,b) land in self.grad."""
        ids, map_np, positions = self.prepare(batch["caption"])
        ids_dev = ids.to(self.dev)
        map_dev = torch.from_numpy(map_np).to(self.dev)
        io = batch["image_ori"]
        return self.run(batch["image"], io["faces"], io["ids"], ids_dev, map_dev, draws["t"], draws["noise"],
                        draws["posterior_eps"], need_grad=need_grad, ema_update=ema_update, positions=positions, ids=ids)

    def run(self, image, faces, ids_person, ids_dev, map_dev, t, noise, posterior_eps, *, need_grad=True,
            ema_update=True, positions=None, ids=None):
        """Device side of the step: only kernel launches on the current stream (CUDA-graph capturable)."""
        B = image.shape[0]
        n_chunks = ids_person.shape[1]
        T = ids_dev.shape[1]
        # Two independent branches until the UNet: (a) face net -> celeb-basis MLP -> CLIP text (small, latency-bound
        # launches that use few SMs) and (b) VAE encode + q_sample (large, throughput-bound convs).  They run on two
        # streams (fork/join with events; a captured graph keeps them as parallel branches).  Branch (a) never launches
        # a grid-barrier kernel (no GroupNorm), so the fused GroupNorm of branch (b) keeps its co-residency guarantee.
        main = torch.cuda.current_stream()
        overlap = self.overlap_branches and self._warm      # first call: sequential, so the GEMM autotuner times alone
        self._warm = True
        if overlap:
            side = self._side_stream()
            fork = torch.cuda.Event()
            fork.record(main)
            side.wait_event(fork)
            ctx_a, lane_a = torch.cuda.stream(side), ops.lane(1)
        else:
            ctx_a, lane_a = contextlib.nullcontext(), contextlib.nullcontext()
        with ctx_a, lane_a:
            v = self.face_features(faces, n_chunks)                                  # (n_chunks*B, 512)
            pre, coef, nrm = ops.celeb_mlp_fwd(v, self.W, self.b, self.es)
            zc = ops.celeb_basis_fwd(coef, self.basis)                               # (F, es, 768)
            tok = ops.embedding_gather(ids_dev.view(-1), self.clip.tok_table)
            emb = ops.embed_inject_fwd(tok, zc.view(-1, zc.shape[-1]), map_dev.view(-1), self.clip.pos_table, B, T)
            context = self.clip.forward(emb, B, need_grad=need_grad)                 # (B*T, 768) fp32
            if overlap:
                join = torch.cuda.Event()
                join.record(side)
        z, _ = self.encode_first_stage(image, posterior_eps)
        noise = noise.contiguous()
        x_noisy = self.q_sample(z, t, noise)
        if overlap:
            main.wait_event(join)
        eps = self.unet.forward(x_noisy, t, context.view(B, T, -1), need_grad=need_grad)
        loss_simple, d_eps = ops.mse_fwd_bwd(eps, noise, 1.0, want_grad=need_grad)   # (B,) per-sample losses
        loss = loss_simple if B == 1 else loss_simple.mean(0, keepdim=True)
        self.last = dict(z=z, context=context.view(B, T, -1), eps=eps, x_noisy=x_noisy, coef=coef, celeb_z=zc,
                         face_feat=v, positions=positions, ids=ids)
        if ema_update:
            self._ema_update(zc, coef, ids_person, B)
        if need_grad:
            dctx = self.unet.backward(d_eps)
            demb = self.clip.backward(dctx.view(B * T, -1))
            dz = ops.embed_inject_bwd(demb, map_dev.view(-1), zc.shape[0] * self.es, B, T)
            dcoef = ops.celeb_basis_bwd(dz.view(zc.shape), self.basis)
            ops.celeb_mlp_bwd(dcoef, coef, nrm, pre, v, self.gW, self.gb)
            self.last.update(d_eps=d_eps, dctx=dctx, demb=demb, dz=dz, dcoef=dcoef)
        return loss

    def _side_stream(self):
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.dev)
        return self._side

    def _ema_update(self, zc, coef, ids_person, B):
        """_momentum_update, training branch (embedding_manager.py:484-489) for the main identity of each sample; the
        identity index is read on the device (no host sync, CUDA-graph safe)."""
        idx = ids_person if ids_person.is_cuda else ids_person.to(self.dev)
        idx = idx.long()
        ops.ema_rows(self.id_embeddings.view(self.max_ids, -1), idx, zc[:B].reshape(B, -1), self.momentum)
        ops.ema_rows(self.id_coefficients.view(self.max_ids, -1), idx, coef[:B].reshape(B, -1), self.momentum)

    # ------------------------------------------------------------------------------------------
    # the step as two stages: a frozen no-grad front end that does not depend on the trained weights (and can therefore
    # be computed for the NEXT batch while this batch trains) and the trainable chain
    # ------------------------------------------------------------------------------------------
    def stage_prefetch(self, image, faces, n_chunks, posterior_eps, z_out=None, v_out=None):
        """get_input's VAE encode + posterior sample (ddpm.py:702-759) and the CosFace features of the face crops
        (meta_net.py:329-346, no_grad): two concurrent branches, neither uses a grid-barrier kernel (lanes 1 / 2)."""
        main = torch.cuda.current_stream()
        side = self._side_stream()
        fork = torch.cuda.Event()
        fork.record(main)
        side.wait_event(fork)
        with torch.cuda.stream(side), ops.lane(1):
            v = self.face_features(faces, n_chunks)
            if v_out is not None:
                v_out.copy_(v)
            join = torch.cuda.Event()
            join.record(side)
        with ops.lane(2):
            z, _ = self.encode_first_stage(image, posterior_eps)
            if z_out is not None:
                z_out.copy_(z)
        main.wait_event(join)
        return (z if z_out is None else z_out), (v if v_out is None else v_out)

    def stage_main(self, z, v, ids_person, ids_dev, map_dev, t, noise, *, need_grad=True, ema_update=True):
        """Everything downstream of the trainable MLP: celeb-basis embeddings -> inject -> CLIP text -> UNet -> loss ->
        backward to (W, b).  Returns the loss; gradients land in self.grad."""
        B, T = z.shape[0], ids_dev.shape[1]
        # the text branch (MLP -> basis -> inject -> 12 CLIP layers, ~110 small launches) runs beside the UNet's prefix
        # (timestep MLP, stem, first ResBlock, first self-attention): the UNet waits for the context at its first
        # cross-attention
        main = torch.cuda.current_stream()
        aux = self._aux_stream()
        fork = torch.cuda.Event()
        fork.record(main)
        aux.wait_event(fork)
        with torch.cuda.stream(aux), ops.lane(3):
            pre, coef, nrm = ops.celeb_mlp_fwd(v, self.W, self.b, self.es)
            zc = ops.celeb_basis_fwd(coef, self.basis)
            tok = ops.embedding_gather(ids_dev.view(-1), self.clip.tok_table)
            emb = ops.embed_inject_fwd(tok, zc.view(-1, zc.shape[-1]), map_dev.view(-1), self.clip.pos_table, B, T)
            context = self.clip.forward(emb, B, need_grad=need_grad)
            ctx_ready = torch.cuda.Event()
            ctx_ready.record(aux)
        noise = noise.contiguous()
        x_noisy = self.q_sample(z, t, noise)
        eps = self.unet.forward(x_noisy, t, context.view(B, T, -1), need_grad=need_grad, context_ready=ctx_ready)
        main.wait_event(ctx_ready)      # (already implied by the UNet's first cross-attention; explicit for the EMA / backward)
        loss_simple, d_eps = ops.mse_fwd_bwd(eps, noise, 1.0, want_grad=need_grad)
        loss = loss_simple if B == 1 else loss_simple.mean(0, keepdim=True)
        self.last = dict(z=z, context=context.view(B, T, -1), eps=eps, x_noisy=x_noisy, coef=coef, celeb_z=zc,
                         face_feat=v, loss_simple=loss_simple)
        if ema_update:
            self._ema_update(zc, coef, ids_person, B)
        if need_grad:
            dctx = self.unet.backward(d_eps)
            demb = self.clip.backward(dctx.view(B * T, -1))
            dz = ops.embed_inject_bwd(demb, map_dev.view(-1), zc.shape[0] * self.es, B, T)
            dcoef = ops.celeb_basis_bwd(dz.view(zc.shape), self.basis)
            ops.celeb_mlp_bwd(dcoef, coef, nrm, pre, v, self.gW, self.gb)
        return loss

    def _aux_stream(self):
        if getattr(self, "_aux", None) is None:
            self._aux = torch.cuda.Stream(device=self.dev, priority=-1)
        return self._aux

    def _prio_stream(self):
        if self._prio is None:
            self._prio = torch.cuda.Stream(device=self.dev, priority=-1)
        return self._prio

    # ---- checkpoint (embedding_manager.py:396-410): the file stable_txt2img.py:230 loads -----------------------
    def gathered_identity_state(self, owned_ids=None):
        """Per-identity EMA state of ALL ranks (each rank updates only the identities it trains; the reference keeps
        them rank-local and saves rank 0's copy only).  owned_ids: identities this rank trained (None = all)."""
        from . import dist as cbd
        if cbd.world_size() > 1 and owned_ids is not None:
            return (cbd.gather_identity_state(self.id_coefficients, list(owned_ids), self.max_ids),
                    cbd.gather_identity_state(self.id_embeddings, list(owned_ids), self.max_ids))
        return self.id_coefficients, self.id_embeddings

    def save(self, path, owned_ids=None):
        """Writes the reference's embedding-manager checkpoint: {"id_coefficients": [max_ids x (es,1,K)]} (test_mode
        'coefficient'), {"id_embeddings": ...} ('embedding') or the MLP state ('image'); fp16 when save_fp16."""
        coef, emb = self.gathered_identity_state(owned_ids)
        cast = (lambda x: x.detach().cpu().half()) if self.save_fp16 else (lambda x: x.detach().cpu().clone())
        out = {}
        if self.test_mode == "coefficient":
            out["id_coefficients"] = [cast(c) for c in coef.unbind(0)]
        elif self.test_mode == "embedding":
            out["id_embeddings"] = [cast(e) for e in emb.unbind(0)]
        else:
            out["meta_id_net"] = {"stylegan_mlp.net.0.weight": self.W.detach().cpu().clone(),
                                  "stylegan_mlp.net.0.bias": self.b.detach().cpu().clone()}
        from . import dist as cbd
        if cbd.rank() == 0:
            torch.save(out, path)
        return out

    def optimizer_step(self, lr=None):
        """torch.optim.AdamW defaults (ddpm.py:1442-1454): betas (.9,.999), eps 1e-8, weight_decay 1e-2."""
        ops.adamw_step(self.flat, self.grad, self.adam_m, self.adam_v, lr=self.lr if lr is None else lr,
                       step_dev=self.step_dev)
