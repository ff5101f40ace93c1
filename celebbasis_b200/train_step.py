"""One CelebBasis training step (SURVEY.md §8 rows a1-a31) on the sm_90a kernels.

    image --VAE encode--> z --q_sample(t, noise)--> x_t --\
    faces --warp/resize--> CosFace R100 --> v -- MLP(W,b) --> coef --basis--> 2 token embeddings      UNet --> eps
    caption --tokenise--> ids --gather--> token rows --inject @placeholder--> +pos --> CLIP text --> context --/
    loss = MSE(eps, noise);  backward: UNet -> d(context) -> CLIP -> d(embeddings) -> d(W), d(b);  AdamW.

This is the function LatentDiffusion.shared_step + loss.backward() + optimizer.step() of the reference performs
(ldm/models/diffusion/ddpm.py:921-936,1069-1116,1442-1454).  Forward and backward are launched back to back so the
whole step can be captured in one CUDA graph; torch is used for buffers, streams and the graph only.
"""
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


class _LatentTrainStep:
    """What both training steps share: the frozen UNet / CLIP text / VAE encoder engines, the noise schedule, the front
    end (VAE encode + posterior sample) and the trainable chain's tail (token gather -> inject of the trained rows -> CLIP
    text -> UNet -> MSE -> UNet / CLIP backward -> gradient of the rows).  A subclass says where the injected rows come
    from (_rows_fwd) and where their gradient goes (_rows_bwd)."""

    def __init__(self, params, state_dict, device, *, tokenizer, dtype=torch.float16, loss_scale=1024.0,
                 vae_res_dtype=torch.float32, lr=5e-3):
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
        self.step_dev = torch.zeros(1, dtype=torch.int32, device=self.dev)
        self.lr = lr
        self._aux = torch.cuda.Stream(device=self.dev, priority=-1)     # stage_main's text branch
        self.tokenizer = tokenizer
        self.scale_factor = float(params["scale_factor"])
        # schedule (ddpm.py:126-178; util.py:21-25: float64 linspace of sqrt(beta), squared)
        T = params["timesteps"]
        betas = torch.linspace(params["linear_start"] ** 0.5, params["linear_end"] ** 0.5, T, dtype=torch.float64) ** 2
        ac = np.cumprod(1.0 - betas.numpy(), axis=0)
        self.sqrt_ac = torch.tensor(np.sqrt(ac), dtype=torch.float32, device=self.dev)
        self.sqrt_1mac = torch.tensor(np.sqrt(1.0 - ac), dtype=torch.float32, device=self.dev)
        self.num_timesteps = T
        self.last = {}
        self.loss_weights = None        # (l_simple_weight, original_elbo_weight, logvar (T,), lvlb_weights (T,))

    def set_loss_weights(self, l_simple_weight, original_elbo_weight, logvar, lvlb_weights):
        """p_losses' loss weights (ddpm.py:1084-1099).  logvar / lvlb_weights: the model's (T,) tables.  Once set, the step
        computes its loss and gradient with cb_diffusion_loss_fwd_bwd instead of cb_mse_fwd_bwd + cb_loss_mean."""
        f32 = dict(dtype=torch.float32, device=self.dev)
        self.loss_weights = (float(l_simple_weight), float(original_elbo_weight),
                             logvar.detach().to(**f32).contiguous(), lvlb_weights.detach().to(**f32).contiguous())

    def _init_flat(self, tensors):
        """The trainable tensors live in ONE flat fp32 buffer (what the data-parallel all-reduce and AdamW operate on);
        returns views of it and of the gradient buffer shaped like `tensors`."""
        self.flat = torch.cat([t.detach().to(self.dev, torch.float32).reshape(-1) for t in tensors]).contiguous()
        self.grad = torch.zeros_like(self.flat)
        self.adam_m = torch.zeros_like(self.flat)
        self.adam_v = torch.zeros_like(self.flat)
        views, grads, off = [], [], 0
        for t in tensors:
            views.append(self.flat[off: off + t.numel()].view(t.shape))
            grads.append(self.grad[off: off + t.numel()].view(t.shape))
            off += t.numel()
        return views, grads

    def tokenize(self, captions):
        return self.tokenizer(captions, truncation=True, max_length=77, return_length=True,
                              return_overflowing_tokens=False, padding="max_length", return_tensors="pt")["input_ids"]

    def encode_first_stage(self, image_nhwc, posterior_eps):
        """get_input (ddpm.py:344-350,702-759): HWC->CHW, VAE encode, posterior sample * scale_factor."""
        x = image_nhwc.permute(0, 3, 1, 2).contiguous().float()   # layout glue exactly as ddpm.py:348-349
        moments = self.vae.encode_moments(x)
        z = ops.posterior_sample(moments, posterior_eps.contiguous(), self.scale_factor)
        return z, moments

    def q_sample(self, z, t, noise):
        """ddpm.py:289-292 per sample (the two coefficients are device scalars gathered by t)."""
        return ops.q_sample(z.contiguous(), noise.contiguous(), t.contiguous(), self.sqrt_ac, self.sqrt_1mac)

    def ema_state(self):
        """Device tensors a step updates besides the gradient (restored after StepGraphs' warm-up steps)."""
        return ()

    def stage_main(self, z, v, ids_person, ids_dev, map_dev, t, noise, *, need_grad=True, ema_update=True):
        """Everything downstream of the frozen front end: the rows to inject -> inject -> CLIP text -> UNet -> loss ->
        backward to the trained tensors.  Returns the loss; gradients land in self.grad."""
        B, T = z.shape[0], ids_dev.shape[1]
        # the text branch (rows -> inject -> 12 CLIP layers, ~110 small launches) runs beside the UNet's prefix (timestep
        # MLP, stem, first ResBlock, first self-attention): the UNet waits for the context at its first cross-attention
        main = torch.cuda.current_stream()
        aux = self._aux
        fork = torch.cuda.Event()
        fork.record(main)
        aux.wait_event(fork)
        with torch.cuda.stream(aux), ops.lane(3):
            rows, saved = self._rows_fwd(v)
            tok = ops.embedding_gather(ids_dev.view(-1), self.clip.tok_table)
            emb = ops.embed_inject_fwd(tok, rows, map_dev.view(-1), self.clip.pos_table, B, T)
            context = self.clip.forward(emb, B, need_grad=need_grad)
            ctx_ready = torch.cuda.Event()
            ctx_ready.record(aux)
        noise = noise.contiguous()
        x_noisy = self.q_sample(z, t, noise)
        eps = self.unet.forward(x_noisy, t, context.view(B, T, -1), need_grad=need_grad, context_ready=ctx_ready)
        main.wait_event(ctx_ready)      # (already implied by the UNet's first cross-attention; explicit for the EMA / backward)
        loss_vlb = None
        if self.loss_weights is None:
            loss_simple, d_eps = ops.mse_fwd_bwd(eps, noise, 1.0, want_grad=need_grad)
            loss = loss_simple if B == 1 else ops.loss_mean(loss_simple)
        else:
            lsw, ew, logvar, lvlb = self.loss_weights
            loss_simple, loss, loss_vlb, d_eps = ops.diffusion_loss_fwd_bwd(eps, noise, t, logvar, lvlb, lsw, ew, 1.0,
                                                                            want_grad=need_grad)
        self.last = dict(z=z, context=context.view(B, T, -1), eps=eps, x_noisy=x_noisy, loss_simple=loss_simple,
                         loss_vlb=loss_vlb, **self._rows_last(saved, v))
        if ema_update:
            self._rows_ema(saved, ids_person, B)
        if need_grad:
            dctx = self.unet.backward(d_eps)
            demb = self.clip.backward(dctx.view(B * T, -1))
            self._rows_bwd(demb, map_dev, B, T, saved, v)
            self._loss_extra(loss)
        return loss

    def _loss_extra(self, loss):
        """Terms of the loss on the trained tensors alone, added to `loss` and to the gradient after the backward."""
        pass

    def _rows_last(self, saved, v):
        return {}

    def _rows_ema(self, saved, ids_person, B):
        pass

    def optimizer_step(self, lr=None):
        """torch.optim.AdamW defaults (ddpm.py:1442-1454): betas (.9,.999), eps 1e-8, weight_decay 1e-2."""
        ops.adamw_step(self.flat, self.grad, self.adam_m, self.adam_v, lr=self.lr if lr is None else lr,
                       step_dev=self.step_dev)


class CelebBasisStep(_LatentTrainStep):
    def __init__(self, params, state_dict, basis, device, *, tokenizer, placeholder="sks", clip_layers=None,
                 dtype=torch.float16, loss_scale=1024.0, vae_res_dtype=torch.float32, lr=5e-3, id_coefficients=None,
                 id_embeddings=None):
        super().__init__(params, state_dict, device, tokenizer=tokenizer, dtype=dtype, loss_scale=loss_scale,
                         vae_res_dtype=vae_res_dtype, lr=lr)
        sd = state_dict
        sub = lambda pre: {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}
        self.face = IResNetEngine(sub("embedding_manager.meta_id_net.id_model."), self.dev, dtype=dtype)
        self._side = torch.cuda.Stream(device=self.dev)      # stage_prefetch's face net, beside the VAE encode
        pc = params["personalization_config"]["params"]
        self.es = pc["num_embeds_per_token"]
        self.K = pc["meta_inner_dim"]
        self.momentum = pc.get("momentum", 0.9)
        self.max_ids = pc.get("max_ids", 10)
        (self.W, self.b), (self.gW, self.gb) = self._init_flat(
            [sd["embedding_manager.meta_id_net.stylegan_mlp.net.0.weight"],
             sd["embedding_manager.meta_id_net.stylegan_mlp.net.0.bias"]])
        self.basis = basis.detach().to(self.dev, torch.float32).contiguous()
        # placeholder: the main identity's string, or the strings of the first, second and third person of a prompt
        # (EmbeddingManagerId.placeholder_strings[:3])
        strings = [placeholder] if isinstance(placeholder, str) else list(placeholder)[:3]
        self.placeholder_tokens = [int(tokenizer(s)["input_ids"][0, 1]) for s in strings]
        self.placeholder_token = self.placeholder_tokens[0]
        self.multi = None           # multi-person EMA lists (enable_multi_person)
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

    def face_features(self, faces, n_chunks):
        x, geo = ops.face_warp_resize(faces.contiguous(), n_chunks, TRANS_MATRIX, out_hw=112, cpad=8, dtype=self.dt)
        feat = self.face.forward(x, geo)
        return ops.l2norm_rows(feat)

    # ------------------------------------------------------------------------------------------
    @staticmethod
    def person_chunks(n_chunks):
        """Face chunk of the first, second and third person of a prompt (embedding_manager.py:298-304): the injected
        rows come from meta[0], meta[1], meta[id_cnt // 2], the EMA coefficients from cef[0], cef[1], cef[1]
        ("in training, the max #id is 2")."""
        return (0, 1, n_chunks // 2), (0, 1, 1)

    def prepare(self, captions, num_ids=None, n_chunks=None):
        """Host side of the step: tokenise, locate the placeholders, build the row map (bit-exact integer path).  Without
        num_ids every prompt has one person (the main identity, face chunk 0); with the per-sample num_ids (1, 2 or 3)
        sample b's j-th placeholder takes the rows of face chunk person_chunks(n_chunks)[0][j]."""
        ids = self.tokenize(captions)
        if num_ids is None:
            map_np, positions = build_inject_map(ids.numpy(), self.placeholder_token, self.es, lambda b: b)
            return ids, map_np, positions
        B = ids.shape[0]
        chunk = self.person_chunks(n_chunks)[0]
        nid = [int(k) for k in num_ids]
        assert all(1 <= k <= len(self.placeholder_tokens) for k in nid), (nid, len(self.placeholder_tokens))
        per_sample = [(self.placeholder_tokens[:k], [(chunk[j] * B + b) * self.es for j in range(k)])
                      for b, k in enumerate(nid)]
        map_np, positions = build_inject_map_multi(ids.numpy(), per_sample, self.es)
        return ids, map_np, positions

    @staticmethod
    def ema_slots(num_ids, n_chunks):
        """The EMA update order of a multi-person batch (embedding_manager.py:321-392: per sample, then its first, second,
        third person) as a fixed-capacity (3B,) list: entry 3b+j is the index of ids[b][j] in the flat (B, n_chunks)
        identity tensor, -1 where sample b has fewer than j+1 persons."""
        nid = [int(k) for k in num_ids]
        slot = np.full(3 * len(nid), -1, dtype=np.int32)
        for b, k in enumerate(nid):
            slot[3 * b: 3 * b + k] = b * n_chunks + np.arange(k)
        return slot

    def enable_multi_person(self, B, n_chunks):
        """Steps from now on take batches whose prompts name one, two or three persons (num_ids per sample): the
        row map comes from prepare(captions, num_ids, n_chunks) and the EMA runs over the list load_ema_slots stages,
        so a captured step replays any mix of 1/2/3-person samples."""
        assert n_chunks >= 2, "two- and three-person prompts take their second identity from face chunk 1"
        emb_chunk, coef_chunk = self.person_chunks(n_chunks)
        src = lambda chunk: torch.tensor([chunk[j] * B + b for b in range(B) for j in range(3)], dtype=torch.int32,
                                         device=self.dev)
        self.multi = dict(B=B, n_chunks=n_chunks, slot=torch.full((3 * B,), -1, dtype=torch.int32, device=self.dev),
                          src_emb=src(emb_chunk), src_coef=src(coef_chunk))

    def load_ema_slots(self, slot):
        self.multi["slot"].copy_(torch.from_numpy(slot), non_blocking=True)

    def forward_backward(self, batch, draws, need_grad=True, ema_update=True):
        """batch: dict as face_id.py:598-644 yields (tensors on self.dev); draws: t (B,), noise, posterior_eps.
        Returns the loss (1-element device tensor).  Gradients of (W,b) land in self.grad.  The same two stages as the
        serial schedule of StepGraphs, run eagerly: the front end, then the chain on its result."""
        io = batch["image_ori"]
        if self.multi is None:
            ids, map_np, positions = self.prepare(batch["caption"])
        else:
            ids, map_np, positions = self.prepare(batch["caption"], io["num_ids"], io["ids"].shape[1])
            self.load_ema_slots(self.ema_slots(io["num_ids"], io["ids"].shape[1]))
        z, v = self.stage_prefetch(batch["image"], io["faces"], io["ids"].shape[1], draws["posterior_eps"])
        loss = self.stage_main(z, v, io["ids"], ids.to(self.dev), torch.from_numpy(map_np).to(self.dev), draws["t"],
                               draws["noise"], need_grad=need_grad, ema_update=ema_update)
        self.last.update(positions=positions, ids=ids)
        return loss

    # ------------------------------------------------------------------------------------------
    # the step as two stages: a frozen no-grad front end that does not depend on the trained weights (and can therefore
    # be computed for the NEXT batch while this batch trains) and the trainable chain
    # ------------------------------------------------------------------------------------------
    def stage_prefetch(self, image, faces, n_chunks, posterior_eps, z_out=None, v_out=None):
        """get_input's VAE encode + posterior sample (ddpm.py:702-759) and the CosFace features of the face crops
        (meta_net.py:329-346, no_grad): two concurrent branches with their own workspaces (lanes 1 / 2)."""
        main = torch.cuda.current_stream()
        side = self._side
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

    # the trainable part of the chain (_LatentTrainStep.stage_main): celeb-basis MLP -> basis -> 2 rows per face
    def _rows_fwd(self, v):
        pre, coef, nrm = ops.celeb_mlp_fwd(v, self.W, self.b, self.es)
        zc = ops.celeb_basis_fwd(coef, self.basis)
        return zc.view(-1, zc.shape[-1]), (pre, coef, nrm, zc)

    def _rows_last(self, saved, v):
        return dict(coef=saved[1], celeb_z=saved[3], face_feat=v)

    def _rows_ema(self, saved, ids_person, B):
        """_momentum_update, training branch (embedding_manager.py:484-489) for the main identity of each sample; the
        identity index is read on the device (no host sync, CUDA-graph safe)."""
        pre, coef, nrm, zc = saved
        idx = (ids_person if ids_person.is_cuda else ids_person.to(self.dev)).long()
        if self.multi is not None:
            mp, F = self.multi, zc.shape[0]
            idx = idx.contiguous()
            ops.ema_rows_sel(self.id_embeddings.view(self.max_ids, -1), idx, mp["slot"], mp["src_emb"],
                             zc.reshape(F, -1), self.momentum)
            ops.ema_rows_sel(self.id_coefficients.view(self.max_ids, -1), idx, mp["slot"], mp["src_coef"],
                             coef.reshape(F, -1), self.momentum)
            return
        ops.ema_rows(self.id_embeddings.view(self.max_ids, -1), idx, zc[:B].reshape(B, -1), self.momentum)
        ops.ema_rows(self.id_coefficients.view(self.max_ids, -1), idx, coef[:B].reshape(B, -1), self.momentum)

    def _rows_bwd(self, demb, map_dev, B, T, saved, v):
        pre, coef, nrm, zc = saved
        dz = ops.embed_inject_bwd(demb, map_dev.view(-1), zc.shape[0] * self.es, B, T)
        dcoef = ops.celeb_basis_bwd(dz.view(zc.shape), self.basis)
        ops.celeb_mlp_bwd(dcoef, coef, nrm, pre, v, self.gW, self.gb)

    def ema_state(self):
        return (self.id_coefficients, self.id_embeddings)

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


class TextualInversionStep(_LatentTrainStep):
    """One Textual Inversion training step (configs/stable-diffusion/v1-finetune.yaml: EmbeddingManager,
    ldm/modules/embedding_manager.py:38-184) on the sm_90a kernels:

        image --VAE encode--> z --q_sample(t, noise)--> x_t ----------------------------------------\
        caption --tokenise--> ids --gather--> token rows --inject the placeholders' rows @map--> +pos --> CLIP text --> UNet
        loss = MSE(eps, noise);  backward: UNet -> d(context) -> CLIP -> d(embeddings) -> d(rows) (summed over occurrences)

    The trained rows of every placeholder (num_vectors_per_token x 768 each, in the manager's dict order) are one flat
    fp32 buffer; `rows` holds them in that order as the (R, 768) z table of the inject kernel.  The row map comes from the
    manager's own host arithmetic (EmbeddingManager.ti_map), so the fused and the eager step inject the same rows."""

    def __init__(self, params, state_dict, placeholder_params, device, *, tokenizer, dtype=torch.float16,
                 loss_scale=1024.0, vae_res_dtype=torch.float32, lr=5e-3):
        super().__init__(params, state_dict, device, tokenizer=tokenizer, dtype=dtype, loss_scale=loss_scale,
                         vae_res_dtype=vae_res_dtype, lr=lr)
        self.params, self.grads = self._init_flat(list(placeholder_params))
        self.rows = self.flat.view(-1, self.clip.hidden)
        self.grad_rows = self.grad.view(-1, self.clip.hidden)
        self.coarse_reg = None

    def set_coarse_reg(self, weight, initial_rows):
        """embedding_reg_weight > 0 (ddpm.py:1101-1107): initial_rows[k] is the initial (nv, 768) rows of the k-th
        placeholder (the engine's parameter order), or None for a placeholder without an initializer word.  The loss
        weights must have been set (set_loss_weights, default values included): the regulariser adds into the loss buffer
        of cb_diffusion_loss_fwd_bwd, not into loss_simple."""
        assert self.loss_weights is not None, "set_loss_weights before set_coarse_reg"
        terms = [(p, g, p0.detach().to(self.dev, torch.float32).reshape(p.shape).contiguous())
                 for p, g, p0 in zip(self.params, self.grads, initial_rows) if p0 is not None]
        self.coarse_reg = (float(weight), len(terms), terms) if terms else None

    def _loss_extra(self, loss):
        if self.coarse_reg is not None:
            w, n_init, terms = self.coarse_reg
            for p, g, p0 in terms:
                ops.ti_coarse_reg(p, p0, g, loss, n_init, w)

    def stage_prefetch(self, image, faces, n_chunks, posterior_eps, z_out=None, v_out=None):
        """get_input's VAE encode + posterior sample (ddpm.py:702-759); there are no face crops."""
        with ops.lane(2):
            z, _ = self.encode_first_stage(image, posterior_eps)
            if z_out is not None:
                z_out.copy_(z)
        return (z if z_out is None else z_out), None

    def _rows_fwd(self, v):
        return self.rows, None

    def _rows_bwd(self, demb, map_dev, B, T, saved, v):
        ops.embed_inject_bwd(demb, map_dev.view(-1), self.rows.shape[0], B, T, out=self.grad_rows)
