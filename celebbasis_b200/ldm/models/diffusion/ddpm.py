"""Host mirror of ldm/models/diffusion/ddpm.py (DDPM :46, LatentDiffusion :439, DiffusionWrapper :1530).

Keeps the surface main.py / main_id_embed.py / scripts/stable_txt2img.py / the DDIM sampler use (SURVEY.md §8b):
constructor keywords of configs/stable-diffusion/aigc_id.yaml, the schedule buffers, `shared_step`, `forward`,
`p_losses`, `apply_model`, `get_input`, `get_learned_conditioning`, `encode/decode_first_stage`, `q_sample`,
`configure_optimizers`, `training_step`, `on_save_checkpoint`, `ema_scope`, the DDPM ancestral sampler (`p_sample`,
`p_sample_loop`, `progressive_denoising`, `sample`: one cb_p_sample launch per step) and `sample_log` / `log_images`
with every panel an AutoencoderKL model can log.  Every tensor operation of the step is a
kernel of libcelebbasis_b200.so reached through the mirrored sub-modules; this file is glue, exactly as in the
reference.  Lightning is optional: without pytorch_lightning the class derives from a minimal stand-in.
"""
import os
from contextlib import contextmanager
from functools import partial

import numpy as np
import torch
import torch.nn as nn

from celebbasis_b200 import ops
from ldm.modules.diffusionmodules.util import extract_into_tensor, make_beta_schedule, noise_like
from ldm.modules.distributions.distributions import DiagonalGaussianDistribution
from ldm.util import cfg_get, count_params, default, exists, instantiate_from_config

try:  # pragma: no cover - pytorch_lightning is not installed in this image
    import pytorch_lightning as pl
    _Base = pl.LightningModule
    from pytorch_lightning.utilities.distributed import rank_zero_only
except Exception:  # minimal LightningModule protocol (what ddpm.py touches)
    class _Base(nn.Module):
        def __init__(self, *a, **k):
            super().__init__()
            self.global_step = 0
            self.current_epoch = 0
            self.trainer = None

        @property
        def device(self):
            for p in self.parameters():
                return p.device
            return torch.device("cpu")

        def log(self, *a, **k):
            pass

        def log_dict(self, d, *a, **k):
            self.last_log = dict(d)

    def rank_zero_only(fn):
        return fn

__conditioning_keys__ = {'concat': 'c_concat', 'crossattn': 'c_crossattn', 'adm': 'y'}


def disabled_train(self, mode=True):
    return self


class _MSEFn(torch.autograd.Function):
    """loss_simple[b] = mean_(c,h,w) (pred - target)^2  (get_loss 'l2' + .mean([1,2,3]), ddpm.py:294-307,1084)."""

    @staticmethod
    def forward(ctx, pred, target):
        need = ctx.needs_input_grad[0]     # (grad mode is off inside Function.forward; this reflects the call site)
        loss, grad = ops.mse_fwd_bwd(pred.float().contiguous(), target.float().contiguous(), 1.0, want_grad=need)
        ctx.B = pred.shape[0]
        if need:
            ctx.save_for_backward(grad)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        (grad,) = ctx.saved_tensors                 # = d(mean_b loss_b)/dpred ; chain rule with dloss per sample
        out = torch.empty_like(grad)
        w = (dloss.float() * ctx.B).tolist() if ctx.B > 1 else None
        if w is None:
            ops.axpby(grad.view(1, -1), float(dloss.item()), out=out.view(1, -1))
        else:
            for b in range(ctx.B):
                ops.axpby(grad[b].view(1, -1), w[b], out=out[b].view(1, -1))
        return out, None


def _row_grid(images, padding=2):
    """n decoded (b, C, H, W) batches -> one (C, b*(H+p)+p, n*(W+p)+p) image, sample k's n images along row k with
    `padding` zero pixels around each: the reference's rearrange('n b c h w -> (b n) c h w') + torchvision make_grid
    (nrow=n, pad_value 0) of ddpm.py:584-587,1365-1368."""
    rows = torch.stack(images, 1)                                # b, n, C, H, W
    b, n, C, H, W = rows.shape
    if C == 1:
        rows, C = rows.expand(b, n, 3, H, W), 3
    grid = rows.new_zeros(C, b, H + padding, n, W + padding)
    grid[:, :, padding:, :, padding:] = rows.permute(2, 0, 3, 1, 4)
    grid = grid.reshape(C, b * (H + padding), n * (W + padding))
    return torch.nn.functional.pad(grid, (0, padding, 0, padding))


def _plain(cfg):
    """OmegaConf node / dict / list -> plain python containers."""
    if isinstance(cfg, dict):
        return {k: _plain(v) for k, v in cfg.items()}
    if isinstance(cfg, (list, tuple)):
        return [_plain(v) for v in cfg]
    return cfg


class _FusedLossFn(torch.autograd.Function):
    """The fused step computes loss AND d(loss)/d(trained tensors) in one CUDA-graph replay; this node hands those
    gradients (`grads`, one per tensor of `params`) to autograd so that the reference's `loss.backward();
    optimizer.step()` contract (Lightning's loop) is unchanged."""

    @staticmethod
    def forward(ctx, loss_dev, grads, *params):
        ctx.save_for_backward(*grads)
        return loss_dev.reshape(()).clone()

    @staticmethod
    def backward(ctx, dloss):
        return (None, None) + tuple(g * dloss for g in ctx.saved_tensors)


class DDPM(_Base):
    def __init__(self, unet_config, timesteps=1000, beta_schedule="linear", loss_type="l2", ckpt_path=None,
                 ignore_keys=[], load_only_unet=False, monitor="val/loss", use_ema=True, first_stage_key="image",
                 image_size=256, channels=3, log_every_t=100, clip_denoised=True, linear_start=1e-4, linear_end=2e-2,
                 cosine_s=8e-3, given_betas=None, original_elbo_weight=0., embedding_reg_weight=0.,
                 unfreeze_model=False, model_lr=0., v_posterior=0., l_simple_weight=1., conditioning_key=None,
                 parameterization="eps", scheduler_config=None, use_positional_encodings=False, learn_logvar=False,
                 logvar_init=0.):
        super().__init__()
        assert parameterization == "eps", "SD-v1 / CelebBasis is eps-prediction"
        self.parameterization = parameterization
        self.cond_stage_model = None
        self.clip_denoised = clip_denoised
        self.log_every_t = log_every_t
        self.first_stage_key = first_stage_key
        self.image_size = image_size
        self.channels = channels
        self.use_positional_encodings = use_positional_encodings
        self.model = DiffusionWrapper(unet_config, conditioning_key)
        count_params(self.model, verbose=True)
        self.use_ema = use_ema
        assert not use_ema, "use_ema: False in every CelebBasis config (aigc_id.yaml:18)"
        self.use_scheduler = scheduler_config is not None
        self.v_posterior = v_posterior
        self.original_elbo_weight = original_elbo_weight
        self.l_simple_weight = l_simple_weight
        self.embedding_reg_weight = embedding_reg_weight
        self.unfreeze_model = unfreeze_model
        self.model_lr = model_lr
        if monitor is not None:
            self.monitor = monitor
        if ckpt_path is not None:
            self.init_from_ckpt(ckpt_path, ignore_keys=ignore_keys, only_model=load_only_unet)
        self.register_schedule(given_betas=given_betas, beta_schedule=beta_schedule, timesteps=timesteps,
                               linear_start=linear_start, linear_end=linear_end, cosine_s=cosine_s)
        self.loss_type = loss_type
        self.learn_logvar = learn_logvar
        self.logvar = torch.full(fill_value=logvar_init, size=(self.num_timesteps,))
        self.learning_rate = 5.0e-03

    def register_schedule(self, given_betas=None, beta_schedule="linear", timesteps=1000, linear_start=1e-4,
                          linear_end=2e-2, cosine_s=8e-3):
        """ddpm.py:126-178: float64 numpy schedule -> fp32 buffers (host arithmetic, init time)."""
        betas = given_betas if exists(given_betas) else make_beta_schedule(
            beta_schedule, timesteps, linear_start=linear_start, linear_end=linear_end, cosine_s=cosine_s)
        alphas = 1. - betas
        alphas_cumprod = np.cumprod(alphas, axis=0)
        alphas_cumprod_prev = np.append(1., alphas_cumprod[:-1])
        self.num_timesteps = int(betas.shape[0])
        self.linear_start, self.linear_end = linear_start, linear_end
        to_torch = partial(torch.tensor, dtype=torch.float32)
        self.register_buffer('betas', to_torch(betas))
        self.register_buffer('alphas_cumprod', to_torch(alphas_cumprod))
        self.register_buffer('alphas_cumprod_prev', to_torch(alphas_cumprod_prev))
        self.register_buffer('sqrt_alphas_cumprod', to_torch(np.sqrt(alphas_cumprod)))
        self.register_buffer('sqrt_one_minus_alphas_cumprod', to_torch(np.sqrt(1. - alphas_cumprod)))
        self.register_buffer('log_one_minus_alphas_cumprod', to_torch(np.log(1. - alphas_cumprod)))
        self.register_buffer('sqrt_recip_alphas_cumprod', to_torch(np.sqrt(1. / alphas_cumprod)))
        self.register_buffer('sqrt_recipm1_alphas_cumprod', to_torch(np.sqrt(1. / alphas_cumprod - 1)))
        posterior_variance = (1 - self.v_posterior) * betas * (1. - alphas_cumprod_prev) / (1. - alphas_cumprod) \
            + self.v_posterior * betas
        self.register_buffer('posterior_variance', to_torch(posterior_variance))
        self.register_buffer('posterior_log_variance_clipped', to_torch(np.log(np.maximum(posterior_variance, 1e-20))))
        self.register_buffer('posterior_mean_coef1', to_torch(betas * np.sqrt(alphas_cumprod_prev) / (1. - alphas_cumprod)))
        self.register_buffer('posterior_mean_coef2', to_torch((1. - alphas_cumprod_prev) * np.sqrt(alphas) / (1. - alphas_cumprod)))
        lvlb = self.betas ** 2 / (2 * self.posterior_variance * to_torch(alphas) * (1 - self.alphas_cumprod))
        lvlb[0] = lvlb[1]
        self.register_buffer('lvlb_weights', lvlb, persistent=False)

    @contextmanager
    def ema_scope(self, context=None):
        yield None   # use_ema is False: the reference's scope is a no-op too (ddpm.py:180-194)

    def init_from_ckpt(self, path, ignore_keys=list(), only_model=False):
        sd = torch.load(path, map_location="cpu")
        if "state_dict" in list(sd.keys()):
            sd = sd["state_dict"]
        for k in list(sd.keys()):
            if any(k.startswith(ik) for ik in ignore_keys):
                del sd[k]
        missing, unexpected = self.load_state_dict(sd, strict=False) if not only_model else self.model.load_state_dict(sd, strict=False)
        print(f"Restored from {path} with {len(missing)} missing and {len(unexpected)} unexpected keys")

    def q_sample(self, x_start, t, noise=None):
        """ddpm.py:289-292 on the device (cb_q_sample)."""
        noise = default(noise, lambda: torch.randn_like(x_start))
        return ops.q_sample(x_start.float().contiguous(), noise.float().contiguous(), t.long().contiguous(),
                            self.sqrt_alphas_cumprod, self.sqrt_one_minus_alphas_cumprod)

    def get_loss(self, pred, target, mean=True):
        assert self.loss_type == 'l2'
        per_sample = _MSEFn.apply(pred, target)
        return per_sample.mean() if mean else per_sample

    def get_input(self, batch, k):
        x = batch[k]
        if len(x.shape) == 3:
            x = x[..., None]
        # 'b h w c -> b c h w' + contiguous + float (ddpm.py:344-350): pure layout glue
        return x.permute(0, 3, 1, 2).to(memory_format=torch.contiguous_format).float()

    def training_step(self, batch, batch_idx):
        loss, loss_dict = self.shared_step(batch)
        self.log_dict(loss_dict, prog_bar=True, logger=True, on_step=True, on_epoch=True)
        self.log("global_step", self.global_step, prog_bar=True, logger=True, on_step=True, on_epoch=False)
        return loss


class LatentDiffusion(DDPM):
    """main class"""

    def __init__(self, first_stage_config, cond_stage_config, personalization_config, num_timesteps_cond=None,
                 cond_stage_key="image", cond_stage_trainable=False, concat_mode=True, cond_stage_forward=None,
                 conditioning_key=None, scale_factor=1.0, scale_by_std=False, *args, **kwargs):
        self.num_timesteps_cond = default(num_timesteps_cond, 1)
        self.scale_by_std = scale_by_std
        self._engine_params = _plain(dict(
            unet_config=kwargs.get("unet_config"), first_stage_config=first_stage_config,
            personalization_config=personalization_config, scale_factor=scale_factor,
            timesteps=kwargs.get("timesteps", 1000), linear_start=kwargs.get("linear_start", 1e-4),
            linear_end=kwargs.get("linear_end", 2e-2)))
        self._fused = None            # StepGraphs of the CUDA-graph training step (built on first use)
        self._fused_sig = None
        self._staged_next = None      # look-ahead batch handed over by the training loop (stage_next_batch)
        self.fused_step = os.environ.get("CB_FUSED_STEP", "1") != "0"
        assert self.num_timesteps_cond <= kwargs['timesteps']
        if conditioning_key is None:
            conditioning_key = 'concat' if concat_mode else 'crossattn'
        ckpt_path = kwargs.pop("ckpt_path", None)
        ignore_keys = kwargs.pop("ignore_keys", [])
        super().__init__(conditioning_key=conditioning_key, *args, **kwargs)
        self.concat_mode = concat_mode
        self.cond_stage_trainable = cond_stage_trainable
        self.cond_stage_key = cond_stage_key
        try:
            self.num_downs = len(cfg_get(first_stage_config, "params", "ddconfig", "ch_mult")) - 1
        except Exception:
            self.num_downs = 0
        assert not scale_by_std
        self.scale_factor = scale_factor
        self.instantiate_first_stage(first_stage_config)
        self.instantiate_cond_stage(cond_stage_config)
        self.cond_stage_forward = cond_stage_forward
        self.clip_denoised = False
        self.bbox_tokenizer = None
        self.restarted_from_ckpt = False
        if ckpt_path is not None:
            self.init_from_ckpt(ckpt_path, ignore_keys)
            self.restarted_from_ckpt = True
        if not self.unfreeze_model:
            self.cond_stage_model.eval()
            self.cond_stage_model.train = disabled_train
            for param in self.cond_stage_model.parameters():
                param.requires_grad = False
            self.model.eval()
            self.model.train = disabled_train
            for param in self.model.parameters():
                param.requires_grad = False
        self.embedding_manager = self.instantiate_embedding_manager(personalization_config, self.cond_stage_model)
        for param in self.embedding_manager.embedding_parameters():
            param.requires_grad = True
        for param in self.embedding_manager.trainable_parameters():
            param.requires_grad = True

    # ---- sub-module construction (ddpm.py:540-576) -----------------------------------------------------------
    def instantiate_first_stage(self, config):
        model = instantiate_from_config(config)
        self.first_stage_model = model.eval()
        self.first_stage_model.train = disabled_train
        for param in self.first_stage_model.parameters():
            param.requires_grad = False

    def instantiate_cond_stage(self, config):
        model = instantiate_from_config(config)
        if not self.cond_stage_trainable:
            self.cond_stage_model = model.eval()
            self.cond_stage_model.train = disabled_train
            for param in self.cond_stage_model.parameters():
                param.requires_grad = False
        else:
            self.cond_stage_model = model

    def instantiate_embedding_manager(self, config, embedder):
        model = instantiate_from_config(config, embedder=embedder)
        ckpt = cfg_get(config, "params", "embedding_manager_ckpt")
        if ckpt:
            model.load(ckpt)
        return model

    # ---- first stage ---------------------------------------------------------------------------------------------
    def get_first_stage_encoding(self, encoder_posterior):
        if isinstance(encoder_posterior, DiagonalGaussianDistribution):
            return encoder_posterior.sample(scale=self.scale_factor)     # scale fused into the sampling kernel
        elif isinstance(encoder_posterior, torch.Tensor):
            return ops.axpby(encoder_posterior.reshape(encoder_posterior.shape[0], -1).float().contiguous(),
                             float(self.scale_factor)).view(encoder_posterior.shape)
        raise NotImplementedError(f"encoder_posterior of type '{type(encoder_posterior)}' not yet implemented")

    @torch.no_grad()
    def encode_first_stage(self, x):
        return self.first_stage_model.encode(x)

    @torch.no_grad()
    def decode_first_stage(self, z, predict_cids=False, force_not_quantize=False):
        z = ops.axpby(z.reshape(z.shape[0], -1).float().contiguous(), 1. / self.scale_factor).view(z.shape)
        return self.first_stage_model.decode(z)

    # ---- conditioning ---------------------------------------------------------------------------------------------
    def get_learned_conditioning(self, c, face_img=None, image_ori=None):
        assert self.cond_stage_forward is None
        c = self.cond_stage_model.encode(c, embedding_manager=self.embedding_manager, face_img=face_img,
                                         image_ori=image_ori)
        if isinstance(c, DiagonalGaussianDistribution):
            c = c.mode()
        return c

    @torch.no_grad()
    def get_input(self, batch, k, return_first_stage_outputs=False, force_c_encode=False, cond_key=None,
                  return_original_cond=False, bs=None):
        x = super().get_input(batch, k)
        if bs is not None:
            x = x[:bs]
        x = x.to(self.device)
        encoder_posterior = self.encode_first_stage(x)
        z = self.get_first_stage_encoding(encoder_posterior).detach()
        cond_key = cond_key or self.cond_stage_key
        assert cond_key in ['caption', 'coordinates_bbox']
        xc = batch[cond_key]
        if not self.cond_stage_trainable or force_c_encode:
            c = self.get_learned_conditioning(xc, face_img=batch.get('image'), image_ori=batch.get('image_ori'))
        else:
            c = xc
        if bs is not None:
            c = c[:bs]
        c = {'caption': c, 'image': batch['image'], 'image_ori': batch.get('image_ori')}
        out = [z, c]
        if return_first_stage_outputs:
            out.extend([x, self.decode_first_stage(z)])
        if return_original_cond:
            out.append(xc)
        return out

    # ---- the training step (ddpm.py:921-936,948-1049,1069-1116) ---------------------------------------------------
    def preprocess_batch(self, batch):
        """RAW batches of the ldm.data.face_id mirror (uint8 images + drawn augmentation parameters) -> the batch dict the
        reference's DataLoader yields, with the pixel work done on this module's device (celebbasis_b200.data_path)."""
        from celebbasis_b200 import data_path
        if data_path.is_raw_batch(batch):
            return data_path.device_augment(batch, self.device)
        return batch

    def shared_step(self, batch, **kwargs):
        batch = self.preprocess_batch(batch)
        if self._fused_applicable(batch):
            return self._fused_shared_step(batch)
        x, c = self.get_input(batch, self.first_stage_key)
        return self(x, c['caption'], face_img=c['image'], image_ori=c['image_ori'])

    # ---- fused training step: the whole of shared_step + backward as CUDA-graph replays ---------------------------
    def stage_next_batch(self, batch):
        """Optional look-ahead hook for the training loop: the batch that the NEXT training_step call will receive (the
        same object).  Its frozen front end (VAE encode, CosFace features) then overlaps this step's UNet work."""
        self._staged_next = batch

    def _fused_applicable(self, batch):
        if not (self.fused_step and self.training and self.cond_stage_trainable and not self.unfreeze_model):
            return False
        if self._textual_inversion():
            return self._ti_fused_applicable(batch)
        io = batch.get("image_ori") if isinstance(batch, dict) else None
        x = batch.get(self.first_stage_key) if isinstance(batch, dict) else None
        if io is None or not torch.is_tensor(x) or x.dim() != 4 or x.shape[-1] != 3 or x.dtype != torch.float32:
            return False
        faces, nid = io.get("faces"), io.get("num_ids")
        if not torch.is_tensor(faces) or faces.shape[:3] != x.shape[:3] or faces.shape[-1] % 3 != 0:
            return False
        if nid is None:
            return False
        nid = torch.as_tensor(nid).cpu()
        k = int(nid.max())
        if int(nid.min()) < 1 or k > 3:
            return False
        if k > 1:       # k persons in a prompt: k placeholders and k identities, the second from face chunk 1 (meta[1])
            ids = io.get("ids")
            if ids is None or ids.shape[-1] < max(2, k) or len(self.embedding_manager.placeholder_strings) < k:
                return False
        if getattr(self.cond_stage_model, "celeb_embeddings", None) is None:
            return False
        return next(self.model.parameters()).is_cuda

    def _textual_inversion(self):
        from ldm.modules.embedding_manager import EmbeddingManager
        return isinstance(self.embedding_manager, EmbeddingManager)

    def _ti_fused_applicable(self, batch):
        """Textual Inversion (v1-finetune.yaml) batches: fp32 (B, H, W, 3) images with one caption each.  Progressive
        words only change the host-built row map from step to step; the manager rejects per_image_tokens when it is
        built."""
        if not isinstance(batch, dict):
            return False
        x, cap = batch.get(self.first_stage_key), batch.get(self.cond_stage_key)
        if not torch.is_tensor(x) or x.dim() != 4 or x.shape[-1] != 3 or x.dtype != torch.float32:
            return False
        if not isinstance(cap, (list, tuple)) or len(cap) != x.shape[0] or not all(isinstance(c, str) for c in cap):
            return False
        return next(self.model.parameters()).is_cuda

    def _ti_params(self):
        em = self.embedding_manager
        return [em.string_to_param_dict[k] for k in em.string_to_token_dict]

    def _ti_prepare(self, eng, captions):
        """Host side of the TI step: tokenise and build the inject map with the manager's own arithmetic (no sync)."""
        ids = eng.tokenize(captions)
        map_np, _ = self.embedding_manager.ti_map(ids.numpy())
        self.embedding_manager.last_map = map_np
        return ids, map_np

    def _fused_build_ti(self, batch):
        from celebbasis_b200.step_graph import StepGraphs
        from celebbasis_b200.train_step import TextualInversionStep
        x = batch[self.first_stage_key]
        B, hw = x.shape[0], x.shape[1]
        params = self._ti_params()
        dev = params[0].device
        em = self.embedding_manager
        eng = TextualInversionStep(self._engine_params, self.state_dict(), [p.detach() for p in params], dev,
                                   tokenizer=self.cond_stage_model.tokenizer, lr=self.learning_rate)
        self._fused_loss_weights(eng, force=self.embedding_reg_weight > 0)
        if self.embedding_reg_weight > 0:
            eng.set_coarse_reg(self.embedding_reg_weight,
                               [em.initial_embeddings[k] if k in em.initial_embeddings else None
                                for k in em.string_to_token_dict])
        # the placeholder parameters alias the engine's flat buffer: FusedAdamW, save() and the graphs see one memory
        for p, view in zip(params, eng.params):
            p.data = view
        T = getattr(self.cond_stage_model, "max_length", 77)
        G = StepGraphs(eng, B=B, T=T, n_chunks=0, image_hw=hw)
        # the capture's row map must not advance the progressive-words counter: the step that follows does, once
        counter = em.progressive_counter
        ids, map_np = self._ti_prepare(eng, batch[self.cond_stage_key])
        em.progressive_counter = counter
        lat = G.noise.shape[-1]
        G.load_next(x, None, torch.zeros(B, 4, lat, lat))
        G.load_step(ids, map_np, torch.zeros(B, dtype=torch.long), torch.zeros_like(G.noise))
        G.capture()
        self._fused, self._fused_sig = G, (B, hw, 0, dev)
        return G

    def _fused_build(self, batch):
        if self._textual_inversion():
            return self._fused_build_ti(batch)
        from celebbasis_b200.step_graph import StepGraphs
        from celebbasis_b200.train_step import CelebBasisStep
        x = batch[self.first_stage_key]
        faces = batch["image_ori"]["faces"]
        B, hw, n_chunks = x.shape[0], x.shape[1], faces.shape[-1] // 3
        em = self.embedding_manager
        lin = em.meta_id_net.stylegan_mlp.net[0]
        dev = lin.weight.device
        eng = CelebBasisStep(self._engine_params, self.state_dict(), self.cond_stage_model.celeb_embeddings, dev,
                             tokenizer=self.cond_stage_model.tokenizer, placeholder=em.placeholder_strings[:3],
                             lr=self.learning_rate, id_coefficients=em.id_coefficients, id_embeddings=em.id_embeddings)
        self._fused_loss_weights(eng)
        multi = self._multi_person(batch)
        if multi:
            eng.enable_multi_person(B, n_chunks)
        # one storage for the trainable tensors and the per-identity EMA state: the optimiser (FusedAdamW on the mirror's
        # parameters), save()/load() of the embedding manager and the graph all see the same memory
        eng.flat[: lin.weight.numel()].copy_(lin.weight.detach().reshape(-1))
        eng.flat[lin.weight.numel():].copy_(lin.bias.detach().reshape(-1))
        lin.weight.data, lin.bias.data = eng.W, eng.b
        em.id_coefficients = list(eng.id_coefficients.unbind(0))
        em.id_embeddings = list(eng.id_embeddings.unbind(0))
        em.moved_to_device = True
        T = getattr(self.cond_stage_model, "max_length", 77)
        G = StepGraphs(eng, B=B, T=T, n_chunks=n_chunks, image_hw=hw)
        ids, map_np, _ = self._cb_prepare(eng, batch)
        lat = G.noise.shape[-1]
        G.load_next(x, faces, torch.zeros(B, 4, lat, lat))
        G.load_step(ids, map_np, torch.zeros(B, dtype=torch.long), torch.zeros_like(G.noise), batch["image_ori"]["ids"])
        G.capture()
        self._fused, self._fused_sig = G, (B, hw, n_chunks, dev, multi)
        return G

    def _fused_loss_weights(self, eng, force=False):
        """Non-default p_losses weights (or `force`: the coarse regulariser needs a loss buffer of its own): the step
        computes its loss and loss_vlb with cb_diffusion_loss_fwd_bwd on the model's logvar and lvlb_weights tables (the
        default keeps cb_mse_fwd_bwd + cb_loss_mean)."""
        if force or self.l_simple_weight != 1. or self.original_elbo_weight != 0. or bool((self.logvar != 0).any()):
            eng.set_loss_weights(self.l_simple_weight, self.original_elbo_weight, self.logvar, self.lvlb_weights)

    def _multi_person(self, batch):
        """True once a batch has named two or three persons: the step then keeps the multi-person map and EMA list, which
        replay any later mix of 1/2/3-person samples.  A run that starts with single-person batches therefore captures
        its graphs a second time at its first multi-person batch (once per run): until then the step makes exactly the
        default configuration's launches.  The trained tensors, the EMA state and the optimiser state (kept by the
        optimiser per parameter) carry over, since the new engine is built from the parameters the old one aliased."""
        return bool(self._fused_sig is not None and len(self._fused_sig) == 5 and self._fused_sig[4]) or \
            int(torch.as_tensor(batch["image_ori"]["num_ids"]).max()) > 1

    def _cb_prepare(self, eng, batch):
        """Host side of the CelebBasis step: tokenise + the bit-exact placeholder row map, and the EMA order of a
        multi-person step."""
        io = batch["image_ori"]
        if eng.multi is None:
            return eng.prepare(batch["caption"])
        n_chunks = io["ids"].shape[1]
        eng.load_ema_slots(eng.ema_slots(io["num_ids"], n_chunks))
        return eng.prepare(batch["caption"], io["num_ids"], n_chunks)

    def _fused_shared_step(self, batch):
        ti = self._textual_inversion()
        faces_of = (lambda b: None) if ti else (lambda b: b["image_ori"]["faces"])
        x = batch[self.first_stage_key]
        B, hw = x.shape[0], x.shape[1]
        G = self._fused
        dev = next(self.model.parameters()).device
        sig = (B, hw, 0, dev) if ti else (B, hw, faces_of(batch).shape[-1] // 3, dev, self._multi_person(batch))
        if G is None or self._fused_sig != sig:
            G = self._fused_build(batch)
        eng = G.eng
        lat_shape = list(G.peps_n.shape)
        if G.next_token is not batch:                         # no look-ahead happened for this batch: front end now
            G.load_next(x, faces_of(batch), torch.randn(lat_shape))   # posterior eps from the CPU generator, as
            G.prefetch(batch)                                          # distributions.py:36 does
        if ti:
            ids, map_np = self._ti_prepare(eng, batch[self.cond_stage_key])
        else:
            ids, map_np, positions = self._cb_prepare(eng, batch)
            self.embedding_manager.last_positions = positions
        t = torch.randint(0, self.num_timesteps, (B,), device=dev).long()
        noise = torch.randn_like(G.z)
        G.load_step(ids, map_np, t, noise, None if ti else batch["image_ori"]["ids"])
        nxt, self._staged_next = self._staged_next, None
        if nxt is not None and (nxt is batch or not self._fused_applicable(nxt)
                                or nxt[self.first_stage_key].shape != x.shape
                                or (not ti and self._multi_person(nxt) != sig[4])):
            nxt = None      # (a batch that switches the step to multi-person prompts has its front end run by the new graphs)
        if nxt is not None:
            G.load_next(nxt[self.first_stage_key], faces_of(nxt), torch.randn(lat_shape))
        loss_dev = G.step(lookahead=nxt is not None, token=nxt)
        if ti:
            loss = _FusedLossFn.apply(loss_dev, eng.grads, *self._ti_params())
        else:
            lin = self.embedding_manager.meta_id_net.stylegan_mlp.net[0]
            loss = _FusedLossFn.apply(loss_dev, (eng.gW, eng.gb), lin.weight, lin.bias)
        loss_simple = eng.last["loss_simple"].detach()
        loss_vlb = eng.last["loss_vlb"]
        prefix = 'train' if self.training else 'val'
        loss_dict = {f'{prefix}/loss_simple': loss_simple.mean(),
                     f'{prefix}/loss_vlb': (self.lvlb_weights.to(dev)[t] * loss_simple).mean() if loss_vlb is None
                     else loss_vlb.detach()[0],
                     f'{prefix}/loss_emb_reg': self.embedding_manager.embedding_neg_loss(),
                     f'{prefix}/loss': loss.detach()}
        return loss, loss_dict

    def forward(self, x, c, face_img=None, image_ori=None, *args, **kwargs):
        t = torch.randint(0, self.num_timesteps, (x.shape[0],), device=self.device).long()
        if self.model.conditioning_key is not None:
            assert c is not None
            if self.cond_stage_trainable:
                c = self.get_learned_conditioning(c, face_img=face_img, image_ori=image_ori)
        return self.p_losses(x, c, t, *args, **kwargs)

    def apply_model(self, x_noisy, t, cond, return_ids=False):
        if not isinstance(cond, dict):
            if not isinstance(cond, list):
                cond = [cond]
            key = 'c_concat' if self.model.conditioning_key == 'concat' else 'c_crossattn'
            cond = {key: cond}
        x_recon = self.model(x_noisy, t, **cond)
        if isinstance(x_recon, tuple) and not return_ids:
            return x_recon[0]
        return x_recon

    def p_losses(self, x_start, cond, t, noise=None):
        noise = default(noise, lambda: torch.randn_like(x_start))
        x_noisy = self.q_sample(x_start=x_start, t=t, noise=noise)
        model_output = self.apply_model(x_noisy, t, cond)
        loss_dict = {}
        prefix = 'train' if self.training else 'val'
        target = noise
        loss_simple = self.get_loss(model_output, target, mean=False)          # (B,) already averaged over (C,H,W)
        loss_dict.update({f'{prefix}/loss_simple': loss_simple.mean()})
        if self.logvar.device != t.device:
            self.logvar = self.logvar.to(t.device)
        logvar_t = self.logvar[t]
        loss = loss_simple / torch.exp(logvar_t) + logvar_t
        loss = self.l_simple_weight * loss.mean()
        loss_vlb = (self.lvlb_weights[t] * loss_simple).mean()
        loss_dict.update({f'{prefix}/loss_vlb': loss_vlb})
        loss = loss + self.original_elbo_weight * loss_vlb
        loss_dict.update({f'{prefix}/loss': loss})
        if self.embedding_reg_weight > 0:
            reg = self.embedding_manager.embedding_to_coarse_loss()
            reg = reg.mean() if torch.is_tensor(reg) else reg       # (nv, nv) for Textual Inversion: the reference's mean
            loss_dict.update({f'{prefix}/loss_emb_reg': reg})
            loss = loss + self.embedding_reg_weight * reg
        neg = self.embedding_manager.embedding_neg_loss()
        loss = loss + neg * 1.
        loss_dict.update({f'{prefix}/loss_emb_reg': neg})
        loss_dict.update({f'{prefix}/loss': loss})
        return loss, loss_dict

    # ---- DDPM ancestral sampling (ddpm.py:1118-1303) ---------------------------------------------------------------
    def _ddpm_unsupported(self, quantize_denoised=False, return_codebook_ids=False, score_corrector=None):
        if score_corrector is not None:
            raise NotImplementedError("score_corrector is not supported: the reference tree ships no score corrector "
                                      "(ddpm.py:1123-1125 calls score_corrector.modify_score)")
        if quantize_denoised:
            raise NotImplementedError("quantize_denoised=True is not supported: the reference calls "
                                      "first_stage_model.quantize (ddpm.py:1139-1140), which AutoencoderKL lacks")
        if return_codebook_ids:
            raise NotImplementedError("return_codebook_ids=True is not supported: the reference raises "
                                      "DeprecationWarning('Support dropped.') there (ddpm.py:1159-1160)")
        if self.num_timesteps_cond > 1:
            raise NotImplementedError("num_timesteps_cond > 1 (shorten_cond_schedule) is not supported: no config sets "
                                      "it, and the reference then q-samples the conditioning every step")

    @torch.no_grad()
    def p_sample(self, x, c, t, clip_denoised=False, repeat_noise=False, return_codebook_ids=False,
                 quantize_denoised=False, return_x0=False, temperature=1., noise_dropout=0., score_corrector=None,
                 corrector_kwargs=None):
        """One ancestral step x_t -> x_{t-1} (ddpm.py:1149-1178): the UNet, the noise_like draw (made at t == 0 too, as
        the reference does), then one cb_p_sample launch for predict_start_from_noise + clamp + q_posterior + noise."""
        self._ddpm_unsupported(quantize_denoised, return_codebook_ids, score_corrector)
        eps = self.apply_model(x, t, c)
        noise = noise_like(x.shape, x.device, repeat_noise)
        if noise_dropout > 0.:
            # the reference rounds noise * temperature before the dropout: do that here, and multiply by 1 in the kernel
            noise = torch.nn.functional.dropout(noise * temperature, p=noise_dropout)
            temperature = 1.
        x_prev, x0 = ops.p_sample(x.float().contiguous(), eps.float().contiguous(), noise.float().contiguous(),
                                  t.to(device=x.device, dtype=torch.long).contiguous(), self.sqrt_recip_alphas_cumprod,
                                  self.sqrt_recipm1_alphas_cumprod, self.posterior_mean_coef1,
                                  self.posterior_mean_coef2, self.posterior_log_variance_clipped,
                                  temperature=temperature, clip_denoised=clip_denoised, want_x0=return_x0)
        return (x_prev, x0) if return_x0 else x_prev

    def _masked_blend(self, img, ts, mask, x0):
        """img_orig = q_sample(x0, ts) (its own randn_like draw, ddpm.py:290); img_orig * mask + (1 - mask) * img in one
        cb_q_sample_masked launch (ddpm.py:1225-1228,1274-1276).  `img` is this step's fresh output: written in place."""
        noise = torch.randn_like(x0)
        return ops.q_sample_masked(x0, noise, ts, self.sqrt_alphas_cumprod, self.sqrt_one_minus_alphas_cumprod, mask,
                                   img, out=img)

    @staticmethod
    def _masked_inputs(mask, x0, img):
        if mask is None:
            return None, x0
        assert x0 is not None
        assert tuple(x0.shape) == tuple(img.shape), (tuple(x0.shape), tuple(img.shape))
        return mask.to(device=img.device, dtype=torch.float32), x0.to(img.device).float().contiguous()

    @staticmethod
    def _slice_cond(cond, batch_size):
        """The reference's conditioning slicing to batch_size (ddpm.py:1198-1203,1293-1298)."""
        if cond is None:
            return None
        if isinstance(cond, dict):
            return {key: cond[key][:batch_size] if not isinstance(cond[key], list) else
                    list(map(lambda x: x[:batch_size], cond[key])) for key in cond}
        return [c[:batch_size] for c in cond] if isinstance(cond, list) else cond[:batch_size]

    @torch.no_grad()
    def progressive_denoising(self, cond, shape, verbose=True, callback=None, quantize_denoised=False,
                              img_callback=None, mask=None, x0=None, temperature=1., noise_dropout=0.,
                              score_corrector=None, corrector_kwargs=None, batch_size=None, x_T=None, start_T=None,
                              log_every_t=None):
        """ddpm.py:1180-1234: ancestral sampling that keeps the x0 predictions; `temperature` is a float or a list
        indexed by the timestep.  Returns (x_0, [x0 prediction at every logged step])."""
        self._ddpm_unsupported(quantize_denoised, False, score_corrector)
        if not log_every_t:
            log_every_t = self.log_every_t
        timesteps = self.num_timesteps
        if batch_size is not None:
            b = batch_size
            shape = [batch_size] + list(shape)
        else:
            b = batch_size = shape[0]
        img = torch.randn(shape, device=self.device) if x_T is None else x_T
        intermediates = []
        cond = self._slice_cond(cond, batch_size)
        if start_T is not None:
            timesteps = min(timesteps, start_T)
        if isinstance(temperature, (int, float)):
            temperature = [float(temperature)] * timesteps
        mask, x0 = self._masked_inputs(mask, x0, img)
        for i in reversed(range(0, timesteps)):
            ts = torch.full((b,), i, device=self.device, dtype=torch.long)
            img, x0_partial = self.p_sample(img, cond, ts, clip_denoised=self.clip_denoised,
                                            quantize_denoised=quantize_denoised, return_x0=True,
                                            temperature=temperature[i], noise_dropout=noise_dropout,
                                            score_corrector=score_corrector, corrector_kwargs=corrector_kwargs)
            if mask is not None:
                img = self._masked_blend(img, ts, mask, x0)
            if i % log_every_t == 0 or i == timesteps - 1:
                intermediates.append(x0_partial)
            if callback:
                callback(i)
            if img_callback:
                img_callback(img, i)
        return img, intermediates

    @torch.no_grad()
    def p_sample_loop(self, cond, shape, return_intermediates=False, x_T=None, verbose=True, callback=None,
                      timesteps=None, quantize_denoised=False, mask=None, x0=None, img_callback=None, start_T=None,
                      log_every_t=None):
        """ddpm.py:1236-1285: min(timesteps, start_T) ancestral steps from x_T (drawn when None), with the masked blend
        after every step when `mask` is given.  Intermediates: x_T, then x_t at every logged step."""
        self._ddpm_unsupported(quantize_denoised)
        if not log_every_t:
            log_every_t = self.log_every_t
        device = self.betas.device
        b = shape[0]
        img = torch.randn(shape, device=device) if x_T is None else x_T
        intermediates = [img]
        if timesteps is None:
            timesteps = self.num_timesteps
        if start_T is not None:
            timesteps = min(timesteps, start_T)
        mask, x0 = self._masked_inputs(mask, x0, img)
        for i in reversed(range(0, timesteps)):
            ts = torch.full((b,), i, device=device, dtype=torch.long)
            img = self.p_sample(img, cond, ts, clip_denoised=self.clip_denoised, quantize_denoised=quantize_denoised)
            if mask is not None:
                img = self._masked_blend(img, ts, mask, x0)
            if i % log_every_t == 0 or i == timesteps - 1:
                intermediates.append(img)
            if callback:
                callback(i)
            if img_callback:
                img_callback(img, i)
        if return_intermediates:
            return img, intermediates
        return img

    @torch.no_grad()
    def sample(self, cond, batch_size=16, return_intermediates=False, x_T=None, verbose=True, timesteps=None,
               quantize_denoised=False, mask=None, x0=None, shape=None, **kwargs):
        """ddpm.py:1287-1303: p_sample_loop over (batch_size, channels, image_size, image_size) with the conditioning
        sliced to batch_size.  Like the reference, other keywords (eta, guidance, start_T, ...) are accepted and unused."""
        if shape is None:
            shape = (batch_size, self.channels, self.image_size, self.image_size)
        cond = self._slice_cond(cond, batch_size)
        return self.p_sample_loop(cond, shape, return_intermediates=return_intermediates, x_T=x_T, verbose=verbose,
                                  timesteps=timesteps, quantize_denoised=quantize_denoised, mask=mask, x0=x0)

    # ---- image logging (ddpm.py:1305-1440; called by main.ImageLogger every batch_frequency steps) --------------------
    @torch.no_grad()
    def sample_log(self, cond, batch_size, ddim, ddim_steps, **kwargs):
        """DDIM samples (ddim=True) or ancestral DDPM samples over all num_timesteps (ddim=False, ddpm.py:1305-1318);
        returns (samples, intermediates)."""
        if not ddim:
            return self.sample(cond=cond, batch_size=batch_size, return_intermediates=True, **kwargs)
        from ldm.models.diffusion.ddim import DDIMSampler
        shape = (self.channels, self.image_size, self.image_size)
        return DDIMSampler(self).sample(ddim_steps, batch_size, shape, cond, verbose=False, **kwargs)

    def _get_denoise_row_from_list(self, samples, desc='', force_no_decoder_quantization=False):
        """Decode every latent of `samples` and lay them out one sample per grid row (ddpm.py:578-588)."""
        return _row_grid([self.decode_first_stage(zd.to(self.device)) for zd in samples])

    @torch.no_grad()
    def log_images(self, batch, N=8, n_row=4, sample=True, ddim_steps=50, ddim_eta=1., return_keys=None,
                   quantize_denoised=True, inpaint=False, plot_denoise_rows=False, plot_progressive_rows=False,
                   plot_diffusion_rows=False, **kwargs):
        """inputs / reconstruction / rendered captions / the forward-diffusion row / samples (DDIM with ddim_steps, or
        DDPM over all timesteps with ddim_steps=None; plain and with guidance 5.0) with their denoise row / the masked-
        sampling panels / the progressive x0 row, as the reference logs them (ddpm.py:1320-1440)."""
        from ldm.util import log_txt_as_img
        use_ddim = ddim_steps is not None
        if sample and plot_denoise_rows and use_ddim:
            # the reference passes the DDIM intermediates dict to _get_denoise_row_from_list, which iterates its keys
            # and fails on the first one (str has no .to): there is no panel to reproduce
            raise NotImplementedError("plot_denoise_rows needs ddim_steps=None (DDPM sampling): with the DDIM sampler "
                                      "the reference's denoise row fails on the intermediates dict")
        batch = self.preprocess_batch(batch)
        log = dict()
        z, c, x, xrec, xc = self.get_input(batch, self.first_stage_key, return_first_stage_outputs=True,
                                           force_c_encode=True, return_original_cond=True, bs=N)
        c = c['caption']
        N = min(x.shape[0], N)
        n_row = min(x.shape[0], n_row)
        log["inputs"] = x
        log["reconstruction"] = xrec
        if self.model.conditioning_key is not None and self.cond_stage_key in ["caption"]:
            log["conditioning"] = log_txt_as_img((x.shape[2], x.shape[3]), batch["caption"][:N])
        if plot_diffusion_rows:
            # q_sample of the first n_row latents at every logged timestep, each with its own randn_like draw
            diffusion_row = list()
            z_start = z[:n_row].float().contiguous()
            for t in range(self.num_timesteps):
                if t % self.log_every_t == 0 or t == self.num_timesteps - 1:
                    tt = torch.full((n_row,), t, device=self.device, dtype=torch.long)
                    noise = torch.randn_like(z_start)
                    z_noisy = self.q_sample(x_start=z_start, t=tt, noise=noise)
                    diffusion_row.append(self.decode_first_stage(z_noisy))
            log["diffusion_row"] = _row_grid(diffusion_row)
        if sample:
            with self.ema_scope("Plotting"):
                samples, z_denoise_row = self.sample_log(cond=c, batch_size=N, ddim=use_ddim, ddim_steps=ddim_steps,
                                                         eta=ddim_eta)
            log["samples"] = self.decode_first_stage(samples)
            if plot_denoise_rows:
                log["denoise_row"] = self._get_denoise_row_from_list(z_denoise_row)
            uc = self.get_learned_conditioning(len(c) * [""])
            sample_scaled, _ = self.sample_log(cond=c, batch_size=N, ddim=ddim_steps is not None, ddim_steps=ddim_steps,
                                               eta=ddim_eta, unconditional_guidance_scale=5.0,
                                               unconditional_conditioning=uc)
            log["samples_scaled"] = self.decode_first_stage(sample_scaled)
            if inpaint:
                # ddpm.py:1405-1425: keep the latent outside a centre square; the reference passes the SAME mask to its
                # outpainting call, so both panels sample the square
                h, w = z.shape[2], z.shape[3]
                mask = torch.ones(N, h, w, device=z.device)
                mask[:, h // 4:3 * h // 4, w // 4:3 * w // 4] = 0.
                mask = mask[:, None, ...]
                with self.ema_scope("Plotting Inpaint"):
                    samples, _ = self.sample_log(cond=c, batch_size=N, ddim=ddim_steps is not None, eta=ddim_eta,
                                                 ddim_steps=ddim_steps, x0=z[:N], mask=mask)
                log["samples_inpainting"] = self.decode_first_stage(samples)
                log["mask"] = mask
                with self.ema_scope("Plotting Outpaint"):
                    samples, _ = self.sample_log(cond=c, batch_size=N, ddim=ddim_steps is not None, eta=ddim_eta,
                                                 ddim_steps=ddim_steps, x0=z[:N], mask=mask)
                log["samples_outpainting"] = self.decode_first_stage(samples)
        if plot_progressive_rows:
            with self.ema_scope("Plotting Progressives"):
                img, progressives = self.progressive_denoising(c, shape=(self.channels, self.image_size,
                                                                         self.image_size), batch_size=N)
            log["progressive_row"] = self._get_denoise_row_from_list(progressives, desc="Progressive Generation")
        if return_keys:
            if np.intersect1d(list(log.keys()), return_keys).shape[0] == 0:
                return log
            return {key: log[key] for key in return_keys}
        return log

    # ---- optimisation / checkpoint cadence (ddpm.py:1442-1454,1519-1528) --------------------------------------------
    def configure_optimizers(self):
        lr = self.learning_rate
        params = list(self.embedding_manager.embedding_parameters()) + list(self.embedding_manager.trainable_parameters())
        from celebbasis_b200.optim import FusedAdamW
        return FusedAdamW([p for p in params if p.requires_grad], lr=lr)

    @rank_zero_only
    def on_save_checkpoint(self, checkpoint):
        checkpoint.clear()
        logdir = getattr(getattr(self, "trainer", None), "checkpoint_callback", None)
        dirpath = getattr(logdir, "dirpath", None) or "."
        if os.path.isdir(dirpath):
            self.embedding_manager.save(os.path.join(dirpath, "embeddings.pt"))
            self.embedding_manager.save(os.path.join(dirpath, f"embeddings_gs-{self.global_step}.pt"))


class DiffusionWrapper(_Base):
    def __init__(self, diff_model_config, conditioning_key):
        super().__init__()
        self.diffusion_model = instantiate_from_config(diff_model_config)
        self.conditioning_key = conditioning_key
        assert self.conditioning_key in [None, 'crossattn']

    def forward(self, x, t, c_concat: list = None, c_crossattn: list = None):
        if self.conditioning_key is None:
            return self.diffusion_model(x, t)
        cc = c_crossattn[0] if len(c_crossattn) == 1 else torch.cat(c_crossattn, 1)
        return self.diffusion_model(x, t, context=cc)
