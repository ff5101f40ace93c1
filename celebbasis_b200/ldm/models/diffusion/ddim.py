"""Host mirror of ldm/models/diffusion/ddim.py (DDIMSampler: make_schedule :25-54, sample :57-111,
ddim_sampling :114-163, p_sample_ddim :166-204, stochastic_encode :207-220, decode :223-241).  The schedule is host
float64 arithmetic as in the reference; the per-step update with classifier-free guidance is one kernel (cb_ddim_step);
the masked (inpaint / outpaint) blend before a step is one kernel (cb_q_sample_masked); the UNet runs through the
mirror."""
import numpy as np
import torch

from celebbasis_b200 import ops
from ldm.modules.diffusionmodules.util import make_ddim_sampling_parameters, make_ddim_timesteps, noise_like

_ORIGINAL_STEPS = ("use_original_steps=True is not supported: the reference's p_sample_ddim then reads "
                   "model.ddim_sigmas_for_original_num_steps, which LatentDiffusion does not define (AttributeError)")


class DDIMSampler(object):
    def __init__(self, model, schedule="linear", **kwargs):
        self.model = model
        self.ddpm_num_timesteps = model.num_timesteps
        self.schedule = schedule

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0., verbose=True):
        self.ddim_timesteps = make_ddim_timesteps(ddim_discr_method=ddim_discretize, num_ddim_timesteps=ddim_num_steps,
                                                  num_ddpm_timesteps=self.ddpm_num_timesteps, verbose=verbose)
        ac = self.model.alphas_cumprod.detach().cpu().double().numpy()
        assert ac.shape[0] == self.ddpm_num_timesteps
        sig, a, a_prev = make_ddim_sampling_parameters(alphacums=ac, ddim_timesteps=self.ddim_timesteps, eta=ddim_eta,
                                                       verbose=verbose)
        self.ddim_sigmas, self.ddim_alphas, self.ddim_alphas_prev = sig, a, a_prev
        self.ddim_sqrt_one_minus_alphas = np.sqrt(1. - a)
        self._encode_tables = None

    @torch.no_grad()
    def sample(self, S, batch_size, shape, conditioning=None, callback=None, normals_sequence=None,
               img_callback=None, quantize_x0=False, eta=0., mask=None, x0=None, temperature=1.,
               noise_dropout=0., score_corrector=None, corrector_kwargs=None, verbose=True, x_T=None,
               log_every_t=100, unconditional_guidance_scale=1., unconditional_conditioning=None, **kwargs):
        self.make_schedule(ddim_num_steps=S, ddim_eta=eta, verbose=verbose)
        C, H, W = shape
        return self.ddim_sampling(conditioning, (batch_size, C, H, W), callback=callback, img_callback=img_callback,
                                  mask=mask, x0=x0, x_T=x_T, log_every_t=log_every_t, temperature=temperature,
                                  unconditional_guidance_scale=unconditional_guidance_scale,
                                  unconditional_conditioning=unconditional_conditioning)

    @torch.no_grad()
    def ddim_sampling(self, cond, shape, x_T=None, ddim_use_original_steps=False, callback=None, mask=None, x0=None,
                      img_callback=None, log_every_t=100, temperature=1., unconditional_guidance_scale=1.,
                      unconditional_conditioning=None, **kwargs):
        if ddim_use_original_steps:
            raise NotImplementedError(_ORIGINAL_STEPS)
        device = self.model.betas.device
        b = shape[0]
        img = torch.randn(shape, device=device) if x_T is None else x_T
        if mask is not None:
            assert x0 is not None
            assert tuple(x0.shape) == tuple(img.shape), (tuple(x0.shape), tuple(img.shape))
            x0 = x0.float().contiguous()
            mask = mask.to(device=img.device, dtype=torch.float32)
        intermediates = {'x_inter': [img], 'pred_x0': [img]}
        time_range = np.flip(self.ddim_timesteps)
        total_steps = self.ddim_timesteps.shape[0]
        for i, step in enumerate(time_range):
            index = total_steps - i - 1
            ts = torch.full((b,), int(step), device=device, dtype=torch.long)
            if mask is not None:
                # img_orig = model.q_sample(x0, ts); img = img_orig * mask + (1 - mask) * img  (ddim.py:144-147):
                # q_sample's own noise draw (ddpm.py:290), then one fused launch
                noise = torch.randn_like(x0)
                img = ops.q_sample_masked(x0, noise, ts, self.model.sqrt_alphas_cumprod,
                                          self.model.sqrt_one_minus_alphas_cumprod, mask, img.float().contiguous())
            img, pred_x0 = self.p_sample_ddim(img, cond, ts, index=index, temperature=temperature,
                                              unconditional_guidance_scale=unconditional_guidance_scale,
                                              unconditional_conditioning=unconditional_conditioning)
            if callback:
                callback(i)
            if img_callback:
                img_callback(pred_x0, i)
            if index % log_every_t == 0 or index == total_steps - 1:
                intermediates['x_inter'].append(img)
                intermediates['pred_x0'].append(pred_x0)
        return img, intermediates

    @torch.no_grad()
    def p_sample_ddim(self, x, c, t, index, repeat_noise=False, use_original_steps=False, quantize_denoised=False,
                      temperature=1., noise_dropout=0., score_corrector=None, corrector_kwargs=None,
                      unconditional_guidance_scale=1., unconditional_conditioning=None):
        if use_original_steps:
            raise NotImplementedError(_ORIGINAL_STEPS)
        b, device = x.shape[0], x.device
        if unconditional_conditioning is None or unconditional_guidance_scale == 1.:
            e_u, e_c = self.model.apply_model(x, t, c), None
        else:
            x_in = torch.cat([x] * 2)            # CFG batch doubling (ddim.py:176-180): layout glue
            t_in = torch.cat([t] * 2)
            c_in = torch.cat([unconditional_conditioning, c])
            e_u, e_c = self.model.apply_model(x_in, t_in, c_in).chunk(2)
            e_u, e_c = e_u.contiguous(), e_c.contiguous()
        sigma = float(self.ddim_sigmas[index])
        noise = None
        if sigma > 0:
            noise = (noise_like(x.shape, device, repeat_noise) * temperature).contiguous()
        return ops.ddim_step(x.contiguous(), e_u, e_c, noise, scale=float(unconditional_guidance_scale),
                             a_t=float(self.ddim_alphas[index]), a_prev=float(self.ddim_alphas_prev[index]),
                             sigma_t=sigma, sqrt_one_minus_at=float(self.ddim_sqrt_one_minus_alphas[index]))

    @torch.no_grad()
    def stochastic_encode(self, x0, t, use_original_steps=False, noise=None):
        """img2img forward noising (ddim.py:207-220): t indexes the DDIM schedule of the last make_schedule (or the DDPM
        schedule with use_original_steps); one cb_q_sample launch on the fp32 tables the reference gathers from."""
        x0 = x0.float().contiguous()
        if noise is None:
            noise = torch.randn_like(x0)
        sqrt_a, sqrt_1ma = self._tables(use_original_steps, x0.device)
        t = t.to(device=x0.device, dtype=torch.long).contiguous()
        assert t.shape == (x0.shape[0],), (tuple(t.shape), tuple(x0.shape))
        return ops.q_sample(x0, noise.float().contiguous(), t, sqrt_a, sqrt_1ma)

    def _tables(self, use_original_steps, device):
        # the reference's fp32 tables: sqrt(alphas_cumprod) / sqrt(1 - alphas_cumprod) of make_schedule (ddim.py:37-38),
        # or torch.sqrt(ddim_alphas) / np.sqrt(1 - ddim_alphas) with ddim_alphas gathered from the fp32 alphas_cumprod
        key = (bool(use_original_steps), str(device))
        if self._encode_tables is None or self._encode_tables[0] != key:
            ac = self.model.alphas_cumprod.detach().float().cpu()
            a = ac if use_original_steps else ac[torch.as_tensor(np.asarray(self.ddim_timesteps, dtype=np.int64))]
            self._encode_tables = (key, (torch.sqrt(a).to(device), torch.sqrt(1. - a).to(device)))
        return self._encode_tables[1]

    @torch.no_grad()
    def decode(self, x_latent, cond, t_start, unconditional_guidance_scale=1.0, unconditional_conditioning=None,
               use_original_steps=False):
        """img2img denoising (ddim.py:223-241): the first t_start DDIM timesteps in reverse, index = total - i - 1, with
        the sigmas of the last make_schedule."""
        if use_original_steps:
            raise NotImplementedError(_ORIGINAL_STEPS)
        timesteps = self.ddim_timesteps[:t_start]
        time_range = np.flip(timesteps)
        total_steps = timesteps.shape[0]
        x_dec = x_latent
        for i, step in enumerate(time_range):
            index = total_steps - i - 1
            ts = torch.full((x_latent.shape[0],), int(step), device=x_latent.device, dtype=torch.long)
            x_dec, _ = self.p_sample_ddim(x_dec, cond, ts, index=index,
                                          unconditional_guidance_scale=unconditional_guidance_scale,
                                          unconditional_conditioning=unconditional_conditioning)
        return x_dec
