"""fp32 restatement of LatentDiffusion's DDPM ancestral sampler (ldm/models/diffusion/ddpm.py): p_sample through
p_mean_variance / predict_start_from_noise / q_posterior for eps-prediction (:231-244,1118-1178), p_sample_loop
(:1236-1285) and progressive_denoising (:1180-1234), with the optional masked blend after every step.  Every random
draw is injected, so the restatement replays the stream the reference recorded (tests/golden/ddpm_sample_tiny.pt).

The tables are register_schedule's (ddpm.py:126-178): float64 numpy arithmetic, stored as fp32.  Each expression is
written in the reference's order, so on one device the restatement and the eager reference round identically."""
import hashlib

import numpy as np
import torch

from oracle import ddim_ref


def digest(t):
    return hashlib.sha1(t.detach().float().contiguous().numpy().tobytes()).hexdigest()[:16]


def regenerate_draws(seed, calls, p_dropout=None):
    """The CPU draws a recorded case made, in order: torch.manual_seed(seed), then for each (function, call site, shape)
    torch.randn(shape) for randn / randn_like, or F.dropout(ones(shape), p_dropout) (the mask over 1 - p) for dropout.
    A fourth entry, when present, is the recorded sha1 prefix of the values and is checked.  The global generator's
    state is restored afterwards."""
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        out = []
        for c in calls:
            fn, shape = c[0], tuple(c[2])
            if fn == "dropout":
                v = torch.nn.functional.dropout(torch.ones(shape), p=p_dropout)
            else:
                assert fn in ("randn", "randn_like"), fn
                v = torch.randn(shape)
            assert len(c) < 4 or digest(v) == c[3], f"draw {len(out)} {c[:3]}: regenerated values differ from the record"
            out.append(v)
    return out


def ddpm_tables(timesteps=1000, linear_start=0.00085, linear_end=0.0120):
    """The fp32 buffers p_sample reads, plus q_sample's two (for the masked blend)."""
    betas = (torch.linspace(linear_start ** 0.5, linear_end ** 0.5, timesteps, dtype=torch.float64) ** 2).numpy()
    alphas = 1. - betas
    ac = np.cumprod(alphas, axis=0)
    ac_prev = np.append(1., ac[:-1])
    post_var = betas * (1. - ac_prev) / (1. - ac)
    f32 = lambda a: torch.tensor(a, dtype=torch.float32)  # noqa: E731
    return {"sqrt_alphas_cumprod": f32(np.sqrt(ac)), "sqrt_one_minus_alphas_cumprod": f32(np.sqrt(1. - ac)),
            "sqrt_recip_alphas_cumprod": f32(np.sqrt(1. / ac)), "sqrt_recipm1_alphas_cumprod": f32(np.sqrt(1. / ac - 1)),
            "posterior_mean_coef1": f32(betas * np.sqrt(ac_prev) / (1. - ac)),
            "posterior_mean_coef2": f32((1. - ac_prev) * np.sqrt(alphas) / (1. - ac)),
            "posterior_log_variance_clipped": f32(np.log(np.maximum(post_var, 1e-20)))}


def _at(tab, name, t):
    return tab[name].to(t.device)[t].view(-1, 1, 1, 1)


def posterior_step(tab, x, eps, t, noise, temperature=1., clip=False, dropout_scale=None):
    """ddpm.py:1149-1178 given the model output `eps` and the noise_like draw `noise`: returns (x_prev, x_recon).
    dropout_scale is F.dropout's multiplier (bernoulli mask / (1 - p)) when noise_dropout > 0."""
    x_recon = _at(tab, "sqrt_recip_alphas_cumprod", t) * x - _at(tab, "sqrt_recipm1_alphas_cumprod", t) * eps
    if clip:
        x_recon = x_recon.clamp(-1., 1.)
    mean = _at(tab, "posterior_mean_coef1", t) * x_recon + _at(tab, "posterior_mean_coef2", t) * x
    log_var = _at(tab, "posterior_log_variance_clipped", t)
    noise = noise * temperature
    if dropout_scale is not None:
        noise = noise * dropout_scale
    nonzero_mask = (1 - (t == 0).float()).view(-1, 1, 1, 1)
    return mean + nonzero_mask * (0.5 * log_var).exp() * noise, x_recon


def p_sample_loop(unet, tab, cond, x_T, timesteps, step_noise, log_every_t, mask=None, x0=None, blend_noise=None,
                  clip=False):
    """ddpm.py:1236-1285 from x_T over reversed(range(timesteps)).  step_noise[k] / blend_noise[k] are step k's
    noise_like and q_sample draws.  Returns (x_0, intermediates = [x_T] + x_t at every logged step)."""
    img, inter = x_T, [x_T]
    for k, i in enumerate(reversed(range(timesteps))):
        t = torch.full((x_T.shape[0],), i, device=x_T.device, dtype=torch.long)
        img, _ = posterior_step(tab, img, unet(img, t, cond), t, step_noise[k], clip=clip)
        if mask is not None:
            img = ddim_ref.masked_blend(tab, x0, t, blend_noise[k], mask, img)
        if i % log_every_t == 0 or i == timesteps - 1:
            inter.append(img)
    return img, inter


def progressive_denoising(unet, tab, cond, x_T, timesteps, step_noise, log_every_t, temperature, dropout_scale=None,
                          clip=False):
    """ddpm.py:1180-1234 without a mask: temperature[i] is the list entry of timestep i, dropout_scale[k] step k's
    dropout multiplier (None: noise_dropout 0).  Returns (x_0, the x0 predictions at every logged step)."""
    img, inter = x_T, []
    for k, i in enumerate(reversed(range(timesteps))):
        t = torch.full((x_T.shape[0],), i, device=x_T.device, dtype=torch.long)
        img, x0 = posterior_step(tab, img, unet(img, t, cond), t, step_noise[k], temperature=temperature[i], clip=clip,
                                 dropout_scale=None if dropout_scale is None else dropout_scale[k])
        if i % log_every_t == 0 or i == timesteps - 1:
            inter.append(x0)
    return img, inter
