"""fp32 restatement of the rest of the reference DDIMSampler (ldm/models/diffusion/ddim.py), next to oracle/torch_ref.py's
ddim_sample: the masked (inpaint / outpaint) branch of ddim_sampling (:144-147), stochastic_encode (:207-220) and decode
(:223-241), with any eta and with or without classifier-free guidance.  Every random draw is injected, so the
restatement replays the stream the reference recorded (tests/golden/ddim_masked_tiny.pt).

The scalar schedule follows the reference's dtypes: ddim_alphas / ddim_alphas_prev are the fp32 alphas_cumprod values,
sigmas are float64, and every per-step coefficient is an fp32 tensor (torch.full in p_sample_ddim)."""
import numpy as np
import torch


def ddim_schedule(sched, steps, eta):
    """make_schedule (ddim.py:25-54) with uniform discretisation: (timesteps, a, a_prev, sigmas, sqrt_one_minus_a)."""
    T = sched["alphas_cumprod"].shape[0]
    ts = np.asarray(list(range(0, T, T // steps))) + 1
    ac = sched["alphas_cumprod"].float().cpu()
    a = ac[torch.as_tensor(ts)]
    a_prev = torch.cat([ac[:1], ac[torch.as_tensor(ts[:-1])]])
    a64, ap64 = a.double().numpy(), a_prev.double().numpy()
    sig = eta * np.sqrt((1 - ap64) / (1 - a64) * (1 - a64 / ap64))
    return ts, a, a_prev, torch.as_tensor(sig), torch.sqrt(1. - a)


def eps_cfg(unet, x, t, cond, uncond, scale):
    if uncond is None or scale == 1.:
        return unet(x, t, cond)
    e_u, e_c = unet(torch.cat([x] * 2), torch.cat([t] * 2), torch.cat([uncond, cond])).chunk(2)
    return e_u + scale * (e_c - e_u)


def p_sample_ddim(unet, sch, x, t, index, cond, uncond, scale, noise):
    """ddim.py:166-204.  `noise` is the noise_like draw of this step (None: the reference drew it, sigma is 0)."""
    _, a, a_prev, sig, s1m = sch
    e = eps_cfg(unet, x, t, cond, uncond, scale)
    dev = x.device
    a_t, a_p = a[index].to(dev), a_prev[index].to(dev)
    sigma_t, sq1m = sig[index].float().to(dev), s1m[index].to(dev)
    pred_x0 = (x - sq1m * e) / a_t.sqrt()
    dir_xt = (1. - a_p - sigma_t ** 2).sqrt() * e
    x_prev = a_p.sqrt() * pred_x0 + dir_xt
    if noise is not None:
        x_prev = x_prev + sigma_t * noise
    return x_prev, pred_x0


def q_sample(sched, x0, t, noise):
    """ddpm.py:289-292: extract(sqrt_ac, t) * x0 + extract(sqrt_1mac, t) * noise."""
    a = sched["sqrt_alphas_cumprod"].to(x0.device)[t].view(-1, 1, 1, 1)
    s = sched["sqrt_one_minus_alphas_cumprod"].to(x0.device)[t].view(-1, 1, 1, 1)
    return a * x0 + s * noise


def masked_blend(sched, x0, t, noise, mask, img):
    """ddim.py:146-147: img_orig = q_sample(x0, t); img_orig * mask + (1 - mask) * img."""
    img_orig = q_sample(sched, x0, t, noise)
    return img_orig * mask + (1. - mask) * img


def ddim_sample(unet, sched, cond, uncond, x_T, steps, scale, eta=0.0, mask=None, x0=None, blend_noise=None,
                step_noise=None):
    """DDIMSampler.sample -> ddim_sampling (ddim.py:57-163).  blend_noise[i] is q_sample's draw before step i (mask
    given), step_noise[i] the noise_like draw of step i (None where sigma is 0)."""
    sch = ddim_schedule(sched, steps, eta)
    ts = sch[0]
    x = x_T
    for i, step in enumerate(np.flip(ts)):
        index = len(ts) - i - 1
        t = torch.full((x.shape[0],), int(step), device=x.device, dtype=torch.long)
        if mask is not None:
            assert x0 is not None
            x = masked_blend(sched, x0, t, blend_noise[i], mask, x)
        x, _ = p_sample_ddim(unet, sch, x, t, index, cond, uncond, scale, None if step_noise is None else step_noise[i])
    return x


def ddim_stochastic_encode(sched, steps, x0, t, noise):
    """ddim.py:207-220 (use_original_steps False): t indexes the DDIM schedule; fp32 tables torch.sqrt(ddim_alphas) and
    np.sqrt(1 - ddim_alphas)."""
    _, a, _, _, s1m = ddim_schedule(sched, steps, 0.0)
    A = torch.sqrt(a).to(x0.device)[t].view(-1, 1, 1, 1)
    S = s1m.to(x0.device)[t].view(-1, 1, 1, 1)
    return A * x0 + S * noise


def ddim_decode(unet, sched, steps, eta, x_latent, cond, t_start, scale=1.0, uncond=None, step_noise=None):
    """ddim.py:223-241: the first t_start DDIM timesteps in reverse, index = total - i - 1, sigmas of make_schedule's eta."""
    sch = ddim_schedule(sched, steps, eta)
    ts = sch[0][:t_start]
    x = x_latent
    for i, step in enumerate(np.flip(ts)):
        index = len(ts) - i - 1
        t = torch.full((x.shape[0],), int(step), device=x.device, dtype=torch.long)
        x, _ = p_sample_ddim(unet, sch, x, t, index, cond, uncond, scale, None if step_noise is None else step_noise[i])
    return x
