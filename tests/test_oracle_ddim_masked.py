"""CPU: masked (inpaint / outpaint) DDIM sampling and the img2img pair stochastic_encode / decode.

  * the fp32 restatement (oracle/ddim_ref.py) reproduces tests/golden/ddim_masked_tiny.pt, which
    `python oracle/make_golden_masked.py` wrote from the UNMODIFIED reference, given the recorded random draws;
  * the mirror's DDIMSampler, with its device launches replaced by their torch arithmetic, draws exactly the stream the
    reference drew (same order, same shapes) and reproduces the same tensors;
  * argument errors and the host-side mask-broadcast strides of cb_q_sample_masked.
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from celebbasis_b200 import ops, synth, workload
from celebbasis_b200.tokenizer import SyntheticCLIPTokenizer
from oracle import ddim_ref, torch_ref


def _rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-30)).item()


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "ddim_masked_tiny.pt"), weights_only=False)


@pytest.fixture(scope="module")
def port():
    params = workload.model_params("tiny")
    om = torch_ref.OracleModel(params, clip_layers=workload.clip_layers("tiny"))
    om.load_state_dict(synth.synth_state_dict(om, seed=0), strict=True)
    om.eval()
    fs = params["first_stage_config"]["params"]
    dec = torch_ref.AutoencoderKLDecode(fs["ddconfig"], fs["embed_dim"])
    dec.load_state_dict(synth.synth_state_dict(dec, seed=0, prefix="first_stage_model."), strict=True)
    return om, dec.eval()


def _cond(om, prompts, pids, coef_seed=3):
    """Eval-branch conditioning (stored identity coefficients) of the restatement, as in test_oracle_golden."""
    g = torch.Generator().manual_seed(coef_seed)
    coefs = [F.normalize(torch.randn(2, 1, 512, generator=g), dim=-1) for _ in range(10)]
    tok = SyntheticCLIPTokenizer()
    tm = om.cond_stage_model.transformer.text_model
    basis = synth.synth_celeb_basis(seed=0)
    uc = tm.forward_embeds(tm.embed_tokens(tok([""] * len(prompts))["input_ids"]))
    ids = tok(prompts)["input_ids"]
    z = torch.cat([torch_ref.celeb_basis(coefs[p].view(1, 2, 1, 512), basis) for p in pids], 0)
    emb, _ = torch_ref.inject_embeddings(ids, tm.embed_tokens(ids), z, tok.word_id("sks"), 2)
    return tm.forward_embeds(emb), uc


def _sites(draws, site):
    return [d[3] for d in draws if d[1] == site]


def _lid_mask(N, h, w):
    mask = torch.ones(N, h, w)
    mask[:, h // 4:3 * h // 4, w // 4:3 * w // 4] = 0.
    return mask[:, None]


# ---------------------------------------------------------------------------------------------------------------------
def test_port_masked_sampling_matches_reference(gold, port):
    om, _ = port
    unet = om.model.diffusion_model
    with torch.no_grad():
        c, uc = _cond(om, gold["prompts"], gold["person_ids"])
        for case in gold["sample"]:
            mask = gold["masks"][case["mask"]]
            x = ddim_ref.ddim_sample(unet, om.sched, c, uc, gold["x_T"], gold["steps"], gold["scale"], eta=case["eta"],
                                     mask=mask, x0=gold["x0"], blend_noise=_sites(case["draws"], "q_sample"),
                                     step_noise=_sites(case["draws"], "noise_like") if case["eta"] > 0 else None)
            assert _rel(x, case["samples"]) < 1e-5, (case["mask"], case["eta"], _rel(x, case["samples"]))


def test_port_img2img_matches_reference(gold, port):
    om, dec = port
    unet = om.model.diffusion_model
    i2i = gold["img2img"]
    B = gold["x0"].shape[0]
    hw = gold["x0"].shape[-1]
    init = torch.rand(B, 3, 8 * hw, 8 * hw, generator=torch.Generator().manual_seed(i2i["init_seed"])) * 2 - 1
    with torch.no_grad():
        c, uc = _cond(om, gold["prompts"], gold["person_ids"])
        for case in i2i["cases"]:
            d = case["draws"]
            assert [x[1] for x in d[:2]] == ["sample", "stochastic_encode"]
            z0 = torch_ref.posterior_sample(om.first_stage_model(init), d[0][3], om.scale_factor)
            t = torch.tensor([i2i["t_enc"]] * B)
            z_enc = ddim_ref.ddim_stochastic_encode(om.sched, i2i["S"], z0, t, d[1][3])
            lat = ddim_ref.ddim_decode(unet, om.sched, i2i["S"], case["eta"], z_enc, c, i2i["t_enc"], scale=gold["scale"],
                                       uncond=uc, step_noise=_sites(d, "noise_like") if case["eta"] > 0 else None)
            ts = ddim_ref.ddim_schedule(om.sched, i2i["S"], case["eta"])[0]
            assert ts.tolist() == case["ddim_timesteps"].tolist()
            assert _rel(z0, case["z0"]) < 1e-5 and _rel(z_enc, case["z_enc"]) < 1e-5
            assert _rel(lat, case["latents"]) < 1e-5, (case["eta"], _rel(lat, case["latents"]))
            if case["img"] is not None:
                img = dec((1. / om.scale_factor) * lat)
                assert _rel(img, case["img"]) < 1e-5, _rel(img, case["img"])


def test_port_log_images_inpaint_matches_reference(gold, port):
    om, dec = port
    unet = om.model.diffusion_model
    li = gold["log_images"]
    N, steps, eta = li["N"], li["ddim_steps"], li["ddim_eta"]
    batch, _ = workload.synth_batch("tiny", B=N, seed=li["batch_seed"])
    # the reference's embedding manager draws three discarded vectors in eval mode (embedding_manager.py:313-315)
    d = [x for x in li["draws"] if x[1] != "forward"]
    assert [x[1] for x in d] == (["sample"] + (["ddim_sampling"] + ["noise_like"] * steps) * 2
                                 + (["ddim_sampling"] + ["q_sample", "noise_like"] * steps) * 2)
    d = [x[3] for x in d]
    P = li["panels"]
    with torch.no_grad():
        x = batch["image"].permute(0, 3, 1, 2).contiguous()
        z = torch_ref.posterior_sample(om.first_stage_model(x), d[0], om.scale_factor)
        assert _rel(z, li["z"]) < 1e-5
        assert _rel(dec((1. / om.scale_factor) * z), P["reconstruction"]) < 1e-5
        ids = batch["image_ori"]["ids"][:, 0].tolist()
        c, uc = _cond(om, batch["caption"], ids)
        k = 1
        for name, u, s in (("samples", None, 1.0), ("samples_scaled", uc, 5.0)):
            x_T, noise = d[k], d[k + 1:k + 1 + steps]
            k += 1 + steps
            lat = ddim_ref.ddim_sample(unet, om.sched, c, u, x_T, steps, s, eta=eta, step_noise=noise)
            assert _rel(dec((1. / om.scale_factor) * lat), P[name]) < 1e-5, name
        mask = _lid_mask(N, z.shape[2], z.shape[3])
        assert torch.equal(mask, P["mask"])
        for name in ("samples_inpainting", "samples_outpainting"):
            x_T, rest = d[k], d[k + 1:k + 1 + 2 * steps]
            k += 1 + 2 * steps
            lat = ddim_ref.ddim_sample(unet, om.sched, c, None, x_T, steps, 1.0, eta=eta, mask=mask, x0=z,
                                       blend_noise=rest[0::2], step_noise=rest[1::2])
            assert _rel(dec((1. / om.scale_factor) * lat), P[name]) < 1e-5, name
        assert k == len(d)


# ---------------------------------------------------------------------------------------------------------------------
class _Replay:
    """torch.randn / torch.randn_like replaced by the next recorded draw; the mirror's calls are logged."""

    def __init__(self, draws):
        self.draws, self.calls = list(draws), []

    def _next(self, fn, shape, device):
        assert self.draws, f"extra draw {fn}{shape}"
        d = self.draws.pop(0)
        self.calls.append((fn, tuple(shape)))
        assert (d[0], d[2]) == (fn, tuple(shape)), (d[:3], fn, shape)
        return d[3].clone().to(device)

    def install(self, monkeypatch):
        def randn(*shape, device=None, **k):
            shp = tuple(shape[0]) if len(shape) == 1 and not isinstance(shape[0], int) else tuple(shape)
            return self._next("randn", shp, device)

        def randn_like(x, **k):
            return self._next("randn_like", x.shape, x.device)
        monkeypatch.setattr(torch, "randn", randn)
        monkeypatch.setattr(torch, "randn_like", randn_like)


class _TorchModel:
    """What DDIMSampler reads from LatentDiffusion, on the CPU restatement."""

    def __init__(self, om):
        self.om = om
        self.num_timesteps = om.sched["alphas_cumprod"].shape[0]
        self.alphas_cumprod = om.sched["alphas_cumprod"]
        self.betas = om.sched["betas"]
        self.sqrt_alphas_cumprod = om.sched["sqrt_alphas_cumprod"]
        self.sqrt_one_minus_alphas_cumprod = om.sched["sqrt_one_minus_alphas_cumprod"]

    def apply_model(self, x, t, c):
        return self.om.model.diffusion_model(x, t, c)


def _torch_ops(monkeypatch):
    """The launches the sampler makes, as their torch arithmetic (the kernels are tested against the same on the GPU)."""
    def ddim_step(x, e_u, e_c, noise, *, scale, a_t, a_prev, sigma_t, sqrt_one_minus_at, want_x0=True):
        e = e_u if e_c is None else e_u + scale * (e_c - e_u)
        p0 = (x - sqrt_one_minus_at * e) / np.sqrt(a_t)
        xp = np.sqrt(a_prev) * p0 + np.sqrt(max(1. - a_prev - sigma_t ** 2, 0.)) * e
        return (xp + sigma_t * noise if noise is not None else xp), p0

    def q_sample_masked(x0, noise, t, sa, s1m, mask, img, out=None):
        ops.mask_strides(mask, tuple(img.shape))
        return ddim_ref.masked_blend({"sqrt_alphas_cumprod": sa, "sqrt_one_minus_alphas_cumprod": s1m}, x0, t, noise,
                                     mask, img)

    def q_sample(x0, noise, t, sa, s1m):
        return sa[t].view(-1, 1, 1, 1) * x0 + s1m[t].view(-1, 1, 1, 1) * noise
    monkeypatch.setattr(ops, "ddim_step", ddim_step)
    monkeypatch.setattr(ops, "q_sample_masked", q_sample_masked)
    monkeypatch.setattr(ops, "q_sample", q_sample)


def _mirror_stream(draws, eta):
    """The draws the mirror consumes: the reference's, minus noise_like at eta 0 (multiplied by sigma 0, so the mirror
    does not draw it)."""
    return [d for d in draws if not (d[1] == "noise_like" and eta == 0)]


def test_mirror_masked_sampling_replays_reference_draws(gold, port, monkeypatch):
    from ldm.models.diffusion.ddim import DDIMSampler
    om, _ = port
    _torch_ops(monkeypatch)
    model = _TorchModel(om)
    B, _, hw, _ = gold["x0"].shape
    with torch.no_grad():
        c, uc = _cond(om, gold["prompts"], gold["person_ids"])
        for case in gold["sample"]:
            exp = _mirror_stream(case["draws"], case["eta"])
            rep = _Replay(exp)
            with monkeypatch.context() as m:
                rep.install(m)
                x, _ = DDIMSampler(model).sample(S=gold["steps"], conditioning=c, batch_size=B, shape=[4, hw, hw],
                                                 verbose=False, unconditional_guidance_scale=gold["scale"],
                                                 unconditional_conditioning=uc, eta=case["eta"], x_T=gold["x_T"],
                                                 mask=gold["masks"][case["mask"]], x0=gold["x0"])
            assert not rep.draws and rep.calls == [(d[0], d[2]) for d in exp]
            # blend draw for step i, then (eta > 0) the DDIM draw of step i
            assert [d[1] for d in exp] == (["q_sample", "noise_like"] if case["eta"] > 0 else ["q_sample"]) * gold["steps"]
            assert _rel(x, case["samples"]) < 1e-5, (case["mask"], case["eta"], _rel(x, case["samples"]))


def test_mirror_img2img_replays_reference_draws(gold, port, monkeypatch):
    from ldm.models.diffusion.ddim import DDIMSampler
    om, _ = port
    _torch_ops(monkeypatch)
    i2i = gold["img2img"]
    B = gold["x0"].shape[0]
    with torch.no_grad():
        c, uc = _cond(om, gold["prompts"], gold["person_ids"])
        for case in i2i["cases"]:
            exp = _mirror_stream(case["draws"][1:], case["eta"])          # [0] is the posterior sample of the encoder
            rep = _Replay(exp)
            sampler = DDIMSampler(_TorchModel(om))
            sampler.make_schedule(ddim_num_steps=i2i["S"], ddim_eta=case["eta"], verbose=False)
            assert np.asarray(sampler.ddim_timesteps).tolist() == case["ddim_timesteps"].tolist()
            with monkeypatch.context() as m:
                rep.install(m)
                z_enc = sampler.stochastic_encode(case["z0"], torch.tensor([i2i["t_enc"]] * B))
                lat = sampler.decode(z_enc, c, i2i["t_enc"], unconditional_guidance_scale=gold["scale"],
                                     unconditional_conditioning=uc)
            assert not rep.draws and rep.calls == [(d[0], d[2]) for d in exp]
            assert _rel(z_enc, case["z_enc"]) < 1e-6
            assert _rel(lat, case["latents"]) < 1e-5, (case["eta"], _rel(lat, case["latents"]))


def test_mask_without_x0_and_original_steps_raise(port):
    from ldm.models.diffusion.ddim import DDIMSampler
    om, _ = port
    sampler = DDIMSampler(_TorchModel(om))
    x = torch.zeros(1, 4, 8, 8)
    with pytest.raises(AssertionError):
        sampler.sample(S=2, batch_size=1, shape=[4, 8, 8], conditioning=None, verbose=False, x_T=x,
                       mask=torch.ones(1, 1, 8, 8))
    sampler.make_schedule(2, verbose=False)
    with pytest.raises(NotImplementedError, match="ddim_sigmas_for_original_num_steps"):
        sampler.decode(x, None, 1, use_original_steps=True)
    with pytest.raises(NotImplementedError, match="ddim_sigmas_for_original_num_steps"):
        sampler.ddim_sampling(None, (1, 4, 8, 8), x_T=x, ddim_use_original_steps=True)
    with pytest.raises(NotImplementedError):
        sampler.p_sample_ddim(x, None, torch.zeros(1, dtype=torch.long), 0, use_original_steps=True)


def test_mask_broadcast_strides():
    B, C, h, w = 3, 4, 8, 16
    assert ops.mask_strides(torch.ones(B, 1, h, w), (B, C, h, w)) == (h * w, 0)        # log_images' (N,1,h,w)
    assert ops.mask_strides(torch.ones(1, 1, h, w), (B, C, h, w)) == (0, 0)
    assert ops.mask_strides(torch.ones(B, C, h, w), (B, C, h, w)) == (C * h * w, h * w)
    assert ops.mask_strides(torch.ones(h, w), (B, C, h, w)) == (0, 0)
    # the strides address the same element torch's broadcast does
    m = torch.rand(B, 1, h, w)
    sb, sc = ops.mask_strides(m, (B, C, h, w))
    flat = m.flatten()
    e = m.expand(B, C, h, w)
    for b, c, y, x in ((0, 0, 0, 0), (2, 3, 7, 15), (1, 2, 3, 4)):
        assert flat[b * sb + c * sc + y * w + x] == e[b, c, y, x]
    with pytest.raises(ValueError):
        ops.mask_strides(torch.ones(B, 1, w, h).transpose(2, 3), (B, C, h, w))          # spatially transposed
    with pytest.raises(ValueError):
        ops.mask_strides(torch.ones(B, 1, 1, 1), (B, C, h, w))                          # spatially broadcast
