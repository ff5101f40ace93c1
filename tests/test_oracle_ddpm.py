"""CPU: the DDPM ancestral sampler of LatentDiffusion (sample, p_sample_loop, progressive_denoising, p_sample) and the
log_images panels it feeds.

  * the fp32 restatement (oracle/ddpm_ref.py) reproduces tests/golden/ddpm_sample_tiny.pt, which
    `python oracle/make_golden_ddpm.py` wrote from the UNMODIFIED reference, given the recorded random draws;
  * the mirror's methods, with the UNet and the two sampler launches replaced by their torch arithmetic, make exactly
    the draws the reference made (function, call site, shape, in order) and reproduce the same tensors;
  * the options the mirror rejects, the DDPM branch of sample_log and the grid layout of the row panels.
"""
import os
import sys

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from celebbasis_b200 import ops, synth, workload
from celebbasis_b200.tokenizer import SyntheticCLIPTokenizer
from oracle import ddim_ref, ddpm_ref, torch_ref


def _rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-30)).item()


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "ddpm_sample_tiny.pt"), weights_only=False)


@pytest.fixture(scope="module")
def tab():
    return ddpm_ref.ddpm_tables()


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


@pytest.fixture(scope="module")
def cond(gold, port):
    return _cond(port[0], gold["prompts"], gold["person_ids"])


def _cond(om, prompts, pids, coef_seed=3):
    """Eval-branch conditioning (stored identity coefficients) of the restatement."""
    g = torch.Generator().manual_seed(coef_seed)
    coefs = [F.normalize(torch.randn(2, 1, 512, generator=g), dim=-1) for _ in range(10)]
    tok = SyntheticCLIPTokenizer()
    tm = om.cond_stage_model.transformer.text_model
    basis = synth.synth_celeb_basis(seed=0)
    ids = tok(prompts)["input_ids"]
    z = torch.cat([torch_ref.celeb_basis(coefs[p].view(1, 2, 1, 512), basis) for p in pids], 0)
    emb, _ = torch_ref.inject_embeddings(ids, tm.embed_tokens(ids), z, tok.word_id("sks"), 2)
    return tm.forward_embeds(emb)


def _draws(rec):
    """[(function, call site, shape, values)] of a recorded case, regenerated from its seed and digest-checked."""
    vals = ddpm_ref.regenerate_draws(rec["seed"], rec["calls"], rec["p_dropout"])
    return [c[:3] + (v,) for c, v in zip(rec["calls"], vals)]


def _sites(draws, site):
    return [d[3] for d in draws if d[1] == site]


def _panel_close(x, ref16):
    """x (fp32) against a panel stored in fp16: the storage rounding (2^-11 relative) plus 1e-5 of the panel's scale."""
    ref = ref16.float()
    assert x.shape == ref.shape, (tuple(x.shape), tuple(ref.shape))
    return bool(((x - ref).abs() <= 2. ** -11 * x.abs() + 1e-5 * ref.abs().max()).all())


# ---------------------------------------------------------------------------------------------------------------------
def test_regenerated_draws_match_the_record(gold):
    for rec in (gold["sample"]["draws"], gold["progressive"]["draws"], gold["log_images"]["draws"]):
        d = _draws(rec)                               # raises on the first digest mismatch
        assert len(d) == len(rec["calls"])
    d = _draws(gold["progressive"]["draws"])
    scales = _sites(d, "p_sample")
    p = gold["progressive"]["noise_dropout"]
    assert len(scales) == gold["progressive"]["start_T"]
    vals = torch.cat([s.flatten() for s in scales]).unique().tolist()
    assert len(vals) == 2 and vals[0] == 0.0 and abs(vals[1] - 1 / (1 - p)) < 1e-6, vals


def test_port_sample_matches_reference(gold, port, tab, cond):
    om, _ = port
    a = gold["sample"]
    d = _draws(a["draws"])
    assert [x[1] for x in d] == ["p_sample_loop"] + ["noise_like"] * 1000
    with torch.no_grad():
        x, inter = ddpm_ref.p_sample_loop(om.model.diffusion_model, tab, cond, d[0][3], 1000, _sites(d, "noise_like"),
                                          gold["log_every_t"])
    assert len(inter) == a["intermediates"].shape[0] == 7
    assert _rel(x, a["samples"]) < 1e-5, _rel(x, a["samples"])
    for k, (p, r) in enumerate(zip(inter, a["intermediates"])):
        assert _rel(p, r) < 1e-5, (k, _rel(p, r))


def test_port_masked_loop_matches_reference(gold, port, tab, cond):
    om, _ = port
    for case in gold["masked"]:
        d = _draws(case["draws"])
        assert [x[1] for x in d] == ["noise_like", "q_sample"] * case["start_T"]
        with torch.no_grad():
            x, inter = ddpm_ref.p_sample_loop(om.model.diffusion_model, tab, cond, gold["x_T"], case["start_T"],
                                              _sites(d, "noise_like"), case["log_every_t"],
                                              mask=gold["masks"][case["mask"]], x0=gold["x0"],
                                              blend_noise=_sites(d, "q_sample"))
        assert len(inter) == case["intermediates"].shape[0] == 7            # x_T, then i = 49, 40, 30, 20, 10, 0
        assert _rel(x, case["samples"]) < 1e-5, (case["mask"], _rel(x, case["samples"]))
        for p, r in zip(inter, case["intermediates"]):
            assert _rel(p, r) < 1e-5, (case["mask"], _rel(p, r))


def test_port_progressive_matches_reference(gold, port, tab, cond):
    om, _ = port
    pc = gold["progressive"]
    d = _draws(pc["draws"])
    assert [x[1] for x in d] == ["progressive_denoising"] + ["noise_like", "p_sample"] * pc["start_T"]
    with torch.no_grad():
        x, inter = ddpm_ref.progressive_denoising(om.model.diffusion_model, tab, cond, d[0][3], pc["start_T"],
                                                  _sites(d, "noise_like"), pc["log_every_t"], pc["temperature"],
                                                  dropout_scale=_sites(d, "p_sample"))
    assert _rel(x, pc["samples"]) < 1e-5, _rel(x, pc["samples"])
    assert len(inter) == pc["intermediates"].shape[0]
    for p, r in zip(inter, pc["intermediates"]):
        assert _rel(p, r) < 1e-5, _rel(p, r)


def test_port_log_images_matches_reference(gold, port, tab):
    """Every latent the reference's log_images decoded, in order, and the panels built from them."""
    om, dec = port
    li = gold["log_images"]
    T, every = 1000, gold["log_every_t"]
    logged = [t for t in range(T) if t % every == 0 or t == T - 1]
    # the reference's embedding manager draws three discarded vectors per encode in eval mode (embedding_manager.py:313)
    d = [x for x in _draws(li["draws"]) if x[1] != "forward"]
    assert [x[1] for x in d] == (["sample"] + ["log_images"] * len(logged) + (["p_sample_loop"] + ["noise_like"] * T) * 2
                                 + ["progressive_denoising"] + ["noise_like"] * T)
    assert li["keys"] == ["inputs", "reconstruction", "conditioning", "diffusion_row", "samples", "denoise_row",
                          "samples_scaled", "progressive_row"]
    N = li["N"]
    batch, _ = workload.synth_batch("tiny", B=N, seed=li["batch_seed"])
    unet = om.model.diffusion_model
    lat = []
    with torch.no_grad():
        x = batch["image"].permute(0, 3, 1, 2).contiguous()
        z = torch_ref.posterior_sample(om.first_stage_model(x), d[0][3], om.scale_factor)
        lat.append(z)                                                    # reconstruction
        for k, t in enumerate(logged):                                   # diffusion row
            lat.append(ddim_ref.q_sample(tab, z[:li["n_row"]], torch.full((li["n_row"],), t), d[1 + k][3]))
        k = 1 + len(logged)
        c = _cond(om, batch["caption"], batch["image_ori"]["ids"][:, 0].tolist())
        runs = []
        for _ in range(2):                                               # samples, then samples_scaled (unguided)
            runs.append(ddpm_ref.p_sample_loop(unet, tab, c, d[k][3], T, [x[3] for x in d[k + 1:k + 1 + T]], every))
            k += 1 + T
        lat += [runs[0][0]] + runs[0][1] + [runs[1][0]]                  # samples, denoise row, samples_scaled
        _, prog = ddpm_ref.progressive_denoising(unet, tab, c, d[k][3], T, [x[3] for x in d[k + 1:k + 1 + T]], every,
                                                 [1.] * T)
        lat += prog
        assert len(lat) == li["decoded"].shape[0]
        for j, (p, r) in enumerate(zip(lat, li["decoded"])):
            assert _rel(p, r) < 1e-5, (j, _rel(p, r))
        from ldm.models.diffusion.ddpm import _row_grid
        img = [dec((1. / om.scale_factor) * v) for v in lat]
        nd = len(logged)
        P = li["panels_fp16"]
        assert _panel_close(img[0], P["reconstruction"])
        rows = {"diffusion_row": _row_grid(img[1:1 + nd]), "denoise_row": _row_grid(img[2 + nd:2 + nd + len(runs[0][1])]),
                "progressive_row": _row_grid(img[-len(prog):])}
        assert _panel_close(img[2 + nd + len(runs[0][1])], P["samples_scaled"])
        for key, grid in rows.items():
            assert tuple(grid.shape) == li["shapes"][key]
            assert _panel_close(grid[:, :P[key].shape[1]], P[key]), key      # the fixture keeps the first grid row


def test_row_grid_is_make_grid_of_the_rearranged_stack():
    tv = pytest.importorskip("torchvision")
    from einops import rearrange
    from ldm.models.diffusion.ddpm import _row_grid
    for n, b, C in ((6, 2, 3), (7, 3, 3), (2, 1, 3), (3, 2, 1)):
        imgs = [torch.randn(b, C, 5, 7) for _ in range(n)]
        rows = rearrange(rearrange(torch.stack(imgs), 'n b c h w -> b n c h w'), 'b n c h w -> (b n) c h w')
        assert torch.equal(_row_grid(imgs), tv.utils.make_grid(rows, nrow=n))


# ---------------------------------------------------------------------------------------------------------------------
_MIRROR_SITE = {"_masked_blend": "q_sample"}     # where the mirror draws q_sample's noise before its fused blend


class _Replay:
    """torch.randn / torch.randn_like / F.dropout return the next recorded draw (dropout: input * recorded multiplier);
    each call's (function, call site, shape) is logged and checked against the record."""

    def __init__(self, draws):
        self.draws, self.calls = list(draws), []

    def _next(self, fn, shape):
        site = sys._getframe(2).f_code.co_name
        site = _MIRROR_SITE.get(site, site)
        assert self.draws, f"extra draw {fn}{shape} at {site}"
        d = self.draws.pop(0)
        self.calls.append((fn, site, tuple(shape)))
        assert (d[0], d[1], tuple(d[2])) == (fn, site, tuple(shape)), (d[:3], fn, site, shape)
        return d[3].clone()

    def install(self, m):
        def randn(*shape, device=None, **k):
            shp = tuple(shape[0]) if len(shape) == 1 and not isinstance(shape[0], int) else tuple(shape)
            return self._next("randn", shp).to(device) if device is not None else self._next("randn", shp)

        def randn_like(x, **k):
            return self._next("randn_like", x.shape).to(x.device)

        o_dropout = torch.nn.functional.dropout

        def dropout(x, p=0.5, training=True, inplace=False):
            if not training or p == 0.:                   # draws nothing (eval-mode dropout layers)
                return o_dropout(x, p=p, training=training, inplace=inplace)
            return x * self._next("dropout", x.shape).to(x.device)
        m.setattr(torch, "randn", randn)
        m.setattr(torch, "randn_like", randn_like)
        m.setattr(torch.nn.functional, "dropout", dropout)


def _torch_ops(m):
    """The two launches the sampler makes, as the restatement's torch arithmetic (the kernel is held bit-exact to the
    same expression on the GPU)."""
    def p_sample(x, eps, noise, t, sr, srm1, c1, c2, lv, *, temperature=1.0, clip_denoised=False, out=None,
                 want_x0=True):
        tb = {"sqrt_recip_alphas_cumprod": sr, "sqrt_recipm1_alphas_cumprod": srm1, "posterior_mean_coef1": c1,
              "posterior_mean_coef2": c2, "posterior_log_variance_clipped": lv}
        xp, x0 = ddpm_ref.posterior_step(tb, x, eps, t, noise, temperature, clip_denoised)
        return xp, (x0 if want_x0 else None)

    def q_sample_masked(x0, noise, t, sa, s1m, mask, img, out=None):
        ops.mask_strides(mask, tuple(img.shape))
        return ddim_ref.masked_blend({"sqrt_alphas_cumprod": sa, "sqrt_one_minus_alphas_cumprod": s1m}, x0, t, noise,
                                     mask, img)
    m.setattr(ops, "p_sample", p_sample)
    m.setattr(ops, "q_sample_masked", q_sample_masked)


def _torch_ld(om, tab, **over):
    """A LatentDiffusion whose UNet is the restatement's and whose schedule buffers are the reference's tables; only the
    sampler's state is set (no engines are built)."""
    from ldm.models.diffusion.ddpm import LatentDiffusion

    class TorchLD(LatentDiffusion):
        def __init__(self):
            nn.Module.__init__(self)
            self.unet = om.model.diffusion_model
            for k, v in tab.items():
                setattr(self, k, v)
            self.betas = torch.zeros(1000)
            self.num_timesteps, self.num_timesteps_cond, self.log_every_t = 1000, 1, 200
            self.clip_denoised, self.channels, self.image_size = False, 4, 8
            for k, v in over.items():
                setattr(self, k, v)

        def apply_model(self, x, t, cond, return_ids=False):
            return self.unet(x, t, cond)
    return TorchLD()


def test_mirror_sample_replays_reference_draws(gold, port, tab, cond, monkeypatch):
    om, _ = port
    ld = _torch_ld(om, tab, log_every_t=gold["log_every_t"])
    a = gold["sample"]
    rep = _Replay(_draws(a["draws"]))
    with monkeypatch.context() as m, torch.no_grad():
        _torch_ops(m)
        rep.install(m)
        x, inter = ld.sample(cond, batch_size=2, return_intermediates=True)
    assert not rep.draws and len(rep.calls) == 1001
    assert _rel(x, a["samples"]) < 1e-5 and len(inter) == a["intermediates"].shape[0]
    for p, r in zip(inter, a["intermediates"]):
        assert _rel(p, r) < 1e-5


def test_mirror_masked_loop_replays_reference_draws(gold, port, tab, cond, monkeypatch):
    om, _ = port
    ld = _torch_ld(om, tab, log_every_t=gold["log_every_t"])
    for case in gold["masked"]:
        rep = _Replay(_draws(case["draws"]))
        seen = []
        with monkeypatch.context() as m, torch.no_grad():
            _torch_ops(m)
            rep.install(m)
            x, inter = ld.p_sample_loop(cond, tuple(gold["x_T"].shape), return_intermediates=True, x_T=gold["x_T"],
                                        mask=gold["masks"][case["mask"]], x0=gold["x0"], start_T=case["start_T"],
                                        log_every_t=case["log_every_t"], callback=seen.append,
                                        img_callback=lambda img, i: seen.append(img.shape))
        assert not rep.draws
        assert seen[:2] == [case["start_T"] - 1, gold["x_T"].shape] and len(seen) == 2 * case["start_T"]
        assert _rel(x, case["samples"]) < 1e-5, (case["mask"], _rel(x, case["samples"]))
        assert len(inter) == case["intermediates"].shape[0]
        for p, r in zip(inter, case["intermediates"]):
            assert _rel(p, r) < 1e-5


def test_mirror_progressive_replays_reference_draws(gold, port, tab, cond, monkeypatch):
    om, _ = port
    ld = _torch_ld(om, tab, log_every_t=gold["log_every_t"])
    pc = gold["progressive"]
    rep = _Replay(_draws(pc["draws"]))
    with monkeypatch.context() as m, torch.no_grad():
        _torch_ops(m)
        rep.install(m)
        x, inter = ld.progressive_denoising(torch.cat([cond, cond]), shape=(4, 8, 8), batch_size=2,
                                            start_T=pc["start_T"], temperature=pc["temperature"],
                                            noise_dropout=pc["noise_dropout"], log_every_t=pc["log_every_t"])
    assert not rep.draws
    assert _rel(x, pc["samples"]) < 1e-5, _rel(x, pc["samples"])
    assert len(inter) == pc["intermediates"].shape[0]
    for p, r in zip(inter, pc["intermediates"]):
        assert _rel(p, r) < 1e-5


def test_conditioning_is_sliced_to_the_batch(port, tab, monkeypatch):
    om, _ = port
    seen = []
    ld = _torch_ld(om, tab)
    ld.apply_model = lambda x, t, c, return_ids=False: (seen.append(c), torch.zeros_like(x))[1]
    c = torch.randn(3, 77, 768)
    with monkeypatch.context() as m, torch.no_grad():
        _torch_ops(m)
        ld.sample(c, batch_size=2, timesteps=1)
        ld.sample([c, c], batch_size=2, timesteps=1)
        ld.sample({"c_crossattn": [c], "y": c}, batch_size=2, timesteps=1)
        ld.progressive_denoising(c, shape=(4, 8, 8), batch_size=2, start_T=1)
    assert torch.equal(seen[0], c[:2]) and [s.shape[0] for s in seen[1]] == [2, 2]
    assert seen[2]["c_crossattn"][0].shape[0] == 2 and seen[2]["y"].shape[0] == 2 and seen[3].shape[0] == 2


def test_sample_log_ddpm_branch_and_rejected_options(port, tab, monkeypatch):
    om, _ = port
    ld = _torch_ld(om, tab)
    calls = []
    monkeypatch.setattr(type(ld), "sample", lambda self, **kw: calls.append(kw) or ("s", "i"))
    assert ld.sample_log(cond="c", batch_size=2, ddim=False, ddim_steps=None, eta=1.0,
                         unconditional_guidance_scale=5.0) == ("s", "i")
    assert calls == [dict(cond="c", batch_size=2, return_intermediates=True, eta=1.0, unconditional_guidance_scale=5.0)]
    monkeypatch.undo()
    x, t = torch.zeros(1, 4, 8, 8), torch.zeros(1, dtype=torch.long)
    with pytest.raises(NotImplementedError, match="quantize"):
        ld.p_sample(x, None, t, quantize_denoised=True)
    with pytest.raises(NotImplementedError, match="score_corrector"):
        ld.p_sample(x, None, t, score_corrector=object())
    with pytest.raises(NotImplementedError, match="codebook"):
        ld.p_sample(x, None, t, return_codebook_ids=True)
    with pytest.raises(NotImplementedError, match="quantize"):
        ld.sample(None, batch_size=1, quantize_denoised=True)
    ld.num_timesteps_cond = 2
    with pytest.raises(NotImplementedError, match="num_timesteps_cond"):
        ld.sample(None, batch_size=1, x_T=x)
    with pytest.raises(NotImplementedError, match="num_timesteps_cond"):
        ld.progressive_denoising(None, shape=(4, 8, 8), batch_size=1, x_T=x)
    with pytest.raises(NotImplementedError, match="plot_denoise_rows"):
        ld.log_images({}, ddim_steps=4, plot_denoise_rows=True)
