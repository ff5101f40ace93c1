"""GPU: DDPM ancestral sampling (LatentDiffusion.p_sample / p_sample_loop / progressive_denoising / sample) and the
log_images panels it feeds (diffusion, denoise and progressive rows).

  * cb_p_sample against the eager fp32 expression: every operation is a separately rounded fp32 op in the reference's
    order, so the kernel is held to BIT-EXACT equality (torch.equal), on the vectorised and scalar routes;
  * the mirror against tests/golden/ddpm_sample_tiny.pt (UNMODIFIED reference, CPU) with the recorded draws replayed;
  * the sampler arithmetic in isolation at the SD-v1 size: the mirror's own eps and noise fed to the fp32 port on the
    same GPU give the bit-identical trajectory;
  * properties: an all-zero mask is plain sampling, every call is bit-reproducible, and a Textual-Inversion model logs
    every DDPM panel.
"""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from celebbasis_b200 import lib
    assert lib.load().cb_device_ok() == 1
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "ddpm_sample_tiny.pt"), weights_only=False)


def rel(a, b):
    a, b = a.float().cpu().flatten(), b.float().cpu().flatten()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


_TABLES = ("sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod", "posterior_mean_coef1", "posterior_mean_coef2",
           "posterior_log_variance_clipped")


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 3, 16])
@pytest.mark.parametrize("hw", [8, 64])
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("temperature", [1.0, 0.7])
def test_p_sample_kernel_bit_exact(dev, B, hw, offset, clip, temperature):
    """offset 0: 16-byte aligned rows (float4 route); offset 1: every tensor starts one float in (scalar route)."""
    from celebbasis_b200 import ops
    from oracle import ddpm_ref
    g = torch.Generator().manual_seed(B * 1000 + hw * 10 + offset + 2 * clip)
    tab = {k: v.to(dev) for k, v in ddpm_ref.ddpm_tables().items()}
    shape = (B, 4, hw, hw)
    n = B * 4 * hw * hw

    def buf(x):                        # x copied into a larger buffer at `offset` (keeps the pointer misaligned)
        b = torch.empty(n + 8, device=dev)
        return b[offset:offset + n].view(shape).copy_(x)
    x = buf(torch.randn(shape, generator=g) * 3)          # x_recon leaves [-1, 1], so the clamp acts
    eps = buf(torch.randn(shape, generator=g))
    noise = buf(torch.randn(shape, generator=g))
    t = torch.randint(0, 1000, (B,), generator=g)
    t[0] = 0
    if B > 1:
        t[-1] = 999
    t = t.to(dev)
    exp_x, exp_x0 = ddpm_ref.posterior_step(tab, x, eps, t, noise, temperature=temperature, clip=clip)
    # fresh outputs inside NaN-filled oversized buffers: nothing outside the outputs may be written
    big = torch.full((n + 64,), float("nan"), device=dev)
    big0 = torch.full((n + 64,), float("nan"), device=dev)
    out = big[16 + offset:16 + offset + n].view(shape)
    out0 = big0[16 + offset:16 + offset + n].view(shape)
    _launch(ops, x, eps, noise, t, tab, temperature, clip, out, out0)
    torch.cuda.synchronize()
    assert torch.equal(out, exp_x) and torch.equal(out0, exp_x0)
    for bb in (big, big0):
        assert torch.isnan(bb[:16 + offset]).all() and torch.isnan(bb[16 + offset + n:]).all()
    if clip:
        assert exp_x0.abs().max().item() <= 1.0
    # in place: x_prev aliases x, no x0
    x2 = buf(x)
    y, none = ops.p_sample(x2, eps, noise, t, *[tab[k] for k in _TABLES], temperature=temperature, clip_denoised=clip,
                           out=x2, want_x0=False)
    assert none is None and y.data_ptr() == x2.data_ptr() and torch.equal(x2, exp_x)


def _launch(ops, x, eps, noise, t, tab, temperature, clip, out, out0):
    """ops.p_sample with an explicit x0 buffer (the wrapper allocates its own), through the raw entry point."""
    from celebbasis_b200 import lib
    import ctypes
    p = lambda a: ctypes.c_void_p(a.data_ptr())  # noqa: E731
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = lib.load().cb_p_sample(p(x), p(eps), p(noise), p(t), *[p(tab[k]) for k in _TABLES], float(temperature),
                                int(clip), p(out), p(out0), x.shape[0], x.numel() // x.shape[0], st)
    assert rc == 0


def test_p_sample_rejects_bad_arguments(dev):
    from celebbasis_b200 import lib
    import ctypes
    L = lib.load()
    x = torch.zeros(2, 4, 8, 8, device=dev)
    tb = torch.zeros(1000, device=dev)
    t = torch.zeros(2, dtype=torch.long, device=dev)
    p = lambda a: ctypes.c_void_p(a.data_ptr()) if a is not None else None  # noqa: E731
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(x_=x, eps=x, noise=x, t_=t, tabs=(tb,) * 5, out=x, B=2, n=256):
        return L.cb_p_sample(p(x_), p(eps), p(noise), p(t_), *[p(a) for a in tabs], 1.0, 0, p(out), None, B, n, st)
    n0 = lib.launch_count()
    assert call(x_=None) < 0 and call(eps=None) < 0 and call(noise=None) < 0 and call(t_=None) < 0
    assert call(tabs=(tb, tb, None, tb, tb)) < 0 and call(tabs=(tb, tb, tb, tb, None)) < 0 and call(out=None) < 0
    assert call(B=0) < 0 and call(n=0) < 0 and call(B=-1) < 0 and call(n=-256) < 0
    torch.cuda.synchronize()
    assert lib.launch_count() == n0
    assert call() == 0 and lib.launch_count() == n0 + 1


# ---------------------------------------------------------------------------------------------------------------------
def _mirror(kind, dev, layers):
    from celebbasis_b200 import synth, workload
    from ldm.models.diffusion.ddpm import LatentDiffusion
    params = workload.model_params(kind)
    params["cond_stage_config"]["params"].update(num_hidden_layers=layers, device="cuda")
    model = LatentDiffusion(**params)
    sd = synth.synth_state_dict(model, seed=0)
    model.load_state_dict(sd, strict=False)
    model = model.to(dev).eval()
    model.cond_stage_model.celeb_embeddings = synth.synth_celeb_basis(seed=0).to(dev)
    g = torch.Generator().manual_seed(3)
    model.embedding_manager.id_coefficients = [F.normalize(torch.randn(2, 1, 512, generator=g), dim=-1)
                                               for _ in range(10)]
    return model


@pytest.fixture(scope="module")
def tiny(dev):
    return _mirror("tiny", dev, 2)


_MIRROR_SITE = {"_masked_blend": "q_sample"}     # where the mirror draws q_sample's noise before its fused blend


class _Replay:
    """torch.randn / torch.randn_like / F.dropout return the next recorded draw on the requested device (dropout: the
    input times the recorded multiplier); (function, call site, shape) must match the record."""

    def __init__(self, draws):
        self.draws = list(draws)

    def _next(self, fn, shape, device):
        site = sys._getframe(2).f_code.co_name
        site = _MIRROR_SITE.get(site, site)
        assert self.draws, f"extra draw {fn}{shape} at {site}"
        d = self.draws.pop(0)
        assert (d[0], d[1], tuple(d[2])) == (fn, site, tuple(shape)), (d[:3], fn, site, shape)
        return d[3].clone().to(device) if device is not None else d[3].clone()

    def install(self, m):
        o_dropout = torch.nn.functional.dropout

        def randn(*shape, device=None, **k):
            shp = tuple(shape[0]) if len(shape) == 1 and not isinstance(shape[0], int) else tuple(shape)
            return self._next("randn", shp, device)

        def randn_like(x, **k):
            return self._next("randn_like", x.shape, x.device)

        def dropout(x, p=0.5, training=True, inplace=False):
            if not training or p == 0.:
                return o_dropout(x, p=p, training=training, inplace=inplace)
            return x * self._next("dropout", x.shape, x.device)
        m.setattr(torch, "randn", randn)
        m.setattr(torch, "randn_like", randn_like)
        m.setattr(torch.nn.functional, "dropout", dropout)


def _draws(rec):
    from oracle import ddpm_ref
    vals = ddpm_ref.regenerate_draws(rec["seed"], rec["calls"], rec["p_dropout"])
    # the reference's embedding manager draws three discarded vectors per encode in eval mode
    # (embedding_manager.py:313-315); the mirror does not
    return [c[:3] + (v,) for c, v in zip(rec["calls"], vals) if c[1] != "forward"]


def _cond(model, gold, golden_dir):
    ref = torch.load(os.path.join(golden_dir, "infer_tiny.pt"))
    B = len(gold["prompts"])
    io = {"faces": None, "ids": [[p, p] for p in gold["person_ids"]], "num_ids": torch.ones(B, dtype=torch.long)}
    c = model.get_learned_conditioning(gold["prompts"], image_ori=io)
    assert rel(c, ref["c"].expand_as(c)) < 2e-3
    return c


# Measured on an H100 80GB HBM3 at a 700 W power limit, relative L2 error against the fixture (worst over the final
# latent and every kept intermediate):
#   (a) sample, 1000 fp16 UNet steps           4.1e-4
#   (b) masked p_sample_loop, 50 steps           1.6e-4 (binary mask), 3.8e-5 (soft mask)
#   (c) progressive_denoising, 60 steps          2.1e-4
#   (d) log_images, the 22 decoded latents       7.4e-4 (the progressive row's x0 predictions); the panels 1.8e-3
# One latent bar serves every case: the 1000-step run measured no worse than 4.1e-4, so it needs nothing looser than
# the short runs.  The panels add the fp16 VAE decode (the masked-DDIM fixture's image bar is 4e-3).
BAR_LATENT, BAR_PANEL = 2e-3, 5e-3


def _report(name, errs):
    print(f"[ddpm-golden] {name}: " + " ".join(f"{e:.2e}" for e in errs))


def test_sample_vs_reference_golden(dev, tiny, gold, golden_dir, monkeypatch):
    a = gold["sample"]
    rep = _Replay(_draws(a["draws"]))
    with torch.no_grad():
        c = _cond(tiny, gold, golden_dir)
        with monkeypatch.context() as m:
            rep.install(m)
            x, inter = tiny.sample(c, batch_size=2, return_intermediates=True)
    assert not rep.draws and len(inter) == a["intermediates"].shape[0]
    errs = [rel(x, a["samples"])] + [rel(p, r) for p, r in zip(inter, a["intermediates"])]
    _report("sample", errs)
    assert max(errs) < BAR_LATENT, errs


def test_masked_loop_vs_reference_golden(dev, tiny, gold, golden_dir, monkeypatch):
    with torch.no_grad():
        c = _cond(tiny, gold, golden_dir)
        for case in gold["masked"]:
            rep = _Replay(_draws(case["draws"]))
            with monkeypatch.context() as m:
                rep.install(m)
                x, inter = tiny.p_sample_loop(c, tuple(gold["x_T"].shape), return_intermediates=True,
                                              x_T=gold["x_T"].to(dev), mask=gold["masks"][case["mask"]].to(dev),
                                              x0=gold["x0"].to(dev), start_T=case["start_T"],
                                              log_every_t=case["log_every_t"])
            assert not rep.draws and len(inter) == case["intermediates"].shape[0]
            errs = [rel(x, case["samples"])] + [rel(p, r) for p, r in zip(inter, case["intermediates"])]
            _report(f"masked {case['mask']}", errs)
            assert max(errs) < BAR_LATENT, (case["mask"], errs)


def test_progressive_vs_reference_golden(dev, tiny, gold, golden_dir, monkeypatch):
    pc = gold["progressive"]
    rep = _Replay(_draws(pc["draws"]))
    with torch.no_grad():
        c = _cond(tiny, gold, golden_dir)
        with monkeypatch.context() as m:
            rep.install(m)
            x, inter = tiny.progressive_denoising(c, shape=(4, 8, 8), batch_size=2, start_T=pc["start_T"],
                                                  temperature=pc["temperature"], noise_dropout=pc["noise_dropout"],
                                                  log_every_t=pc["log_every_t"])
    assert not rep.draws and len(inter) == pc["intermediates"].shape[0]
    errs = [rel(x, pc["samples"])] + [rel(p, r) for p, r in zip(inter, pc["intermediates"])]
    _report("progressive", errs)
    assert max(errs) < BAR_LATENT, errs


def test_log_images_ddpm_rows_vs_reference_golden(dev, tiny, gold, monkeypatch):
    from celebbasis_b200 import workload
    li = gold["log_images"]
    batch, _ = workload.synth_batch("tiny", B=li["N"], seed=li["batch_seed"])
    batch = {"image": batch["image"].to(dev), "caption": batch["caption"],
             "image_ori": {"faces": None, "ids": batch["image_ori"]["ids"], "num_ids": batch["image_ori"]["num_ids"]}}
    rep = _Replay(_draws(li["draws"]))
    decoded = []
    orig = tiny.decode_first_stage
    with monkeypatch.context() as m, torch.no_grad():
        rep.install(m)
        m.setattr(tiny, "decode_first_stage", lambda z, *a, **k: (decoded.append(z.clone()), orig(z, *a, **k))[1])
        log = tiny.log_images(batch, N=li["N"], n_row=li["n_row"], ddim_steps=None, plot_diffusion_rows=True,
                              plot_progressive_rows=True, plot_denoise_rows=True)
    assert not rep.draws
    assert list(log.keys()) == li["keys"]
    assert {k: tuple(v.shape) for k, v in log.items()} == li["shapes"]
    assert all(torch.isfinite(v).all() for v in log.values())
    assert len(decoded) == li["decoded"].shape[0]
    lat = [rel(p, r) for p, r in zip(decoded, li["decoded"])]
    pan = [rel(log[k][:, :v.shape[1]], v.float()) for k, v in li["panels_fp16"].items()]   # rows: the first grid row
    _report("log_images latents", lat)
    _report("log_images panels", pan)
    assert max(lat) < BAR_LATENT and max(pan) < BAR_PANEL, (lat, pan)


# ---------------------------------------------------------------------------------------------------------------------
def test_zero_mask_is_plain_sampling_and_calls_repeat(dev, tiny, gold, golden_dir, monkeypatch):
    x_T, x0 = gold["x_T"].to(dev), gold["x0"].to(dev)
    shape = tuple(x_T.shape)
    with torch.no_grad():
        c = _cond(tiny, gold, golden_dir)

        def run(**kw):
            torch.manual_seed(5)
            return tiny.p_sample_loop(c, shape, x_T=x_T, start_T=20, **kw)
        # the masked loop also draws q_sample's noise (randn_like) every step: noise_like's randn draws come from a
        # generator of their own, so both runs see the same step noise
        o_randn = torch.randn
        with monkeypatch.context() as m:
            gen = torch.Generator(device=dev)
            m.setattr(torch, "randn", lambda *a, **k: o_randn(*a, generator=gen, **k))
            gen.manual_seed(4)
            plain = run()
            gen.manual_seed(4)
            zero = run(mask=torch.zeros(shape[0], 1, shape[2], shape[3], device=dev), x0=x0)
        assert torch.equal(plain, zero)

        def prog():
            torch.manual_seed(6)
            return tiny.progressive_denoising(c, shape=shape[1:], batch_size=shape[0], start_T=20,
                                              temperature=[0.8] * 20, noise_dropout=0.2)[0]
        for fn in (run, lambda: run(mask=gold["masks"]["soft"].to(dev), x0=x0), prog,
                   lambda: (torch.manual_seed(7), tiny.sample(c, batch_size=2, timesteps=20))[1]):
            a, b = fn(), fn()
            assert torch.equal(a, b)


def test_sampler_arithmetic_at_sd_size_vs_port(dev, monkeypatch):
    """Full SD-v1 model, batch 8, 64x64 latent, the first 60 timesteps from a given x_T: the mirror's own per-step eps
    and noise_like draws, fed to the fp32 port's posterior step on the same GPU, give the same trajectory bit for
    bit (the kernel is the eager expression, rounded op by op)."""
    from oracle import ddpm_ref
    model = _mirror("full", dev, 12)
    n, T = 8, 60
    g = torch.Generator().manual_seed(31)
    x_T = torch.randn(n, 4, 64, 64, generator=g).to(dev)
    eps_seen, traj = [], []
    orig = model.apply_model
    with torch.no_grad():
        c = model.get_learned_conditioning(["a photo of sks person"] * n,
                                           image_ori={"faces": None, "ids": [[3, 3]] * n,
                                                      "num_ids": torch.ones(n, dtype=torch.long)})
        with monkeypatch.context() as m:
            m.setattr(model, "apply_model", lambda x, t, cc: (lambda e: (eps_seen.append(e.clone()), e)[1])(orig(x, t, cc)))
            noise_seen = []
            o_randn = torch.randn

            def randn(*a, **k):
                r = o_randn(*a, **k)
                noise_seen.append(r.clone())
                return r
            m.setattr(torch, "randn", randn)
            torch.manual_seed(8)
            x = model.p_sample_loop(c, (n, 4, 64, 64), x_T=x_T, start_T=T, img_callback=lambda im, i: traj.append(im.clone()))
    assert len(eps_seen) == len(noise_seen) == len(traj) == T
    tab = {k: getattr(model, k) for k in _TABLES}
    ref_tab = ddpm_ref.ddpm_tables()
    assert all(torch.equal(tab[k].cpu(), ref_tab[k]) for k in _TABLES)
    y = x_T
    for k, i in enumerate(reversed(range(T))):
        t = torch.full((n,), i, device=dev, dtype=torch.long)
        y, _ = ddpm_ref.posterior_step(tab, y, eps_seen[k], t, noise_seen[k])
        assert torch.equal(y, traj[k]), (i, rel(y, traj[k]))
    assert torch.equal(y, x) and torch.isfinite(x).all()


def test_textual_inversion_model_logs_ddpm_panels(dev):
    """A v1-finetune (Textual Inversion) model: log_images with ddim_steps=None and every row, and sample()."""
    from celebbasis_b200 import synth, workload
    from ldm.models.diffusion.ddpm import LatentDiffusion
    params = workload.ti_model_params("tiny")
    params["cond_stage_config"]["params"].update(num_hidden_layers=2, device="cuda")
    model = LatentDiffusion(**params)
    model.load_state_dict(synth.synth_state_dict(model, seed=0), strict=False)
    model = model.to(dev).eval()
    g = torch.Generator().manual_seed(9)
    batch = {"image": (torch.rand(2, 64, 64, 3, generator=g) * 2 - 1).to(dev),
             "caption": ["a photo of *", "a rendition of a *"]}
    torch.manual_seed(10)
    with torch.no_grad():
        log = model.log_images(batch, N=2, n_row=2, ddim_steps=None, plot_diffusion_rows=True,
                               plot_progressive_rows=True, plot_denoise_rows=True)
        c = model.get_learned_conditioning(batch["caption"])
        s = model.sample(c, batch_size=2)
    every, T = model.log_every_t, model.num_timesteps
    nd = len([t for t in range(T) if t % every == 0 or t == T - 1])
    assert log["diffusion_row"].shape == (3, 2 * 66 + 2, nd * 66 + 2)
    assert log["denoise_row"].shape == (3, 2 * 66 + 2, (nd + 1) * 66 + 2)
    assert log["progressive_row"].shape == log["diffusion_row"].shape
    assert log["samples"].shape == log["samples_scaled"].shape == (2, 3, 64, 64)
    assert s.shape == (2, 4, 8, 8)
    assert all(torch.isfinite(v).all() for v in log.values()) and torch.isfinite(s).all()
