"""GPU: masked (inpaint / outpaint) DDIM sampling, img2img (stochastic_encode + decode) and log_images(inpaint=True).

  * cb_q_sample_masked against the eager fp32 expression: every operation is a separately rounded fp32 op in the
    reference's order, so the kernel is held to BIT-EXACT equality (torch.equal), on the vectorised and scalar routes;
  * the mirror against tests/golden/ddim_masked_tiny.pt (UNMODIFIED reference, CPU) with the recorded draws replayed;
  * properties: an all-zero mask is plain sampling, and every call is bit-reproducible;
  * img2img at the txt2img size (UNet batch 16 under CFG, VAE encode at batch 8) against the fp32 port on the same GPU.
"""
import os

import numpy as np
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
    return torch.load(os.path.join(golden_dir, "ddim_masked_tiny.pt"), weights_only=False)


def rel(a, b):
    a, b = a.float().cpu().flatten(), b.float().cpu().flatten()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _eager_blend(x0, noise, t, sa, s1m, mask, img):
    a = sa[t].view(-1, 1, 1, 1)
    s = s1m[t].view(-1, 1, 1, 1)
    img_orig = a * x0 + s * noise
    return img_orig * mask + (1. - mask) * img


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 3, 16])
@pytest.mark.parametrize("hw", [8, 64])
@pytest.mark.parametrize("mkind", ["b1hw_binary", "11hw_soft", "bchw_soft", "b1hw_soft"])
@pytest.mark.parametrize("offset", [0, 1])
def test_q_sample_masked_kernel_bit_exact(dev, B, hw, mkind, offset):
    """offset 0: 16-byte aligned rows (float4 route); offset 1: every tensor starts one float in (scalar route)."""
    from celebbasis_b200 import ops
    from oracle import torch_ref
    g = torch.Generator().manual_seed(B * 1000 + hw + offset)
    sched = torch_ref.make_schedule()
    sa, s1m = sched["sqrt_alphas_cumprod"].to(dev), sched["sqrt_one_minus_alphas_cumprod"].to(dev)
    C = 4
    shape = (B, C, hw, hw)
    n = B * C * hw * hw

    def buf(x):                        # x copied into a larger buffer at `offset` (keeps the pointer misaligned)
        b = torch.empty(n + 8, device=dev)
        v = b[offset:offset + n].view(shape)
        v.copy_(x)
        return v
    x0 = buf(torch.randn(shape, generator=g))
    noise = buf(torch.randn(shape, generator=g))
    img = buf(torch.randn(shape, generator=g))
    t = torch.randint(0, 1000, (B,), generator=g).to(dev)                     # per-sample timesteps
    if mkind == "b1hw_binary":
        mask = (torch.rand(B, 1, hw, hw, generator=g) > 0.5).float()
    elif mkind == "b1hw_soft":
        mask = torch.rand(B, 1, hw, hw, generator=g)
    elif mkind == "11hw_soft":
        mask = torch.rand(1, 1, hw, hw, generator=g)
    else:
        mask = torch.rand(B, C, hw, hw, generator=g)
    mb = torch.empty(mask.numel() + 8, device=dev)
    mask = mb[offset:offset + mask.numel()].view(mask.shape).copy_(mask.to(dev))
    exp = _eager_blend(x0, noise, t, sa, s1m, mask, img)
    # fresh output inside a NaN-filled oversized buffer: nothing outside the output may be written
    big = torch.full((n + 64,), float("nan"), device=dev)
    out = big[16 + offset:16 + offset + n].view(shape)
    ops.q_sample_masked(x0, noise, t, sa, s1m, mask, img, out=out)
    torch.cuda.synchronize()
    assert torch.equal(out, exp)
    assert torch.isnan(big[:16 + offset]).all() and torch.isnan(big[16 + offset + n:]).all()
    # in place: out aliases img
    img2 = img.clone() if offset == 0 else buf(img)
    ops.q_sample_masked(x0, noise, t, sa, s1m, mask, img2, out=img2)
    assert torch.equal(img2, exp)


def test_q_sample_masked_rejects_bad_arguments(dev):
    from celebbasis_b200 import lib, ops
    import ctypes
    L = lib.load()
    x = torch.zeros(2, 4, 8, 8, device=dev)
    t = torch.zeros(2, dtype=torch.long, device=dev)
    p = lambda a: ctypes.c_void_p(a.data_ptr())  # noqa: E731
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    n0 = lib.launch_count()
    assert L.cb_q_sample_masked(p(x), p(x), p(t), p(x), p(x), None, 0, 0, p(x), p(x), 2, 4, 64, st) < 0
    assert L.cb_q_sample_masked(p(x), p(x), p(t), p(x), p(x), p(x), 0, 0, p(x), p(x), 0, 4, 64, st) < 0
    assert L.cb_q_sample_masked(p(x), p(x), p(t), p(x), p(x), p(x), -4, 0, p(x), p(x), 2, 4, 64, st) < 0
    assert lib.launch_count() == n0
    with pytest.raises(ValueError):
        ops.q_sample_masked(x, x, t, x.flatten(), x.flatten(), torch.ones(2, 1, 8, 8, device=dev).transpose(2, 3), x)


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
    return model, sd


@pytest.fixture(scope="module")
def tiny(dev):
    return _mirror("tiny", dev, 2)[0]


class _Replay:
    """torch.randn / torch.randn_like return the next recorded draw (shape-checked) on the requested device."""

    def __init__(self, draws):
        self.draws = list(draws)

    def _next(self, fn, shape, device):
        assert self.draws, f"extra draw {fn}{shape}"
        d = self.draws.pop(0)
        assert (d[0], d[2]) == (fn, tuple(shape)), (d[:3], fn, shape)
        return d[3].clone().to(device) if device is not None else d[3].clone()

    def install(self, m):
        def randn(*shape, device=None, **k):
            shp = tuple(shape[0]) if len(shape) == 1 and not isinstance(shape[0], int) else tuple(shape)
            return self._next("randn", shp, device)

        def randn_like(x, **k):
            return self._next("randn_like", x.shape, x.device)
        m.setattr(torch, "randn", randn)
        m.setattr(torch, "randn_like", randn_like)


def _stream(draws, eta):
    # the reference's three discarded test-mode draws of the embedding manager (embedding_manager.py:313-315), and its
    # noise_like draws at eta 0 (multiplied by sigma 0), are not drawn by the mirror
    return [d for d in draws if d[1] != "forward" and not (d[1] == "noise_like" and eta == 0)]


def _cond(model, gold, golden_dir):
    ref = torch.load(os.path.join(golden_dir, "infer_tiny.pt"))
    B = gold["x0"].shape[0]
    io = {"faces": None, "ids": [[p, p] for p in gold["person_ids"]], "num_ids": torch.ones(B, dtype=torch.long)}
    uc = model.get_learned_conditioning([""] * B)
    c = model.get_learned_conditioning(gold["prompts"], image_ori=io)
    # the fixture's conditioning is infer_tiny.pt's (same prompt / identity), rows repeated
    assert rel(uc, ref["uc"].expand_as(uc)) < 2e-3 and rel(c, ref["c"].expand_as(c)) < 2e-3
    return c, uc


def test_masked_sampling_vs_reference_golden(dev, tiny, gold, golden_dir, monkeypatch):
    from ldm.models.diffusion.ddim import DDIMSampler
    B, _, hw, _ = gold["x0"].shape
    with torch.no_grad():
        c, uc = _cond(tiny, gold, golden_dir)
        for case in gold["sample"]:
            rep = _Replay(_stream(case["draws"], case["eta"]))
            with monkeypatch.context() as m:
                rep.install(m)
                x, _ = DDIMSampler(tiny).sample(S=gold["steps"], conditioning=c, batch_size=B, shape=[4, hw, hw],
                                                verbose=False, unconditional_guidance_scale=gold["scale"],
                                                unconditional_conditioning=uc, eta=case["eta"],
                                                x_T=gold["x_T"].to(dev), mask=gold["masks"][case["mask"]].to(dev),
                                                x0=gold["x0"].to(dev))
            assert not rep.draws
            assert rel(x, case["samples"]) < 3e-3, (case["mask"], case["eta"], rel(x, case["samples"]))


def test_img2img_vs_reference_golden(dev, tiny, gold, golden_dir, monkeypatch):
    from ldm.models.diffusion.ddim import DDIMSampler
    i2i = gold["img2img"]
    B, _, hw, _ = gold["x0"].shape
    init = (torch.rand(B, 3, 8 * hw, 8 * hw, generator=torch.Generator().manual_seed(i2i["init_seed"])) * 2 - 1).to(dev)
    with torch.no_grad():
        c, uc = _cond(tiny, gold, golden_dir)
        for case in i2i["cases"]:
            rep = _Replay(_stream(case["draws"], case["eta"]))
            with monkeypatch.context() as m:
                rep.install(m)
                z0 = tiny.get_first_stage_encoding(tiny.encode_first_stage(init))
                sampler = DDIMSampler(tiny)
                sampler.make_schedule(ddim_num_steps=i2i["S"], ddim_eta=case["eta"], verbose=False)
                z_enc = sampler.stochastic_encode(z0, torch.tensor([i2i["t_enc"]] * B, device=dev))
                lat = sampler.decode(z_enc, c, i2i["t_enc"], unconditional_guidance_scale=gold["scale"],
                                     unconditional_conditioning=uc)
            assert not rep.draws
            assert rel(z0, case["z0"]) < 2e-3 and rel(z_enc, case["z_enc"]) < 2e-3, (rel(z0, case["z0"]),
                                                                                      rel(z_enc, case["z_enc"]))
            assert rel(lat, case["latents"]) < 3e-3, (case["eta"], rel(lat, case["latents"]))
            if case["img"] is not None:
                img = tiny.decode_first_stage(lat)
                assert rel(img, case["img"]) < 4e-3, rel(img, case["img"])


def test_log_images_inpaint_vs_reference_golden(dev, tiny, gold, monkeypatch):
    from celebbasis_b200 import workload
    li = gold["log_images"]
    batch, _ = workload.synth_batch("tiny", B=li["N"], seed=li["batch_seed"])
    batch = {"image": batch["image"].to(dev), "caption": batch["caption"],
             "image_ori": {"faces": None, "ids": batch["image_ori"]["ids"], "num_ids": batch["image_ori"]["num_ids"]}}
    rep = _Replay(_stream(li["draws"], li["ddim_eta"]))
    with monkeypatch.context() as m, torch.no_grad():
        rep.install(m)
        log = tiny.log_images(batch, N=li["N"], inpaint=True, ddim_steps=li["ddim_steps"])
    assert not rep.draws
    for k in ("samples_inpainting", "mask", "samples_outpainting"):
        assert k in log
    assert torch.equal(log["mask"].cpu(), li["panels"]["mask"])
    for k, v in li["panels"].items():
        if k != "mask":
            assert rel(log[k], v) < 4e-3, (k, rel(log[k], v))


# ---------------------------------------------------------------------------------------------------------------------
def test_zero_mask_is_plain_sampling_and_calls_repeat(dev, tiny, gold, golden_dir):
    from ldm.models.diffusion.ddim import DDIMSampler
    B, _, hw, _ = gold["x0"].shape
    x_T, x0 = gold["x_T"].to(dev), gold["x0"].to(dev)
    kw = dict(S=gold["steps"], batch_size=B, shape=[4, hw, hw], verbose=False, unconditional_guidance_scale=gold["scale"])
    with torch.no_grad():
        c, uc = _cond(tiny, gold, golden_dir)
        plain, _ = DDIMSampler(tiny).sample(conditioning=c, unconditional_conditioning=uc, eta=0.0, x_T=x_T, **kw)
        zero, _ = DDIMSampler(tiny).sample(conditioning=c, unconditional_conditioning=uc, eta=0.0, x_T=x_T,
                                           mask=torch.zeros(B, 1, hw, hw, device=dev), x0=x0, **kw)
        assert torch.equal(plain, zero)

        def masked(eta):
            torch.manual_seed(11)
            return DDIMSampler(tiny).sample(conditioning=c, unconditional_conditioning=uc, eta=eta, x_T=x_T,
                                            mask=gold["masks"]["soft"].to(dev), x0=x0, **kw)[0]

        def img2img():
            torch.manual_seed(12)
            s = DDIMSampler(tiny)
            s.make_schedule(8, ddim_eta=1.0, verbose=False)
            z = s.stochastic_encode(x0, torch.full((B,), 6, device=dev, dtype=torch.long))
            return s.decode(z, c, 6, unconditional_guidance_scale=5.0, unconditional_conditioning=uc)
        for fn in (lambda: masked(0.0), lambda: masked(1.0), img2img):
            a, b = fn(), fn()
            assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------------
def test_img2img_txt2img_size_vs_port(dev, monkeypatch):
    """n_samples 8 => UNet batch 16 under CFG 10; 512x512 seeded init images VAE-encoded at batch 8 with supplied
    posterior eps; S = 8, t_enc = 4; decode of two of the images; against the fp32 port on the same GPU."""
    from celebbasis_b200 import synth, workload
    from celebbasis_b200.tokenizer import SyntheticCLIPTokenizer
    from ldm.models.diffusion.ddim import DDIMSampler
    from oracle import ddim_ref, torch_ref
    model, sd = _mirror("full", dev, 12)
    g = torch.Generator().manual_seed(3)
    coefs = [F.normalize(torch.randn(2, 1, 512, generator=g), dim=-1) for _ in range(10)]
    n, S, t_enc, scale = 8, 8, 4, 10.0
    prompts = ["a photo of sks person"] * n
    image_ori = {"faces": None, "ids": [[3, 3]] * n, "num_ids": torch.ones(n, dtype=torch.long)}
    gi = torch.Generator().manual_seed(21)
    init = (torch.rand(n, 3, 512, 512, generator=gi) * 2 - 1).to(dev)
    eps = torch.randn(n, 4, 64, 64, generator=gi).to(dev)
    noise = torch.randn(n, 4, 64, 64, generator=gi).to(dev)
    with torch.no_grad():
        uc = model.get_learned_conditioning([""] * n)
        c = model.get_learned_conditioning(prompts, image_ori=image_ori)
        post = model.encode_first_stage(init)
        with monkeypatch.context() as m:
            m.setattr(torch, "randn", lambda *a, **k: eps.clone())
            z0 = model.get_first_stage_encoding(post)
        sampler = DDIMSampler(model)
        sampler.make_schedule(ddim_num_steps=S, ddim_eta=0.0, verbose=False)
        tt = torch.full((n,), t_enc, device=dev, dtype=torch.long)
        z_enc = sampler.stochastic_encode(z0, tt, noise=noise)
        lat = sampler.decode(z_enc, c, t_enc, unconditional_guidance_scale=scale, unconditional_conditioning=uc)
        img = model.decode_first_stage(lat[:2].contiguous())
    del model, post
    torch.cuda.empty_cache()
    om = torch_ref.OracleModel(workload.model_params("full"), clip_layers=12)
    om.load_state_dict({k: v for k, v in sd.items() if k in om.state_dict()})
    om = om.to(dev).eval()
    tm = om.cond_stage_model.transformer.text_model
    tok = SyntheticCLIPTokenizer()
    with torch.no_grad():
        uc_r = tm.forward_embeds(tm.embed_tokens(tok([""] * n)["input_ids"].to(dev)))
        ids = tok(prompts)["input_ids"]
        zc = torch_ref.celeb_basis(coefs[3].view(1, 2, 1, 512).to(dev).repeat(n, 1, 1, 1), synth.synth_celeb_basis(seed=0).to(dev))
        emb, _ = torch_ref.inject_embeddings(ids, tm.embed_tokens(ids.to(dev)), zc, tok.word_id("sks"), 2)
        c_r = tm.forward_embeds(emb)
        z0_r = torch_ref.posterior_sample(om.first_stage_model(init), eps, om.scale_factor)
        z_enc_r = ddim_ref.ddim_stochastic_encode(om.sched, S, z0_r, tt, noise)
        lat_r = ddim_ref.ddim_decode(om.model.diffusion_model, om.sched, S, 0.0, z_enc_r, c_r, t_enc, scale=scale,
                                     uncond=uc_r)
        fs = workload.model_params("full")["first_stage_config"]["params"]
        dec = torch_ref.AutoencoderKLDecode(fs["ddconfig"], fs["embed_dim"])
        dec.load_state_dict({k[len("first_stage_model."):]: v for k, v in sd.items()
                             if k.startswith("first_stage_model.") and k[len("first_stage_model."):] in dec.state_dict()})
        img_r = dec.to(dev)((1. / om.scale_factor) * lat_r[:2])
    assert rel(c, c_r) < 2e-3 and rel(uc, uc_r) < 2e-3
    assert rel(z0, z0_r) < 2e-3, rel(z0, z0_r)                   # the training step's z bar
    assert rel(lat, lat_r) < 3e-3, rel(lat, lat_r)
    assert img.shape == img_r.shape == (2, 3, 512, 512) and rel(img, img_r) < 5e-3, rel(img, img_r)
