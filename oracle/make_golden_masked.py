"""Generate tests/golden/ddim_masked_tiny.pt by running the UNMODIFIED reference (through oracle/ref_shim.py) on CPU, in
the tiny configuration of `python oracle/make_golden.py infer`:

    python oracle/make_golden_masked.py

  (a) DDIMSampler.sample with classifier-free guidance, `mask` and `x0` (ddim.py:57-163, the blend of :144-147), at eta 0
      and 1, with a binary non-rectangular (B,1,h,w) mask and a soft (1,1,h,w) mask;
  (b) img2img: encode_first_stage + get_first_stage_encoding of a seeded image, make_schedule + stochastic_encode at
      t_enc = int(0.75 * S) + decode with CFG (ddim.py:207-241), decode_first_stage, at eta 0 and 1;
  (c) LatentDiffusion.log_images(batch, N=2, inpaint=True, ddim_steps=4) (ddpm.py:1320-1440) panels.

Every torch.randn / torch.randn_like call the reference makes (x_T, q_sample's noise, noise_like, the posterior sample)
is recorded in order with its shape, so the port and the mirror can replay the same stream.
"""
import contextlib
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np
import torch
import torch.nn.functional as F

from celebbasis_b200 import synth, workload
from oracle import ref_shim

GOLD = os.path.join(ROOT, "tests", "golden")


@contextlib.contextmanager
def record_draws(draws):
    """Wrap torch.randn / torch.randn_like: each draw runs unchanged and is appended to `draws` as (function, calling
    function's name, shape, tensor); the call site tells noise_like (ddim.py:200) from q_sample (ddpm.py:290),
    stochastic_encode (ddim.py:218), the posterior sample (distributions.py:36), x_T (ddim.py:123) and the three
    discarded test-mode draws of the embedding manager (embedding_manager.py:313-315)."""
    o_randn, o_randn_like = torch.randn, torch.randn_like

    def site():
        f = sys._getframe(2)
        while f.f_code.co_name in ("<lambda>", "default"):     # noise_like's / q_sample's default-noise lambdas
            f = f.f_back
        return f.f_code.co_name

    def randn(*a, **k):
        out = o_randn(*a, **k)
        draws.append(("randn", site(), tuple(out.shape), out.detach().clone()))
        return out

    def randn_like(x, *a, **k):
        out = o_randn_like(x, *a, **k)
        draws.append(("randn_like", site(), tuple(out.shape), out.detach().clone()))
        return out
    torch.randn, torch.randn_like = randn, randn_like
    try:
        yield draws
    finally:
        torch.randn, torch.randn_like = o_randn, o_randn_like


def masks(B, hw):
    """A binary non-rectangular (B,1,h,w) mask (a disc and its complement-shifted twin; 1 = keep x0) and a soft
    (1,1,h,w) ramp with values strictly inside (0, 1)."""
    yy, xx = torch.meshgrid(torch.arange(hw, dtype=torch.float32), torch.arange(hw, dtype=torch.float32), indexing="ij")
    c = (hw - 1) / 2
    disc = ((yy - c) ** 2 + (xx - c) ** 2 <= (hw / 3) ** 2)
    tri = (xx + yy) < hw                                        # lower-left triangle
    binary = torch.stack([(~disc).float(), tri.float()] + [(~disc).float()] * (B - 2), 0)[:B, None]
    soft = torch.sigmoid((xx - c) / 1.5 + 0.5 * (yy - c) / 1.5)[None, None]
    return binary.contiguous(), soft.contiguous()


def run_masked(kind="tiny", steps=4, scale=5.0):
    torch.manual_seed(0)
    basis = synth.synth_celeb_basis(seed=0)
    model = ref_shim.build_reference(workload.model_params(kind), seed=0, clip_layers=workload.clip_layers(kind),
                                     celeb_basis=basis)
    model.eval()
    from ldm.models.diffusion.ddim import DDIMSampler

    def register_buffer(self, name, attr):            # ddim.py:19-23 hard-codes .to("cuda"); same values on the CPU
        setattr(self, name, attr)
    DDIMSampler.register_buffer = register_buffer
    g = torch.Generator().manual_seed(3)
    coefs = [F.normalize(torch.randn(2, 1, 512, generator=g), dim=-1) for _ in range(10)]
    model.embedding_manager.id_coefficients = [c.clone() for c in coefs]
    hw = workload.model_params(kind)["image_size"]
    B = 2
    pids = [3, 3]          # the prompt and identity of infer_tiny.pt, whose c / uc rows pin this conditioning
    prompts = ["a photo of sks person"] * B
    image_ori = {"faces": None, "ids": torch.tensor([[p, p] for p in pids]), "num_ids": torch.ones(B, dtype=torch.long)}
    out = {"kind": kind, "steps": steps, "scale": scale, "coef_seed": 3, "prompts": prompts, "person_ids": pids}
    with torch.no_grad():
        uc = model.get_learned_conditioning([""] * B)
        c = model.get_learned_conditioning(prompts, image_ori=image_ori)
        x0 = torch.randn(B, 4, hw, hw, generator=g)
        x_T = torch.randn(B, 4, hw, hw, generator=g)
        ref = torch.load(os.path.join(GOLD, f"infer_{kind}.pt"))
        assert torch.equal(c, ref["c"].expand_as(c)) and torch.equal(uc, ref["uc"].expand_as(uc))
        out.update(x0=x0.clone(), x_T=x_T.clone())
        binary, soft = masks(B, hw)
        out["masks"] = {"binary": binary, "soft": soft}
        # (a) masked sampling
        out["sample"] = []
        for mname, mask in (("binary", binary), ("soft", soft)):
            for eta in (0.0, 1.0):
                torch.manual_seed(100 + len(out["sample"]))
                with record_draws([]) as draws:
                    samples, _ = DDIMSampler(model).sample(S=steps, conditioning=c, batch_size=B, shape=[4, hw, hw],
                                                           verbose=False, unconditional_guidance_scale=scale,
                                                           unconditional_conditioning=uc, eta=eta, x_T=x_T.clone(),
                                                           mask=mask, x0=x0)
                out["sample"].append({"mask": mname, "eta": eta, "samples": samples.clone(), "draws": draws})
                print(f"[masked] {mname} eta={eta}: |x|={samples.norm().item():.6f} draws={[d[1:3] for d in draws]}")
        # (b) img2img: scripts/img2img.py-style encode -> stochastic_encode -> decode -> decode_first_stage
        S = 8
        t_enc = int(0.75 * S)
        init = torch.rand(B, 3, 8 * hw, 8 * hw, generator=torch.Generator().manual_seed(4)) * 2 - 1
        out["img2img"] = {"S": S, "t_enc": t_enc, "init_seed": 4, "cases": []}
        for eta in (0.0, 1.0):
            torch.manual_seed(200 + len(out["img2img"]["cases"]))
            with record_draws([]) as draws:
                z0 = model.get_first_stage_encoding(model.encode_first_stage(init))
                sampler = DDIMSampler(model)
                sampler.make_schedule(ddim_num_steps=S, ddim_eta=eta, verbose=False)
                z_enc = sampler.stochastic_encode(z0, torch.tensor([t_enc] * B))
                lat = sampler.decode(z_enc, c, t_enc, unconditional_guidance_scale=scale, unconditional_conditioning=uc)
            img = model.decode_first_stage(lat)
            out["img2img"]["cases"].append({"eta": eta, "z0": z0.clone(), "z_enc": z_enc.clone(), "latents": lat.clone(),
                                            "img": img.clone() if eta == 0 else None, "draws": draws,
                                            "ddim_timesteps": torch.as_tensor(np.asarray(sampler.ddim_timesteps).copy())})
            print(f"[img2img] eta={eta}: |z_enc|={z_enc.norm().item():.6f} |lat|={lat.norm().item():.6f} "
                  f"draws={[d[1:3] for d in draws]}")
        # (c) log_images(inpaint=True): the ImageLogger calls it with the module in eval mode.  The batch is
        # workload.synth_batch(kind, B=2, seed=1234) without faces (the eval branch reads only the identity ids);
        # "inputs" is that batch's image, so only its shape is stored
        batch, _ = workload.synth_batch(kind, B=B, seed=1234)
        batch["image_ori"]["faces"] = None
        cap = {}
        orig_fse = model.get_first_stage_encoding

        def fse(post):
            z = orig_fse(post)
            cap["z"] = z.detach().clone()
            return z
        model.get_first_stage_encoding = fse
        torch.manual_seed(300)
        with record_draws([]) as draws:
            log = model.log_images(batch, N=2, inpaint=True, ddim_steps=4)
        model.get_first_stage_encoding = orig_fse
        keys = ["reconstruction", "samples", "samples_scaled", "samples_inpainting", "mask",
                "samples_outpainting"]
        assert torch.equal(log["inputs"], batch["image"].permute(0, 3, 1, 2))
        out["log_images"] = {"batch_seed": 1234, "N": 2, "ddim_steps": 4, "ddim_eta": 1.0, "z": cap["z"], "draws": draws,
                             "panels": {k: log[k].detach().clone() for k in keys}}
        print(f"[log_images] keys={sorted(log.keys())} draws={[d[1:3] for d in draws]}")
    os.makedirs(GOLD, exist_ok=True)
    torch.save(out, os.path.join(GOLD, f"ddim_masked_{kind}.pt"), _use_new_zipfile_serialization=False)
    print(f"[masked/{kind}] written {os.path.getsize(os.path.join(GOLD, f'ddim_masked_{kind}.pt'))} bytes")


if __name__ == "__main__":
    run_masked("tiny")
