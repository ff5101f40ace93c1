"""Generate tests/golden/ddpm_sample_tiny.pt by running the UNMODIFIED reference (through oracle/ref_shim.py) on CPU, in
the tiny configuration (workload.model_params("tiny"), 1000 timesteps):

    python oracle/make_golden_ddpm.py

  (a) LatentDiffusion.sample(c, batch_size=2, return_intermediates=True) over all 1000 steps (ddpm.py:1287-1303);
  (b) p_sample_loop with a given x_T, start_T = 50, log_every_t = 10 and the binary (B,1,h,w) and soft (1,1,h,w) masks of
      the masked-DDIM fixture (the blend of ddpm.py:1274-1276);
  (c) progressive_denoising with start_T = 60, a per-timestep temperature list and noise_dropout = 0.3
      (ddpm.py:1180-1234);
  (d) log_images(N=2, n_row=2, ddim_steps=None, plot_diffusion_rows/plot_progressive_rows/plot_denoise_rows=True)
      (ddpm.py:1320-1440): every latent it decodes, in order, and the panels.

Every torch.randn / torch.randn_like call (make_golden_masked.record_draws) and every F.dropout call is recorded in
order with its call site and shape.  One 1000-step loop draws 2 KB per step, so the draws are not stored: each case
stores its torch.manual_seed and, per draw, (function, call site, shape, sha1 of the values); ddpm_ref.regenerate_draws
replays the seed through the same calls and checks every digest.  This script checks that the regenerated stream is
the recorded one bit for bit before it writes the file.  The image panels are stored in fp16, the three row panels cut
to the first sample's grid row, and every latent log_images decodes in fp32; the file stays under 1 MB.
"""
import contextlib
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch
import torch.nn.functional as F

from celebbasis_b200 import synth, workload
from oracle import ddpm_ref, ref_shim
from oracle.make_golden_masked import masks, record_draws

GOLD = os.path.join(ROOT, "tests", "golden")


@contextlib.contextmanager
def record_dropout(draws):
    """F.dropout recorded as ("dropout", calling function, shape, multiplier): the multiplier is the bernoulli mask over
    (1 - p) that the call drew, re-drawn from the same generator state as F.dropout(ones) and checked against the
    call's own output (dropout is input * multiplier)."""
    o_dropout = F.dropout

    def dropout(x, p=0.5, training=True, inplace=False):
        if not training or p == 0.:                 # no draw (the eval-mode nn.Dropout layers of the UNet and CLIP)
            return o_dropout(x, p=p, training=training, inplace=inplace)
        state = torch.get_rng_state()
        out = o_dropout(x, p=p, training=training, inplace=inplace)
        after = torch.get_rng_state()
        torch.set_rng_state(state)
        scale = o_dropout(torch.ones_like(x), p=p, training=training)
        assert torch.equal(torch.get_rng_state(), after) and torch.equal(x * scale, out)
        draws.append(("dropout", sys._getframe(1).f_code.co_name, tuple(out.shape), scale))
        return out
    F.dropout = torch.nn.functional.dropout = dropout
    try:
        yield draws
    finally:
        F.dropout = torch.nn.functional.dropout = o_dropout


@contextlib.contextmanager
def recorded(seed, p_dropout=None):
    """torch.manual_seed(seed), then every draw recorded; yields the list and checks, on exit, that the regenerated
    stream is bit-identical."""
    torch.manual_seed(seed)
    draws = []
    with record_draws(draws), record_dropout(draws):
        yield draws
    regen = ddpm_ref.regenerate_draws(seed, [d[:3] for d in draws], p_dropout)
    assert len(regen) == len(draws) and all(torch.equal(r, d[3]) for r, d in zip(regen, draws))


def _first_row(key, panel, hw=64, padding=2):
    """Row panels keep only the first sample's grid row (with the padding above and below it); the others are whole."""
    return panel[:, :hw + 2 * padding].clone() if key.endswith("_row") else panel


def compact(seed, draws, p_dropout=None):
    return {"seed": seed, "p_dropout": p_dropout, "calls": [d[:3] + (ddpm_ref.digest(d[3]),) for d in draws]}


def run_ddpm(kind="tiny"):
    torch.manual_seed(0)
    basis = synth.synth_celeb_basis(seed=0)
    model = ref_shim.build_reference(workload.model_params(kind), seed=0, clip_layers=workload.clip_layers(kind),
                                     celeb_basis=basis)
    model.eval()
    g = torch.Generator().manual_seed(3)
    coefs = [F.normalize(torch.randn(2, 1, 512, generator=g), dim=-1) for _ in range(10)]
    model.embedding_manager.id_coefficients = [c.clone() for c in coefs]
    hw = workload.model_params(kind)["image_size"]
    B = 2
    pids = [3, 3]          # the prompt and identity of infer_tiny.pt, whose c rows pin this conditioning
    prompts = ["a photo of sks person"] * B
    image_ori = {"faces": None, "ids": torch.tensor([[p, p] for p in pids]), "num_ids": torch.ones(B, dtype=torch.long)}
    out = {"kind": kind, "coef_seed": 3, "prompts": prompts, "person_ids": pids, "log_every_t": model.log_every_t,
           "clip_denoised": model.clip_denoised}
    with torch.no_grad():
        c = model.get_learned_conditioning(prompts, image_ori=image_ori)
        ref = torch.load(os.path.join(GOLD, f"infer_{kind}.pt"))
        assert torch.equal(c, ref["c"].expand_as(c))
        # (a) sample over all timesteps
        with recorded(400) as draws:
            x, inter = model.sample(c, batch_size=B, return_intermediates=True, verbose=False)
        out["sample"] = {"samples": x.clone(), "intermediates": torch.stack(inter), "draws": compact(400, draws)}
        print(f"[ddpm] sample: |x|={x.norm().item():.6f} intermediates={len(inter)} draws={len(draws)}")
        # (b) masked p_sample_loop from a given x_T over the first 50 timesteps
        x0 = torch.randn(B, 4, hw, hw, generator=g)
        x_T = torch.randn(B, 4, hw, hw, generator=g)
        binary, soft = masks(B, hw)
        out.update(x0=x0.clone(), x_T=x_T.clone(), masks={"binary": binary, "soft": soft})
        out["masked"] = []
        for k, (mname, mask) in enumerate((("binary", binary), ("soft", soft))):
            with recorded(410 + k) as draws:
                x, inter = model.p_sample_loop(c, (B, 4, hw, hw), return_intermediates=True, x_T=x_T.clone(),
                                               verbose=False, mask=mask, x0=x0, start_T=50, log_every_t=10)
            out["masked"].append({"mask": mname, "start_T": 50, "log_every_t": 10, "samples": x.clone(),
                                  "intermediates": torch.stack(inter), "draws": compact(410 + k, draws)})
            print(f"[ddpm] masked {mname}: |x|={x.norm().item():.6f} draws={len(draws)}")
        # (c) progressive denoising with a per-timestep temperature and noise dropout
        T, p = 60, 0.3
        temps = [0.5 + 0.01 * i for i in range(T)]
        with recorded(420, p) as draws:
            x, inter = model.progressive_denoising(c, shape=(4, hw, hw), batch_size=B, verbose=False, start_T=T,
                                                   temperature=temps, noise_dropout=p, log_every_t=20)
        out["progressive"] = {"start_T": T, "temperature": temps, "noise_dropout": p, "log_every_t": 20,
                              "samples": x.clone(), "intermediates": torch.stack(inter), "draws": compact(420, draws, p)}
        print(f"[ddpm] progressive: |x|={x.norm().item():.6f} draws={len(draws)}")
        # (d) log_images with the DDPM sampler and all three row panels.  The batch is workload.synth_batch(kind, B=2,
        # seed=1234) without faces (the eval branch reads only the identity ids); every latent log_images decodes is
        # captured in order
        batch, _ = workload.synth_batch(kind, B=B, seed=1234)
        batch["image_ori"]["faces"] = None
        decoded = []
        orig_dfs = model.decode_first_stage

        def dfs(z, *a, **k):
            decoded.append(z.detach().clone())
            return orig_dfs(z, *a, **k)
        model.decode_first_stage = dfs
        with recorded(430) as draws:
            log = model.log_images(batch, N=2, n_row=2, ddim_steps=None, plot_diffusion_rows=True,
                                   plot_progressive_rows=True, plot_denoise_rows=True)
        model.decode_first_stage = orig_dfs
        assert torch.equal(log["inputs"], batch["image"].permute(0, 3, 1, 2))
        keep = ["reconstruction", "diffusion_row", "denoise_row", "samples_scaled", "progressive_row"]
        out["log_images"] = {"batch_seed": 1234, "N": 2, "n_row": 2, "decoded": torch.stack(decoded),
                             "draws": compact(430, draws), "keys": list(log.keys()),
                             "shapes": {k: tuple(v.shape) for k, v in log.items()},
                             "panels_fp16": {k: _first_row(k, log[k]).detach().half() for k in keep}}
        print(f"[ddpm] log_images: keys={list(log.keys())} decoded={len(decoded)} draws={len(draws)}")
    os.makedirs(GOLD, exist_ok=True)
    path = os.path.join(GOLD, f"ddpm_sample_{kind}.pt")
    torch.save(out, path, _use_new_zipfile_serialization=False)
    print(f"[ddpm/{kind}] written {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    run_ddpm("tiny")
