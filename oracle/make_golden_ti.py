"""Generate tests/golden/ti_train_tiny.pt by running the UNMODIFIED reference's Textual Inversion workflow on the CPU.

    python oracle/make_golden_ti.py

Two parts:
  * ldm.data.personalized.PersonalizedBase (v1-finetune.yaml's dataset) over seeded synthetic PNGs
    (workload.synth_photo_files: non-square, modes RGB / RGBA / L / P): every `interpolation`, centre crop on and off,
    per-image-token mixing and a coarse class text.  Recorded per item: the caption, the flip draw, the image tensor and a
    digest of the random / numpy / torch generator states after the item.
  * LatentDiffusion with v1-finetune.yaml's personalization config (EmbeddingManager, '*', initializer word 'person',
    2 vectors per token) on the tiny model: `steps` optimiser steps of shared_step -> backward -> torch.optim.AdamW
    (configure_optimizers) on batch-size-2 batches of that dataset, with t, noise and the posterior eps replayed.
    Recorded: the draws, the captions, the losses, the initial and the trained placeholder rows.
"""
import hashlib
import os
import pickle
import random
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np
import torch

from celebbasis_b200 import workload
from oracle import ref_shim

GOLD = os.path.join(ROOT, "tests", "golden")
DATA_SIZE = 24
DATA_CASES = ([dict(interpolation=i, center_crop=c) for i in ("linear", "bilinear", "bicubic", "lanczos")
               for c in (False, True)]
              + [dict(interpolation="bicubic", per_image_tokens=True, mixing_prob=0.5),
                 dict(interpolation="bilinear", coarse_class_text="person", center_crop=True)])
DATA_INDICES = (0, 1, 2, 3, 5, 10)
DATA_SEED = 11
TRAIN = dict(steps=12, B=2, lr=5e-3, seed=3, size=64)


def rng_digest():
    return hashlib.sha1(pickle.dumps((random.getstate(), np.random.get_state()[1].tobytes(), np.random.get_state()[2],
                                      torch.get_rng_state().numpy().tobytes()))).hexdigest()


def seed_all(seed):
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)


def _reference_dataset_class():
    # Pillow 10 removed the LINEAR alias the reference's filter table names; before that it was BILINEAR
    import PIL.Image
    if not hasattr(PIL.Image, "LINEAR"):
        PIL.Image.LINEAR = PIL.Image.BILINEAR
    ref_shim.install_stubs(2)
    from ldm.data.personalized import PersonalizedBase
    return PersonalizedBase


def run_data(root):
    PersonalizedBase = _reference_dataset_class()
    cases = []
    for kw in DATA_CASES:
        seed_all(DATA_SEED)
        ds = PersonalizedBase(root, size=DATA_SIZE, repeats=4, **kw)
        items = []
        for i in DATA_INDICES:
            before = torch.get_rng_state()
            ex = ds[i]
            after, digest = torch.get_rng_state(), rng_digest()
            # the item's one torch draw is the flip's torch.rand(1): replay it from the saved state
            torch.set_rng_state(before)
            flip_draw = float(torch.rand(1))
            torch.set_rng_state(after)
            items.append({"index": i, "caption": ex["caption"], "image": torch.from_numpy(ex["image"].copy()),
                          "flip_draw": flip_draw, "rng_digest": digest})
        cases.append({"kwargs": kw, "len": len(ds), "items": items})
        print(f"[ti-data] {kw}: {[it['caption'] for it in items[:2]]}")
    return cases


def run_train(root):
    PersonalizedBase = _reference_dataset_class()
    kind = "tiny"
    steps, B, lr = TRAIN["steps"], TRAIN["B"], TRAIN["lr"]
    seed_all(TRAIN["seed"])
    ds = PersonalizedBase(root, size=TRAIN["size"], repeats=100, interpolation="bicubic", flip_p=0.5)
    batches = [torch.utils.data.default_collate([ds[s * B + j] for j in range(B)]) for s in range(steps)]
    torch.manual_seed(0)
    torch.set_num_threads(os.cpu_count())
    model = ref_shim.build_reference(workload.ti_model_params(kind), seed=0, clip_layers=workload.clip_layers(kind))
    em = model.embedding_manager
    model.learning_rate = lr
    opt = model.configure_optimizers()
    opt = opt[0] if isinstance(opt, (list, tuple)) else opt
    params0 = {k: v.detach().clone() for k, v in em.string_to_param_dict.items()}
    lat = TRAIN["size"] // 8
    g = torch.Generator().manual_seed(29)
    draws, losses = [], []
    t0 = time.time()
    for s in range(steps):
        d = {"t": torch.randint(0, 1000, (B,), generator=g).long(), "noise": torch.randn(B, 4, lat, lat, generator=g),
             "posterior_eps": torch.randn(B, 4, lat, lat, generator=g)}
        with ref_shim.replay_randomness(d["t"], d["noise"], d["posterior_eps"]):
            loss, _ = model.shared_step(batches[s])
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
        draws.append(d)
    print(f"[ti-train] {steps} steps in {time.time() - t0:.1f}s; losses {losses[0]:.6f} .. {losses[-1]:.6f} "
          f"optimizer {type(opt).__name__}")
    return {"kind": kind, **TRAIN, "captions": [b["caption"] for b in batches], "draws": draws,
            "losses": torch.tensor(losses, dtype=torch.float64), "params0": params0,
            "params_final": {k: v.detach().clone() for k, v in em.string_to_param_dict.items()},
            "tokens": {k: int(v) for k, v in em.string_to_token_dict.items()}, "optimizer": type(opt).__name__}


def main():
    with tempfile.TemporaryDirectory() as td:
        workload.synth_photo_files(td, seed=0)
        files = os.listdir(td)
        out = {"photo_seed": 0, "files": files, "size": DATA_SIZE, "indices": list(DATA_INDICES), "seed": DATA_SEED,
               "data": run_data(td), "train": run_train(td)}
    os.makedirs(GOLD, exist_ok=True)
    torch.save(out, os.path.join(GOLD, "ti_train_tiny.pt"), _use_new_zipfile_serialization=False)
    print("[ti] wrote", os.path.join(GOLD, "ti_train_tiny.pt"))


if __name__ == "__main__":
    main()
