"""Training throughput of the step options that run on the fused CUDA-graph step besides the default configuration, on
one GPU at the full SD-v1 sizes with synthetic weights:

  cb_weights        CelebBasis, batch 1, l_simple_weight 0.5, original_elbo_weight 1e-2, logvar_init 0.1
  cb_persons        CelebBasis, batch 2, four face crops per sample, prompts naming 1, 2 or 3 persons from step to step
  ti_options        Textual Inversion, batch 2, num_vectors_per_token 2, two placeholders (one without an initializer
                    word), embedding_reg_weight 1e-2, progressive words, the loss weights above

For each option set, alternates rounds of the fused step (with the look-ahead front end Trainer.fit enables) and of
the eager per-module route (model.fused_step = False) in one process, each round `--steps` x (shared_step -> backward
-> optimiser step), timed with CUDA events around a device synchronise.  Prints the card name and power limit beside
the numbers, and one JSON line.

    python tools/bench_fused_options.py --steps 10 --rounds 2
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch

from bench_ti import card

WEIGHTS = dict(l_simple_weight=0.5, original_elbo_weight=1e-2, logvar_init=0.1)
CAPTIONS = {1: "a photo of a face of sks person", 2: "a photo of sks person and ks person",
            3: "a photo of sks and ks and ata together"}


def option_set(name):
    """(model params, B, host batch maker) of one option set."""
    from celebbasis_b200 import workload
    if name == "ti_options":
        p = workload.ti_model_params("full", num_vectors_per_token=2)
        p["personalization_config"]["params"].update(placeholder_strings=["*", "sks"], initializer_words=["person"],
                                                     progressive_words=True)
        p["embedding_reg_weight"] = 1e-2
        caps = ["a photo of *", "a photo of sks and *", "a sks photo", "* in a photo of sks"]

        def make(g, i, B):
            return {"image": torch.rand(B, 512, 512, 3, generator=g) * 2 - 1,
                    "caption": [caps[(i + b) % len(caps)] for b in range(B)]}
        B = 2
    else:
        p = workload.model_params("full")
        B = 1 if name == "cb_weights" else 2
        mix = [[1, 1]] if name == "cb_weights" else [[1, 2], [3, 1], [2, 3], [2, 2]]
        n_chunks = 2 if name == "cb_weights" else 4

        def make(g, i, B):
            nid = torch.tensor(mix[i % len(mix)][:B], dtype=torch.long)
            return {"image": torch.rand(B, 512, 512, 3, generator=g) * 2 - 1, "caption": [CAPTIONS[int(k)] for k in nid],
                    "image_ori": {"faces": torch.rand(B, 512, 512, 3 * n_chunks, generator=g) * 2 - 1,
                                  "ids": torch.stack([torch.randperm(10, generator=g)[:n_chunks] for _ in range(B)]),
                                  "num_ids": nid}}
    p["cond_stage_config"]["params"].update(device="cuda")
    p.update(WEIGHTS)
    return p, B, make


def to_dev(h, dev):
    out = {k: (v.to(dev, non_blocking=True) if torch.is_tensor(v) else v) for k, v in h.items() if k != "image_ori"}
    if "image_ori" in h:
        io = h["image_ori"]
        out["image_ori"] = {"faces": io["faces"].to(dev, non_blocking=True), "ids": io["ids"], "num_ids": io["num_ids"]}
    return out


def bench(name, args, dev):
    from celebbasis_b200 import synth
    from ldm.models.diffusion.ddpm import LatentDiffusion
    torch.manual_seed(0)
    params, B, make = option_set(name)
    model = LatentDiffusion(**params)
    model.load_state_dict(synth.synth_state_dict(model, seed=0), strict=False)
    model = model.to(dev).train()
    if not model._textual_inversion():
        model.cond_stage_model.celeb_embeddings = synth.synth_celeb_basis(seed=0).to(dev)
    model.learning_rate = 5e-3
    opt = model.configure_optimizers()
    g = torch.Generator().manual_seed(1)
    host = [make(g, i, B) for i in range(4)]
    for h in host:
        h["image"] = h["image"].pin_memory()
        if "image_ori" in h:
            h["image_ori"]["faces"] = h["image_ori"]["faces"].pin_memory()
    staged = {}

    def step(i, fused):
        b = staged.pop(i, None) or to_dev(host[i % len(host)], dev)
        if fused:                           # the same object the next step receives, as Trainer.fit stages it
            staged[i + 1] = to_dev(host[(i + 1) % len(host)], dev)
            model.stage_next_batch(staged[i + 1])
        loss, _ = model.shared_step(b)
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)

    def round_(fused):
        model.fused_step = fused
        model._staged_next = None
        staged.clear()
        for i in range(args.warmup):
            step(i, fused)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.steps):
            step(i, fused)
        e1.record()
        torch.cuda.synchronize()
        return args.steps * 1000.0 / e0.elapsed_time(e1)

    res = {"fused": [], "eager": []}
    for r in range(args.rounds):
        for mode in ("fused", "eager"):
            res[mode].append(round_(mode == "fused"))
            print(f"[bench_fused_options] {name} round {r} {mode}: {res[mode][-1]:.2f} steps/s", file=sys.stderr)
    assert model._fused is not None, f"the fused step did not engage for {name}"
    out = {"option_set": name, "batch": B, "fused_steps_per_s": max(res["fused"]),
           "eager_steps_per_s": max(res["eager"]), "fused_rounds": res["fused"], "eager_rounds": res["eager"]}
    del model, opt
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--sets", default="cb_weights,cb_persons,ti_options")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_fused_options.py needs a GPU"
    dev = torch.device("cuda:0")
    results = [bench(name, args, dev) for name in args.sets.split(",")]
    name = card()
    for r in results:
        print(f"[bench_fused_options] {name}: {r['option_set']}: fused {r['fused_steps_per_s']:.2f} steps/s, eager "
              f"{r['eager_steps_per_s']:.2f} steps/s ({r['fused_steps_per_s'] / r['eager_steps_per_s']:.2f}x)",
              file=sys.stderr)
    print(json.dumps({"workload": "SD-v1 full size, 512x512, synthetic weights", "card": name, "results": results}))


if __name__ == "__main__":
    main()
