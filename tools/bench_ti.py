"""Textual Inversion training throughput (configs/stable-diffusion/v1-finetune.yaml) on one GPU: the full SD-v1 model
with synthetic weights at v1-finetune's batch size of 2, 512x512 images.

Alternates rounds of the fused CUDA-graph step (with the look-ahead VAE encode the training loop's stage_next_batch
enables) and of the eager per-module path (CB_FUSED_STEP=0 semantics: model.fused_step = False) in one process, each round
`--steps` x (shared_step -> backward -> FusedAdamW step), timed with CUDA events around a device synchronise.  Prints the
card name and power limit beside the numbers, and one JSON line.

    python tools/bench_ti.py --steps 20 --rounds 3
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:                  # nvidia-smi missing: say so rather than guess
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ti.py needs a GPU"
    from celebbasis_b200 import synth, workload
    from ldm.models.diffusion.ddpm import LatentDiffusion
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    B = args.batch
    params = workload.ti_model_params("full")
    params["cond_stage_config"]["params"].update(device="cuda")
    model = LatentDiffusion(**params)
    model.load_state_dict(synth.synth_state_dict(model, seed=0), strict=False)
    model = model.to(dev).train()
    model.learning_rate = 5e-3
    opt = model.configure_optimizers()
    g = torch.Generator().manual_seed(1)
    captions = ["a photo of *", "a rendering of a *", "a close-up photo of the *", "a good photo of a *"]
    host = [{"image": (torch.rand(B, 512, 512, 3, generator=g) * 2 - 1).pin_memory(),
             "caption": [captions[(i + j) % len(captions)] for j in range(B)]} for i in range(4)]

    def batch(i):
        h = host[i % len(host)]
        return {"image": h["image"].to(dev, non_blocking=True), "caption": h["caption"]}

    staged = {}

    def step(i, fused):
        b = staged.pop(i, None) or batch(i)
        if fused:                           # the same object the next step receives, as Trainer.fit stages it
            staged[i + 1] = batch(i + 1)
            model.stage_next_batch(staged[i + 1])
        loss, _ = model.shared_step(b)
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        return loss

    def round_(fused, n):
        model.fused_step = fused
        model._staged_next = None
        staged.clear()
        for i in range(args.warmup):
            step(i, fused)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(n):
            step(i, fused)
        e1.record()
        torch.cuda.synchronize()
        return n * 1000.0 / e0.elapsed_time(e1)

    res = {"fused": [], "eager": []}
    for r in range(args.rounds):
        for mode in ("fused", "eager"):
            res[mode].append(round_(mode == "fused", args.steps))
            print(f"[bench_ti] round {r} {mode}: {res[mode][-1]:.2f} steps/s", file=sys.stderr)
    assert model._fused is not None, "the fused TI step did not engage"
    name = card()
    out = {"workload": f"textual inversion, SD-v1 full size, 512x512, batch {B}", "card": name,
           "fused_steps_per_s": max(res["fused"]), "eager_steps_per_s": max(res["eager"]),
           "fused_rounds": res["fused"], "eager_rounds": res["eager"],
           "graph_launches_per_step": model._fused.launches["pipe"]}
    print(f"[bench_ti] {name}: fused {out['fused_steps_per_s']:.2f} steps/s, eager {out['eager_steps_per_s']:.2f} "
          f"steps/s ({out['fused_steps_per_s'] / out['eager_steps_per_s']:.2f}x)", file=sys.stderr)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
