"""GPU probe: the full CelebBasis training step (CelebBasisStep) vs the reference-generated golden fixtures."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tools_out")
os.makedirs(OUT, exist_ok=True)

import torch

from celebbasis_b200 import synth, workload
from celebbasis_b200.tokenizer import SyntheticCLIPTokenizer
from celebbasis_b200.train_step import CelebBasisStep
from oracle import torch_ref


def emit(rec):
    with open(os.path.join(OUT, "step_probe.jsonl"), "a") as f:
        f.write(json.dumps(rec) + "\n")
    print(json.dumps(rec), flush=True)


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def run(kind, vae_res=torch.float32):
    dev = torch.device("cuda:0")
    gold = torch.load(os.path.join(ROOT, "tests", "golden", f"step_{kind}.pt"))
    params = workload.model_params(kind)
    t0 = time.time()
    om = torch_ref.OracleModel(params, clip_layers=workload.clip_layers(kind))   # only used to enumerate keys/shapes
    sd = synth.synth_state_dict(om, seed=0)
    del om
    basis = synth.synth_celeb_basis(seed=0)
    eng = CelebBasisStep(params, sd, basis, dev, tokenizer=SyntheticCLIPTokenizer(), vae_res_dtype=vae_res)
    torch.cuda.synchronize()
    t_build = time.time() - t0
    batch, draws = workload.synth_batch(kind, B=1, seed=1234)
    bdev = {"image": batch["image"].to(dev), "caption": batch["caption"],
            "image_ori": {"faces": batch["image_ori"]["faces"].to(dev), "ids": batch["image_ori"]["ids"],
                          "num_ids": batch["image_ori"]["num_ids"]}}
    ddev = {k: v.to(dev) for k, v in draws.items()}
    t0 = time.time()
    loss = eng.forward_backward(bdev, ddev)
    torch.cuda.synchronize()
    t_first = time.time() - t0
    L = eng.last
    rec = dict(case=f"step_{kind}_vaeres_{str(vae_res)[6:]}", loss=loss.item(), loss_ref=gold["loss"].item(),
               loss_rel=abs(loss.item() - gold["loss"].item()) / abs(gold["loss"].item()),
               z_rel=rel(L["z"], gold["z"]), face_rel=rel(L["face_feat"], torch.nn.functional.normalize(gold["face_feat"], dim=-1)),
               coef_rel=rel(L["coef"].view(-1), gold["celeb_coef"].view(-1)), celebz_rel=rel(L["celeb_z"], gold["celeb_z"]),
               ctx_rel=rel(L["context"], gold["context"]), xnoisy_rel=rel(L["x_noisy"], gold["x_noisy"]),
               eps_rel=rel(L["eps"], gold["eps"]), gb_rel=rel(eng.gb, gold["gb"]),
               gW_norm=eng.gW.norm().item(), gW_norm_ref=gold["gW_norm"].item(),
               positions=[[f.tolist() for f in p] for p in L["positions"]],
               t_build_s=round(t_build, 2), t_first_s=round(t_first, 3))
    if "gW" in gold:
        rec["gW_rel"] = rel(eng.gW, gold["gW"])
    else:
        rec["gW_sample_rel"] = rel(eng.gW.flatten()[::131], gold["gW_sample"])
    emit(rec)
    torch.cuda.synchronize()
    t0 = time.time()
    n = 5
    for _ in range(n):
        eng.forward_backward(bdev, ddev)
        eng.optimizer_step()
    torch.cuda.synchronize()
    emit(dict(case=f"step_{kind}_eager_warm", s_per_step=round((time.time() - t0) / n, 4),
              peak_mem_gb=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)))


if __name__ == "__main__":
    for w in (sys.argv[1:] or ["tiny", "full"]):
        try:
            if w == "full16":
                run("full", torch.float16)
            else:
                run(w)
        except Exception as e:  # noqa
            import traceback
            traceback.print_exc()
            emit(dict(case=w, ok=False, error=repr(e)[:600]))
