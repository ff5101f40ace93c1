"""GPU probe: locate gradient error along the backward chain by comparing against the fp32 oracle run on the GPU."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tools_out")
os.makedirs(OUT, exist_ok=True)
import torch

torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False
from celebbasis_b200 import ops, synth, workload
from celebbasis_b200.tokenizer import SyntheticCLIPTokenizer
from celebbasis_b200.train_step import CelebBasisStep
from oracle import torch_ref


def rel(a, b):
    a, b = a.float().cpu().flatten(), b.float().cpu().flatten()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _tap(fn, out, key, pick):
    def wrapped(*args, **kw):
        r = fn(*args, **kw)
        out[key] = r if pick is None else r[pick]
        return r
    return wrapped


def run(kind, loss_scale=1024.0, dtype=torch.float16):
    dev = torch.device("cuda:0")
    params = workload.model_params(kind)
    om = torch_ref.OracleModel(params, clip_layers=workload.clip_layers(kind))
    sd = synth.synth_state_dict(om, seed=0)
    om.load_state_dict(sd)
    om = om.to(dev).eval()
    basis = synth.synth_celeb_basis(seed=0)
    tok = SyntheticCLIPTokenizer()
    batch, draws = workload.synth_batch(kind, B=1, seed=1234)
    bdev = {"image": batch["image"].to(dev), "caption": batch["caption"],
            "image_ori": {"faces": batch["image_ori"]["faces"].to(dev), "ids": batch["image_ori"]["ids"],
                          "num_ids": batch["image_ori"]["num_ids"]}}
    ddev = {k: v.to(dev) for k, v in draws.items()}
    W, b = om.trainable()
    W.requires_grad_(True); b.requires_grad_(True)
    ids = tok(batch["caption"])["input_ids"]
    out = om.step(bdev, ddev, ids, basis, tok.word_id("sks"))
    out["loss"].backward()
    eng = CelebBasisStep(params, sd, basis, dev, tokenizer=tok, loss_scale=loss_scale, dtype=dtype)
    # the backward's intermediate gradients, taken from the calls that produce them: (owner, function, key, output)
    taps = [(ops, "mse_fwd_bwd", "d_eps", 1), (eng.unet, "backward", "dctx", None), (eng.clip, "backward", "demb", None),
            (ops, "embed_inject_bwd", "dz", None), (ops, "celeb_basis_bwd", "dcoef", None)]
    L, originals = {}, [getattr(owner, name) for owner, name, _, _ in taps]
    for (owner, name, key, pick), fn in zip(taps, originals):
        setattr(owner, name, _tap(fn, L, key, pick))
    try:
        loss = eng.forward_backward(bdev, ddev)
    finally:
        for (owner, name, _, _), fn in zip(taps, originals):
            setattr(owner, name, fn)
    L.update(eng.last)
    rec = dict(case=f"grad_{kind}_S{loss_scale}_{str(dtype)[6:]}", loss=loss.item(), loss_ref=out["loss"].item(),
               eps_rel=rel(L["eps"], out["eps"]), ctx_rel=rel(L["context"], out["context"]),
               d_eps_rel=rel(L["d_eps"], out["eps"].grad), dctx_rel=rel(L["dctx"], out["context"].grad),
               demb_rel=rel(L["demb"], out["emb"].grad),
               dz_rel=rel(L["dz"].view(-1, 2, 768)[:1], out["celeb_z"].grad[:1]),
               dcoef_rel=rel(L["dcoef"][:1], out["coef"].grad[:1]),
               gW_rel=rel(eng.gW, W.grad), gb_rel=rel(eng.gb, b.grad),
               dctx_norm=out["context"].grad.norm().item(), demb_norm=out["emb"].grad.norm().item(),
               dcoef_norm=out["coef"].grad.norm().item(), gW_norm=W.grad.norm().item())
    # isolate stages: feed the oracle's upstream gradient into each of our backward stages
    with open(os.path.join(OUT, "grad_probe.jsonl"), "a") as f:
        f.write(json.dumps(rec) + "\n")
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    args = sys.argv[1:] or ["tiny"]
    for a in args:
        try:
            if a == "tiny":
                run("tiny")
            elif a == "full":
                run("full")
            elif a == "full_bf16":
                run("full", dtype=torch.bfloat16)
            elif a == "full_S64":
                run("full", loss_scale=65536.0)
        except Exception as e:  # noqa
            import traceback
            traceback.print_exc()
            print(json.dumps(dict(case=a, error=repr(e)[:500])))
