"""GPU probe: UNetEngine forward/backward vs the plain-torch fp32 oracle on the same synthetic weights."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tools_out")
os.makedirs(OUT, exist_ok=True)

import torch

torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False

from celebbasis_b200 import synth
from celebbasis_b200.unet_engine import UNetEngine
from oracle import torch_ref

CFGS = {
    "tiny": dict(in_channels=4, out_channels=4, model_channels=64, attention_resolutions=[4, 2, 1], num_res_blocks=1,
                 channel_mult=[1, 2, 4, 4], num_heads=8, context_dim=768),
    "full": dict(in_channels=4, out_channels=4, model_channels=320, attention_resolutions=[4, 2, 1], num_res_blocks=2,
                 channel_mult=[1, 2, 4, 4], num_heads=8, context_dim=768),
}


def emit(rec):
    with open(os.path.join(OUT, "unet_probe.jsonl"), "a") as f:
        f.write(json.dumps(rec) + "\n")
    print(json.dumps(rec), flush=True)


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


def run(name, B=1, res=64, dtype=torch.float16):
    cfg = CFGS[name]
    dev = torch.device("cuda:0")
    ref = torch_ref.UNetModel(**cfg)
    sd = synth.synth_state_dict(ref, seed=0, prefix="model.diffusion_model.")
    ref.load_state_dict(sd, strict=True)
    ref = ref.to(dev).float()
    g = torch.Generator().manual_seed(7)
    x = torch.randn(B, 4, res, res, generator=g).to(dev)
    t = torch.randint(0, 1000, (B,), generator=g).to(dev)
    ctx = torch.randn(B, 77, 768, generator=g).to(dev).requires_grad_(True)
    noise = torch.randn(B, 4, res, res, generator=g).to(dev)
    t0 = time.time()
    eps_ref = ref(x, t, ctx)
    loss_ref = torch_ref.eps_loss(eps_ref, noise)
    loss_ref.backward()
    torch.cuda.synchronize()
    t_ref = time.time() - t0

    eng = UNetEngine(cfg, sd, dev, dtype=dtype)
    torch.cuda.synchronize()
    t0 = time.time()
    eps = eng.forward(x, t, ctx.detach())
    torch.cuda.synchronize()
    t_fwd = time.time() - t0
    loss = torch_ref.eps_loss(eps, noise)
    d_eps = 2.0 * (eps - noise) / eps.numel()
    t0 = time.time()
    dctx = eng.backward(d_eps)
    torch.cuda.synchronize()
    t_bwd = time.time() - t0
    emit(dict(case=f"unet_{name}_B{B}_{res}_{str(dtype)[6:]}", eps_rel=rel(eps, eps_ref.detach()),
              loss=loss.item(), loss_ref=loss_ref.item(), loss_rel=abs(loss.item() - loss_ref.item()) / abs(loss_ref.item()),
              dctx_rel=rel(dctx, ctx.grad), dctx_norm=ctx.grad.norm().item(), eps_norm=eps_ref.norm().item(),
              finite=bool(torch.isfinite(eps).all() and torch.isfinite(dctx).all()),
              t_ref_s=round(t_ref, 3), t_fwd_s=round(t_fwd, 3), t_bwd_s=round(t_bwd, 3)))
    # second pass timing (warm)
    torch.cuda.synchronize()
    t0 = time.time()
    for _ in range(3):
        eps = eng.forward(x, t, ctx.detach())
        dctx = eng.backward(d_eps)
    torch.cuda.synchronize()
    emit(dict(case=f"unet_{name}_B{B}_warm", s_per_fwdbwd=round((time.time() - t0) / 3, 4)))


if __name__ == "__main__":
    which = sys.argv[1:] or ["tiny", "full"]
    for w in which:
        try:
            if w == "tiny":
                run("tiny", B=2, res=32)
            elif w == "full":
                run("full", B=1, res=64)
            elif w == "full_bf16":
                run("full", B=1, res=64, dtype=torch.bfloat16)
        except Exception as e:  # noqa
            import traceback
            traceback.print_exc()
            emit(dict(case=w, ok=False, error=repr(e)[:500]))
