"""BASELINE config 5: attention / conv microbench sweep with both roofline fractions per row (SURVEY 8d definitions:
algorithmic FLOPs and bytes, recompute not counted; peaks from the H100 SXM data sheet).  One JSON line per case."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from celebbasis_b200 import ops
from celebbasis_b200.unet_engine import _Attn
dev = torch.device("cuda:0")
g = torch.Generator().manual_seed(0)
rnd = lambda *s: torch.randn(*s, generator=g).half().to(dev)
PEAK_TF, PEAK_GB = 989.0, 3350.0      # H100 SXM data sheet, dense BF16 / HBM3 (700 W); never reached
out_path = os.path.join(ROOT, "tools_out", "microbench_sweep.jsonl")
os.makedirs(os.path.dirname(out_path), exist_ok=True)
open(out_path, "w").close()

def timeit(fn, n=10):
    fn(); torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        for _ in range(n):
            fn()
    gr.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        gr.replay()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000 / (5 * n)

def emit(case, us, flops, bytes_):
    tf, gb = flops / us / 1e6, bytes_ / us / 1e3
    rec = dict(case=case, us=round(us, 2), tflops=round(tf, 1), frac_tensor=round(tf / PEAK_TF, 4), gbs=round(gb, 1),
               frac_hbm=round(gb / PEAK_GB, 4), bound="tensor" if flops / (PEAK_TF * 1e12) > bytes_ / (PEAK_GB * 1e9) else "hbm")
    print(json.dumps(rec), flush=True)
    with open(out_path, "a") as f:
        f.write(json.dumps(rec) + "\n")

H = 8
for N in (1024, 4096):
    for C in (320, 640, 1280):
        dh = C // H
        for kind, nk in (("self", N), ("cross", 77)):
            q, k, v, dO = rnd(N, C), rnd(nk, C), rnd(nk, C), rnd(N, C)
            o = torch.empty_like(q); dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
            st = {}
            def f():
                st["s"] = _Attn.fwd(q, k, v, images=1, heads=H, dh=dh, nq=N, nk=nk, scale=dh ** -0.5, out=o)
            def b():
                _Attn.bwd(dO, q, k, v, st["s"], images=1, heads=H, dh=dh, nq=N, nk=nk, scale=dh ** -0.5, dq=dq, dk=dk, dv=dv)
            core_bytes = 2 * (2 * N * C + 2 * nk * C)            # q, o + k, v (16-bit)
            emit(f"sdpa_fwd_{kind}_N{N}_C{C}", timeit(f), 4.0 * N * nk * C, core_bytes)
            emit(f"sdpa_bwd_{kind}_N{N}_C{C}", timeit(b), 8.0 * N * nk * C, 2 * core_bytes + 2 * N * C)

def conv(cin, cout, h):
    x = torch.randn(h * h, cin, generator=g).to(dev)                  # fp32 residual stream, as in the UNet
    gm, bt = torch.ones(cin, device=dev), torch.zeros(cin, device=dev)
    w = ops.pack_conv_weight(torch.randn(cout, cin, 3, 3, generator=g).to(dev) * 0.02, torch.float16)
    geo = ops.Geo(1, h, h)
    out = torch.empty(h * h, cout, dtype=torch.float16, device=dev)
    def f():
        n16, _ = ops.groupnorm(x, geo, gm, bt, silu=True)
        ops.conv2d(n16, geo, w, cout, out=out)
    dy = rnd(h * h, cout)
    dx = torch.empty(h * h, cin, dtype=torch.float16, device=dev)
    def d():
        ops.conv2d_dgrad(dy, geo, w, cin, out=dx)
    fl = 18.0 * cin * cout * h * h
    by = 2 * cin * h * h + 2 * cout * h * h + 18 * cin * cout
    emit(f"gn_silu_conv3x3_fwd_{cin}->{cout}@{h}", timeit(f), fl, by)
    emit(f"conv3x3_dgrad_{cout}->{cin}@{h}", timeit(d), fl, by)

for (c, h) in ((320, 64), (640, 32), (1280, 16), (1280, 8)):
    conv(c, c, h)
for (ci, co, h) in ((640, 320, 64), (960, 320, 64), (1920, 640, 32), (2560, 1280, 16), (2560, 1280, 8)):
    conv(ci, co, h)
