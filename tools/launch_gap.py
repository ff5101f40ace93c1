"""How long does one kernel node cost inside a CUDA graph? (per-node time of 100-node graphs of tiny launches)"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from celebbasis_b200 import ops
dev = torch.device("cuda:0")
g = torch.Generator().manual_seed(0)
rnd = lambda *s: torch.randn(*s, generator=g).half().to(dev)

def per_node(name, fn, n=100):
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
    print(f"{name}: {e0.elapsed_time(e1) * 1000 / (5 * n):.2f} us per node", flush=True)

a = torch.randn(64, 256, device=dev); b = torch.empty_like(a)
per_node("axpby 64x256 f32", lambda: ops.axpby(a, 2.0, out=b))
x, w = rnd(128, 64), rnd(64, 64); o = torch.empty(128, 64, dtype=torch.float16, device=dev)
per_node("linear 128x64x64 (1 CTA)", lambda: ops.linear(x, w, out=o))
x2, w2 = rnd(4096, 320), rnd(320, 320); o2 = torch.empty(4096, 320, dtype=torch.float16, device=dev)
per_node("linear 4096x320x320 (64 CTAs)", lambda: ops.linear(x2, w2, out=o2))
x3, w3 = rnd(4096, 320), rnd(2560, 320); o3 = torch.empty(4096, 2560, dtype=torch.float16, device=dev)
per_node("linear 4096x2560x320 (512 CTAs)", lambda: ops.linear(x3, w3, out=o3))
xn = torch.randn(4096, 320, device=dev); gm = torch.ones(320, device=dev); bt = torch.zeros(320, device=dev)
per_node("layernorm 4096x320", lambda: ops.layernorm(xn, gm, bt))
per_node("groupnorm 4096x320 (cluster, 1 kernel)", lambda: ops.groupnorm(xn, ops.Geo(1, 64, 64), gm, bt))
per_node("torch add (reference point)", lambda: torch.add(a, 1.0, out=b))
