"""GPU microbench of representative cb_gemm shapes of the training step (CUDA-graph replay => pure device time)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from celebbasis_b200 import ops

dev = torch.device("cuda:0")
g = torch.Generator().manual_seed(0)
out_path = os.path.join(ROOT, "tools_out", "gemm_shapes.jsonl")
os.makedirs(os.path.dirname(out_path), exist_ok=True)


def rnd(*s):
    return torch.randn(*s, generator=g).half().to(dev)


def timeit(name, fn, flops, bytes_):
    fn()
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        for _ in range(10):
            fn()
    for _ in range(2):
        gr.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        gr.replay()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1000 / 50
    rec = dict(case=name, us=round(us, 2), tflops=round(flops / us / 1e6, 1), gbs=round(bytes_ / us / 1e3, 1))
    print(json.dumps(rec), flush=True)
    with open(out_path, "a") as f:
        f.write(json.dumps(rec) + "\n")


def conv(n, h, cin, cout, tag=""):
    x = rnd(n * h * h, cin)
    w = ops.pack_conv_weight(torch.randn(cout, cin, 3, 3, generator=g).to(dev) * 0.02, torch.float16)
    geo = ops.Geo(n, h, h)
    out = torch.empty(n * h * h, cout, dtype=torch.float16, device=dev)
    timeit(f"conv3x3{tag}_{n}x{h}x{h}_{cin}->{cout}", lambda: ops.conv2d(x, geo, w, cout, out=out),
           18.0 * cin * cout * n * h * h, 2 * (n * h * h * (cin + cout) + 9 * cin * cout))


def lin(M, N, K):
    x, w = rnd(M, K), rnd(N, K)
    out = torch.empty(M, N, dtype=torch.float16, device=dev)
    timeit(f"linear_{M}x{N}x{K}", lambda: ops.linear(x, w, out=out), 2.0 * M * N * K, 2 * (M * K + N * K + M * N))
    dy = rnd(M, N)
    o2 = torch.empty(M, K, dtype=torch.float16, device=dev)
    timeit(f"lin_dgrad_{M}x{K}x{N}", lambda: ops.linear_dgrad(dy, w, out=o2), 2.0 * M * N * K, 2 * (M * K + N * K + M * N))


which = sys.argv[1:] or ["unet", "misc"]
if "unet" in which:
    conv(1, 64, 320, 320); conv(1, 64, 640, 320); conv(1, 64, 640, 640)
    conv(1, 32, 640, 640); conv(1, 32, 1280, 640); conv(1, 32, 1280, 1280)
    conv(1, 16, 1280, 1280); conv(1, 16, 2560, 1280)
    conv(1, 8, 1280, 1280); conv(1, 8, 2560, 1280)
    lin(4096, 320, 320); lin(4096, 2560, 320); lin(4096, 320, 1280); lin(4096, 960, 320)
    lin(1024, 640, 640); lin(1024, 5120, 640); lin(256, 1280, 1280); lin(256, 10240, 1280); lin(64, 1280, 1280)
    lin(77, 2560, 768); lin(77, 768, 768); lin(77, 3072, 768); lin(1, 17920, 1280)
if "misc" in which:
    conv(2, 56, 64, 64, "_r100"); conv(2, 28, 128, 128, "_r100"); conv(2, 14, 256, 256, "_r100"); conv(2, 7, 512, 512, "_r100")
    conv(1, 512, 128, 128, "_vae"); conv(1, 256, 256, 256, "_vae"); conv(1, 128, 512, 512, "_vae"); conv(1, 64, 512, 512, "_vae")
