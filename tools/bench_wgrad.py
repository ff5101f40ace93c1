"""Time of each parameter-gradient kernel (cb_wgrad.cu, and ops.linear_wgrad on cb_gemm) at SD-v1 UNet / CLIP shapes,
batch 2 at 512x512 (64^2 latent), fp16 operands: CUDA events around `--iters` launches after `--warmup` launches, best of
`--rounds`.  Prints the card name and power limit beside the numbers, and one JSON line.

    python tools/bench_wgrad.py --iters 50 --rounds 3
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
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                  # nvidia-smi missing: say so rather than guess
        return f"unknown ({e})"


def time_us(fn, iters, warmup, rounds):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = float("inf")
    for _ in range(rounds):
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        best = min(best, e0.elapsed_time(e1) * 1000.0 / iters)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_wgrad.py needs a GPU"
    from celebbasis_b200 import ops
    torch.manual_seed(0)
    f16 = torch.float16
    res = {}

    def rnd(*shape, dtype=f16):
        return torch.randn(*shape, device="cuda").to(dtype)

    # convolutions: (name, N, H, W, cin, cout, k, stride, pad); flops = 2 * N*OH*OW * cout * cin * k*k
    for name, N, H, W, cin, cout, k, s, p in [
            ("conv3x3_320_64sq", 2, 64, 64, 320, 320, 3, 1, 1), ("down3x3s2_320_64sq", 2, 64, 64, 320, 320, 3, 2, 1),
            ("conv1x1_640to320_64sq", 2, 64, 64, 640, 320, 1, 1, 0), ("conv3x3_1280_16sq", 2, 16, 16, 1280, 1280, 3, 1, 1),
            ("conv3x3_2560to1280_8sq", 2, 8, 8, 2560, 1280, 3, 1, 1)]:
        oh, ow = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
        x, dy, geo = rnd(N * H * W, cin), rnd(N * oh * ow, cout), ops.Geo(N, H, W)
        out = torch.empty(cout, cin, k, k, device="cuda")
        us = time_us(lambda: ops.conv2d_wgrad(x, geo, dy, ksize=k, stride=s, pad=p, out=out), args.iters, args.warmup,
                     args.rounds)
        res[name] = {"us": round(us, 2), "tflops": round(2.0 * N * oh * ow * cout * cin * k * k / us / 1e6, 1)}
    # linear: (name, rows, in, out)
    for name, M, K, Nn in [("linear_320to2560_8192rows", 8192, 320, 2560), ("linear_768to3072_154rows", 154, 768, 3072)]:
        x, dy = rnd(M, K), rnd(M, Nn)
        out = torch.empty(Nn, K, device="cuda")
        us = time_us(lambda: ops.linear_wgrad(x, dy, out=out), args.iters, args.warmup, args.rounds)
        res[name] = {"us": round(us, 2), "tflops": round(2.0 * M * K * Nn / us / 1e6, 1)}
    # reductions: bytes = what the kernel reads
    x = rnd(8192, 320)
    us = time_us(lambda: ops.colsum(x, groups=2), args.iters, args.warmup, args.rounds)
    res["colsum_per_image_8192x320"] = {"us": round(us, 2), "gbps": round(x.numel() * 2 / us / 1e3, 1)}
    xf, dyf = rnd(8192, 320, dtype=torch.float32), rnd(8192, 320)
    gamma, beta = torch.ones(320, device="cuda"), torch.zeros(320, device="cuda")
    geo = ops.Geo(2, 64, 64)
    _, st = ops.groupnorm(xf, geo, gamma, beta, silu=True)
    us = time_us(lambda: ops.groupnorm_affine_bwd(dyf, xf, geo, gamma, beta, st, silu=True), args.iters, args.warmup,
                 args.rounds)
    res["gn_silu_affine_bwd_8192x320"] = {"us": round(us, 2), "gbps": round(xf.numel() * 6 / us / 1e3, 1)}
    _, lst = ops.layernorm(xf, gamma, beta)
    us = time_us(lambda: ops.layernorm_affine_bwd(dyf, xf, lst), args.iters, args.warmup, args.rounds)
    res["ln_affine_bwd_8192x320"] = {"us": round(us, 2), "gbps": round(xf.numel() * 6 / us / 1e3, 1)}
    ids = torch.randint(0, 49408, (154,), device="cuda")
    dout = torch.randn(154, 768, device="cuda")
    table = torch.zeros(49408, 768, device="cuda")
    us = time_us(lambda: ops.embedding_bwd(ids, dout, 49408, out=table), args.iters, args.warmup, args.rounds)
    res["embedding_bwd_154x768"] = {"us": round(us, 2)}
    print(f"card: {card()}")
    for k, v in res.items():
        print(f"  {k:30s} {v}")
    print(json.dumps({"metric": "parameter-gradient kernel time (us, best of rounds)", "card": card(),
                      "iters": args.iters, "rounds": args.rounds, "kernels": res}))


if __name__ == "__main__":
    main()
