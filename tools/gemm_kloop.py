"""Where the time of ONE cb_gemm launch goes, warm and cold L2: per-CTA clock stamps (desc.debug_timeline) of the step's
deep-K / small-M shapes and two VAE shapes -> setup, first tile latency, k-loop time, accumulator drain, epilogue.

The k-loop is also given per 64-deep k-iteration, in SM clocks (`kloop_clk_per_kiter`), next to the clocks the MMAs of
one k-iteration of the launch's 128 x BN tile take at the data-sheet tensor rate (`mma_clk_per_kiter`: 4096 fp16 flop
per clock and SM, the rate behind 989 TFLOP/s at 1830 MHz, so 4 * BN clocks).  The tile width and the number of
k-slices are read off the launch itself: the CTA count of the launch as tuned, and of the same descriptor with one slice.

The epilogue is split at the first 8-column unit of the stamping thread (`epi_first`, `epi_rest`): a first unit that
costs much more than the rest points at instruction fetch, an even cost per unit at the loads and stores.  Besides the
plain fp16 outputs the cases cover the epilogues the step runs: fp32 output with an fp32 residual, per-column bias,
per-image bias rows, a second destination, the GEGLU FF-in projection and one cluster split-K launch.
"""
import ctypes, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from celebbasis_b200 import lib, ops
dev = torch.device("cuda:0")
g = torch.Generator().manual_seed(0)
rnd = lambda *s: torch.randn(*s, generator=g).half().to(dev)
flush_buf = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
GHZ = 1.965
print(json.dumps({"card": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()}))


def ctas_of(desc, buf):
    buf.zero_()
    t = lib.GemmDesc.from_buffer_copy(bytes(desc))
    t.debug_timeline = buf.data_ptr()
    lib.check(lib.load().cb_gemm(ctypes.byref(t), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "ctas")
    torch.cuda.synchronize()
    return int((buf.view(-1, 8)[:, 7] != 0).sum().item())


def launch_shape(fn, m_tiles, N, buf):
    """(tile width, k-slices) of the launch fn makes, from its CTA count with and without the library's split."""
    ops.GEMM_RECORD = []
    fn()
    rec, ops.GEMM_RECORD = ops.GEMM_RECORD, None
    desc = lib.GemmDesc.from_buffer_copy(rec[-1][0])
    n = ctas_of(desc, buf)
    desc.splits = 1
    tiles = ctas_of(desc, buf)
    # untuned: of the widths giving this tile count the narrowest, which the library's cost model prefers
    bns = [desc.tile_n] if desc.tile_n else [bn for bn in (64, 128, 160, 256) if -(-N // bn) * m_tiles == tiles]
    return (bns[0] if bns else None), n // tiles


def report(name, fn, kiters_total, m_tiles, N, cold, ncta_max=8192):
    fn(); fn()
    torch.cuda.synchronize()
    buf = torch.zeros(ncta_max * 8, dtype=torch.int64, device=dev)
    bn, splits = launch_shape(fn, m_tiles, N, buf)
    buf.zero_()
    if cold:
        flush_buf.fill_(1)
        torch.cuda.synchronize()
    ops.GEMM_DEBUG_TIMELINE = buf
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); fn(); e1.record()
    torch.cuda.synchronize()
    ops.GEMM_DEBUG_TIMELINE = None
    t = buf.view(-1, 8).cpu()
    t = t[t[:, 0] > 0]
    d = lambda a, b: ((t[:, b] - t[:, a]).double() / GHZ / 1000.0)
    win = [v for k, v in ops._TUNE.items()][-1] if ops._TUNE else None
    n = t.shape[0]
    span_us = float(t[:, 7].max() - t[:, 7].min()) / 1000.0
    kiters_cta = kiters_total / splits
    kloop_clk = (t[:, 3] - t[:, 2]).double().mean().item()
    print(json.dumps({"case": name, "l2": "cold" if cold else "warm", "ctas": n, "tuned": win, "event_us": round(e0.elapsed_time(e1) * 1e3, 2),
                      "cta_start_spread_us": round(span_us, 2), "setup": round(d(0, 1).mean().item(), 2),
                      "first_full": round(d(1, 2).mean().item(), 2), "kloop": round(d(2, 3).mean().item(), 2),
                      "kloop_max": round(d(2, 3).max().item(), 2), "drain": round(d(3, 4).mean().item(), 2),
                      "epilogue": round(d(4, 5).mean().item(), 2), "epilogue_max": round(d(4, 5).max().item(), 2),
                      "epi_first": round(d(4, 6).mean().item(), 2), "epi_rest": round(d(6, 5).mean().item(), 2),
                      "cta_total": round(d(0, 5).mean().item(), 2), "cta_total_max": round(d(0, 5).max().item(), 2),
                      "kiters_total": kiters_total, "tile_n": bn, "splits": splits, "kiters_per_cta": round(kiters_cta, 2),
                      "kloop_clk_per_kiter": round(kloop_clk / kiters_cta, 1),
                      "mma_clk_per_kiter": 4 * bn if bn else None}), flush=True)


def conv_m_tiles(n, h):
    bw = min(h, 128)
    bh = min(128 // bw, h)
    bi = max(1, min(128 // (bw * bh), n))
    return -(-h // bw) * -(-h // bh) * -(-n // bi)


def both(name, fn, kiters_total, m_tiles, N):
    for cold in (False, True):
        report(name, fn, kiters_total, m_tiles, N, cold)


def conv(n, h, cin, cout, out_dtype=torch.float16, residual=False, bias=None, tag="", **kw):
    x = rnd(n * h * h, cin)
    w = ops.pack_conv_weight(torch.randn(cout, cin, 3, 3, generator=g).to(dev) * 0.02, torch.float16)
    out = torch.empty(n * h * h, cout, dtype=out_dtype, device=dev)
    res = torch.randn(n * h * h, cout, generator=g).to(dev, out_dtype) if residual else None
    b = torch.randn(*((n, cout) if bias == "image" else (cout,)), generator=g).to(dev) if bias else None
    fn = lambda: ops.conv2d(x, ops.Geo(n, h, h), w, cout, b, out=out, residual=res, bias_per_image=bias == "image", **kw)
    both(f"conv3x3 {n}x{h}x{h} {cin}->{cout}{tag}", fn, 9 * cin // 64, conv_m_tiles(n, h), cout)
    return fn


def lin(M, N, K, out_dtype=torch.float16, residual=False, bias=False, tag=""):
    x, w = rnd(M, K), rnd(N, K)
    out = torch.empty(M, N, dtype=out_dtype, device=dev)
    res = torch.randn(M, N, generator=g).to(dev, out_dtype) if residual else None
    b = torch.randn(N, generator=g).to(dev) if bias else None
    both(f"linear {M}x{N}x{K}{tag}", lambda: ops.linear(x, w, b, out=out, residual=res), K // 64, -(-M // 128), N)


def geglu(M, N, K):
    x, w, b = rnd(M, K), rnd(N, K), torch.randn(N, generator=g).to(dev)
    both(f"geglu {M}x{N}x{K}", lambda: ops.linear_geglu(x, w, b), K // 64, -(-M // 128), N)


def cluster_splitk(n, h, cin, cout):
    """the launch of conv(n, h, cin, cout) with its k-slices reduced inside a thread-block cluster"""
    x = rnd(n * h * h, cin)
    w = ops.pack_conv_weight(torch.randn(cout, cin, 3, 3, generator=g).to(dev) * 0.02, torch.float16)
    out = torch.empty(n * h * h, cout, dtype=torch.float16, device=dev)
    ops.GEMM_RECORD = []
    ops.conv2d(x, ops.Geo(n, h, h), w, cout, out=out)
    rec, ops.GEMM_RECORD = ops.GEMM_RECORD, None
    desc = lib.GemmDesc.from_buffer_copy(rec[-1][0])
    desc.tile_n, desc.splits, desc.stages, desc.cta_pair, desc.splitk_cluster = 128, 0, 0, 0, 1
    raw = bytes(desc)
    both(f"conv3x3 {n}x{h}x{h} {cin}->{cout} cluster split-K", lambda: ops._gemm(lib.GemmDesc.from_buffer_copy(raw), "cluster"),
         9 * cin // 64, conv_m_tiles(n, h), cout)


conv(1, 16, 1280, 1280); conv(1, 8, 1280, 1280); conv(1, 32, 640, 640); conv(1, 64, 320, 320); conv(1, 16, 2560, 1280)
conv(1, 128, 512, 512); conv(1, 512, 128, 128)
lin(256, 1280, 1280); lin(77, 768, 768); lin(1024, 640, 640); lin(4096, 320, 320); lin(256, 10240, 1280); lin(256, 1280, 5120)
# the epilogues the step runs besides a plain 16-bit store
conv(1, 512, 128, 128, torch.float32, residual=True, tag=" f32 out + f32 residual")
lin(4096, 320, 320, torch.float32, residual=True, tag=" f32 out + f32 residual")
lin(4096, 320, 320, bias=True, tag=" + bias")
conv(2, 32, 640, 640, bias="image", tag=" + per-image bias")
conv(1, 64, 320, 320, bias=True, tag=" + bias + D2", out2=torch.empty(64 * 64, 320, dtype=torch.float16, device=dev))
geglu(4096, 2560, 320)
cluster_splitk(1, 16, 1280, 1280)
