"""Per-CTA %globaltimer timeline of one cb_gemm launch (setup / first load / main loop / epilogue)."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from celebbasis_b200 import ops
dev = torch.device("cuda:0")
g = torch.Generator().manual_seed(0)
rnd = lambda *s: torch.randn(*s, generator=g).half().to(dev)

def report(name, fn, ncta_max=4096):
    fn(); fn()
    torch.cuda.synchronize()
    buf = torch.zeros(ncta_max * 8, dtype=torch.int64, device=dev)
    ops.GEMM_DEBUG_TIMELINE = buf
    fn()
    torch.cuda.synchronize()
    ops.GEMM_DEBUG_TIMELINE = None
    t = buf.view(-1, 8).cpu()
    t = t[t[:, 0] > 0]
    GHZ = 1.965
    d = lambda a, b: ((t[:, b] - t[:, a]).double() / GHZ / 1000.0)
    g0 = t[:, 7].min()
    print(f"{name}: ctas={t.shape[0]} cta_start_spread={(t[:, 7].max() - g0) / 1000:.2f}us | per-CTA (SM clock @1.965GHz, mean/max us): "
          f"setup={d(0,1).mean():.2f} first_full={d(1,2).mean():.2f} mainloop_issue={d(2,3).mean():.2f}/{d(2,3).max():.2f} "
          f"mma_drain={d(3,4).mean():.2f} epilogue={d(4,5).mean():.2f}/{d(4,5).max():.2f} first_unit={d(4,6).mean():.2f} "
          f"total={d(0,5).mean():.2f}/{d(0,5).max():.2f}")


def conv(n, h, cin, cout):
    x = rnd(n * h * h, cin)
    w = ops.pack_conv_weight(torch.randn(cout, cin, 3, 3, generator=g).to(dev) * 0.02, torch.float16)
    out = torch.empty(n * h * h, cout, dtype=torch.float16, device=dev)
    report(f"conv {n}x{h}x{h} {cin}->{cout}", lambda: ops.conv2d(x, ops.Geo(n, h, h), w, cout, out=out))

def lin(M, N, K):
    x, w = rnd(M, K), rnd(N, K)
    out = torch.empty(M, N, dtype=torch.float16, device=dev)
    report(f"linear {M}x{N}x{K}", lambda: ops.linear(x, w, out=out))

conv(1, 64, 320, 320); conv(1, 32, 640, 640); conv(1, 8, 1280, 1280); conv(1, 128, 512, 512)
lin(4096, 320, 320); lin(4096, 2560, 320); lin(77, 768, 768); lin(1024, 640, 640)


def gaps(name, fn, n=6, ncta_max=1024):
    """Capture n back-to-back launches in one CUDA graph, each with its own timeline buffer; print kernel spans/gaps."""
    fn(); fn()
    torch.cuda.synchronize()
    bufs = [torch.zeros(ncta_max * 8, dtype=torch.int64, device=dev) for _ in range(n)]
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        for b in bufs:
            ops.GEMM_DEBUG_TIMELINE = b
            fn()
    ops.GEMM_DEBUG_TIMELINE = None
    gr.replay(); gr.replay()
    torch.cuda.synchronize()
    spans = []
    for b in bufs:
        t = b.view(-1, 8).cpu()
        t = t[t[:, 0] > 0]
        spans.append((int(t[:, 0].min()), int(t[:, 5].max()), int(t[:, 0].max())))
    base = spans[0][0]
    txt = " ".join(f"[{(s - base) / 1000:.1f}-{(e - base) / 1000:.1f} (last cta start {(ls - base) / 1000:.1f})]" for s, e, ls in spans)
    print(f"{name}: {txt}")


def conv_fn(n, h, cin, cout):
    x = rnd(n * h * h, cin)
    w = ops.pack_conv_weight(torch.randn(cout, cin, 3, 3, generator=g).to(dev) * 0.02, torch.float16)
    out = torch.empty(n * h * h, cout, dtype=torch.float16, device=dev)
    return lambda: ops.conv2d(x, ops.Geo(n, h, h), w, cout, out=out)


gaps("graph conv 64x64 320->320", conv_fn(1, 64, 320, 320))
gaps("graph conv 8x8 1280->1280", conv_fn(1, 8, 1280, 1280))
x_, w_ = rnd(4096, 320), rnd(320, 320)
o_ = torch.empty(4096, 320, dtype=torch.float16, device=dev)
gaps("graph linear 4096x320x320", lambda: ops.linear(x_, w_, out=o_))
