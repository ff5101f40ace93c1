"""One launch each of the hot kernels between cudaProfilerStart/Stop (for `ncu --set full --profile-from-start off`):
implicit-GEMM conv (UNet 64x64 320->320, VAE 128x128 512->512), a projection GEMM, flash attention forward and the two
backward kernels at the UNet's 4096-token / 1024-token self-attention shapes, cluster GroupNorm(+SiLU) fwd/bwd."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from celebbasis_b200 import ops
dev = torch.device("cuda:0")
g = torch.Generator().manual_seed(0)
rnd = lambda *s: torch.randn(*s, generator=g).half().to(dev)
work = []

def conv(n, h, cin, cout):
    x = rnd(n * h * h, cin)
    w = ops.pack_conv_weight(torch.randn(cout, cin, 3, 3, generator=g).to(dev) * 0.02, torch.float16)
    out = torch.empty(n * h * h, cout, dtype=torch.float16, device=dev)
    work.append(lambda: ops.conv2d(x, ops.Geo(n, h, h), w, cout, out=out))

def lin(M, N, K):
    x, w = rnd(M, K), rnd(N, K)
    out = torch.empty(M, N, dtype=torch.float16, device=dev)
    work.append(lambda: ops.linear(x, w, out=out))

def attn(nq, dh, H=8):
    C = H * dh
    q, k, v, dO = rnd(nq, C), rnd(nq, C), rnd(nq, C), rnd(nq, C)
    o = torch.empty_like(q); dq, dk, dv = torch.empty_like(q), torch.empty_like(q), torch.empty_like(q)
    st = {}
    def f():
        st["lse"] = ops.attention_fwd(q, k, v, o, images=1, heads=H, dh=dh, nq=nq, nk=nq, scale=dh ** -0.5, want_lse=True)[1]
    def b():
        ops.attention_bwd(q, k, v, o, dO, st["lse"], dq, dk, dv, images=1, heads=H, dh=dh, nq=nq, nk=nq, scale=dh ** -0.5)
    work.append(f); work.append(b)

def gn(hw, c):
    x = torch.randn(hw * hw, c, device=dev); gm = torch.ones(c, device=dev); bt = torch.zeros(c, device=dev)
    dy = rnd(hw * hw, c)
    st = {}
    def f():
        st["s"] = ops.groupnorm(x, ops.Geo(1, hw, hw), gm, bt, silu=True)[1]
    work.append(f)
    work.append(lambda: ops.groupnorm_bwd(dy, x, ops.Geo(1, hw, hw), gm, bt, st["s"], silu=True))

conv(1, 64, 320, 320); conv(1, 128, 512, 512); conv(1, 16, 1280, 1280); conv(1, 64, 640, 640); lin(4096, 2560, 320); lin(77, 768, 768)
attn(4096, 40); attn(1024, 80)
gn(64, 320); gn(32, 640)
for _ in range(2):
    for w in work:
        w()
torch.cuda.synchronize()
torch.cuda.cudart().cudaProfilerStart()
for w in work:
    w()
torch.cuda.synchronize()
torch.cuda.cudart().cudaProfilerStop()
print("done")
