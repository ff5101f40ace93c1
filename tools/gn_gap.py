"""Per-node time of GroupNorm forward / backward at the UNet and VAE shapes (CUDA-graph replay), labelled with the route
each call takes: "cluster" (one launch) or "pair" (statistics + apply launches)."""
import ctypes, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from celebbasis_b200 import lib, ops
dev = torch.device("cuda:0")
_plan = (ctypes.c_int32 * 4)()


def route(N, HW, C, bytes_per_elem):
    rc = lib.load().cb_groupnorm_cluster_plan(N, HW, C, 32, bytes_per_elem, ctypes.cast(_plan, ctypes.c_void_p))
    return "cluster" if rc == 1 else "pair"

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

xn = torch.randn(4096, 320, device=dev); gm = torch.ones(320, device=dev); bt = torch.zeros(320, device=dev)
per_node(f"groupnorm 4096x320 [{route(1, 4096, 320, 4)}]", lambda: ops.groupnorm(xn, ops.Geo(1, 64, 64), gm, bt))
for (hw, c) in ((64, 320), (64, 640), (32, 640), (32, 1280), (16, 1280), (16, 2560), (8, 1280), (8, 2560), (64, 960)):
    xs = torch.randn(hw * hw, c, device=dev); g2 = torch.ones(c, device=dev); b2 = torch.zeros(c, device=dev)
    per_node(f"groupnorm+silu {hw}x{hw}x{c} [{route(1, hw * hw, c, 4)}]", lambda: ops.groupnorm(xs, ops.Geo(1, hw, hw), g2, b2, silu=True))
    y, stt = ops.groupnorm(xs, ops.Geo(1, hw, hw), g2, b2, silu=True)
    dy = torch.randn(hw * hw, c, device=dev).half()
    per_node(f"groupnorm_bwd  {hw}x{hw}x{c} [{route(1, hw * hw, c, 4 + 2)}]", lambda: ops.groupnorm_bwd(dy, xs, ops.Geo(1, hw, hw), g2, b2, stt, silu=True))

# VAE-size tensors
for (hw, c, dt) in ((512, 128, torch.float32), (256, 256, torch.float32), (256, 128, torch.float32), (128, 512, torch.float32), (128, 256, torch.float32)):
    xs = torch.randn(hw * hw, c, device=dev).to(dt); g2 = torch.ones(c, device=dev); b2 = torch.zeros(c, device=dev)
    per_node(f"groupnorm+silu {hw}x{hw}x{c} {str(dt)[6:]} [{route(1, hw * hw, c, 4)}]", lambda: ops.groupnorm(xs, ops.Geo(1, hw, hw), g2, b2, silu=True), n=10)
