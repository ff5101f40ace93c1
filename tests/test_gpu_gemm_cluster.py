"""GPU: the split-K hand-off of cb_gemm.  The k-slices of a tile are added in slice order whichever CTA arrives last and
whichever path (global workspace or thread-block cluster) reduces them, so forced configurations that only move data
must give bit-identical outputs; convolutions at the UNet's split-K shapes are checked against fp32 torch."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from celebbasis_b200 import lib
    assert lib.load().cb_device_ok() == 1, "tests must run on an sm_90 device"
    return torch.device("cuda:0")


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def rnd(*shape, dtype=torch.float16, scale=1.0, seed=[100]):
    seed[0] += 1
    g = torch.Generator().manual_seed(seed[0])
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


class forced:
    """Every cb_gemm launch inside the block runs with the given descriptor knobs."""

    def __init__(self, **kw):
        self.kw = kw

    def __enter__(self):
        from celebbasis_b200 import ops
        self.orig = orig = ops._gemm

        def run(d, what):
            for k, v in self.kw.items():
                setattr(d, k, v)
            return orig(d, what)
        ops._gemm = run

    def __exit__(self, *exc):
        from celebbasis_b200 import ops
        ops._gemm = self.orig


def counters_zero():
    from celebbasis_b200 import ops
    torch.cuda.synchronize()
    ws = ops._splitk_workspace(torch.cuda.current_device())
    return int(ws[:65536].view(torch.int32).count_nonzero().item()) == 0


@pytest.mark.parametrize("cluster", [0, 1])
@pytest.mark.parametrize("splits", [2, 5, 8])
@pytest.mark.parametrize("out_dtype", [torch.float16, torch.float32])
def test_splitk_m_tiles_are_independent(dev, cluster, splits, out_dtype):
    """An M=256 linear (two M tiles) with bias + residual equals, bit for bit, two M=128 launches of its halves."""
    from celebbasis_b200 import ops
    x, w = rnd(256, 2560), rnd(640, 2560, scale=0.05)
    bias, res = rnd(640, dtype=torch.float32), rnd(256, 640, dtype=out_dtype)
    with forced(tile_n=160, splits=splits, splitk_cluster=cluster):
        y = ops.linear(x, w, bias, out_dtype=out_dtype, residual=res)
        lo = ops.linear(x[:128].contiguous(), w, bias, out_dtype=out_dtype, residual=res[:128].contiguous())
        hi = ops.linear(x[128:].contiguous(), w, bias, out_dtype=out_dtype, residual=res[128:].contiguous())
    assert torch.equal(y, torch.cat([lo, hi]))
    assert rel(y, x.float() @ w.float().t() + bias + res.float()) < 2e-3
    assert counters_zero()


@pytest.mark.parametrize("bn,splits", [(64, 6), (128, 4), (160, 8), (128, 12)])
def test_splitk_paths_bit_identical(dev, bn, splits):
    """Workspace (L2) and cluster (DSMEM) reduction of the same k-slices give the same bits; repeated launches leave the
    per-tile arrival counters at zero."""
    from celebbasis_b200 import ops
    x, w = rnd(300, 3072), rnd(1000, 3072, scale=0.05)       # ragged M (3 M tiles) and N
    bias, res = rnd(1000, dtype=torch.float32), rnd(300, 1000, dtype=torch.float32)
    outs = []
    for cluster in (0, 1):
        with forced(tile_n=bn, splits=splits, splitk_cluster=cluster):
            for _ in range(3):
                outs.append(ops.linear(x, w, bias, out_dtype=torch.float32, residual=res))
    assert all(torch.equal(outs[0], o) for o in outs[1:])
    assert rel(outs[0], x.float() @ w.float().t() + bias + res) < 2e-3
    assert counters_zero()


@pytest.mark.parametrize("n,h,cin,cout", [(1, 16, 1280, 1280), (1, 64, 320, 320), (2, 16, 640, 1280), (1, 16, 1280, 1000)])
def test_conv_and_dgrad_at_splitk_shapes(dev, n, h, cin, cout):
    """The UNet's 16^2 and 64^2 convolutions (library split), two images at 16^2, ragged N; forward (K-major B) and dgrad
    (MN-major B, flipped taps) against fp32 torch."""
    from celebbasis_b200 import ops
    g = ops.Geo(n, h, h)
    x = rnd(g.rows, cin)
    wt = torch.randn(cout, cin, 3, 3, device="cuda") * (9 * cin) ** -0.5
    pk = ops.pack_conv_weight(wt, torch.float16)
    b = rnd(cout, dtype=torch.float32)
    y, _ = ops.conv2d(x, g, pk, cout, bias=b, out_dtype=torch.float32)
    xr = x.float().view(n, h, h, cin).permute(0, 3, 1, 2)
    ref = F.conv2d(xr, wt.half().float(), b, padding=1).permute(0, 2, 3, 1).reshape(-1, cout)
    assert rel(y, ref) < 2e-3
    dy = rnd(g.rows, cout)
    dx, _ = ops.conv2d_dgrad(dy, g, pk, cin, out_dtype=torch.float32)
    refd = F.conv_transpose2d(dy.float().view(n, h, h, cout).permute(0, 3, 1, 2), wt.half().float(), padding=1)
    assert rel(dx, refd.permute(0, 2, 3, 1).reshape(-1, cin)) < 2e-3
    assert counters_zero()
