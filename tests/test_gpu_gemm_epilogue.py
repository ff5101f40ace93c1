"""GPU: every epilogue feature of cb_gemm against a reference built from the kernel's own raw accumulator.

The reference launch is the same descriptor with an fp32 D, alpha 1 and no epilogue feature: the same tile width and the
same k-slices, so the same products summed in the same order.  The epilogue is then restated in fp32 torch.  Outputs go
into NaN-filled buffers with a wider row pitch and spare rows, and nothing outside [M, N] (or its transpose) may change.
Without an activation, and with alpha a power of two, the outputs must equal the reference bit for bit; with an
activation (fast-math exp / erf in the kernel) they must be within 2 ulp of the output dtype, plus 2^-21 of the
pre-activation for the cancellation in 1 + erf(x) at large negative x.  A D2 affine may be a fused multiply-add: 1 ulp.
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32
MANT = {F16: 10, BF16: 7, F32: 23}
EMIN = {F16: -14, BF16: -126, F32: -126}


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from celebbasis_b200 import lib
    assert lib.load().cb_device_ok() == 1, "tests must run on an sm_90 device"
    return torch.device("cuda:0")


def rnd(*shape, dtype=F16, scale=1.0, seed=[7000]):
    seed[0] += 1
    g = torch.Generator().manual_seed(seed[0])
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


def nan_buf(rows, cols, dtype):
    return torch.full((rows, cols), float("nan"), dtype=dtype, device="cuda")


def pitch(n, dtype, extra=8):
    """a row pitch > n that keeps rows 16-byte aligned"""
    per = 16 // torch.empty((), dtype=dtype).element_size()
    return (n + per - 1) // per * per + extra


def ulp(y, dtype):
    _, e = torch.frexp(y.double())
    return torch.exp2((torch.clamp(e - 1, min=EMIN[dtype]) - MANT[dtype]).double())


def act_ref(v, act, slope):
    from celebbasis_b200 import lib
    if act == lib.CB_ACT_SILU:
        return v / (1.0 + torch.exp(-v))
    if act == lib.CB_ACT_GELU:
        return 0.5 * v * (1.0 + torch.erf(v * 0.70710678118654752))
    if act == lib.CB_ACT_QUICK_GELU:
        return v / (1.0 + torch.exp(-1.702 * v))
    if act == lib.CB_ACT_PRELU:
        return torch.where(v > 0, v, v * slope)
    return v


def dt(t):
    from celebbasis_b200 import lib
    return {F16: lib.CB_F16, BF16: lib.CB_BF16, F32: lib.CB_F32}[t]


def launch(d):
    from celebbasis_b200 import lib, ops
    ws = ops._splitk_workspace(torch.cuda.current_device())
    d.splitk_ws, d.splitk_ws_bytes = ws.data_ptr(), ws.numel()
    lib.check(lib.load().cb_gemm(ctypes.byref(d), ops._st()), "cb_gemm(epilogue sweep)")


def check_close(out, ref, pre, dtype, exact, what, tol_ulp=2):
    assert not torch.isnan(out).any(), f"{what}: unwritten elements"
    if exact:
        bad = (out.float() != ref.to(dtype).float()).sum().item()
        assert bad == 0, f"{what}: {bad} elements differ from the reference"
    else:
        diff = (out.double() - ref.double()).abs()
        tol = tol_ulp * ulp(ref, dtype) + 2.0 ** -21 * pre.double().abs()
        bad = (diff > tol).sum().item()
        assert bad == 0, f"{what}: {bad} elements off by more than {tol_ulp} ulp (max {diff.max().item():.3e})"


def check_untouched(buf, rows, cols, what):
    mask = torch.ones_like(buf, dtype=torch.bool)
    mask[:rows, :cols] = False
    assert torch.isnan(buf[mask].float()).all(), f"{what}: written outside [{rows}, {cols}]"


# (name, geometry, N, K, tile_n, d dtype, residual dtype, bias, act, alpha, d2, special, splits, cluster)
#   geometry: ("lin", M) or ("conv", images, height, width); bias: None / "col" / "image"; d2: None / "plain" / "affine";
#   special: None / "glu" / "trans" / "unaligned"
def _cases():
    from celebbasis_b200 import lib
    A = lib
    c = []
    add = lambda *a: c.append(a)
    # tile widths, output and residual dtypes, ragged M and N
    for bn in (64, 128, 160, 256):
        for n in ((72, 77, 200) if bn != 256 else (300,)):
            add(f"lin bn{bn} n{n}", ("lin", 300), n, 192, bn, F16, None, None, 0, 1.0, None, None, 0, 0)
    for m in (1, 77, 300):
        add(f"lin m{m}", ("lin", m), 200, 128, 128, F32, F32, "col", 0, 1.0, None, None, 0, 0)
    for dd in (F16, BF16, F32):
        for rd in (None, F16, BF16, F32):
            add(f"dtype d{dd} r{rd}", ("lin", 300), 200, 320, 160, dd, rd, "col", 0, 0.5, None, None, 0, 0)
    # activations (16-bit outputs), alpha, per-image bias
    for act in (A.CB_ACT_SILU, A.CB_ACT_GELU, A.CB_ACT_QUICK_GELU, A.CB_ACT_PRELU):
        add(f"act{act}", ("lin", 300), 200, 256, 128, F16, F16, "col", act, 0.25, None, None, 0, 0)
    add("act bf16", ("lin", 77), 77, 256, 64, BF16, None, "col", A.CB_ACT_SILU, 1.0, None, None, 0, 0)
    add("alpha 2", ("lin", 300), 256, 192, 256, F32, F32, None, 0, 2.0, None, None, 0, 0)
    add("bias per image lin", ("lin", 300), 200, 128, 128, F16, F16, "image", 0, 1.0, None, None, 0, 0)
    # second destination
    add("d2 plain", ("lin", 300), 200, 128, 128, F32, F32, "col", 0, 1.0, "plain", None, 0, 0)
    add("d2 affine", ("lin", 77), 77, 128, 64, F16, None, "col", A.CB_ACT_PRELU, 1.0, "affine", None, 0, 0)
    add("d2 affine conv", ("conv", 2, 20, 20), 160, 64, 160, F32, F32, "image", 0, 1.0, "affine", None, 0, 0)
    # GEGLU, transposed D, unaligned rows
    add("glu bn128", ("lin", 300), 192, 128, 128, F16, None, "col", 0, 1.0, None, "glu", 0, 0)
    add("glu bn256 nobias", ("lin", 77), 256, 192, 256, BF16, None, None, 0, 1.0, None, "glu", 0, 0)
    add("trans", ("lin", 300), 77, 128, 64, F16, None, None, 0, 1.0, None, "trans", 0, 0)
    add("trans bn128", ("lin", 200), 200, 128, 128, F32, None, "col", 0, 0.5, None, "trans", 0, 0)
    add("unaligned", ("lin", 77), 200, 128, 128, F16, F16, "col", 0, 1.0, None, "unaligned", 0, 0)
    # split-K through L2 and through a cluster
    for cl in (0, 1):
        add(f"splitk cl{cl}", ("lin", 77), 200, 2560, 64, F16, F32, "col", 0, 1.0, None, None, 4, cl)
        add(f"splitk bn128 cl{cl}", ("lin", 300), 77, 1536, 128, F32, F32, "col", A.CB_ACT_GELU, 1.0, None, None, 3, cl)
    add("splitk d2", ("lin", 77), 200, 2560, 160, F16, None, "col", 0, 1.0, "affine", None, 5, 1)
    # conv boxes spanning several rows (out_w < 128) or several images, with edge tiles
    add("conv rows", ("conv", 3, 24, 24), 200, 64, 128, F16, F16, "col", 0, 1.0, None, None, 0, 0)
    add("conv images", ("conv", 5, 6, 6), 77, 64, 64, F32, F32, "image", 0, 1.0, None, None, 0, 0)
    add("conv rect", ("conv", 2, 12, 28), 128, 128, 128, F16, None, "image", A.CB_ACT_SILU, 1.0, None, None, 0, 0)
    add("conv wide", ("conv", 1, 9, 140), 72, 64, 64, BF16, BF16, "col", 0, 1.0, None, None, 0, 0)
    return c


CASES = _cases()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_epilogue_against_raw_accumulator(dev, case):
    from celebbasis_b200 import lib, ops
    name, geo, N, K, bn, ddt, rdt, bias_kind, act, alpha, d2, special, splits, cluster = case
    glu, trans = special == "glu", special == "trans"

    def desc():
        d = lib.GemmDesc()
        d.N, d.K, d.batch, d.ab_dtype = N, K, 1, lib.CB_F16
        d.A, d.lda, d.a_major = x.data_ptr(), K, lib.CB_MAJOR_K
        d.B, d.ldb, d.b_major = w.data_ptr(), K, lib.CB_MAJOR_K
        if geo[0] == "conv":
            d.M = M
            d.conv, d.img_n, d.img_h, d.img_w, d.out_h, d.out_w = 1, n_img, oh, ow, oh, ow
            d.kh = d.kw = 3
            d.stride, d.pad_top, d.pad_left, d.b_tap_rows = 1, 1, 1, N
        else:
            d.M = M
        d.tile_n, d.splits, d.splitk_cluster, d.alpha = bn, splits, cluster, 1.0
        return d

    if geo[0] == "conv":
        _, n_img, oh, ow = geo
        M, rows_per_img = n_img * oh * ow, oh * ow
        x, w = rnd(M, K), rnd(9 * N, K, scale=0.05)
    else:
        M, rows_per_img = geo[1], 50
        x, w = rnd(M, K), rnd(N, K, scale=0.1)

    # raw accumulator of the same launch
    S = torch.zeros(M, N, dtype=F32, device=dev)
    d = desc()
    d.D, d.d_dtype, d.ldd = S.data_ptr(), lib.CB_F32, N
    if glu:
        d.splits = 1
    launch(d)

    d = desc()
    d.alpha, d.act = alpha, act
    v = S * alpha
    if bias_kind == "col":
        bias = rnd(N, dtype=F32)
        d.bias, d.ldbias = bias.data_ptr(), N
        v = v + bias
    elif bias_kind == "image":
        nb = (M + rows_per_img - 1) // rows_per_img
        ldb = N + 12
        bias = rnd(nb, ldb, dtype=F32)
        d.bias, d.ldbias, d.bias_row_div = bias.data_ptr(), ldb, rows_per_img
        v = v + bias[torch.arange(M, device=dev) // rows_per_img, :N]
    pre = v
    slope = None
    if act == lib.CB_ACT_PRELU:
        slope = rnd(N, dtype=F32, scale=0.2)
        d.act_param = slope.data_ptr()
    v = act_ref(v, act, slope)
    if rdt is not None:
        ldr = pitch(N, rdt, 16)
        R = rnd(M, ldr, dtype=rdt)
        d.R, d.r_dtype, d.ldr = R.data_ptr(), dt(rdt), ldr
        v = v + R[:, :N].float()
    exact = act == lib.CB_ACT_NONE

    if glu:
        D = nan_buf(M + 3, pitch(N, ddt), ddt)
        D2 = nan_buf(M + 3, pitch(N // 2, ddt), ddt)
        d.D, d.d_dtype, d.ldd = D.data_ptr(), dt(ddt), D.shape[1]
        d.D2, d.d2_dtype, d.ldd2, d.glu = D2.data_ptr(), dt(ddt), D2.shape[1], 1
        launch(d)
        torch.cuda.synchronize()
        check_close(D[:M, :N], v, pre, ddt, True, "glu D")
        check_untouched(D, M, N, "glu D")
        val = v.view(M, N // 64, 2, 32)
        u = (val[:, :, 0] * act_ref(val[:, :, 1], lib.CB_ACT_GELU, None)).reshape(M, N // 2)
        check_close(D2[:M, :N // 2], u, val[:, :, 1].reshape(M, N // 2), ddt, False, "glu D2")
        check_untouched(D2, M, N // 2, "glu D2")
        return

    if trans:
        D = nan_buf(N + 3, pitch(M, ddt), ddt)
        d.D, d.d_dtype, d.ldd, d.d_transposed = D.data_ptr(), dt(ddt), D.shape[1], 1
    else:
        ldd = N + 1 if special == "unaligned" else pitch(N, ddt)
        D = nan_buf(M + 3, ldd, ddt)
        d.D, d.d_dtype, d.ldd = D.data_ptr(), dt(ddt), ldd
    D2 = None
    if d2 is not None:
        d2dt = BF16 if ddt == F16 else F16
        D2 = nan_buf(M + 3, pitch(N, d2dt), d2dt)
        d.D2, d.d2_dtype, d.ldd2 = D2.data_ptr(), dt(d2dt), D2.shape[1]
        if d2 == "affine":
            sc, sh = rnd(N, dtype=F32), rnd(N, dtype=F32)
            d.d2_scale, d.d2_shift = sc.data_ptr(), sh.data_ptr()
    launch(d)
    torch.cuda.synchronize()
    if trans:
        check_close(D[:N, :M], v.t(), pre.t(), ddt, exact, "D^T")
        check_untouched(D, N, M, "D^T")
    else:
        check_close(D[:M, :N], v, pre, ddt, exact, "D")
        check_untouched(D, M, N, "D")
    if D2 is not None:
        ref2 = v if d2 == "plain" else (v.double() * sc.double() + sh.double()).float()
        check_close(D2[:M, :N], ref2, pre, d2dt, exact and d2 == "plain", "D2", tol_ulp=1 if exact else 2)
        check_untouched(D2, M, N, "D2")
