"""The HBM-bound pointwise, layout and celeb-basis kernels (cb_elementwise.cu, cb_embed.cu, cb_prep.cu) against the
operation each one implements, evaluated in fp64 on the same stored inputs.

Covered: every dtype pairing of every entry that takes dtypes, row pitches wider than the row, column slices and
in-place outputs, one-row and odd shapes, grid-stride loops (every family has a case past its grid cap: 32 CTAs per SM
of 256 threads for the pointwise kernels, 16 per SM in cb_prep.cu, 1184 CTAs for AdamW / DDIM, 64 per sample for
q_sample, 8 per row for ema_rows), activations past the saturation of __expf / __fdividef, softmax rows from 1 to 4096
columns with causal periods, the interleaved GEGLU layout, the 16-face unroll and the K / D tails of the celeb-basis
chain, 200 AdamW steps.

Poisoning.  Every output sits in a NaN-filled buffer: in a wider row pitch (and at a column offset) where the entry
takes a pitch, followed by a NaN guard tail everywhere.  After each call the guard must still be NaN, and pad columns
the kernel documents as zero must be exactly 0.  Every case is launched twice; both results must be the same bits.

Error model, per element:
- moves and casts (upsample forward, zero insertion, NCHW <-> NHWC, embedding gather, embed-inject forward,
  cb_convert_f32, cb_pack_conv_weight, axpby with a = 1 and no y) must equal, bit for bit, torch evaluating the same
  fp32 expression and casting with round-to-nearest-even;
- everything else must satisfy |X - X_ref| <= k * u * X_abs + floor, where u is the unit roundoff of the stored
  dtype of X (2^-24 fp32, 2^-11 fp16, 2^-8 bf16), X_abs is the same expression evaluated on absolute values (the
  quantity rounding errors scale with: |a x| + |b y| for axpby, 0.5 |x| (1 + |erf(x / sqrt 2)|) for GELU,
  0.5 (1 + |erf|) + |x pdf| for its derivative, P (|dP| + sum |dP| P) for the softmax backward, ...) and floor covers
  16-bit subnormals: 2^-25 (half the fp16 subnormal step) for fp16, 2^-126 for fp32 and bf16.  Two bounds are wider
  and say why where they are used: activations (__fdividef returns 0 once its denominator passes 2^126, so SiLU of
  x < -87.3 flushes values below 2^-119 to zero) and the timestep embedding, whose reference is fp64 cos / sin of the
  fp32 argument the reference code forms (torch's fp32 exp and product): the kernel forms its fp32 argument
  t * exp(-ln(max_period) k / half) with its own rounding, so X_abs = |X| + (2^-24 / u) (1 + |arg|).
The k of each quantity is in K below; a quantity stored in fp32 has its own k, since fp32 arithmetic errors are not
hidden under a 16-bit rounding there.
"""
import ctypes
import math
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as tF

pytestmark = pytest.mark.gpu

F16, BF16, F32, F64 = torch.float16, torch.bfloat16, torch.float32, torch.float64
DTYPES = (F16, BF16, F32)
NAN = float("nan")
U = {F32: 2.0 ** -24, F16: 2.0 ** -11, BF16: 2.0 ** -8}
FLOOR = {F32: 2.0 ** -126, F16: 2.0 ** -25, BF16: 2.0 ** -126}
CODE = {F16: 0, BF16: 1, F32: 2}
ACT_NONE, ACT_SILU, ACT_GELU, ACT_QUICK_GELU = 0, 1, 2, 3

# k of each checked quantity, (16-bit output, fp32 output): the bound is k * u of the stored dtype.  The inputs are
# seeded and the library is bit-reproducible, so every error is deterministic.  Next to each k: the worst error
# measured over every case of this file, in units of u, fp16 / bf16 / fp32, on an H100 80GB HBM3 at a 700 W power limit.
K = {
    "axpby": (1.25, 2.5),         # 1.00 / 1.00 / 1.66
    "act": (1.25, 96.0),          # 1.00 / 1.00 / 65.7   fp32: __expf(x) is off by ~|x| ulp, |x| up to 88 before it saturates
    "act_grad": (1.25, 96.0),     # 1.00 / 1.00 / 62.9
    "geglu": (1.25, None),        # 1.00 / 1.00
    "geglu_grad": (1.25, None),   # 1.00 / 1.00
    "softmax": (1.25, None),      # 0.98 / 1.00
    "softmax_grad": (1.25, None),  # 0.86 / 1.00
    "upsample_grad": (1.25, 2.5),  # 1.00 / 0.92 / 1.60
    "mse_loss": (None, 8.0),      # - / - / 4.25
    "mse_grad": (None, 4.0),      # - / - / 2.52
    "timestep": (2.0, 4.0),       # 1.31 / 0.98 / 2.51
    "affine_act": (1.25, 2.5),    # 1.00 / 0.99 / 1.56
    "face_warp": (1.25, 1.0),     # 0.93 / 0.97 / 0.61
    "l2norm": (None, 4.0),        # - / - / 2.23
    "celeb_pre": (None, 1.5),     # - / - / 0.72
    "celeb_coef": (None, 1.0),    # - / - / 0.44
    "celeb_nrm": (None, 1.0),     # - / - / 0.33
    "celeb_z": (None, 1.5),       # - / - / 0.86
    "celeb_dcoef": (None, 1.5),   # - / - / 0.94
    "celeb_dW": (None, 0.125),    # - / - / 0.016   X_abs of dW / db bounds every term of the chain rule, so it is loose
    "celeb_db": (None, 0.125),    # - / - / 0.0084
    "inject_grad": (None, 4.0),   # - / - / 2.11
    "adamw": (None, 4.0),         # - / - / 1.05
    "posterior": (None, 6.0),     # - / - / 3.25
    "q_sample": (None, 3.0),      # - / - / 1.93
    "ddim": (None, 8.0),          # - / - / 4.51
    "ema": (None, 1.5),           # - / - / 0.67
}
WORST = {}       # (quantity, dtype) -> (worst error of this run in units of u, its case)


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from celebbasis_b200 import lib
    lb = lib.load()
    assert lb.cb_device_ok() == 1, "tests must run on an sm_90 device"
    yield lb
    for (name, dt), (w, what) in sorted(WORST.items()):
        print(f"[worst] {name:14s} {dt:8s} {w:9.4f}  {what}")


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def gen(name):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()))


def st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def P(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def ok(rc, L):
    assert rc == 0, f"rc={rc}: {L.cb_last_error().decode()}"


def dn(t):
    return t.to(F64)


def rup(a, b):
    return (a + b - 1) // b * b


def bits(t):
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


# ------------------------------------------------------------------------------------------------ poisoned outputs
class Out:
    """A NaN-filled buffer holding a [rows][cols] view at column col0 of an ld-wide row (or a flat [n] view when cols is
    None), followed by a guard of spare elements.  intact(): everything outside the view still holds NaN."""

    def __init__(self, dtype, rows, cols=None, ld=None, col0=0, guard=64, fill=NAN):
        self.dtype = dtype
        if cols is None:
            self.buf = torch.full((rows + guard,), NAN, dtype=dtype, device="cuda")
            self.v = self.buf[:rows]
        else:
            ld = ld or cols
            assert col0 + cols <= ld
            n = rows * ld + guard
            self.buf = torch.full((n,), NAN, dtype=dtype, device="cuda")
            self.v = self.buf[:rows * ld].view(rows, ld)[:, col0:col0 + cols]
        if fill is not None and not (isinstance(fill, float) and math.isnan(fill)):
            self.v.copy_(fill)
        self.mask = torch.ones(self.buf.shape, dtype=torch.bool, device="cuda")
        self._view_of(self.mask).fill_(False)

    def _view_of(self, t):
        return t.as_strided(self.v.shape, self.v.stride(), self.v.storage_offset())

    def ld(self):
        return self.v.stride(0)

    def intact(self):
        return bool(torch.isnan(self.buf[self.mask]).all())


def twice(make, launch):
    """make() -> fresh list of Out (and any in/out state), launch(outs); runs twice, requires the same bits in every
    buffer and an intact guard, returns the first run's outputs."""
    a = make()
    launch(a)
    b = make()
    launch(b)
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert x.intact(), "a write landed outside the output"
        assert torch.equal(bits(x.buf), bits(y.buf)), "two launches of the same case differ"
    return a


def check(name, got, ref, absref, what, floor=None):
    """|got - ref| <= k u X_abs + floor, element-wise; records the worst (|d| - floor) / (u X_abs)."""
    dt = got.dtype
    k = K[name][1 if dt == F32 else 0]
    fl = FLOOR[dt] if floor is None else floor
    assert torch.isfinite(got).all(), f"{name} {what}: non-finite element"
    diff = (dn(got) - ref).abs()
    ex = ((diff - fl).clamp_min(0) / (U[dt] * absref)).nan_to_num(nan=0.0, posinf=math.inf)
    worst = ex.max().item() if ex.numel() else 0.0
    key = (name, str(dt).split(".")[-1])
    WORST[key] = max(WORST.get(key, (0.0, "")), (worst, what))
    assert worst <= k, f"{name} {what}: error {worst:.3f} u > {k} u"


def exact(got, want, what):
    assert got.dtype == want.dtype and got.shape == want.shape
    bad = bits(got) != bits(want.contiguous())
    if bad.any():
        i = tuple(int(x) for x in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.numel()} elements differ, first at {i}: "
                             f"{got[i].item()} != {want[i].item()}")


def values(shape, dtype, g, scale=1.0):
    return (torch.randn(shape, generator=g) * scale).to(dtype).cuda()


# ================================================================================================ axpby2d
AX_A, AX_B = 0.7, -1.3


def _axpby_case(L, xd, yd, od, rows, cols, *, with_y, a=AX_A, b=AX_B, ldx=None, ldy=None, ldo=None, col0=0, what=""):
    g = gen(f"axpby{xd}{yd}{od}{rows}{cols}{with_y}{a}")
    ldx, ldy = ldx or cols, ldy or cols
    xs = values((rows, ldx), xd, g, 3.0)
    ys = values((rows, ldy), yd, g, 3.0) if with_y else None
    x, y = xs[:, :cols], (ys[:, :cols] if with_y else None)

    def launch(o):
        ok(L.cb_axpby2d(P(x), CODE[xd], ldx, a, P(y), CODE[yd] if with_y else 0, ldy if with_y else 0, b, P(o[0].v),
                        CODE[od], o[0].ld(), rows, cols, st()), L)

    o = twice(lambda: [Out(od, rows, cols, ldo or cols, col0)], launch)[0].v
    fa, fb = float(np.float32(a)), float(np.float32(b))
    if a == 1.0 and not with_y:
        exact(o, x.float().to(od), what)
        return
    ref = fa * dn(x) + (fb * dn(y) if with_y else 0.0)
    absr = abs(fa) * dn(x).abs() + (abs(fb) * dn(y).abs() if with_y else 0.0)
    check("axpby", o, ref, absr, what)


@pytest.mark.parametrize("with_y", [False, True])
@pytest.mark.parametrize("od", DTYPES)
@pytest.mark.parametrize("yd", DTYPES)
@pytest.mark.parametrize("xd", DTYPES)
def test_axpby2d_dtypes_and_pitches(L, xd, yd, od, with_y):
    """a x + b y into a column slice of a wider buffer, with ldx, ldy and ldo all wider than cols"""
    _axpby_case(L, xd, yd, od, 37, 52, with_y=with_y, ldx=60, ldy=68, ldo=72, col0=8,
                what=f"{xd}/{yd}->{od} y={with_y}")


@pytest.mark.parametrize("od", DTYPES)
@pytest.mark.parametrize("xd", DTYPES)
def test_axpby2d_cast_is_exact(L, xd, od):
    """a = 1 and no y: the cast / strided copy (skip concat into a column slice) is round-to-nearest-even exact"""
    _axpby_case(L, xd, xd, od, 29, 40, with_y=False, a=1.0, ldx=44, ldo=96, col0=52, what=f"cast {xd}->{od}")


def test_axpby2d_one_row_and_past_grid_cap(L):
    _axpby_case(L, F16, BF16, F32, 1, 4, with_y=True, what="1x4")
    _axpby_case(L, F32, F16, BF16, 1, 4, with_y=False, what="1x4 no y")
    rows = (32 * sms() * 256 * 4) // 4000 + 3
    _axpby_case(L, F32, F16, BF16, rows, 4000, with_y=True, ldo=4008, what="past the grid cap")


@pytest.mark.parametrize("dt", DTYPES)
def test_axpby2d_in_place(L, dt):
    """out = x (the in-place gradient add of the UNet skip branch)"""
    g = gen(f"axpby_inplace{dt}")
    rows, cols, ld = 33, 44, 52
    x0 = values((rows, ld), dt, g, 2.0)
    y = values((rows, cols), F32, g, 2.0)
    outs = []
    for _ in range(2):
        x = x0.clone()
        ok(L.cb_axpby2d(P(x), CODE[dt], ld, AX_A, P(y), CODE[F32], cols, AX_B, P(x), CODE[dt], ld, rows, cols, st()), L)
        outs.append(x)
    torch.cuda.synchronize()
    assert torch.equal(bits(outs[0]), bits(outs[1]))
    exact(outs[0][:, cols:], x0[:, cols:], "pad columns of the in-place buffer")
    fa, fb = float(np.float32(AX_A)), float(np.float32(AX_B))
    check("axpby", outs[0][:, :cols], fa * dn(x0[:, :cols]) + fb * dn(y),
          abs(fa) * dn(x0[:, :cols]).abs() + abs(fb) * dn(y).abs(), f"in place {dt}")


# ================================================================================================ activations
ACT_FLOOR = {F32: 2.0 ** -119, BF16: 2.0 ** -119, F16: FLOOR[F16]}
EDGE = [0.0, -0.0, 90.0, -90.0, 88.5, -88.5, 87.0, -87.0, 60.0, -60.0, 20.0, -20.0, 5.0, -5.0, 1.0, -1.0, 1e-3, -1e-3]


def _act_input(n, dt, g):
    x = torch.randn(n, generator=g, dtype=F64) * 6.0
    x[:len(EDGE)] = torch.tensor(EDGE, dtype=F64)
    x[len(EDGE):len(EDGE) + 64] = torch.linspace(-100, 100, 64, dtype=F64)
    return x.to(dt).cuda()


def _act_ref(x, act):
    """(f(x), f_abs(x), f'(x), f'_abs(x)) in fp64"""
    if act == ACT_NONE:
        one = torch.ones_like(x)
        return x, x.abs(), one, one
    if act in (ACT_SILU, ACT_QUICK_GELU):
        c = 1.0 if act == ACT_SILU else float(np.float32(1.702))
        s = torch.sigmoid(c * x)
        y = x * s
        return y, y.abs(), s * (1 + c * x * (1 - s)), s * (1 + c * x.abs() * (1 - s))
    e = torch.erf(x / math.sqrt(2.0))
    pdf = torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    return 0.5 * x * (1 + e), 0.5 * x.abs() * (1 + e.abs()), 0.5 * (1 + e) + x * pdf, 0.5 * (1 + e.abs()) + (x * pdf).abs()


ACTS = [ACT_NONE, ACT_SILU, ACT_GELU, ACT_QUICK_GELU]


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("yd", DTYPES)
@pytest.mark.parametrize("xd", DTYPES)
def test_act_fwd(L, xd, yd, act):
    n = 12345
    x = _act_input(n, xd, gen(f"act{xd}{act}"))

    def launch(o):
        ok(L.cb_act_fwd(P(x), CODE[xd], P(o[0].v), CODE[yd], n, act, st()), L)

    y = twice(lambda: [Out(yd, n)], launch)[0].v
    ref, absr, _, _ = _act_ref(dn(x), act)
    check("act", y, ref, absr, f"act {act} {xd}->{yd}", ACT_FLOOR[yd])


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("dxd", DTYPES)
@pytest.mark.parametrize("xd", DTYPES)
@pytest.mark.parametrize("gd", DTYPES)
def test_act_bwd(L, gd, xd, dxd, act):
    n = 4097
    g = gen(f"actb{gd}{xd}{act}")
    x = _act_input(n, xd, g)
    dy = values((n,), gd, g)

    def launch(o):
        ok(L.cb_act_bwd(P(dy), CODE[gd], P(x), CODE[xd], P(o[0].v), CODE[dxd], n, act, st()), L)

    dx = twice(lambda: [Out(dxd, n)], launch)[0].v
    _, _, d, dabs = _act_ref(dn(x), act)
    check("act_grad", dx, dn(dy) * d, dn(dy).abs() * dabs, f"act' {act} {gd}/{xd}->{dxd}",
          ACT_FLOOR[dxd] * (1 + dn(dy).abs()))


@pytest.mark.parametrize("act", [ACT_SILU, ACT_GELU])
def test_act_past_grid_cap(L, act):
    n = 32 * sms() * 256 + 1001
    g = gen(f"actcap{act}")
    x = _act_input(n, F16, g)
    dy = values((n,), BF16, g)
    o = twice(lambda: [Out(BF16, n), Out(F32, n)],
              lambda o: (ok(L.cb_act_fwd(P(x), CODE[F16], P(o[0].v), CODE[BF16], n, act, st()), L),
                         ok(L.cb_act_bwd(P(dy), CODE[BF16], P(x), CODE[F16], P(o[1].v), CODE[F32], n, act, st()), L)))
    ref, absr, d, dabs = _act_ref(dn(x), act)
    check("act", o[0].v, ref, absr, "past the grid cap", ACT_FLOOR[BF16])
    check("act_grad", o[1].v, dn(dy) * d, dn(dy).abs() * dabs, "past the grid cap", ACT_FLOOR[F32] * (1 + dn(dy).abs()))


# ================================================================================================ GEGLU
def _interleave_cols(t):
    """[M][values | gates] -> the interleaved layout, through ops.glu_interleave_rows on the transpose"""
    from celebbasis_b200 import ops
    return ops.glu_interleave_rows(t.t().contiguous()).t().contiguous()


def _deinterleave_cols(t):
    M, F2 = t.shape
    g = t.reshape(M, F2 // 64, 2, 32)
    return torch.cat([g[:, :, 0].reshape(M, -1), g[:, :, 1].reshape(M, -1)], 1)


def _gelu_parts(g):
    e = torch.erf(g / math.sqrt(2.0))
    pdf = torch.exp(-0.5 * g * g) / math.sqrt(2 * math.pi)
    return (0.5 * g * (1 + e), 0.5 * g.abs() * (1 + e.abs()), 0.5 * (1 + e) + g * pdf,
            0.5 * (1 + e.abs()) + (g * pdf).abs())


GEGLU_F = [32, 1280, 5120]


@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("F", GEGLU_F)
@pytest.mark.parametrize("dt", [F16, BF16])
def test_geglu_fwd(L, dt, F, il):
    M = 37
    plain = values((M, 2 * F), dt, gen(f"geglu{dt}{F}"), 3.0)
    inp = _interleave_cols(plain) if il else plain

    def launch(o):
        ok(L.cb_geglu_fwd(P(inp), P(o[0].v), CODE[dt], M, F, il, st()), L)

    out = twice(lambda: [Out(dt, M, F)], launch)[0].v
    a, gg = dn(plain[:, :F]), dn(plain[:, F:])
    ge, gabs, _, _ = _gelu_parts(gg)
    check("geglu", out, a * ge, a.abs() * gabs, f"{dt} F={F} il={il}")


@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("F", GEGLU_F)
@pytest.mark.parametrize("gd", [F16, BF16])
@pytest.mark.parametrize("dt", [F16, BF16])
def test_geglu_bwd(L, dt, gd, F, il):
    M = 29
    g = gen(f"geglub{dt}{gd}{F}")
    plain = values((M, 2 * F), dt, g, 3.0)
    inp = _interleave_cols(plain) if il else plain
    dout = values((M, F), gd, g)

    def launch(o):
        ok(L.cb_geglu_bwd(P(dout), P(inp), P(o[0].v), CODE[dt], CODE[gd], M, F, il, st()), L)

    din = twice(lambda: [Out(gd, M, 2 * F)], launch)[0].v
    din = _deinterleave_cols(din) if il else din
    a, gg, d = dn(plain[:, :F]), dn(plain[:, F:]), dn(dout)
    ge, gabs, gp, gpabs = _gelu_parts(gg)
    what = f"{dt}/{gd} F={F} il={il}"
    check("geglu_grad", din[:, :F], d * ge, d.abs() * gabs, what + " d value")
    check("geglu_grad", din[:, F:], d * a * gp, (d * a).abs() * gpabs, what + " d gate")


# ================================================================================================ softmax
SM_COLS = [1, 3, 64, 77, 128, 129, 256, 1000, 4096]


def _scores(rows, ncols, g):
    """rows cycling through: spread up to +-150, flat, near-one-hot, mild normal"""
    s = torch.empty(rows, ncols, dtype=F64)
    for r in range(rows):
        kind = r % 4
        if kind == 0:
            s[r] = (torch.rand(ncols, generator=g, dtype=F64) * 2 - 1) * 150
        elif kind == 1:
            s[r] = 0.375
        elif kind == 2:
            s[r] = torch.randn(ncols, generator=g, dtype=F64) - 12.0
            s[r, int(torch.randint(ncols, (1,), generator=g))] = 9.0
        else:
            s[r] = torch.randn(ncols, generator=g, dtype=F64) * 3
    return s


def _softmax_ref(s, ncols, causal_period):
    rows = s.shape[0]
    lim = torch.full((rows,), ncols, dtype=torch.long)
    if causal_period:
        lim = torch.clamp(torch.arange(rows) % causal_period + 1, max=ncols)
    mask = torch.arange(ncols)[None, :] < lim[:, None]
    return torch.softmax(s.masked_fill(~mask.to(s.device), -math.inf), -1)


def _softmax_case(L, dt, ncols, ld, rows, causal_period, what):
    g = gen(f"sm{dt}{ncols}{ld}{causal_period}")
    s = torch.full((rows, ld), NAN, dtype=dt, device="cuda")
    s[:, :ncols] = _scores(rows, ncols, g).to(dt).cuda()

    def launch(o):
        ok(L.cb_softmax_fwd(P(s), P(o[0].v), CODE[dt], rows, ncols, ld, causal_period, st()), L)

    p = twice(lambda: [Out(dt, rows, ld)], launch)[0].v
    exact(p[:, ncols:], torch.zeros_like(p[:, ncols:]), f"softmax pad columns {what}")
    ref = _softmax_ref(dn(s[:, :ncols]), ncols, causal_period)
    check("softmax", p[:, :ncols], ref, ref, what)


@pytest.mark.parametrize("pad", ["round8", "plus24"])
@pytest.mark.parametrize("ncols", SM_COLS)
@pytest.mark.parametrize("dt", [F16, BF16])
def test_softmax_fwd(L, dt, ncols, pad):
    ld = rup(ncols, 8) if pad == "round8" else ncols + 24
    _softmax_case(L, dt, ncols, ld, 12, 0, f"{dt} ncols={ncols} ld={ld}")


@pytest.mark.parametrize("ncols,period", [(77, 77), (77, 20), (64, 100), (3, 5)])
@pytest.mark.parametrize("dt", [F16, BF16])
def test_softmax_fwd_causal(L, dt, ncols, period):
    """row r sees columns <= r % period; several periods per launch"""
    _softmax_case(L, dt, ncols, rup(ncols, 8), 3 * period + 2, period, f"{dt} causal ncols={ncols} period={period}")


@pytest.mark.parametrize("pad", ["round8", "plus24"])
@pytest.mark.parametrize("ncols", SM_COLS)
@pytest.mark.parametrize("gd", [F16, BF16])
@pytest.mark.parametrize("pd", [F16, BF16])
def test_softmax_bwd(L, pd, gd, ncols, pad):
    ld = rup(ncols, 8) if pad == "round8" else ncols + 24
    rows = 12
    g = gen(f"smb{pd}{gd}{ncols}{ld}")
    p = torch.full((rows, ld), NAN, dtype=pd, device="cuda")
    p[:, :ncols] = torch.softmax(_scores(rows, ncols, g), -1).to(pd).cuda()
    dp = torch.full((rows, ld), NAN, dtype=gd, device="cuda")
    dp[:, :ncols] = values((rows, ncols), gd, g, 2.0)

    def launch(o):
        ok(L.cb_softmax_bwd(P(dp), P(p), P(o[0].v), CODE[pd], CODE[gd], rows, ncols, ld, st()), L)

    ds = twice(lambda: [Out(gd, rows, ld)], launch)[0].v
    exact(ds[:, ncols:], torch.zeros_like(ds[:, ncols:]), "softmax_bwd pad columns")
    Pd, dP = dn(p[:, :ncols]), dn(dp[:, :ncols])
    ref = Pd * (dP - (dP * Pd).sum(-1, keepdim=True))
    absr = Pd * (dP.abs() + (dP.abs() * Pd).sum(-1, keepdim=True))
    check("softmax_grad", ds[:, :ncols], ref, absr, f"{pd}/{gd} ncols={ncols} ld={ld}")


# ================================================================================================ upsample / zero insert
def _nhwc(N, H, W, C, dt, g, scale=1.0):
    return values((N * H * W, C), dt, g, scale)


def _up_ref(x, N, H, W, C):
    return x.view(N, H, 1, W, 1, C).expand(N, H, 2, W, 2, C).reshape(N * 4 * H * W, C)


UP_SHAPES = [(2, 5, 7, 4), (3, 1, 3, 12), (2, 300, 300, 8)]     # the last one is past the grid cap


@pytest.mark.parametrize("shape", UP_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("dt", DTYPES)
def test_upsample2x_fwd_and_zero_insert(L, dt, shape):
    N, H, W, C = shape
    x = _nhwc(N, H, W, C, dt, gen(f"up{dt}{shape}"))
    o = twice(lambda: [Out(dt, 4 * N * H * W, C), Out(dt, 4 * N * H * W, C)],
              lambda o: (ok(L.cb_upsample2x_fwd(P(x), P(o[0].v), CODE[dt], N, H, W, C, st()), L),
                         ok(L.cb_zero_insert2x(P(x), P(o[1].v), CODE[dt], N, H, W, C, st()), L)))
    exact(o[0].v, _up_ref(x, N, H, W, C), f"upsample {dt} {shape}")
    z = torch.zeros(N, H, 2, W, 2, C, dtype=dt, device="cuda")
    z[:, :, 0, :, 0] = x.view(N, H, W, C)
    exact(o[1].v, z.reshape(-1, C), f"zero insert {dt} {shape}")


@pytest.mark.parametrize("shape", UP_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("acc", [0, 1])
@pytest.mark.parametrize("dxd", DTYPES)
@pytest.mark.parametrize("gd", DTYPES)
def test_upsample2x_bwd(L, gd, dxd, acc, shape):
    N, H, W, C = shape
    if shape == UP_SHAPES[-1] and (gd, dxd) not in ((F16, F32), (BF16, F16)):
        pytest.skip("the grid-stride case runs for two dtype pairs")
    g = gen(f"upb{gd}{dxd}{acc}{shape}")
    dy = _nhwc(N, 2 * H, 2 * W, C, gd, g)
    prior = _nhwc(N, H, W, C, dxd, g, 4.0)

    def launch(o):
        ok(L.cb_upsample2x_bwd(P(dy), CODE[gd], P(o[0].v), CODE[dxd], N, H, W, C, acc, st()), L)

    dx = twice(lambda: [Out(dxd, N * H * W, C, fill=prior if acc else NAN)], launch)[0].v
    d = dn(dy).view(N, H, 2, W, 2, C)
    ref = d.sum((2, 4)).reshape(-1, C)
    absr = d.abs().sum((2, 4)).reshape(-1, C)
    if acc:
        ref, absr = ref + dn(prior), absr + dn(prior).abs()
    check("upsample_grad", dx, ref, absr, f"{gd}->{dxd} acc={acc} {shape}")


# ================================================================================================ NCHW <-> NHWC
LAYOUT = [(2, 3, 5, 7), (1, 4, 9, 9), (3, 8, 4, 6), (1, 8, 512, 512)]      # the last one is past the grid cap


@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("shape", LAYOUT, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("dt", DTYPES)
def test_nchw_nhwc(L, dt, shape, padded):
    N, C, H, W = shape
    cpad = rup(C, 8) + 8 if padded else C
    x = torch.randn(N, C, H, W, generator=gen(f"lay{shape}")).cuda()
    o = twice(lambda: [Out(dt, N * H * W, cpad)],
              lambda o: ok(L.cb_nchw_to_nhwc(P(x), P(o[0].v), CODE[dt], N, C, H * W, cpad, st()), L))[0].v
    want = torch.zeros(N * H * W, cpad, dtype=dt, device="cuda")
    want[:, :C] = x.permute(0, 2, 3, 1).reshape(-1, C).to(dt)
    exact(o, want, f"nchw->nhwc {dt} {shape} cpad={cpad}")
    # back: the pad channels of the source hold NaN, which a read of them would carry into the output
    src = torch.full((N * H * W, cpad), NAN, dtype=dt, device="cuda")
    src[:, :C] = want[:, :C]
    back = twice(lambda: [Out(F32, N * C * H * W)],
                 lambda o: ok(L.cb_nhwc_to_nchw(P(src), CODE[dt], P(o[0].v), N, C, H * W, cpad, st()), L))[0].v
    exact(back, want[:, :C].float().view(N, H, W, C).permute(0, 3, 1, 2).reshape(-1), f"nhwc->nchw {dt} {shape}")


# ================================================================================================ MSE
@pytest.mark.parametrize("per_sample", [1, 1000, 4 * 64 * 64, 4 * 96 * 96])
@pytest.mark.parametrize("B", [1, 3, 16])
def test_mse_fwd_bwd(L, B, per_sample):
    g = gen(f"mse{B}{per_sample}")
    pred = values((B, per_sample), F32, g, 2.0)
    target = values((B, per_sample), F32, g)
    gscale = 0.37
    for want_grad in (True, False):
        def launch(o):
            ok(L.cb_mse_fwd_bwd(P(pred), P(target), P(o[0].v), P(o[1].v) if want_grad else None, B, per_sample,
                                gscale, st()), L)

        o = twice(lambda: [Out(F32, B), Out(F32, B * per_sample)], launch)
        d = dn(pred) - dn(target)
        check("mse_loss", o[0].v, (d * d).mean(1), (d * d).mean(1), f"B={B} n={per_sample}")
        if want_grad:
            ginv = float(np.float32(1.0 / float(np.float32(B) * np.float32(per_sample))))
            check("mse_grad", o[1].v.view(B, -1), 2 * d * ginv * float(np.float32(gscale)),
                  2 * (dn(pred).abs() + dn(target).abs()) * ginv * float(np.float32(gscale)), f"B={B} n={per_sample}")
        else:
            assert torch.isnan(o[1].buf).all(), "want_grad=False wrote a gradient"


# ================================================================================================ timestep embedding
@pytest.mark.parametrize("max_period", [10000.0, 777.0])
@pytest.mark.parametrize("dim", [320, 321, 2, 3])
@pytest.mark.parametrize("dt", DTYPES)
def test_timestep_embedding(L, dt, dim, max_period):
    t = torch.tensor([0, 999, 1, 500, 999, 37, 998, 250], dtype=torch.int64)
    B, half = t.numel(), dim // 2
    td = t.cuda()
    o = twice(lambda: [Out(dt, B, dim)],
              lambda o: ok(L.cb_timestep_embedding(P(td), P(o[0].v), CODE[dt], B, dim, max_period, st()), L))[0].v
    # the reference code's fp32 argument (diffusionmodules/util.py:151-171), then fp64 cos / sin of it
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=F32) / half)
    arg = (t[:, None].float() * freqs[None]).double().cuda()
    ref = torch.cat([torch.cos(arg), torch.sin(arg)], 1)
    absr = ref.abs() + (U[F32] / U[dt]) * torch.cat([1 + arg.abs(), 1 + arg.abs()], 1)
    check("timestep", o[:, :2 * half], ref, absr, f"{dt} dim={dim} max_period={max_period}")
    if dim % 2:
        exact(o[:, -1], torch.zeros(B, dtype=dt, device="cuda"), "odd dim: last column")


# ================================================================================================ channel affine + PReLU
@pytest.mark.parametrize("mode", ["affine", "slope", "both"])
@pytest.mark.parametrize("yd", DTYPES)
@pytest.mark.parametrize("xd", DTYPES)
def test_channel_affine_act(L, xd, yd, mode):
    _affine_case(L, xd, yd, mode, 37, 24, inplace=False)


def _affine_case(L, xd, yd, mode, rows, C, inplace):
    g = gen(f"aff{xd}{yd}{mode}{rows}")
    x0 = values((rows, C), xd, g, 3.0)
    scale = (torch.rand(C, generator=g) * 2 - 0.5).cuda() if mode != "slope" else None
    shift = torch.randn(C, generator=g).cuda() if mode != "slope" else None
    slope = (torch.rand(C, generator=g) - 0.5).cuda() if mode != "affine" else None

    def launch(o):
        x = o[0].v if inplace else x0
        ok(L.cb_channel_affine_act(P(x), CODE[xd], P(o[0].v), CODE[yd], P(scale), P(shift), P(slope), rows, C, st()), L)

    y = twice(lambda: [Out(yd, rows, C, fill=x0 if inplace else NAN)], launch)[0].v
    v, va = dn(x0), dn(x0).abs()
    if scale is not None:
        v, va = v * dn(scale) + dn(shift), va * dn(scale).abs() + dn(shift).abs()
    if slope is not None:
        neg = v < 0
        v = torch.where(neg, v * dn(slope), v)
        va = torch.where(neg, va * dn(slope).abs(), va)
    check("affine_act", y, v, va, f"{xd}->{yd} {mode} rows={rows} inplace={inplace}")


@pytest.mark.parametrize("dt", DTYPES)
def test_channel_affine_act_in_place_and_past_cap(L, dt):
    _affine_case(L, dt, dt, "both", 37, 24, inplace=True)
    _affine_case(L, dt, dt, "slope", 32 * sms() * 256 * 4 // 256 + 7, 256, inplace=True)


# ================================================================================================ face warp + resize
def _rot_shift(theta, dx, dy):
    from celebbasis_b200.train_step import TRANS_MATRIX
    m = torch.tensor(TRANS_MATRIX, dtype=F64).view(2, 3)
    c, s = math.cos(theta), math.sin(theta)
    r = torch.tensor([[c, -s, dx], [s, c, dy], [0, 0, 1]], dtype=F64)
    return (m @ r).float()        # the kernel takes fp32 entries


@pytest.mark.parametrize("out_hw", [112, 17])
@pytest.mark.parametrize("n_chunks", [1, 2])
@pytest.mark.parametrize("dt", DTYPES)
def test_face_warp_resize(L, dt, n_chunks, out_hw):
    B, H, W, cpad = 2, 40, 56, 8
    faces = (torch.rand(B, H, W, 3 * n_chunks, generator=gen(f"face{n_chunks}"), dtype=F32) * 2 - 1).cuda()
    m = _rot_shift(0.3, 0.25, -0.2)
    arr = (ctypes.c_float * 6)(*m.flatten().tolist())
    nimg = n_chunks * B
    o = twice(lambda: [Out(dt, nimg * out_hw * out_hw, cpad)],
              lambda o: ok(L.cb_face_warp_resize(P(faces), P(o[0].v), CODE[dt], B, H, W, n_chunks, out_hw, cpad, arr,
                                                 st()), L))[0].v
    img = torch.cat(dn(faces).permute(0, 3, 1, 2).chunk(n_chunks, 1), 0)      # image f = chunk * B + b

    def warp(im):
        grid = tF.affine_grid(dn(m)[None].expand(nimg, 2, 3).cuda(), list(im.shape), align_corners=True)
        w = tF.grid_sample(im, grid, mode="bilinear", padding_mode="zeros", align_corners=True)
        return tF.interpolate(w, size=(out_hw, out_hw), mode="bilinear", align_corners=True).permute(0, 2, 3, 1)

    ref = warp(img).reshape(-1, 3)
    # fp32 sampling coordinates are off by ~(H + W) 2^-24 pixels; one pixel step changes a value by up to 2 max|img|
    absr = warp(img.abs()).reshape(-1, 3) + (U[F32] / U[dt]) * (H + W) * 2 * img.abs().max()
    got = o.view(-1, cpad)
    check("face_warp", got[:, :3], ref, absr, f"{dt} chunks={n_chunks} out={out_hw}")
    exact(got[:, 3:], torch.zeros_like(got[:, 3:]), "face_warp pad channels")


# ================================================================================================ l2norm rows
@pytest.mark.parametrize("D", [1, 7, 255, 256, 257, 512, 4100])
def test_l2norm_rows(L, D):
    rows = 5
    x = values((rows, D), F32, gen(f"l2{D}"), 3.0)
    x[2] = 0
    o = twice(lambda: [Out(F32, rows * D)], lambda o: ok(L.cb_l2norm_rows(P(x), P(o[0].v), rows, D, st()), L))[0].v
    o = o.view(rows, D)
    xd = dn(x)
    nrm = xd.norm(dim=1, keepdim=True).clamp_min(1e-12)
    check("l2norm", o, xd / nrm, xd.abs() / nrm, f"D={D}")
    exact(o[2], torch.zeros(D, device="cuda"), "zero row")


# ================================================================================================ convert / pack
def _f32_specials(n, g):
    x = torch.randn(n, generator=g) * 100
    sp = torch.tensor([65504.0, 65520.0, 70000.0, -1e5, 3e38, 6.1e-5, 3e-6, 5.96e-8, 2.98e-8, 1e-9, -4e-7, 0.0, -0.0,
                       1e-40, 1.5, 2.0 ** -24, 2.0 ** -25 * 1.0001])
    x[:sp.numel()] = sp
    k = min(1000, n - sp.numel())
    x[sp.numel():sp.numel() + k] = torch.randn(k, generator=g) * 1e-6       # fp16 subnormal range
    return x.cuda()


@pytest.mark.parametrize("scale", [1.0, 0.37])
@pytest.mark.parametrize("dt", DTYPES)
def test_convert_f32(L, dt, scale):
    n = 16 * sms() * 256 + 4097          # past the cb_prep.cu grid cap
    x = _f32_specials(n, gen(f"conv{dt}"))
    o = twice(lambda: [Out(dt, n)], lambda o: ok(L.cb_convert_f32(P(x), P(o[0].v), CODE[dt], n, scale, st()), L))[0].v
    exact(o, (x * torch.tensor(scale, dtype=F32)).to(dt), f"convert {dt} scale={scale}")


@pytest.mark.parametrize("oscale", [False, True])
@pytest.mark.parametrize("shape", [(8, 5, 1, 1, 8, 8), (6, 3, 3, 3, 16, 8), (7, 4, 1, 3, 8, 12), (64, 48, 3, 3, 64, 48)],
                         ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("dt", DTYPES)
def test_pack_conv_weight(L, dt, shape, oscale):
    cout, cin, kh, kw, cout_pad, cin_pad = shape
    g = gen(f"pack{shape}")
    w = _f32_specials(cout * cin * kh * kw, g).view(cout, cin, kh, kw)
    sc = (torch.rand(cout, generator=g) + 0.5).cuda() if oscale else None
    rows = kh * kw * cout_pad
    o = twice(lambda: [Out(dt, rows, cin_pad)],
              lambda o: ok(L.cb_pack_conv_weight(P(w), P(o[0].v), CODE[dt], cout, cin, kh, kw, cout_pad, cin_pad, P(sc),
                                                 st()), L))[0].v
    want = torch.zeros(kh * kw, cout_pad, cin_pad, dtype=F32, device="cuda")
    ws = w * sc.view(-1, 1, 1, 1) if oscale else w
    want[:, :cout, :cin] = ws.permute(2, 3, 0, 1).reshape(kh * kw, cout, cin)
    exact(o, want.view(rows, cin_pad).to(dt), f"pack {dt} {shape} oscale={oscale}")


# ================================================================================================ embedding gather
@pytest.mark.parametrize("D", [4, 768])
def test_embedding_gather(L, D):
    V = 50
    table = values((V, D), F32, gen(f"emb{D}"))
    ids = torch.tensor([0, V - 1, 7, 0, -3, V + 5, 13, V - 1, 2 ** 40], dtype=torch.int64, device="cuda")
    n = ids.numel()
    o = twice(lambda: [Out(F32, n * D)],
              lambda o: ok(L.cb_embedding_gather(P(ids), P(table), P(o[0].v), n, D, V, st()), L))[0].v
    exact(o.view(n, D), table[ids.clamp(0, V - 1)], f"gather D={D}")     # ids outside [0, V) take the nearest row


# ================================================================================================ celeb-basis chain
SLOPE = 0.2
IN_DIM = 512


def _celeb_cases():
    Ks, Ds = [5, 7, 14, 100, 512], [100, 768, 1024]
    out = []
    for F in (1, 2, 5, 16):
        for es in (1, 2, 3):
            for i, K_ in enumerate(Ks):
                out.append((F, es, K_, Ds[(i + es) % 3], (F + es + i) % 2 == 1))
    return out


@pytest.mark.parametrize("F,es,Kc,D,neg", _celeb_cases(), ids=lambda v: str(v))
def test_celeb_chain(L, F, es, Kc, D, neg):
    """mlp_fwd -> basis_fwd -> basis_bwd -> mlp_bwd against fp64 autograd of linear, LeakyReLU(0.2), normalize and the
    basis contraction; `neg` shifts the bias so most pre-activations are negative"""
    g = gen(f"celeb{F}{es}{Kc}{D}{neg}")
    od = es * Kc
    v = values((F, IN_DIM), F32, g)
    W = values((od, IN_DIM), F32, g, 0.05)
    b = values((od,), F32, g, 0.5) - (2.0 if neg else 0.0)
    basis = values((es, Kc + 1, D), F32, g)
    dz = values((F, es, D), F32, g)
    gscale = 1.0 / 1024

    def launch(o):
        pre, coef, nrm, z, dcoef, ws, dW, db = (t.v for t in o)
        ok(L.cb_celeb_mlp_fwd(P(v), P(W), P(b), P(pre), P(coef), P(nrm), F, IN_DIM, Kc, es, SLOPE, st()), L)
        ok(L.cb_celeb_basis_fwd(P(coef), P(basis), P(z), F, es, Kc, D, st()), L)
        ok(L.cb_celeb_basis_bwd(P(dz), P(basis), P(dcoef), F, es, Kc, D, st()), L)
        ok(L.cb_celeb_mlp_bwd(P(dcoef), P(coef), P(nrm), P(pre), P(v), P(ws), P(dW), P(db), F, IN_DIM, Kc, es, SLOPE,
                              gscale, st()), L)

    o = twice(lambda: [Out(F32, F * od), Out(F32, F * od), Out(F32, F * es), Out(F32, F * es * D), Out(F32, F * od),
                       Out(F32, F * od), Out(F32, od * IN_DIM), Out(F32, od)], launch)
    pre, coef, nrm, z, dcoef, _, dW, db = (t.v for t in o)
    what = f"F={F} es={es} K={Kc} D={D} neg={neg}"
    # fp64 chain; the LeakyReLU branch follows the sign of the kernel's pre-activation (the two agree except within
    # rounding of 0, where both branches give the same value but different derivatives)
    vd, Wd, bd, Bd = dn(v), dn(W).requires_grad_(), dn(b).requires_grad_(), dn(basis)
    pre_r = vd @ Wd.t() + bd
    pos = (pre > 0).view(F, od)
    act = pre_r * torch.where(pos, 1.0, SLOPE)
    a3 = act.view(F, es, Kc)
    nrm_r = a3.norm(dim=2).clamp_min(1e-12)
    coef_r = a3 / nrm_r[..., None]
    z_r = torch.einsum("fek,ekc->fec", coef_r, Bd[:, 1:]) + Bd[:, 0]
    (z_r * dn(dz)).sum().mul(float(np.float32(gscale))).backward()
    with torch.no_grad():
        pre_a = vd.abs() @ Wd.abs().t() + bd.abs()
        act_a = (pre_a * torch.where(pos, 1.0, SLOPE)).view(F, es, Kc)
        nrm_a = act_a.norm(dim=2)
        coef_a = act_a / nrm_r[..., None] + coef_r.abs() * (nrm_a / nrm_r)[..., None]
        z_a = torch.einsum("fek,ekc->fec", coef_a, Bd[:, 1:].abs()) + Bd[:, 0].abs()
        dcoef_r = torch.einsum("fec,ekc->fek", dn(dz), Bd[:, 1:])
        dcoef_a = torch.einsum("fec,ekc->fek", dn(dz).abs(), Bd[:, 1:].abs())
        dpre_a = (dcoef_a + coef_a * (coef_a * dcoef_a).sum(2, keepdim=True)) / nrm_r[..., None]
        dpre_a = dpre_a.reshape(F, od) * torch.where(pos, 1.0, SLOPE) * gscale
        check("celeb_pre", pre.view(F, od), pre_r, pre_a, what)
        check("celeb_coef", coef.view(F, es, Kc), coef_r, coef_a, what)
        check("celeb_nrm", nrm.view(F, es), nrm_r, nrm_a, what)
        check("celeb_z", z.view(F, es, D), z_r, z_a, what)
        check("celeb_dcoef", dcoef.view(F, es, Kc), dcoef_r, dcoef_a, what)
        check("celeb_dW", dW.view(od, IN_DIM), Wd.grad, dpre_a.t() @ vd.abs(), what)
        check("celeb_db", db, bd.grad, dpre_a.sum(0), what)


def test_celeb_mlp_rejects_17_faces(L):
    buf = torch.zeros(1 << 16, device="cuda")
    n0 = L.cb_launch_count()
    assert L.cb_celeb_mlp_fwd(P(buf), P(buf), P(buf), P(buf), P(buf), P(buf), 17, IN_DIM, 8, 1, SLOPE, st()) == -1
    assert L.cb_launch_count() == n0


# ================================================================================================ embed inject
@pytest.mark.parametrize("B", [1, 4])
def test_embed_inject(L, B):
    from celebbasis_b200.train_step import build_inject_map
    T, D, reps, ph = 77, 768, 2, 42
    g = gen(f"inject{B}")
    ids = torch.randint(1000, 4000, (B, T), generator=g).numpy()
    ids[:, 5] = ph
    if B > 1:
        ids[1, 20] = ph              # a prompt naming the identity twice
        ids[3, 9] = ph
    sample = [0, 0, 2, 0][:B]        # z rows 0, 1 feed prompts 0, 1, 3 (>= 3 uses); rows 2, 3 stay unused
    m, _ = build_inject_map(ids, ph, reps, lambda b: sample[b])
    n_z = 6
    mp = torch.from_numpy(np.ascontiguousarray(m)).cuda()
    tok = values((B * T, D), F32, g)
    z = values((n_z, D), F32, g)
    pos = values((T, D), F32, g)
    dout = values((B * T, D), F32, g)
    o = twice(lambda: [Out(F32, B * T * D), Out(F32, n_z * D)],
              lambda o: (ok(L.cb_embed_inject_fwd(P(tok), P(z), P(mp), P(pos), P(o[0].v), B, T, D, st()), L),
                         ok(L.cb_embed_inject_bwd(P(dout), P(mp), P(o[1].v), n_z, B, T, D, st()), L)))
    mflat = mp.view(-1).long()
    rows = torch.arange(B * T, device="cuda")
    src = torch.where((mflat >= 0)[:, None], tok[(rows // T) * T + mflat.clamp_min(0)], z[(-(mflat + 1)).clamp_min(0)])
    exact(o[0].v.view(B * T, D), src + pos.repeat(B, 1), f"inject fwd B={B}")
    use = torch.zeros(n_z, B * T, dtype=F64, device="cuda")
    zr = mflat < 0
    use[(-(mflat[zr] + 1)), rows[zr]] = 1.0
    counts = use.sum(1)
    if B > 1:
        assert counts[:2].min() >= 3 and (counts == 0).any() and (counts == 1).any()
    dz = o[1].v.view(n_z, D)
    check("inject_grad", dz, use @ dn(dout), use @ dn(dout).abs(), f"inject bwd B={B}")
    exact(dz[counts == 0], torch.zeros_like(dz[counts == 0]), "unused z rows")


# ================================================================================================ AdamW
@pytest.mark.parametrize("gmode", ["normal", "zero", "tiny"])
@pytest.mark.parametrize("wd", [0.0, 1e-2])
@pytest.mark.parametrize("n", [1, 1000, 1184 * 256 + 5])
def test_adamw_200_steps(L, n, wd, gmode):
    lr, b1, b2, eps, steps = 1e-3, 0.9, 0.999, 1e-8, 200
    f = lambda x: float(np.float32(x))
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(f"adamw{n}{wd}{gmode}".encode()))
    p0 = torch.randn(n, generator=g, device="cuda")
    states, step_dev = [], torch.zeros(1, dtype=torch.int32, device="cuda")
    for path in ("host", "device"):
        p, m, v = p0.clone(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
        states.append((p, m, v))
    pr, mr, vr = dn(p0), torch.zeros(n, dtype=F64, device="cuda"), torch.zeros(n, dtype=F64, device="cuda")
    pa, ma, va = pr.abs(), mr.clone(), vr.clone()
    for t in range(1, steps + 1):
        if gmode == "normal":
            gr = torch.randn(n, generator=g, device="cuda") * 0.1
        else:
            gr = torch.full((n,), 0.0 if gmode == "zero" else 1e-20, device="cuda")
        for path, (p, m, v) in zip(("host", "device"), states):
            ok(L.cb_adamw_step(P(p), P(gr), P(m), P(v), n, lr, b1, b2, eps, wd, t if path == "host" else 0,
                               P(step_dev) if path == "device" else None, st()), L)
        gd = dn(gr)
        bc1, bc2s = 1 - f(b1) ** t, math.sqrt(1 - f(b2) ** t)
        mr = f(b1) * mr + (1 - f(b1)) * gd
        vr = f(b2) * vr + (1 - f(b2)) * gd * gd
        ma = f(b1) * ma + (1 - f(b1)) * gd.abs() + mr.abs()
        va = f(b2) * va + (1 - f(b2)) * gd * gd + vr
        upd = (f(lr) / bc1) * (mr / (vr.sqrt() / bc2s + f(eps)))
        pr = pr * (1 - f(lr) * f(wd)) - upd
        pa = pa * (1 - f(lr) * f(wd)) + upd.abs() + pr.abs()
    torch.cuda.synchronize()
    assert int(step_dev.item()) == steps
    for a, b in zip(states[0], states[1]):
        assert torch.equal(bits(a), bits(b)), "host-step and device-step AdamW differ"
    what = f"n={n} wd={wd} g={gmode}"
    check("adamw", states[0][0], pr, pa, what)
    check("adamw", states[0][1], mr, ma, what + " m")
    check("adamw", states[0][2], vr, va, what + " v", floor=steps * 2.0 ** -149)    # v is subnormal for 1e-20 gradients


# ================================================================================================ diffusion helpers
def test_posterior_sample(L):
    N, Cz, HW, scale = 3, 4, 4 * 37 * 41, 0.18215
    g = gen("posterior")
    mom = values((N, 2 * Cz, HW), F32, g, 2.0)
    mom[:, Cz:] = (torch.rand(N, Cz, HW, generator=g) * 100 - 60).cuda()     # logvar in [-60, 40]
    e = values((N * Cz * HW,), F32, g)
    o = twice(lambda: [Out(F32, N * Cz * HW)],
              lambda o: ok(L.cb_posterior_sample(P(mom), P(e), P(o[0].v), N, Cz, HW, scale, st()), L))[0].v
    mean, lv = dn(mom[:, :Cz]).reshape(-1), dn(mom[:, Cz:]).clamp(-30, 20).reshape(-1)
    s = float(np.float32(scale))
    std = torch.exp(0.5 * lv)
    check("posterior", o, s * (mean + std * dn(e)), s * (mean.abs() + std * dn(e).abs()), "logvar in [-60, 40]")


def _schedule():
    betas = torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=F64) ** 2
    ac = torch.cumprod(1 - betas, 0)
    return ac.sqrt().float().cuda(), (1 - ac).sqrt().float().cuda()


@pytest.mark.parametrize("per_sample", [4 * 64 * 64 + 4 * 37, 1000])
def test_q_sample(L, per_sample):
    B = 16
    g = gen(f"q{per_sample}")
    t = torch.tensor([0, 999] + torch.randperm(998, generator=g)[:B - 2].add(1).tolist(), dtype=torch.int64).cuda()
    sa, s1 = _schedule()
    x0 = values((B, per_sample), F32, g)
    nz = values((B, per_sample), F32, g)
    o = twice(lambda: [Out(F32, B * per_sample)],
              lambda o: ok(L.cb_q_sample(P(x0), P(nz), P(t), P(sa), P(s1), P(o[0].v), B, per_sample, st()), L))[0].v
    a, s = dn(sa[t])[:, None], dn(s1[t])[:, None]
    check("q_sample", o.view(B, -1), a * dn(x0) + s * dn(nz), a * dn(x0).abs() + s * dn(nz).abs(), f"n={per_sample}")


@pytest.mark.parametrize("a_prev,sigma", [(0.6, 0.2), (0.9, 0.5)], ids=["dir", "clamped-dir"])
@pytest.mark.parametrize("opt", ["none", "cond", "noise", "x0", "all"])
@pytest.mark.parametrize("n", [1001, 1184 * 256 + 333])
def test_ddim_step(L, n, opt, a_prev, sigma):
    g = gen(f"ddim{n}{opt}{a_prev}")
    x, eu, ec, nz = (values((n,), F32, g) for _ in range(4))
    use_c, use_n, use_x0 = opt in ("cond", "all"), opt in ("noise", "all"), opt in ("x0", "all")
    scale, a_t = 7.5, 0.3
    s1m = math.sqrt(1 - a_t)

    def launch(o):
        ok(L.cb_ddim_step(P(x), P(eu), P(ec) if use_c else None, P(nz) if use_n else None, P(o[0].v),
                          P(o[1].v) if use_x0 else None, n, scale, a_t, a_prev, sigma, s1m, st()), L)

    o = twice(lambda: [Out(F32, n), Out(F32, n)], launch)
    f = lambda v: float(np.float32(v))
    sg, sat, sap = f(sigma), math.sqrt(f(a_t)), math.sqrt(f(a_prev))
    dirc = math.sqrt(max(1 - f(a_prev) - sg * sg, 0.0))
    e, ea = dn(eu), dn(eu).abs()
    if use_c:
        e, ea = e + f(scale) * (dn(ec) - e), ea + f(scale) * (dn(ec).abs() + ea)
    p0 = (dn(x) - f(s1m) * e) / sat
    p0a = (dn(x).abs() + f(s1m) * ea) / sat
    xp, xpa = sap * p0 + dirc * e, sap * p0a + dirc * ea
    if use_n:
        xp, xpa = xp + sg * dn(nz), xpa + sg * dn(nz).abs()
    what = f"n={n} {opt} a_prev={a_prev} sigma={sigma}"
    check("ddim", o[0].v, xp, xpa, what)
    if use_x0:
        check("ddim", o[1].v, p0, p0a, what + " pred_x0")
    else:
        assert torch.isnan(o[1].buf).all(), "pred_x0 written though not requested"


# ================================================================================================ EMA rows
@pytest.mark.parametrize("momentum", [0.0, 1.0, 0.99, 0.5])
@pytest.mark.parametrize("idx_stride", [1, 2])
def test_ema_rows(L, idx_stride, momentum):
    B, row, n_rows = 16, 8 * 256 + 37, 10
    g = gen(f"ema{idx_stride}{momentum}")
    ids = [3, 1, 3, 0, 3, 7, -1, 1, 12, 9, 3, 0, 10, 1, 7, 3]      # repeats in several orders; -1, 10, 12 are skipped
    idx = torch.full((B, idx_stride), -5, dtype=torch.int64)
    idx[:, 0] = torch.tensor(ids)
    idx = idx.cuda()
    table0 = values((n_rows, row), F32, g)
    src = values((B, row), F32, g, 3.0)

    def launch(o):
        ok(L.cb_ema_rows(P(o[0].v), P(idx), idx_stride, P(src), B, row, n_rows, momentum, st()), L)

    t = twice(lambda: [Out(F32, n_rows * row, fill=table0.view(-1))], launch)[0].v.view(n_rows, row)
    m = float(np.float32(momentum))
    ref, ra = dn(table0).clone(), dn(table0).abs()
    for b, i in enumerate(ids):
        if 0 <= i < n_rows:
            ref[i] = m * ref[i] + (1 - m) * dn(src[b])
            ra[i] = m * ra[i] + (1 - m) * dn(src[b]).abs()
    untouched = [i for i in range(n_rows) if i not in ids]
    exact(t[untouched], table0[untouched], "rows no sample names")
    if momentum == 1.0:
        exact(t, table0, "momentum 1")
    check("ema", t, ref, ra + ref.abs() * 16, f"stride={idx_stride} m={momentum}")
