"""GPU: the flash-attention kernels (cb_attention_fwd, cb_attention_bwd, cb_attention_bwd_dq) and the routes of
unet_engine._Attn against softmax(Q K^T * scale [+ top-left causal mask]) V evaluated in fp64 on the same 16-bit inputs.

What a full-size training step never runs is covered here: every head-dim instantiation (k16 steps 1..8) in fp16 and
bf16, one-row and ragged lengths on both sides of the 64 / 128 tile edges, more key blocks than the 4-stage K/V ring,
several images with ragged nq / nk, causal tiles with nq > 128 and nq != nk, the lazy rescale of the running maximum,
scaled scores far beyond fp32's exp range, near-one-hot and exactly flat rows.

Every output goes into a NaN-filled buffer with a wider row pitch (q / k / v and the gradients are column slices of
fused buffers, as the engines keep them).  After each call: the result matches the reference; the columns
[nk, round_up(nk, 8)) of P and dS are exactly 0; in O, dQ, dK and dV every element outside rows x [0, heads * d) still
holds NaN.  P and dS columns past round_up(nk, 8) are not checked: the kernels may zero them up to the end of the last
visited key block.

Error measure.  u is the unit roundoff of the operand dtype (2^-11 fp16, 2^-8 bf16).  Every element of an output X is
checked against the fp64 reference with

    |X - X_ref| <= k * u * X_abs + floor

where X_abs is the expression of X evaluated on absolute values -- the quantity rounding errors scale with:
    O: P |V|        dV: P^T |dO|        dS: P o (|dO| |V|^T + rowsum(|dO| o P |V|)) * scale
    P: P            dQ: dS_abs |K|      dK: dS_abs^T |Q|
and floor covers values below the 16-bit normal range.  Storing one costs up to f absolute: f = 2^-25 (half the fp16
subnormal step) in fp16, f = 2^-126 (fp32's flush-to-zero threshold, which bf16 shares) in bf16.  The kernels store
P and dS in 16 bits before the MMA that consumes them, so f is carried through that product over the keys (queries)
each row sees: floor = f for P and dS, f (1 + M |V|) for O, f (1 + M |K|) for dQ, f (1 + M^T |Q|) for dK and
f (1 + M^T |dO|) for dV, with M the 0/1 mask of visible keys.  An element-wise bound catches an error that is
confined to one row or one key, which a norm-wise ratio over the whole tensor averages away.  It is also the only
meaningful bound for near-one-hot rows, where dS is a difference of nearly equal terms: there the error is bounded
against |P| (|dP| + |delta|), not against ||dS||.  lse is compared by absolute error over max(1, |lse|).
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
FLOOR = {torch.float16: 2.0 ** -25, torch.bfloat16: 2.0 ** -126}

# k of each checked quantity: the tolerance is k * u for fp16 and bf16 alike.  The inputs are seeded and the library is
# bit-reproducible, so every error is deterministic.  Next to each k: the worst error measured over every case of this
# file (kernels and _Attn routes), in units of u, fp16 / bf16, on an H100 80GB HBM3.
K = {
    "o": 3.0,       # 1.48 / 1.56   O, one- and two-pass forward and every _Attn route
    "lse": 0.003,   # 0.0011 / 0.0001   |lse - lse_ref| / max(1, |lse_ref|): fp32 arithmetic on exact inputs
    "p": 2.0,       # 0.996 / 0.996   exported probabilities (two-pass forward)
    "dq": 1.0,      # 0.32 / 0.39
    "dk": 1.5,      # 0.58 / 0.69
    "dv": 4.0,      # 1.84 / 1.96
    "ds": 1.5,      # 0.65 / 0.67   exported dS (attention_bwd_dq)
}


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from celebbasis_b200 import lib
    assert lib.load().cb_device_ok() == 1, "tests must run on an sm_90 device"
    return torch.device("cuda:0")


def _round_up(a, b):
    return (a + b - 1) // b * b


# ------------------------------------------------------------------------------------------------ buffers and inputs
def _poisoned(dtype, *shapes):
    """NaN-filled buffer of max(rows) + 2 rows and sum(cols) + 24 columns, and one view per (rows, cols) shape: rows
    [1, rows + 1), consecutive column slices from column 8.  Returns the views and a check that everything outside them
    still holds NaN."""
    rows = max(r for r, _ in shapes)
    buf = torch.full((rows + 2, sum(c for _, c in shapes) + 24), float("nan"), dtype=dtype, device="cuda")
    outside = torch.ones(buf.shape, dtype=torch.bool, device="cuda")
    views, c0 = [], 8
    for r, c in shapes:
        views.append(buf[1:r + 1, c0:c0 + c])
        outside[1:r + 1, c0:c0 + c] = False
        c0 += c
    return views, lambda: bool(torch.isnan(buf[outside]).all())


def _inputs(dtype, images, heads, nq, nk, d, seed):
    """q / k / v as column slices of one fused [rows][3C + 8] projection buffer, dO as a slice of a [rows][C + 8] one."""
    C = heads * d
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(images * max(nq, nk), 3 * C + 8, generator=g).to(dtype).cuda()
    dO = torch.randn(images * nq, C + 8, generator=g).to(dtype).cuda()
    return qkv[:images * nq, :C], qkv[:images * nk, C:2 * C], qkv[:images * nk, 2 * C:3 * C], dO[:, :C]


def _reference(q, k, v, dO, *, images, heads, nq, nk, d, scale, causal):
    """fp64 softmax(Q K^T * scale) V, its fp64 autograd gradients, dS = P o (dP - rowsum(dO o O)) * scale, the
    absolute-value expression of each and its floor.  Returns {name: (value, value_abs, floor)} in the kernels' layouts
    (lse: the value alone)."""
    f = FLOOR[q.dtype]
    sp = lambda t, n: t.double().reshape(images, n, heads, d).permute(0, 2, 1, 3)
    Q, Kt, V = sp(q, nq).requires_grad_(), sp(k, nk).requires_grad_(), sp(v, nk).requires_grad_()
    G = sp(dO, nq)
    s = Q @ Kt.transpose(-1, -2) * scale
    if causal:
        s = s.masked_fill(torch.ones(nq, nk, dtype=torch.bool, device=s.device).triu_(1), float("-inf"))
    P = torch.softmax(s, -1)
    O = P @ V
    O.backward(G)
    with torch.no_grad():
        s, P, O = s.detach(), P.detach(), O.detach()
        aQ, aK, aV, aG = Q.detach().abs(), Kt.detach().abs(), V.detach().abs(), G.abs()
        M = torch.isfinite(s).double()            # the keys each query sees
        Oa = P @ aV
        dS = P * (G @ V.detach().transpose(-1, -2) - (G * O).sum(-1, keepdim=True)) * scale
        dSa = P * (aG @ aV.transpose(-1, -2) + (aG * Oa).sum(-1, keepdim=True)) * scale
        back = lambda t, n: t.permute(0, 2, 1, 3).reshape(images * n, heads * d)
        flat = lambda t: t.reshape(images * heads * nq, nk)
        return {
            "o": (back(O, nq), back(Oa, nq), f * (1 + back(M @ aV, nq))),
            "lse": torch.logsumexp(s, -1).reshape(-1),
            "p": (flat(P), flat(P), f),
            "dq": (back(Q.grad, nq), back(dSa @ aK, nq), f * (1 + back(M @ aK, nq))),
            "dk": (back(Kt.grad, nk), back(dSa.transpose(-1, -2) @ aQ, nk), f * (1 + back(M.transpose(-1, -2) @ aQ, nk))),
            "dv": (back(V.grad, nk), back(P.transpose(-1, -2) @ aG, nk), f * (1 + back(M.transpose(-1, -2) @ aG, nk))),
            "ds": (flat(dS), flat(dSa), f),
        }


def _excess(name, got, ref):
    """max over elements of (|X - X_ref| - floor) / (u X_abs): the k this output needs (0 if every error is under the
    floor, inf if an element with X_abs = 0 is off by more than the floor)."""
    value, absval, floor = ref
    diff = (got.double() - value).abs()
    assert torch.isfinite(diff).all(), f"{name}: non-finite element"
    ex = (diff - floor).clamp_min(0) / (U[got.dtype] * absval)
    return ex.nan_to_num(nan=0.0, posinf=math.inf).max().item()


def _lse_excess(got, ref, dtype):
    assert torch.isfinite(got).all(), "lse: non-finite element"
    return ((got.double() - ref).abs() / ref.abs().clamp_min(1.0)).max().item() / U[dtype]


def _assert_within(errs, table):
    bad = {n: (round(e, 4), table[n]) for n, e in errs.items() if not e <= table[n]}
    assert not bad, f"error / u above k: {bad}"


# ------------------------------------------------------------------------------------------------ kernel calls
def _fwd_with_p(q, k, v, o, lse, P, *, images, heads, nq, nk, d, scale, causal):
    """Two-pass forward through the C ABI with a caller-owned P buffer (row pitch P.shape[1])."""
    from celebbasis_b200 import lib
    L = lib.load()
    code = lib.CB_BF16 if q.dtype == torch.bfloat16 else lib.CB_F16
    lib.check(L.cb_attention_fwd(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
                                 o.data_ptr(), o.stride(0), lse.data_ptr(), P.data_ptr(), P.shape[1], code, images, heads,
                                 nq, nk, d, scale, 1 if causal else 0, torch.cuda.current_stream().cuda_stream),
              "cb_attention_fwd")


def _run_kernels(q, k, v, dO, *, images, heads, nq, nk, d, scale, causal):
    """One call of each entry point into NaN-poisoned buffers with wider row pitches: the one-pass forward (O, lse), the
    two-pass forward (O, lse, P), attention_bwd (dq, dk, dv) and attention_bwd_dq (dq, dS).  Asserts that nothing was
    written outside the outputs and that the P / dS columns [nk, round_up(nk, 8)) are zero."""
    from celebbasis_b200 import ops
    dt, C = q.dtype, heads * d
    kw = dict(images=images, heads=heads, nq=nq, nk=nk, scale=scale, causal=causal)
    ldr = _round_up(nk, 8)
    ldw = ldr + 72                        # P / dS row pitch wider than the kernels need
    (o,), o_ok = _poisoned(dt, (images * nq, C))
    _, lse = ops.attention_fwd(q, k, v, o, dh=d, want_lse=True, **kw)
    (o2,), o2_ok = _poisoned(dt, (images * nq, C))
    lse2 = torch.full((images * heads * nq,), float("nan"), dtype=torch.float32, device="cuda")
    P = torch.full((images * heads * nq, ldw), float("nan"), dtype=dt, device="cuda")
    _fwd_with_p(q, k, v, o2, lse2, P, d=d, **kw)
    (dq, dk, dv), g_ok = _poisoned(dt, (images * nq, C), (images * nk, C), (images * nk, C))
    ops.attention_bwd(q, k, v, o, dO, lse, dq, dk, dv, dh=d, **kw)
    (dq2,), dq2_ok = _poisoned(dt, (images * nq, C))
    dS = torch.full((images * heads * nq, ldw), float("nan"), dtype=dt, device="cuda")
    ops.attention_bwd_dq(q, k, v, o, dO, lse, dq2, dS, dh=d, **kw)
    torch.cuda.synchronize()
    for name, ok in (("O", o_ok), ("O (two-pass)", o2_ok), ("dq/dk/dv", g_ok), ("dq (bwd_dq)", dq2_ok)):
        assert ok(), f"{name}: written outside rows x [0, heads * d)"
    assert bool((P[:, nk:ldr] == 0).all()), "P: columns [nk, round_up(nk, 8)) not zero"
    assert bool((dS[:, nk:ldr] == 0).all()), "dS: columns [nk, round_up(nk, 8)) not zero"
    return {"o": o, "lse": lse, "o2": o2, "lse2": lse2, "p": P[:, :ldr], "dq": dq, "dk": dk, "dv": dv, "dq2": dq2,
            "ds": dS[:, :ldr]}


def _check_kernels(dtype, images, heads, nq, nk, d, *, causal=False, scale=None, seed=0, design=None, repeat=False):
    """Runs every entry point on one shape and returns {quantity: error / u}; `design(q, k)` may rewrite q and k."""
    scale = d ** -0.5 if scale is None else scale
    shape = dict(images=images, heads=heads, nq=nq, nk=nk, d=d)
    q, k, v, dO = _inputs(dtype, images, heads, nq, nk, d, seed=seed)
    if design is not None:
        design(q, k)
    kw = dict(shape, scale=scale, causal=causal)
    ref = _reference(q, k, v, dO, **kw)
    got = _run_kernels(q, k, v, dO, **kw)
    # dQ of attention_bwd_dq is the same MODE 0 launch as in attention_bwd: exporting dS must not change it
    assert torch.equal(got["dq2"], got["dq"])
    if repeat:   # no atomics, fixed summation order: a second run gives the same bits
        again = _run_kernels(q, k, v, dO, **kw)
        for name in got:
            assert torch.equal(got[name], again[name]), f"{name} differs between two identical calls"
    return {
        "o": max(_excess("o", got["o"], ref["o"]), _excess("o2", got["o2"], ref["o"])),
        "lse": max(_lse_excess(got["lse"], ref["lse"], dtype), _lse_excess(got["lse2"], ref["lse"], dtype)),
        "p": _excess("p", got["p"][:, :nk], ref["p"]),
        "dq": _excess("dq", got["dq"], ref["dq"]),
        "dk": _excess("dk", got["dk"], ref["dk"]),
        "dv": _excess("dv", got["dv"], ref["dv"]),
        "ds": _excess("ds", got["ds"][:, :nk], ref["ds"]),
    }


DTYPES = [pytest.param(torch.float16, id="f16"), pytest.param(torch.bfloat16, id="bf16")]


# ------------------------------------------------------------------------------------------------ A + E: instantiations
# KS = ceil(d / 16) = 1..8; d = 24 / 72 / 120 leave the last k16 step half filled in the first / second 64-column box,
# d = 72..120 fill the second box only partly.  One shape ragged in nq and nk, non-causal; every call runs twice.
_A = [(dt, d) for dt in (torch.float16, torch.bfloat16) for d in (8, 16, 24, 32, 48, 64, 72, 96, 112, 120, 128)] + \
     [(torch.bfloat16, 40), (torch.bfloat16, 80)]


@pytest.mark.parametrize("dtype,d", _A, ids=[f"{'bf16' if dt == torch.bfloat16 else 'f16'}-d{d}" for dt, d in _A])
def test_head_dim_instantiations(dev, dtype, d):
    _assert_within(_check_kernels(dtype, 2, 3, 200, 330, d, seed=d, repeat=True), K)


# ------------------------------------------------------------------------------------------------ B: length edges
# nq on both sides of the 64-row warpgroup and 128-row CTA edges, nk from one key to more key blocks than the 4-stage ring
# (577 = 10 blocks: the ring phase wraps twice, four times in two-pass mode), three images so that a read or write
# across an image boundary shows.
_B_PAIRS = [(1, 1), (1, 577), (4, 9), (16, 8), (63, 63), (64, 64), (65, 65), (127, 255), (128, 256), (129, 257),
            (65, 320), (128, 577), (63, 77), (129, 1), (4, 64), (127, 65)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("d", [32, 64])
@pytest.mark.parametrize("nq,nk", _B_PAIRS)
def test_length_edges(dev, nq, nk, d, dtype):
    _assert_within(_check_kernels(dtype, 3, 2, nq, nk, d, seed=nq * 1000 + nk), K)


# the tiny workload's attention: 8 heads over 64 / 128 / 256 channels at 8^2 / 4^2 / 2^2 tokens, self and 77-key cross
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("d,n", [(8, 64), (16, 16), (32, 4)])
@pytest.mark.parametrize("cross", [False, True], ids=["self", "cross77"])
def test_tiny_workload_shapes(dev, d, n, cross, dtype):
    _assert_within(_check_kernels(dtype, 3, 8, n, 77 if cross else n, d, seed=d), K)


# ------------------------------------------------------------------------------------------------ C: causal
# top-left aligned mask (key <= query).  nq > 128 with P export is where a query tile visits fewer key blocks than P has.
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("nq,nk", [(1, 1), (65, 7), (129, 129), (300, 300), (200, 330), (330, 200)])
def test_causal(dev, nq, nk, dtype):
    _assert_within(_check_kernels(dtype, 2, 2, nq, nk, 64, causal=True, seed=nq + nk), K)


# ------------------------------------------------------------------------------------------------ D: wide score ranges
def _wide_scores(q, k, *, images, heads, nq, nk, d, seed):
    """Rewrites q and k so that consecutive query rows cycle through six regimes inside every 128-row tile (scale 1/8):
    (i)   key block j scores 7 j higher than block j - 1 (10.1 in log2 units): the running maximum moves, and O and l are
          rescaled, on every block;
    (ii)  the row maximum is key 0 (+2 over the rest of block 0), later blocks 7 j lower;
    (iii) the maximum lies only in the last key block (+10);
    (iv)  scores spread over [-150, 150]: exp without the maximum subtracted overflows fp32;
    (v)   one key 15 above the rest: nearly one-hot (the hot key is in block 0, block 3 or the last block);
    (vi)  q = 0: exactly flat.
    The structure lives in channels 0..7; the other channels carry N(0, 1/4) noise in regimes (i)..(v)."""
    g = torch.Generator().manual_seed(seed)
    Qh = torch.randn(images, nq, heads, d, generator=g) * 0.5
    Kh = torch.randn(images, nk, heads, d, generator=g) * 0.5
    Qh[..., :8] = 0
    Kh[..., :8] = 0
    blk = torch.arange(nk) // 64
    Kh[..., 0] = blk.to(Kh.dtype)[None, :, None]
    Kh[:, 0, :, 1] = 1
    Kh[:, blk == blk[-1], :, 2] = 1
    Kh[..., 3] = torch.randint(-32, 33, (images, nk, heads), generator=g) / 32
    for j, hot in enumerate((37, 200, nk - 1)):
        Kh[:, hot, :, 5 + j] = 1
    for r in range(nq):
        regime = r % 6
        if regime == 0:
            Qh[:, r, :, 0] = 56
        elif regime == 1:
            Qh[:, r, :, 0], Qh[:, r, :, 1] = -56, 16
        elif regime == 2:
            Qh[:, r, :, 2] = 80
        elif regime == 3:
            Qh[:, r, :, 3] = 1200
        elif regime == 4:
            Qh[:, r, :, 5 + (r // 6) % 3] = 120
        else:
            Qh[:, r] = 0
    q.copy_(Qh.reshape(images * nq, heads * d))
    k.copy_(Kh.reshape(images * nk, heads * d))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("d", [64, 128])
def test_wide_score_ranges(dev, d, dtype):
    shape = dict(images=1, heads=2, nq=200, nk=333, d=d)        # 6 key blocks, two query tiles
    design = lambda q, k: _wide_scores(q, k, seed=d, **shape)
    _assert_within(_check_kernels(dtype, *shape.values(), scale=0.125, seed=d, design=design), K)


# ------------------------------------------------------------------------------------------------ F: _Attn routes
# (route, nq, nk, dh, FLASH, FLASH_BWD, causal, state the forward must return)
_ROUTES = [
    ("flash-lse", 200, 256, 64, True, True, False, "lse"),
    ("p+lse", 200, 255, 64, True, True, False, "p+lse"),
    ("materialised", 200, 255, 64, False, True, False, "P"),
    ("materialised", 200, 256, 64, False, True, False, "P"),
    ("materialised-d160", 200, 255, 160, True, True, False, "P"),
    ("materialised-d160", 200, 256, 160, True, True, False, "P"),
    ("flash-fwd-P", 200, 255, 64, True, False, False, "P"),
    ("flash-fwd-P", 200, 256, 64, True, False, False, "P"),
    ("p+lse-causal", 200, 200, 64, True, True, True, "p+lse"),
    ("flash-fwd-P-causal", 200, 200, 64, True, False, True, "P"),
]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("route,nq,nk,dh,flash,flash_bwd,causal,kind", _ROUTES,
                         ids=[f"{r[0]}-nk{r[2]}-d{r[3]}" for r in _ROUTES])
def test_attn_routes(dev, route, nq, nk, dh, flash, flash_bwd, causal, kind, dtype):
    """unet_engine._Attn forward + backward on each of its routes.  Where the forward keeps P, it is handed memory that
    held NaN, so a P element the forward leaves unwritten reaches dV."""
    from celebbasis_b200.unet_engine import _Attn
    images, heads, scale = 2, 2, dh ** -0.5
    shape = dict(images=images, heads=heads, nq=nq, nk=nk)
    C = heads * dh
    q, k, v, dO = _inputs(dtype, images, heads, nq, nk, dh, seed=nk + dh)
    ref = _reference(q, k, v, dO, d=dh, scale=scale, causal=causal, **shape)
    saved = (_Attn.FLASH, _Attn.FLASH_BWD)
    try:
        _Attn.FLASH, _Attn.FLASH_BWD = flash, flash_bwd
        (o,), o_ok = _poisoned(dtype, (images * nq, C))
        dirty = torch.full((images * heads * nq, _round_up(nk, 8)), float("nan"), dtype=dtype, device="cuda")
        dirty_ptr = dirty.data_ptr()
        del dirty                         # the caching allocator hands this block to the next allocation of its size
        state = _Attn.fwd(q, k, v, images=images, heads=heads, dh=dh, nq=nq, nk=nk, scale=scale, out=o, causal=causal)
        got_kind = state[0] if isinstance(state, tuple) else "P"
        assert got_kind == kind, (got_kind, kind)
        if flash and kind != "lse":
            P = state[1] if isinstance(state, tuple) else state
            assert P.data_ptr() == dirty_ptr, "P did not get the NaN-filled block"
        (dq, dk, dv), g_ok = _poisoned(dtype, (images * nq, C), (images * nk, C), (images * nk, C))
        _Attn.bwd(dO, q, k, v, state, images=images, heads=heads, dh=dh, nq=nq, nk=nk, scale=scale, dq=dq, dk=dk, dv=dv)
        torch.cuda.synchronize()
    finally:
        _Attn.FLASH, _Attn.FLASH_BWD = saved
    assert o_ok() and g_ok(), "written outside rows x [0, heads * dh)"
    _assert_within({n: _excess(n, t, ref[n]) for n, t in (("o", o), ("dq", dq), ("dk", dk), ("dv", dv))}, K)
