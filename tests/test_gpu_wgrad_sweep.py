"""The parameter-gradient kernels (cb_wgrad.cu: cb_conv_wgrad, cb_colsum, cb_groupnorm_affine_bwd,
cb_layernorm_affine_bwd, cb_embedding_bwd; ops.linear_wgrad over cb_gemm) against the same sums evaluated in fp64 on
the same stored inputs.

Cases: every UNet convolution geometry (3x3 stride 1, the 3x3 stride-2 Downsample with padding 1, 1x1 skip /
proj_in / proj_out) at the SD-v1 channel counts, batches 1-4, N*H*W that are not multiples of the 64-row k-chunk, Cin /
Cout off the 128 x 128 tile, fp16 and bf16; the UNet and CLIP linear shapes; GroupNorm affine gradients with and without
the fused SiLU over every x / dy dtype pair; LayerNorm affine gradients; bias, per-image and position-embedding column
sums; the token-embedding gradient with repeated and out-of-range ids.

Bounds, elementwise, with u = 2^-24 and T the sum of the magnitudes of the terms that form the output (evaluated in
fp64 next to the reference):
- conv / linear weight gradients (wgmma, fp32 accumulation, split-K slices added in slice order):
  |dW - ref| <= kgemm(K) u T, T = sum |dy| |x|, K = the reduction length N*H*W (rows for a linear layer).  Products of
  two 16-bit values are exact in fp32, but the tensor cores' fp32 accumulation does not round to nearest, so the error
  grows with the length of one accumulator chain: kgemm(K) = 16 + K / 256.  Worst ratio |dW - ref| / (u T) measured on
  an H100 80GB HBM3 at a 700 W power limit: 16.3, at K = 8192 in one unsplit chain (linear 320 -> 2560, fp16).
- column sums: S = min(8, max(1, rows // 1024)) CTAs of a cluster each hold 32 row lanes; an output is a chain of
  ceil(rows / (32 S)) + 32 + S fp32 additions followed by the scale by alpha, at most ceil(rows / 32) + 40, so
  |out - ref| <= (ceil(rows / 32) + 42) u T, T = |alpha| sum |x|.  The cases cover S = 1, 3, 4, 7 and 8.
- norm affine gradients: the same chain over the terms dz * xh (dgamma) and dz (dbeta), where xh = (x - mean) * rstd
  and silu' each add a few roundings per term: |out - ref| <= (ceil(rows / 32) + 42 + KTERM (1 + |z|)) u T, T = sum of
  the term magnitudes, z the SiLU input (0 without SiLU).  The reference takes the fp32 mean / rstd the library's forward
  saved as exact.
- embedding gradient: a chain of (count of the id) fp32 additions: |out - ref| <= (count + 2) u T.

Poisoning: every output buffer is NaN-filled before the call; no output may stay NaN, and embedding rows that no id
selects must keep their NaN.  Every case runs twice and must give the same bits.
"""
import ctypes
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

F16, BF16, F32, F64 = torch.float16, torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -24
KTERM = 16.0


def kgemm(k):
    return 16.0 + k / 256.0


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from celebbasis_b200 import lib, ops
    assert lib.load().cb_device_ok() == 1
    return lib, ops


def _same_bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _check(out, ref, bound, what):
    assert not torch.isnan(out).any(), f"{what}: NaN left in the output"
    err = (out.double() - ref).abs()
    ratio = (err / bound.clamp_min(1e-300)).max().item()
    bad = (err > bound).nonzero()
    assert bad.numel() == 0, f"{what}: {bad.shape[0]} elements over the bound, worst ratio {ratio:.3g} at {bad[0].tolist()}"


def _rand(shape, dtype, gen, scale=1.0):
    return (torch.randn(shape, generator=gen, device="cuda", dtype=F32) * scale).to(dtype)


# ================================================================================ convolution weight gradient
# (N, H, W, cin, cout, k, stride, pad)
CONV = [
    # SD-v1 UNet geometries
    (2, 64, 64, 320, 320, 3, 1, 1),      # ResBlock conv at 64^2: K = N*H*W = 8192
    (2, 64, 64, 8, 320, 3, 1, 1),        # conv_in, 4 latent channels padded to 8
    (2, 64, 64, 320, 8, 3, 1, 1),        # out conv, 4 channels padded to 8
    (2, 64, 64, 320, 320, 3, 2, 1),      # Downsample 64 -> 32
    (2, 32, 32, 640, 640, 3, 2, 1),      # Downsample 32 -> 16
    (2, 64, 64, 640, 320, 1, 1, 0),      # skip connection at 64^2
    (2, 64, 64, 320, 320, 1, 1, 0),      # proj_in / proj_out
    (2, 32, 32, 960, 640, 3, 1, 1),      # output block ResBlock at 32^2
    (2, 16, 16, 1280, 1280, 3, 1, 1),
    (2, 8, 8, 2560, 1280, 3, 1, 1),      # output block at 8^2: deep N, K = 128
    (2, 8, 8, 2560, 1280, 1, 1, 0),
    # batches 1-4, N*H*W tails, channels off the tile
    (1, 9, 7, 40, 72, 3, 1, 1),
    (3, 5, 11, 136, 200, 3, 1, 1),
    (4, 13, 6, 24, 136, 3, 2, 1),
    (1, 7, 9, 16, 8, 3, 2, 1),
    (3, 17, 3, 264, 56, 1, 1, 0),
    (4, 33, 31, 64, 96, 3, 1, 1),
    (1, 1, 1, 8, 8, 3, 1, 1),
]


def _conv_ref(x, dy, N, H, W, cin, cout, k, stride, pad):
    OH = (H + 2 * pad - k) // stride + 1
    OW = (W + 2 * pad - k) // stride + 1
    xn = x.view(N, H, W, cin).permute(0, 3, 1, 2).to(F64)
    dn = dy.view(N, OH, OW, cout).permute(0, 3, 1, 2).to(F64)
    g = torch.nn.grad.conv2d_weight
    ref = g(xn, (cout, cin, k, k), dn, stride=stride, padding=pad)
    mag = g(xn.abs(), (cout, cin, k, k), dn.abs(), stride=stride, padding=pad)
    return ref, mag, OH, OW


@pytest.mark.parametrize("dtype", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", CONV, ids=lambda c: "n{}_{}x{}_{}to{}_k{}s{}p{}".format(*c))
def test_conv_wgrad(env, case, dtype):
    lib, ops = env
    N, H, W, cin, cout, k, stride, pad = case
    gen = torch.Generator(device="cuda").manual_seed(hash(case) & 0xFFFF)
    OH = (H + 2 * pad - k) // stride + 1
    OW = (W + 2 * pad - k) // stride + 1
    x = _rand((N * H * W, cin), dtype, gen)
    dy = _rand((N * OH * OW, cout), dtype, gen, 0.5)
    alpha = 1.0 / 1024
    geo = ops.Geo(N, H, W)
    outs = []
    for _ in range(2):
        out = torch.full((cout, cin, k, k), float("nan"), dtype=F32, device="cuda")
        ops.conv2d_wgrad(x, geo, dy, ksize=k, stride=stride, pad=pad, alpha=alpha, out=out)
        outs.append(out)
    torch.cuda.synchronize()
    assert _same_bits(outs[0], outs[1]), "two runs gave different bits"
    ref, mag, _, _ = _conv_ref(x, dy, N, H, W, cin, cout, k, stride, pad)
    _check(outs[0], ref * alpha, kgemm(N * OH * OW) * U * mag * alpha, f"conv_wgrad {case} {dtype}")


def test_conv_wgrad_rejects_unaligned_channels(env):
    lib, ops = env
    x = torch.zeros(64, 12, dtype=F16, device="cuda")
    dy = torch.zeros(64, 16, dtype=F16, device="cuda")
    with pytest.raises(lib.CelebBasisB200Error):
        ops.conv2d_wgrad(x, ops.Geo(1, 8, 8), dy, ksize=3, stride=1, pad=1)


# ================================================================================ linear weight gradient
# (rows, in, out): CLIP (77 tokens x batch), UNet attention / feed-forward, time embedding (rows = batch)
LINEAR = [(154, 768, 768), (154, 768, 3072), (154, 3072, 768), (8192, 320, 320), (8192, 320, 2560), (2048, 1280, 640),
          (154, 768, 320), (2, 320, 1280), (2, 1280, 1280), (100, 72, 40), (77, 8, 24)]


@pytest.mark.parametrize("dtype", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", LINEAR, ids=lambda c: "m{}_in{}_out{}".format(*c))
def test_linear_wgrad(env, case, dtype):
    lib, ops = env
    M, K, N = case
    gen = torch.Generator(device="cuda").manual_seed(M * 7 + K * 3 + N)
    x = _rand((M, K), dtype, gen)
    dy = _rand((M, N), dtype, gen, 0.5)
    alpha = 1.0 / 1024
    outs = []
    for _ in range(2):
        out = torch.full((N, K), float("nan"), dtype=F32, device="cuda")
        ops.linear_wgrad(x, dy, alpha=alpha, out=out)
        outs.append(out)
    torch.cuda.synchronize()
    assert _same_bits(outs[0], outs[1]), "two runs gave different bits"
    ref = dy.to(F64).t() @ x.to(F64)
    mag = dy.to(F64).abs().t() @ x.to(F64).abs()
    _check(outs[0], ref * alpha, kgemm(M) * U * mag * alpha, f"linear_wgrad {case} {dtype}")


# ================================================================================ column sums
# (rows, C, groups)
COLSUM = [(8192, 320, 1), (8192, 320, 2), (4096 * 3, 640, 3), (256, 1280, 4), (2, 77 * 768, 1), (1000, 33, 1),
          (31, 8, 1), (4 * 63, 1281, 4), (3 * 1024 + 5, 72, 1), (2 * (7 * 1024 + 9), 40, 2)]


@pytest.mark.parametrize("dtype", [F32, F16, BF16], ids=["f32", "f16", "bf16"])
@pytest.mark.parametrize("case", COLSUM, ids=lambda c: "r{}_c{}_g{}".format(*c))
def test_colsum(env, case, dtype):
    lib, ops = env
    rows, C, groups = case
    gen = torch.Generator(device="cuda").manual_seed(rows + C + groups)
    ld = C + 8                                   # a row pitch wider than C, NaN in the gap
    buf = torch.full((rows, ld), float("nan"), dtype=dtype, device="cuda")
    buf[:, :C] = _rand((rows, C), dtype, gen)
    x = buf[:, :C]
    alpha = 0.75
    outs = []
    for _ in range(2):
        out = torch.full((groups, C), float("nan"), dtype=F32, device="cuda")
        ops.colsum(x, groups=groups, alpha=alpha, out=out)
        outs.append(out)
    torch.cuda.synchronize()
    assert _same_bits(outs[0], outs[1])
    xg = x.to(F64).view(groups, rows // groups, C)
    ref = alpha * xg.sum(1)
    chain = math.ceil(rows / groups / 32) + 42
    _check(outs[0], ref, chain * U * alpha * xg.abs().sum(1), f"colsum {case} {dtype}")


# ================================================================================ norm affine gradients
# (N, HW, C, G)
GN = [(2, 4096, 320, 32), (2, 1024, 640, 32), (1, 64, 1280, 32), (2, 64, 2560, 32), (3, 100, 80, 8), (4, 7, 64, 16),
      (3, 1100, 64, 32)]
DT_PAIRS = [(F16, F16), (F32, F16), (F32, F32), (BF16, BF16), (F32, BF16), (F16, F32)]   # (x, dy)


@pytest.mark.parametrize("silu", [False, True], ids=["plain", "silu"])
@pytest.mark.parametrize("dts", DT_PAIRS, ids=lambda p: "x{}_dy{}".format(*(str(t).split(".")[-1] for t in p)))
@pytest.mark.parametrize("case", GN, ids=lambda c: "n{}_hw{}_c{}_g{}".format(*c))
def test_groupnorm_affine_bwd(env, case, dts, silu):
    lib, ops = env
    N, HW, C, G = case
    xdt, gdt = dts
    gen = torch.Generator(device="cuda").manual_seed(N * HW + C + G)
    x = (_rand((N * HW, C), F32, gen, 2.0) + 0.5).to(xdt)
    dy = _rand((N * HW, C), gdt, gen, 0.25)
    gamma = 1.0 + 0.3 * torch.randn(C, generator=gen, device="cuda")
    beta = 0.2 * torch.randn(C, generator=gen, device="cuda")
    geo = ops.Geo(N, 1, HW)
    _, stats = ops.groupnorm(x, geo, gamma, beta, groups=G, silu=silu, out_dtype=F16)
    L = lib.load()
    alpha = 1.0 / 1024
    outs = []
    for _ in range(2):
        dg = torch.full((C,), float("nan"), dtype=F32, device="cuda")
        db = torch.full((C,), float("nan"), dtype=F32, device="cuda")
        lib.check(L.cb_groupnorm_affine_bwd(dy.data_ptr(), ops._dt(dy), x.data_ptr(), ops._dt(x), gamma.data_ptr(),
                                            beta.data_ptr(), stats.mean.data_ptr(), stats.rstd.data_ptr(), dg.data_ptr(),
                                            db.data_ptr(), N, HW, C, G, 1 if silu else 0, alpha, None), "gn_affine")
        outs.append((dg, db))
    torch.cuda.synchronize()
    assert _same_bits(outs[0][0], outs[1][0]) and _same_bits(outs[0][1], outs[1][1])
    cpg = C // G
    m = stats.mean.to(F64).view(N, G).repeat_interleave(cpg, 1).repeat_interleave(HW, 0)
    r = stats.rstd.to(F64).view(N, G).repeat_interleave(cpg, 1).repeat_interleave(HW, 0)
    xh = (x.to(F64) - m) * r
    dz = dy.to(F64)
    zmag = torch.zeros_like(xh)
    if silu:
        z = xh * gamma.to(F64) + beta.to(F64)
        s = torch.sigmoid(z)
        dz = dz * s * (1 + z * (1 - s))
        zmag = z.abs()
    chain = math.ceil(N * HW / 32) + 42
    for what, term, out in (("dgamma", dz * xh, outs[0][0]), ("dbeta", dz, outs[0][1])):
        bound = U * alpha * (chain * term.abs().sum(0) + KTERM * (term.abs() * (1 + zmag)).sum(0))
        _check(out, alpha * term.sum(0), bound, f"gn {what} {case} {dts} silu={silu}")


# (M, C)
LN = [(8192, 320), (2048, 640), (154, 768), (77, 768), (1000, 72), (3, 1280), (7 * 1024 + 3, 64)]


@pytest.mark.parametrize("dts", [(F32, F32), (F32, F16), (F32, BF16), (F16, F16)],
                         ids=lambda p: "x{}_dy{}".format(*(str(t).split(".")[-1] for t in p)))
@pytest.mark.parametrize("case", LN, ids=lambda c: "m{}_c{}".format(*c))
def test_layernorm_affine_bwd(env, case, dts):
    lib, ops = env
    M, C = case
    xdt, gdt = dts
    gen = torch.Generator(device="cuda").manual_seed(M + C)
    x = (_rand((M, C), F32, gen, 3.0) - 1.0).to(xdt)
    dy = _rand((M, C), gdt, gen, 0.25)
    gamma = 1.0 + 0.3 * torch.randn(C, generator=gen, device="cuda")
    beta = 0.2 * torch.randn(C, generator=gen, device="cuda")
    _, stats = ops.layernorm(x, gamma, beta, out_dtype=F16)
    outs = []
    for _ in range(2):
        dg, db = ops.layernorm_affine_bwd(dy, x, stats, alpha=0.5)
        outs.append((dg, db))
    torch.cuda.synchronize()
    assert _same_bits(outs[0][0], outs[1][0]) and _same_bits(outs[0][1], outs[1][1])
    xh = (x.to(F64) - stats.mean.to(F64)[:, None]) * stats.rstd.to(F64)[:, None]
    dz = dy.to(F64)
    chain = math.ceil(M / 32) + 42
    for what, term, out in (("dgamma", dz * xh, outs[0][0]), ("dbeta", dz, outs[0][1])):
        bound = U * 0.5 * (chain + KTERM) * term.abs().sum(0)
        _check(out, 0.5 * term.sum(0), bound, f"ln {what} {case} {dts}")


def test_layernorm_affine_bwd_poisoned_outputs(env):
    """The raw entry point writes every column of both NaN-filled outputs, and either output may be omitted."""
    lib, ops = env
    M, C = 300, 200
    gen = torch.Generator(device="cuda").manual_seed(5)
    x = _rand((M, C), F32, gen)
    dy = _rand((M, C), F16, gen)
    _, stats = ops.layernorm(x, torch.ones(C, device="cuda"), torch.zeros(C, device="cuda"))
    L = lib.load()
    dg = torch.full((C + 16,), float("nan"), device="cuda")
    db = torch.full((C + 16,), float("nan"), device="cuda")
    lib.check(L.cb_layernorm_affine_bwd(dy.data_ptr(), ops._dt(dy), x.data_ptr(), ops._dt(x), stats.mean.data_ptr(),
                                        stats.rstd.data_ptr(), dg.data_ptr(), None, M, C, 1.0, None), "ln_affine")
    lib.check(L.cb_layernorm_affine_bwd(dy.data_ptr(), ops._dt(dy), x.data_ptr(), ops._dt(x), stats.mean.data_ptr(),
                                        stats.rstd.data_ptr(), None, db.data_ptr(), M, C, 1.0, None), "ln_affine")
    torch.cuda.synchronize()
    assert not dg[:C].isnan().any() and dg[C:].isnan().all()
    assert not db[:C].isnan().any() and db[C:].isnan().all()
    ref_g, ref_b = ops.layernorm_affine_bwd(dy, x, stats)
    assert _same_bits(dg[:C], ref_g) and _same_bits(db[:C], ref_b)


# ================================================================================ embedding gradients
@pytest.mark.parametrize("case", [(154, 49408, 768, 0), (50, 10, 64, 1), (77, 300, 1024, 2), (7, 3, 8, 3)],
                         ids=lambda c: "n{}_v{}_d{}".format(*c[:3]))
def test_embedding_bwd(env, case):
    lib, ops = env
    n, V, D, seed = case
    gen = torch.Generator(device="cuda").manual_seed(seed)
    # CLIP-like prompts: start / end / padding tokens repeat; a few ids outside [0, V) take the nearest row
    ids = torch.randint(0, V, (n,), generator=gen, device="cuda")
    ids[:: max(1, n // 5)] = V - 1
    ids[1] = V + 5
    if n > 3:
        ids[2] = -3
    dout = torch.randn(n, D, generator=gen, device="cuda")
    alpha = 1.0 / 1024
    outs = []
    for _ in range(2):
        out = torch.full((V, D), float("nan"), device="cuda")
        ops.embedding_bwd(ids, dout, V, alpha=alpha, out=out)
        outs.append(out)
    torch.cuda.synchronize()
    assert torch.equal(outs[0].isnan(), outs[1].isnan())
    assert torch.equal(torch.nan_to_num(outs[0]).view(torch.int32), torch.nan_to_num(outs[1]).view(torch.int32))
    cl = ids.clamp(0, V - 1)
    used = torch.zeros(V, dtype=torch.bool, device="cuda")
    used[cl] = True
    assert not outs[0][used].isnan().any() and outs[0][~used].isnan().all()
    ref = torch.zeros(V, D, dtype=F64, device="cuda").index_add_(0, cl, dout.to(F64)) * alpha
    mag = torch.zeros(V, D, dtype=F64, device="cuda").index_add_(0, cl, dout.to(F64).abs()) * alpha
    cnt = torch.bincount(cl, minlength=V).to(F64)[:, None]
    _check(outs[0][used], ref[used], ((cnt + 2) * U * mag)[used], f"embedding_bwd {case}")


def test_position_embedding_grad_is_batch_colsum(env):
    """The position-embedding gradient of a [B][T][D] embedding output: one cb_colsum over its [B][T*D] view."""
    lib, ops = env
    B, T, D = 3, 77, 768
    gen = torch.Generator(device="cuda").manual_seed(11)
    dout = torch.randn(B, T, D, generator=gen, device="cuda")
    g = ops.colsum(dout.view(B, T * D)).view(T, D)
    ref = dout.to(F64).sum(0)
    _check(g, ref, (math.ceil(B / 32) + 42) * U * dout.to(F64).abs().sum(0), "position embedding")


def test_conv_wgrad_ws_bytes_matches_use(env):
    """The workspace query: a 1x1 stride-1 unpadded convolution reads x directly; the others gather N*OH*OW*cin*k*k
    16-bit elements."""
    lib, ops = env
    L = lib.load()
    col, sk = ctypes.c_longlong(-1), ctypes.c_longlong(-1)
    lib.check(L.cb_conv_wgrad_ws_bytes(2, 64, 64, 320, 320, 1, 1, 0, ctypes.byref(col), ctypes.byref(sk)), "ws")
    assert col.value == 0 and sk.value >= 0
    lib.check(L.cb_conv_wgrad_ws_bytes(2, 64, 64, 320, 320, 3, 2, 1, ctypes.byref(col), ctypes.byref(sk)), "ws")
    assert col.value == 2 * 32 * 32 * 320 * 9 * 2
    assert L.cb_conv_wgrad_ws_bytes(2, 64, 64, 320, 320, 5, 1, 2, ctypes.byref(col), ctypes.byref(sk)) == -1
