"""The cb_gemm main loop against the same product evaluated in fp64 on the same 16-bit operands.

Covered: every kernel instantiation (tile width, operand majors, ring depth, kExt) with K in each of the four tail
batches of the last 64-chunk (1, 2, 3 or 4 k16 MMAs), K below 16, ragged M and N; two-level batches with their own
strides for A, B, D and the residual, transposed D; split-K through the L2 workspace and through a cluster, with
batches, MN-major operands, uneven and clamped splits and 16 slices; convolutions (3x3 stride 1 / 2 with symmetric and
(0, 1) padding, 1x1 stride 2, multi-image, odd and > 128-wide output boxes, input rows wider than Cin, padded weight
packs) and their dgrad (flipped taps, MN-major weights, stride 2 through zero insertion) in fp16 and bf16.

Poisoning.  Operands sit in NaN-filled buffers: past K in the row pitch of a K-major operand, past M / N in the row
pitch of an MN-major one, in spare rows and in the gaps between batch slices (input channels past Cin, weight-pack
columns past Cin).  A read outside the operand the descriptor describes turns its outputs into NaN.  The weight pack's
padding rows (b_tap_rows > Cout) stay zero: the kernel may read them against the TMA zero fill of A.  D is fp32 (alpha 1,
no bias or activation) in a NaN-filled buffer with a wider row pitch, spare rows and NaN gaps between batch slices;
nothing outside the described output may change.

Two value modes for every case:
- exact: small integers (|x| <= 4 in fp16, <= 3 in bf16) times power-of-two row scales of A and column scales of B.
  Every product and partial sum of an output is an integer multiple of the same power of two below 2^24, so any
  summation order gives the exact result and D must equal the fp64 reference exactly.  A dropped, duplicated or
  misplaced product, a wrong tap, a wrong batch offset or a non-zero out-of-bounds fill fails deterministically.
- gauss: normal values times per-row scales of A and per-column scales of B of 2^[-12, 12] (fp16, with subnormal
  entries) or 2^[-40, 40] (bf16); a convolution scales the activation per image and the weights per output column.  Every element must satisfy |D - ref| <= k * 2^-24 * (|A| @ |B|); KTOL holds k.

Every case is launched twice and both results must be the same bits.  For split-K shapes, every configuration the host
autotuner may pick (tile widths of its candidate list, ring depth 0 / 3 / 6, cluster or L2 reduction) must give the
same bits, since the autotuner's choice depends on timing noise.
"""
import math
import os
import re
import shutil
import subprocess
import zlib
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F

F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32
NAN = float("nan")
U = 2.0 ** -24

# k of the gauss-mode bound |D - ref| <= k * 2^-24 * (|A| @ |B|), per operand dtype.  The inputs are seeded and the
# library is bit-reproducible, so every error is deterministic.  Beside each k: the worst ratio measured over every case
# of this file per effective K (K x taps), on an H100 80GB HBM3 at a 700 W power limit.
KTOL = {
    F16: 12.0,   # K < 64: 3.57 | 64-511: 4.95 | 512-2047: 6.29 | >= 2048: 2.34
    BF16: 9.0,   # K < 64: 1.81 | 64-511: 3.44 | 512-2047: 4.39 | >= 2048: 1.08
}
WORST = {}       # (dtype, K range) -> (worst ratio of this run, its case)


def k_range(k):
    return "K < 64" if k < 64 else "64-511" if k < 512 else "512-2047" if k < 2048 else ">= 2048"


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from celebbasis_b200 import lib
    assert lib.load().cb_device_ok() == 1, "tests must run on an sm_90 device"
    return torch.device("cuda:0")


def rnd(name):
    """the seeded generator of one case and mode"""
    return torch.Generator().manual_seed(zlib.crc32(name.encode()))


def rup(a, b):
    return (a + b - 1) // b * b


# ------------------------------------------------------------------------------------------------ values and checks
def operand(shape, dtype, mode, g, scale_dim):
    """16-bit values on the host: exact-mode integers or gauss-mode normals, times a power-of-two scale per index of
    `scale_dim` (rows of A, columns of B).  In gauss mode the first index gets the smallest and the last the largest
    scale, so fp16 operands always hold subnormal entries."""
    if mode == "exact":
        lim = 4 if dtype == F16 else 3
        v = torch.randint(-lim, lim + 1, shape, generator=g).double()
        lo, hi = -2, 2
    else:
        v = torch.randn(shape, generator=g, dtype=torch.float64)
        lo, hi = (-12, 12) if dtype == F16 else (-40, 40)
    e = torch.randint(lo, hi + 1, (shape[scale_dim],), generator=g)
    if mode != "exact":
        e[0], e[-1] = lo, hi
    view = [1] * len(shape)
    view[scale_dim] = -1
    return (v * torch.exp2(e.double()).view(view)).to(dtype)


def ratio(out, ref, absref):
    """|out - ref| in units of 2^-24 (|A| @ |B|); an output whose products are all zero must be exactly zero"""
    diff = (out.double() - ref).abs()
    scale = U * absref
    return torch.where(scale > 0, diff / torch.where(scale > 0, scale, 1.0),
                       torch.where(diff > 0, math.inf, 0.0))


def check(out, ref, absref, dtype, mode, keff, what):
    nan = torch.isnan(out)
    assert not nan.any(), f"{what}: {int(nan.sum())} of {out.numel()} outputs unwritten or NaN"
    if mode == "exact":
        bad = out.double() != ref
        if bad.any():
            i = tuple(int(x) for x in bad.nonzero()[0])
            raise AssertionError(f"{what}: {int(bad.sum())} of {out.numel()} outputs differ from the exact result, "
                                 f"first at {i}: {out[i].item()} != {ref[i].item()}")
    else:
        r = ratio(out, ref, absref)
        worst = r.max().item()
        key = (str(dtype).split(".")[-1], k_range(keff))
        WORST[key] = max(WORST.get(key, (0.0, "")), (worst, what))
        assert worst <= KTOL[dtype], f"{what}: error {worst:.2f} x 2^-24 |A||B| > {KTOL[dtype]}"


def nan_buf(n, dtype):
    return torch.full((n,), NAN, dtype=dtype, device="cuda")


class Placed:
    """[images][heads][rows][cols] at element offsets zo * s2 + zi * s1 + r * ld + c of a NaN-filled buffer.
    side_by_side: the heads of an image share rows (s1 = head width), as the fused q / k / v / dO buffers of the
    attention layers keep them; otherwise every slice has its own rows and NaN rows separate slices and images, with
    s2 != heads * s1."""

    def __init__(self, images, heads, rows, cols, dtype, side_by_side=False):
        w = rup(cols, 8)
        if side_by_side:
            self.ld = heads * w + 8
            self.s1, self.s2 = w, (rows + 2) * self.ld
        else:
            self.ld = w + 8
            self.s1 = (rows + 3) * self.ld
            self.s2 = heads * self.s1 + 5 * self.ld
        self.shape = (images, heads, rows, cols)
        self.buf = nan_buf((images - 1) * self.s2 + (heads - 1) * self.s1 + (rows + 2) * self.ld, dtype)

    def view(self, buf=None):
        return (self.buf if buf is None else buf).as_strided(self.shape, (self.s2, self.s1, self.ld, 1))

    def outside_is_nan(self):
        inside = torch.zeros(self.buf.shape, dtype=torch.bool, device=self.buf.device)
        self.view(inside).fill_(True)
        return bool(torch.isnan(self.buf[~inside]).all())


def same_bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def launch(d):
    import ctypes
    from celebbasis_b200 import lib, ops
    ws = ops._splitk_workspace(torch.cuda.current_device())
    d.splitk_ws, d.splitk_ws_bytes = ws.data_ptr(), ws.numel()
    lib.check(lib.load().cb_gemm(ctypes.byref(d), ops._st()), "cb_gemm(main-loop sweep)")


# ------------------------------------------------------------------------------------------------ host dispatch model
def picked_bn(N, tile_n, a_mn, b_mn):
    """the tile width cb_gemm runs for an explicit tile_n (pick_bn), None where its cost model decides"""
    if N <= 64:
        return 64
    if tile_n == 256 and N >= 256 and not a_mn:
        return 256
    return tile_n if tile_n in ((64, 128) if b_mn else (64, 128, 160)) else None


def instantiation(N, tile_n, stages, a_mn, b_mn, ext):
    """(BN, A_MN, B_MN, ring stages, kExt) of the kernel cb_gemm launches, None where the library chooses"""
    bn = picked_bn(N, tile_n, a_mn, b_mn)
    if bn is None:
        return None
    st = 4 if bn == 256 else (stages if stages in (3, 6) else None)
    return None if st is None else (bn, a_mn, b_mn, st, ext)


def cluster_fits(bn, splits, stages):
    """cluster_sk_fits: the exchange buffer fits the TMA ring behind the staged accumulator tile"""
    stage = rup(128 * (bn + 4) * 4, 1024)
    ring = stages * (128 * 64 * 2 + bn * 64 * 2)
    return stage + splits * ((bn // 8 + splits - 1) // splits) * 128 * 32 <= ring


def autotune_configs(N, M, a_mn, b_mn):
    """(tile_n, stages, cluster) of every configuration the host autotuner (ops._autotune) may pick"""
    bns = [64] if N <= 64 else ([64, 128] if b_mn else [64, 128, 160])
    if N >= 256 and not a_mn and M >= 1024:
        bns.append(256)
    return [(0, 0, 0)] + [(bn, st, cl) for bn in bns for st in (0, 3, 6) for cl in (0, 1)]


# ------------------------------------------------------------------------------------------------ GEMM cases
@dataclass(frozen=True)
class Gemm:
    name: str
    dtype: torch.dtype
    M: int
    N: int
    K: int
    a_mn: bool = False
    b_mn: bool = False
    tile_n: int = 0
    stages: int = 0
    ext: bool = False          # a plain fp32 copy in D2 forces the kExt instantiation
    heads: int = 1             # batch_inner; batch = heads * images
    images: int = 1
    side: bool = False         # B and D keep the heads of an image side by side in their rows
    trans: bool = False        # D[b][n][m]
    resid: bool = False        # fp32 residual with its own batch strides (exact mode only)
    splits: int = 0
    cluster: int = 0

    @property
    def inst(self):
        return instantiation(self.N, self.tile_n, self.stages, self.a_mn, self.b_mn, self.ext)


class GemmRun:
    """Operands, reference and output buffers of one GEMM case in one value mode."""

    def __init__(self, c, mode):
        self.c, self.mode = c, mode
        g = rnd(f"{c.name}/{mode}")
        io, hd = c.images, c.heads
        A = operand((io, hd, c.M, c.K), c.dtype, mode, g, 2)
        B = operand((io, hd, c.K, c.N), c.dtype, mode, g, 3)
        self.pa = Placed(io, hd, *((c.K, c.M) if c.a_mn else (c.M, c.K)), c.dtype)
        self.pb = Placed(io, hd, *((c.K, c.N) if c.b_mn else (c.N, c.K)), c.dtype, c.side)
        self.pa.view().copy_((A.transpose(2, 3) if c.a_mn else A).cuda())
        self.pb.view().copy_((B if c.b_mn else B.transpose(2, 3)).cuda())
        A64, B64 = A.cuda().double(), B.cuda().double()
        self.ref, self.absref = A64 @ B64, A64.abs() @ B64.abs()
        self.R = None
        if c.resid:
            assert mode == "exact"
            self.R = Placed(io, hd, c.M, c.N, F32)
            self.R.view().copy_(torch.randint(-64, 65, (io, hd, c.M, c.N), generator=g).float().cuda())
            self.ref = self.ref + self.R.view().double()

    def desc(self, D, D2=None, tile_n=None, stages=None, splits=None, cluster=None):
        from celebbasis_b200 import lib
        c = self.c
        d = lib.GemmDesc()
        d.M, d.N, d.K, d.batch = c.M, c.N, c.K, c.heads * c.images
        d.ab_dtype = lib.CB_F16 if c.dtype == F16 else lib.CB_BF16
        d.batch_inner = c.heads if d.batch > 1 else 0
        pa, pb = self.pa, self.pb
        d.A, d.lda, d.a_batch_stride, d.a_batch_stride2 = pa.buf.data_ptr(), pa.ld, pa.s1, pa.s2
        d.a_major = lib.CB_MAJOR_MN if c.a_mn else lib.CB_MAJOR_K
        d.B, d.ldb, d.b_batch_stride, d.b_batch_stride2 = pb.buf.data_ptr(), pb.ld, pb.s1, pb.s2
        d.b_major = lib.CB_MAJOR_MN if c.b_mn else lib.CB_MAJOR_K
        d.D, d.d_dtype, d.ldd, d.d_batch_stride, d.d_batch_stride2 = D.buf.data_ptr(), lib.CB_F32, D.ld, D.s1, D.s2
        d.d_transposed = int(c.trans)
        if self.R is not None:
            R = self.R
            d.R, d.r_dtype, d.ldr, d.r_batch_stride, d.r_batch_stride2 = R.buf.data_ptr(), lib.CB_F32, R.ld, R.s1, R.s2
        if D2 is not None:
            d.D2, d.d2_dtype, d.ldd2 = D2.buf.data_ptr(), lib.CB_F32, D2.ld
        d.alpha = 1.0
        d.tile_n = c.tile_n if tile_n is None else tile_n
        d.stages = c.stages if stages is None else stages
        d.splits = c.splits if splits is None else splits
        d.splitk_cluster = c.cluster if cluster is None else cluster
        return d

    def out_buffers(self):
        c = self.c
        rows, cols = (c.N, c.M) if c.trans else (c.M, c.N)
        D = Placed(c.images, c.heads, rows, cols, F32, c.side and not c.trans)
        D2 = Placed(1, 1, c.M, c.N, F32) if c.ext else None
        return D, D2

    def run(self, **kw):
        D, D2 = self.out_buffers()
        launch(self.desc(D, D2, **kw))
        return D, D2

    def check(self, D, D2, what):
        c = self.c
        out = D.view()
        if c.trans:
            out = out.transpose(2, 3)
        check(out, self.ref, self.absref, c.dtype, self.mode, c.K, what)
        assert D.outside_is_nan(), f"{what}: D written outside its {c.images} x {c.heads} slices"
        if D2 is not None:
            assert same_bits(D2.view()[0, 0], D.view()[0, 0]), f"{what}: the D2 copy differs from D"
            assert D2.outside_is_nan(), f"{what}: D2 written outside [M, N]"


def run_gemm_case(c, mode):
    r = GemmRun(c, mode)
    D, D2 = r.run()
    torch.cuda.synchronize()
    r.check(D, D2, f"{c.name} [{mode}]")
    E, E2 = r.run()
    assert same_bits(D.buf, E.buf), f"{c.name} [{mode}]: a second launch gave different bits"
    if D2 is not None:
        assert same_bits(D2.buf, E2.buf)


# every (BN, A_MN, B_MN, stages, kExt) that launch() can dispatch, with seven shapes each: K = 1 and 8 (below one k16
# step; lda is 16 bytes past K either way), K % 64 in each of the tail batches (1, 2, 3 or 4 k16 MMAs: 77, 158, 47,
# 252) and a multiple of 64 (320); ragged M and N against the 128-row and BN-column tiles
MAJORS = ((False, False, (64, 128, 160)), (False, True, (64, 128)), (True, True, (64, 128)))
INSTANTIATIONS = [(bn, a, b, st, ext) for a, b, widths in MAJORS for bn in widths for st in (3, 6)
                  for ext in (False, True)] + \
                 [(256, False, b, 4, ext) for b in (False, True) for ext in (False, True)]
INST_K = (1, 8, 77, 158, 47, 252, 320)
INST_M = (1, 65, 129, 300, 65, 300, 129)
INST_N = {64: (8, 72, 77, 200, 300, 64, 130), 128: (72, 77, 200, 300, 130, 160, 257),
          160: (72, 77, 200, 300, 130, 160, 257), 256: (256, 300, 520, 257, 300, 256, 390)}


def inst_name(inst):
    bn, a, b, st, ext = inst
    return f"bn{bn}-{'MN' if a else 'K'}{'MN' if b else 'K'}-s{st}{'-ext' if ext else ''}"


def inst_cases(inst):
    bn, a, b, st, ext = inst
    return [Gemm(f"{inst_name(inst)} {m}x{n}x{k}", (F16, BF16)[i % 2], m, n, k, a, b, bn, st if bn != 256 else 0, ext)
            for i, (m, n, k) in enumerate(zip(INST_M, INST_N[bn], INST_K))]


def _batch_cases():
    c = []
    for a, b in ((False, False), (False, True), (True, True)):
        mj = f"{'MN' if a else 'K'}{'MN' if b else 'K'}"
        for i, (hd, io, m, n, k, side) in enumerate(((1, 2, 65, 40, 77, False), (3, 1, 129, 77, 64, True),
                                                       (8, 5, 40, 80, 40, True), (3, 2, 200, 130, 150, False),
                                                       (1, 5, 77, 64, 200, True))):
            c.append(Gemm(f"batch {mj} {hd}x{io} {m}x{n}x{k}", (F16, BF16)[i % 2], m, n, k, a, b,
                          heads=hd, images=io, side=side))
        c.append(Gemm(f"batch {mj} trans", (BF16, F16)[a], 77 + 53 * a, 40 + 32 * b, 64 + 13 * b, a, b,
                      heads=3, images=2, trans=True))
    # cross-attention of the UNet: nk = 77 keys as K of P.V and as M of dV = P^T dO (both operands MN-major)
    for d, hd in ((40, 8), (160, 2)):
        c.append(Gemm(f"attn P.V d{d}", F16, 256, d, 77, False, True, heads=hd, images=2, side=True))
        c.append(Gemm(f"attn dV d{d}", BF16, 77, d, 256, True, True, heads=hd, images=2, side=True))
    return c


RESID_CASES = [
    Gemm("resid KK 3x2", F16, 77, 72, 100, heads=3, images=2, resid=True),
    Gemm("resid MNMN 1x5", BF16, 130, 64, 77, True, True, heads=1, images=5, resid=True),
    Gemm("resid KMN 8x2 side", F16, 64, 40, 130, False, True, heads=8, images=2, side=True, resid=True),
]


def _splitk_cases():
    c = []
    for cl in (0, 1):
        c += [
            Gemm(f"splitk 4 of 40 cl{cl}", F16, 77, 200, 2560, tile_n=64, stages=6, splits=4, cluster=cl),
            Gemm(f"splitk 6 of 40 (uneven) cl{cl}", BF16, 77, 200, 2560, tile_n=64, stages=6, splits=6, cluster=cl),
            Gemm(f"splitk 64 of 10 (clamped) cl{cl}", F16, 130, 72, 640, tile_n=64, stages=6, splits=64, cluster=cl),
            Gemm(f"splitk batch 3x2 cl{cl}", BF16, 130, 72, 1024, tile_n=128, stages=6, splits=3, cluster=cl,
                 heads=3, images=2),
            Gemm(f"splitk MNMN batch 2x2 cl{cl}", F16, 77, 80, 1000, True, True, tile_n=128, stages=6, splits=5,
                 cluster=cl, heads=2, images=2, side=True),
            Gemm(f"splitk KMN cl{cl}", BF16, 200, 320, 1280, False, True, tile_n=128, stages=6, splits=4, cluster=cl),
            Gemm(f"splitk bn160 cl{cl}", F16, 300, 330, 1536, tile_n=160, stages=6, splits=2, cluster=cl),
            Gemm(f"splitk 16 slices cl{cl}", BF16, 77, 128, 2048, tile_n=64, stages=6, splits=16, cluster=cl),
            Gemm(f"splitk 3-stage cl{cl}", F16, 77, 64, 1536, tile_n=64, stages=3, splits=4, cluster=cl),
        ]
    return c


REGRESSION_CASES = [
    # a 256-wide tile requested with MN-major A: there is no such instantiation, the library picks the width
    Gemm("tile_n 256 with MN-major A", F16, 200, 300, 150, True, True, tile_n=256, heads=2, images=1),
    Gemm("tile_n 256 with MN-major A bf16", BF16, 77, 520, 77, True, True, tile_n=256, stages=6),
]

INST_CASES = [c for inst in INSTANTIATIONS for c in inst_cases(inst)]
GEMM_CASES = _batch_cases() + _splitk_cases() + REGRESSION_CASES


# ------------------------------------------------------------------------------------------------ convolution cases
@dataclass(frozen=True)
class Conv:
    name: str
    dtype: torch.dtype
    n: int
    cin: int
    cout: int
    k: int
    stride: int
    pad: tuple                 # (top, bottom, left, right)
    oh: int                    # output size of the forward convolution
    ow: int
    extra: int = 0             # input rows / columns past the smallest input that gives (oh, ow)
    lda: int = 0               # row pitch of the activation (0: Cin rounded up to 8, plus 8)
    cin_pad: int = 0
    cout_pad: int = 0
    dgrad: int = 0             # 1: dgrad of a stride-1 convolution, 2: of a stride-2 one through zero insertion
    tile_n: int = 0
    stages: int = 0
    splits: int = 0
    cluster: int = 0

    @property
    def inst(self):
        return instantiation(self.cin if self.dgrad else self.cout, self.tile_n, self.stages, False, bool(self.dgrad),
                             False)


def conv_ref(x, w, stride, pt, pl, oh, ow):
    """fp64 convolution of an NHWC image x with w[co][ci][k][k] read at input pixel (o * stride + r - pt, ...), zero
    outside the image; rows of the result in (image, oh, ow) raster order"""
    k = w.shape[2]
    xn = x.permute(0, 3, 1, 2)
    pb = max(0, (oh - 1) * stride + k - pt - xn.shape[2])
    pr = max(0, (ow - 1) * stride + k - pl - xn.shape[3])
    y = F.conv2d(F.pad(xn, (pl, pr, pt, pb)), w, stride=stride)[:, :, :oh, :ow]
    return y.permute(0, 2, 3, 1).reshape(-1, w.shape[0])


class ConvRun:
    def __init__(self, c, mode):
        from celebbasis_b200 import ops
        self.c, self.mode = c, mode
        g = rnd(f"{c.name}/{mode}")
        k, s = c.k, c.stride
        pt, pb, pl, pr = c.pad
        h = (c.oh - 1) * s + k - pt - pb + c.extra
        w_ = (c.ow - 1) * s + k - pl - pr + c.extra
        assert h >= 1 and w_ >= 1
        cin_pad, cout_pad = c.cin_pad or c.cin, c.cout_pad or c.cout
        # weights: gauss / exact values times a power-of-two scale per GEMM output column (Cout, or Cin for dgrad)
        wt = operand((c.cout, c.cin, k, k), c.dtype, mode, g, 1 if c.dgrad else 0)
        pack = ops.pack_conv_weight(wt.float().cuda(), c.dtype, cin_pad=cin_pad, cout_pad=cout_pad)
        assert not pack.view(k * k, cout_pad, cin_pad)[:, c.cout:].any(), "pack padding rows must be zero"
        pack[:, c.cin:] = NAN                          # past Cin: outside both the K-major and the MN-major operand
        self.pack, self.cin_pad, self.cout_pad = pack, cin_pad, cout_pad
        w64 = wt.cuda().double()
        if not c.dgrad:
            self.img = (c.n, h, w_)
            self.out = (c.oh, c.ow)
            self.K, self.N = c.cin, c.cout
            self.geo = (s, pt, pl)
        else:
            # the stride-1 dgrad reads dy (oh x ow) with flipped taps and writes dx of the forward input's size
            assert k == 3 and c.pad == (1, 1, 1, 1)
            self.K, self.N = c.cout, c.cin
            self.img = (c.n, c.oh, c.ow) if c.dgrad == 1 else (c.n, 2 * c.oh, 2 * c.ow)
            self.out = self.img[1:]
            self.geo = (1, k - 1 - pt, k - 1 - pl)
        # A: the activation (dy for dgrad) with a power-of-two scale per image.  The taps of one output read different
        # pixels, so a scale per pixel would not be common to all products of an output (exact mode would not be exact
        # and in gauss mode a single product could dominate its sum); exact mode uses plain integers.
        hw = (c.oh, c.ow) if c.dgrad else (h, w_)
        if mode == "gauss":
            x = operand((c.n, hw[0] * hw[1] * self.K), c.dtype, mode, g, 0)
        else:
            lim = 4 if c.dtype == F16 else 3
            x = torch.randint(-lim, lim + 1, (c.n, hw[0] * hw[1] * self.K), generator=g).to(c.dtype)
        x = x.view(-1, self.K).cuda()
        x64 = x.double().view(c.n, *hw, self.K)
        if c.dgrad == 2:
            z, _ = ops.zero_insert2x(x, ops.Geo(c.n, c.oh, c.ow))
            x = z
            self.ref = self._t(F.conv_transpose2d(x64.permute(0, 3, 1, 2), w64, stride=2, padding=1, output_padding=1))
            self.absref = self._t(F.conv_transpose2d(x64.abs().permute(0, 3, 1, 2), w64.abs(), stride=2, padding=1,
                                                     output_padding=1))
        else:
            wr = w64.flip(2, 3).transpose(0, 1) if c.dgrad else w64
            self.ref = conv_ref(x64, wr, *self.geo, *self.out)
            self.absref = conv_ref(x64.abs(), wr.abs(), *self.geo, *self.out)
        lda = c.lda or rup(self.K, 8) + 8
        self.xbuf = nan_buf((x.shape[0] + 2) * lda, c.dtype)
        self.xbuf[:x.shape[0] * lda].view(-1, lda)[:, :self.K] = x
        self.lda = lda
        self.M = c.n * self.out[0] * self.out[1]

    @staticmethod
    def _t(y):
        return y.permute(0, 2, 3, 1).reshape(-1, y.shape[1])

    def run(self, tile_n=None, stages=None, splits=None, cluster=None):
        from celebbasis_b200 import lib
        c = self.c
        D = Placed(1, 1, self.M, self.N, F32)
        d = lib.GemmDesc()
        d.M, d.N, d.K, d.batch = self.M, self.N, self.K, 1
        d.ab_dtype = lib.CB_F16 if c.dtype == F16 else lib.CB_BF16
        d.A, d.lda, d.a_major = self.xbuf.data_ptr(), self.lda, lib.CB_MAJOR_K
        d.B, d.ldb = self.pack.data_ptr(), self.cin_pad
        d.b_major = lib.CB_MAJOR_MN if c.dgrad else lib.CB_MAJOR_K
        d.conv = 1
        d.img_n, d.img_h, d.img_w = self.img
        d.out_h, d.out_w = self.out
        d.kh = d.kw = c.k
        d.stride, d.pad_top, d.pad_left = self.geo
        d.b_tap_rows, d.flip_taps = self.cout_pad, int(bool(c.dgrad))
        d.D, d.d_dtype, d.ldd = D.buf.data_ptr(), lib.CB_F32, D.ld
        d.alpha = 1.0
        d.tile_n = c.tile_n if tile_n is None else tile_n
        d.stages = c.stages if stages is None else stages
        d.splits = c.splits if splits is None else splits
        d.splitk_cluster = c.cluster if cluster is None else cluster
        launch(d)
        return D

    def check(self, D, what):
        check(D.view()[0, 0], self.ref, self.absref, self.c.dtype, self.mode, self.K * self.c.k ** 2, what)
        assert D.outside_is_nan(), f"{what}: D written outside [M, N]"


CONV_CASES = [
    Conv("3x3 s1 cin8 7x7 x3", F16, 3, 8, 40, 3, 1, (1, 1, 1, 1), 7, 7),
    Conv("3x3 s1 cin40 13x5 x3 lda48", BF16, 3, 40, 72, 3, 1, (1, 1, 1, 1), 13, 5, lda=48),
    Conv("3x3 s2 cin72 2x2 x3", F16, 3, 72, 77, 3, 2, (1, 1, 1, 1), 2, 2),
    Conv("3x3 s2 p01 cin320 7x7 padded pack", BF16, 1, 320, 200, 3, 2, (0, 1, 0, 1), 7, 7, cin_pad=328,
         cout_pad=208, tile_n=128, stages=3),
    Conv("3x3 s2 p01 cin8 9x140", F16, 1, 8, 72, 3, 2, (0, 1, 0, 1), 9, 140, extra=1),
    Conv("3x3 s2 cin8 13x5 x3 odd input", BF16, 3, 8, 40, 3, 2, (1, 1, 1, 1), 13, 5, extra=1),
    Conv("1x1 s2 cin40 13x5 x3", F16, 3, 40, 130, 1, 2, (0, 0, 0, 0), 13, 5, tile_n=160, stages=6),
    Conv("1x1 s2 cin320 7x7 lda336", BF16, 1, 320, 64, 1, 2, (0, 0, 0, 0), 7, 7, lda=336),
    Conv("1x1 s2 cin72 2x2 x3 padded pack", F16, 3, 72, 256, 1, 2, (0, 0, 0, 0), 2, 2, cin_pad=80, cout_pad=264,
         tile_n=256),
    Conv("3x3 s1 cin72 9x140", BF16, 1, 72, 40, 3, 1, (1, 1, 1, 1), 9, 140),
    Conv("3x3 s1 cin8 1x1 x3", F16, 3, 8, 64, 3, 1, (1, 1, 1, 1), 1, 1),
    Conv("3x3 s1 cin320 2x2", BF16, 1, 320, 320, 3, 1, (1, 1, 1, 1), 2, 2, tile_n=256),
    # dgrad: K = Cout (4 with the 16-row pack of the UNet's output conv), MN-major weights, flipped taps
    Conv("dgrad cout4 pack16 13x5", F16, 1, 320, 4, 3, 1, (1, 1, 1, 1), 13, 5, cout_pad=16, lda=8, dgrad=1),
    Conv("dgrad cout4 pack16 7x7 x3 bf16", BF16, 3, 40, 4, 3, 1, (1, 1, 1, 1), 7, 7, cout_pad=16, lda=8, dgrad=1),
    Conv("dgrad cout77 7x7 x3", BF16, 3, 40, 77, 3, 1, (1, 1, 1, 1), 7, 7, cin_pad=48, dgrad=1),
    Conv("dgrad cout320 2x2 x3", F16, 3, 72, 320, 3, 1, (1, 1, 1, 1), 2, 2, dgrad=1, tile_n=128, stages=6),
    Conv("dgrad cout1280 7x7 x2", BF16, 2, 130, 1280, 3, 1, (1, 1, 1, 1), 7, 7, cin_pad=136, dgrad=1),
    Conv("dgrad cout1280 9x140 fp16", F16, 1, 40, 1280, 3, 1, (1, 1, 1, 1), 9, 140, dgrad=1, tile_n=64, stages=3),
    Conv("dgrad s2 cout320 4x4 x2", F16, 2, 72, 320, 3, 2, (1, 1, 1, 1), 4, 4, dgrad=2),
    Conv("dgrad s2 cout64 7x7", BF16, 1, 40, 64, 3, 2, (1, 1, 1, 1), 7, 7, dgrad=2),
]

# shapes whose bits must not depend on the configuration the autotuner picks: split-K by request and by the library's
# own choice (splits = 0, as the autotuner launches them), plain and batched, convolution and dgrad
CONFIG_CASES = [
    Gemm("cfg KK splits 4", F16, 77, 200, 2560, splits=4),
    Gemm("cfg KK library split", BF16, 77, 330, 2560),
    Gemm("cfg KMN library split", F16, 256, 320, 1280, False, True),
    Gemm("cfg MNMN batch splits 3", BF16, 77, 80, 1024, True, True, heads=3, images=2, side=True, splits=3),
    Gemm("cfg KK large", F16, 1024, 320, 320),
    Conv("cfg conv library split", BF16, 1, 640, 320, 3, 1, (1, 1, 1, 1), 8, 8),
    Conv("cfg dgrad splits 6", F16, 1, 320, 640, 3, 1, (1, 1, 1, 1), 8, 8, dgrad=1, splits=6),
]


def _cluster_cases_fit():
    for c in GEMM_CASES:
        if c.cluster:
            bn = picked_bn(c.N, c.tile_n, c.a_mn, c.b_mn)
            kiters = (c.K + 63) // 64
            per = -(-kiters // min(c.splits, kiters))
            s = -(-kiters // per)
            assert 2 <= s <= 16 and cluster_fits(bn, s, c.stages), f"{c.name}: cluster split-K would fall back to L2"


_cluster_cases_fit()


# ------------------------------------------------------------------------------------------------ GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["exact", "gauss"])
@pytest.mark.parametrize("inst", INSTANTIATIONS, ids=inst_name)
def test_instantiation(dev, inst, mode):
    for c in inst_cases(inst):
        run_gemm_case(c, mode)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["exact", "gauss"])
@pytest.mark.parametrize("case", GEMM_CASES, ids=lambda c: c.name)
def test_gemm(dev, case, mode):
    run_gemm_case(case, mode)


@pytest.mark.gpu
@pytest.mark.parametrize("case", RESID_CASES, ids=lambda c: c.name)
def test_batched_residual(dev, case):
    run_gemm_case(case, "exact")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["exact", "gauss"])
@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: c.name)
def test_conv(dev, case, mode):
    r = ConvRun(case, mode)
    D = r.run()
    torch.cuda.synchronize()
    r.check(D, f"{case.name} [{mode}]")
    assert same_bits(D.buf, r.run().buf), f"{case.name} [{mode}]: a second launch gave different bits"


@pytest.mark.gpu
@pytest.mark.parametrize("case", CONFIG_CASES, ids=lambda c: c.name)
def test_bits_do_not_depend_on_the_autotuned_configuration(dev, case):
    """ops._autotune times tile width, ring depth and cluster vs L2 reduction and keeps the fastest; none of them may
    change a bit of the result."""
    conv = isinstance(case, Conv)
    r = ConvRun(case, "gauss") if conv else GemmRun(case, "gauss")
    M = r.M if conv else case.M
    N = r.N if conv else case.N
    first = None
    for tile_n, stages, cluster in autotune_configs(N, M, False if conv else case.a_mn,
                                                    bool(case.dgrad) if conv else case.b_mn):
        what = f"{case.name} tile_n {tile_n} stages {stages} cluster {cluster}"
        D = r.run(tile_n=tile_n, stages=stages, cluster=cluster)
        if conv:
            r.check(D, what)
        else:
            D = D[0]
            r.check(D, None, what)
        if first is None:
            first = D
        assert same_bits(first.buf, D.buf), f"{what}: different bits from the library's own configuration"


@pytest.mark.gpu
def test_dispatch_matches_the_table(dev):
    """The kernel each forced case launches is the instantiation the table assigns to it (the dispatch model above),
    read from the kernel names the profiler records."""
    cases = [(c, GemmRun(c, "exact")) for inst in INSTANTIATIONS for c in inst_cases(inst)[:1]]
    cases += [(c, ConvRun(c, "exact")) for c in CONV_CASES if c.inst is not None]
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _, r in cases:
            r.run()
        torch.cuda.synchronize()
    names = [e for e in prof.events() if "cb_gemm_kernel" in e.name]
    names = [parse_kernel_name(e.name) for e in sorted(names, key=lambda e: e.time_range.start)]
    assert names == [c.inst for c, _ in cases]


def parse_kernel_name(name):
    """(BN, A_MN, B_MN, stages, kExt) of a demangled cb_gemm_kernel<...> name ("(int)128" / "128", "(bool)1" / "true")"""
    args = re.search(r"cb_gemm_kernel<([^>]*)>", name).group(1).split(",")
    v = [re.sub(r"^\(\w+\)", "", a.strip()) for a in args]
    b = lambda s: s in ("1", "true")
    return (int(v[0]), b(v[1]), b(v[2]), int(v[3]), b(v[4]))


# ------------------------------------------------------------------------------------------------ CPU tests
def round_sig(x, bits):
    """x rounded to `bits` significant bits (round to nearest even), exponent range unlimited"""
    m, e = torch.frexp(x)
    return torch.ldexp(torch.round(m * 2.0 ** bits) / 2.0 ** bits, e)


@pytest.mark.parametrize("dtype", [F16, BF16])
def test_bound_rejects_16bit_partial_sums(dtype):
    """The gauss-mode bound is tight enough to fail a main loop whose running sum is rounded to fp16 precision
    (11 significant bits) after every 64-deep k-iteration, and loose enough to pass one that adds each k16 step's
    products exactly and rounds the running sum to fp32, at every K range the GPU cases use."""
    for K in (47, 320, 1280, 2560):
        g = rnd(f"bound {dtype} {K}")
        A = operand((96, K), dtype, "gauss", g, 0).double()
        B = operand((K, 80), dtype, "gauss", g, 1).double()
        ref, absref = A @ B, A.abs() @ B.abs()
        acc16 = torch.zeros_like(ref)
        for k0 in range(0, K, 64):
            acc16 = round_sig(acc16 + A[:, k0:k0 + 64] @ B[k0:k0 + 64], 11)
        acc32 = torch.zeros_like(ref, dtype=F32)
        for k0 in range(0, K, 16):
            acc32 = (acc32.double() + A[:, k0:k0 + 16] @ B[k0:k0 + 16]).float()
        assert ratio(acc16, ref, absref).max() > KTOL[dtype], f"K={K}: 16-bit partial sums pass the bound"
        assert ratio(acc32, ref, absref).max() <= KTOL[dtype], f"K={K}: an fp32 main loop fails the bound"


def _tool(name):
    found = shutil.which(name)
    if found:
        return found
    cand = os.path.join("/usr/local/cuda/bin", name)
    return cand if os.path.exists(cand) else None


def test_every_compiled_instantiation_has_cases(tmp_path):
    """Every cb_gemm_kernel<BN, A_MN, B_MN, stages, kExt> in the compiled code is a row of INSTANTIATIONS and every row
    is compiled; each row's cases run that instantiation (dispatch model, checked on the GPU by
    test_dispatch_matches_the_table) with K in every tail batch, K below 16, and ragged M and N."""
    from celebbasis_b200 import build
    cuobjdump, cufilt = _tool("cuobjdump"), _tool("cu++filt")
    if cuobjdump is None or cufilt is None:
        pytest.skip("cuobjdump / cu++filt not available")
    src = os.path.join(build.CSRC, "cb_gemm.cu")
    obj = os.path.join(build.OBJ, "cb_gemm.o")
    stamp = obj + ".sha1"
    if not (os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == build._digest(src)):
        nvcc = _tool("nvcc")
        if nvcc is None:
            pytest.skip("no up-to-date cb_gemm.o and no nvcc")
        obj = str(tmp_path / "cb_gemm.o")
        r = subprocess.run([nvcc, *build.NVCC_FLAGS, "-c", src, "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-4000:]
    r = subprocess.run([cuobjdump, "-symbols", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    mangled = sorted(set(re.findall(r"\S*cb_gemm_kernel\S*", r.stdout)))
    assert mangled, "no cb_gemm_kernel symbol in the compiled code"
    r = subprocess.run([cufilt], input="\n".join(mangled) + "\n", capture_output=True, text=True)
    compiled = {parse_kernel_name(line) for line in r.stdout.splitlines() if "cb_gemm_kernel" in line}
    assert len(compiled) == len(mangled)
    assert compiled - set(INSTANTIATIONS) == set(), "instantiations without cases"
    assert set(INSTANTIATIONS) - compiled == set(), "table rows that are not compiled"
    for inst in INSTANTIATIONS:
        cases = inst_cases(inst)
        assert all(c.inst == inst for c in cases), inst
        tails = {(c.K % 64 + 15) // 16 for c in cases}          # k16 MMAs of the last chunk, 0: a multiple of 64
        assert tails == {0, 1, 2, 3, 4} and min(c.K for c in cases) < 16, inst
        assert any(c.M % 128 and c.M > 128 for c in cases) and any(c.N % inst[0] and c.N > inst[0] for c in cases)
        assert {c.dtype for c in cases} == {F16, BF16}
