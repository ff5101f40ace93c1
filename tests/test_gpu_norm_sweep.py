"""GroupNorm and LayerNorm (cb_norm.cu, cb_layernorm.cu) against the same operation evaluated in fp64 on the same stored
inputs, on every launch route and every compiled instantiation.

Routes.  GroupNorm forward runs the cluster kernel (gn_cluster_fwd_kernel) when cb_groupnorm_cluster_plan finds a slab
plan, else the TMA-streamed pair (gn_stats_tma_kernel + gn_apply_tma_kernel); the backward runs gn_cluster_bwd_kernel or
gn_bwd_stats_kernel + gn_bwd_apply_kernel.  LayerNorm runs ln_fwd_q_kernel / ln_bwd_q_kernel<..., W, Q> with the
(warps per row, quads per lane) plan of ln_plan (mirrored below) for fp32 x, 16-byte aligned pointers and C % 4 == 0,
else the warp-per-row ln_fwd_kernel / ln_bwd_kernel of cb_norm.cu (C <= 2048, CB_ERR_ARG beyond).  Every row of CASES
states the route it must take: a CPU test derives it from cb_groupnorm_cluster_plan and the ln_plan mirror, and a GPU
test reads the kernels the profiler records.  A CPU test lists every gn_* / ln_* instantiation in the compiled objects
and requires a case for each.

Error model, with u = 2^-24 and per group (GroupNorm) or row (LayerNorm) mean mu, variance s2, r = 1 / sqrt(s2 + eps),
and c = mu^2 / (s2 + eps) for GroupNorm (its variance is the one-pass E[x^2] - mu^2, so the relative error of the
squares' sum is amplified by 1 + c) or c = 0 for LayerNorm (two passes):
- mean_out, rstd_out (always fp32): |mean - mu| <= K u mean|x|,  |rstd - r| / r <= K u (1 + c);
- y and dx: |out - ref| <= half an ulp of the output dtype at the result + K u T, where T is the magnitude of the terms
  that form it.  Forward: T = |g xh| (1 + c) + |b| + |g| r mean|x| (the last two carry the statistics' errors into y),
  times |silu'(z)| plus |silu(z)| (1 + |z|) where SiLU is fused.  Backward, fed fp32 statistics m, r that the reference
  uses as exact: T = r (|dz g| + mean|dz g| + |xh| mean(|dz g| xa) + xa |mean(dz g xh)|) with xa = (|x| + |m|) r, the
  magnitude of xh's operands; with SiLU, |dz g| is |dy g| (s + |z s (1 - s)| + (|g| xa + |b|) / 2), the magnitude of
  silu'(z) and of its change under z's rounding error.  An accumulating call adds |dx before|.
K below holds the constants; a CPU test shows they are tight: an fp32 emulation of the kernels passes every case at
reduced size, and seven kinds of wrong kernel each fail at least one case.

Poisoning.  Every output (y, dx, dx_lp, mean, rstd) sits in a NaN-filled allocation with guard regions before and
after it; inputs sit in NaN-filled allocations too, so an over-read turns outputs into NaN.  Nothing outside an output
may change and nothing inside it may stay NaN.  The GroupNorm workspace is filled with 0xFF bytes (NaN floats) before
every call.  Every case runs twice and must give the same bits.
"""
import ctypes
import math
import os
import re
import shutil
import subprocess
import zlib
from dataclasses import dataclass, replace

import numpy as np
import pytest
import torch

F16, BF16, F32, F64 = torch.float16, torch.bfloat16, torch.float32, torch.float64
DTYPES = (F32, F16, BF16)
CODE = {F16: 0, BF16: 1, F32: 2}
NAME = {F32: "f32", F16: "f16", BF16: "bf16"}
CTYPE = {"float": F32, "__half": F16, "__nv_bfloat16": BF16}
MANT = {F32: 24, F16: 11, BF16: 8}               # significand bits
EMIN = {F32: -126, F16: -14, BF16: -126}         # smallest normal exponent
U = 2.0 ** -24
CB_ERR_ARG = -1
WS_BYTES = 131072                                # CB_GN_WS_BYTES
GUARD = 256                                      # guard elements before and after every buffer (>= 512 bytes)

# K of each bound, per quantity and route family.  The inputs are seeded and the library is bit-reproducible, so every
# error is deterministic.  Beside each K: the worst ratio measured over every case of this file, per output dtype
# f32 / f16 / bf16, on an H100 80GB HBM3 at a 700 W power limit.
K = {
    ("mean", "gn_cluster"): 8.0,    # 3.89
    ("mean", "gn_pair"): 12.0,      # 6.16
    ("mean", "ln_q"): 5.0,          # 2.45
    ("mean", "ln_fallback"): 4.0,   # 1.92
    ("rstd", "gn_cluster"): 6.0,    # 2.86
    ("rstd", "gn_pair"): 11.0,      # 5.45
    ("rstd", "ln_q"): 6.0,          # 3.02
    ("rstd", "ln_fallback"): 5.0,   # 2.43
    ("y", "gn_cluster"): 5.5,       # 1.48 / 2.67 / 2.05
    ("y", "gn_pair"): 8.0,          # 1.40 / 3.92 / 1.04
    ("y", "ln_q"): 6.0,             # 3.03 / 2.15 / 1.62
    ("y", "ln_fallback"): 6.0,      # 2.80 / 1.55 / 0.90
    ("dx", "gn_cluster"): 5.0,      # 2.32 / 1.31 / 0.87
    ("dx", "gn_pair"): 5.0,         # 2.50 / 1.07 / 0.76
    ("dx", "ln_q"): 4.0,            # 1.92 / 1.03 / 0.70
    ("dx", "ln_fallback"): 3.5,     # 1.68 / 1.35 / 0.54
}
WORST = {}       # (quantity, family, dtype) -> (worst ratio of this run, its case)


# ================================================================================================ routes
def ln_plan(M, C):
    """(warps per row, quads per lane) of cb_layernorm.cu's ln_plan, or None where the fallback takes the shape"""
    if C % 4:
        return None
    wpr = 4 if (M <= 1024 and C >= 512) or M <= 256 else 1
    q = -(-(C // 4) // (32 * wpr))
    if q <= 3:
        return wpr, 3
    if q <= 10:
        return wpr, 10
    q4 = -(-(C // 4) // 128)
    if wpr == 1 and q4 <= 10:
        return 4, 3 if q4 <= 3 else 10
    return None


def gn_plan(N, HW, C, G, bytes_per_elem):
    """cb_groupnorm_cluster_plan: (S, gpc, rows per CTA, smem) or None (the kernel pair takes the shape)"""
    from celebbasis_b200 import lib
    plan = (ctypes.c_int * 4)()
    rc = lib.load().cb_groupnorm_cluster_plan(N, HW, C, G, bytes_per_elem, ctypes.cast(plan, ctypes.c_void_p))
    assert rc in (0, 1), (rc, N, HW, C, G)
    return tuple(plan) if rc == 1 else None


def esize(dt):
    return 4 if dt == F32 else 2


def family(route):
    return "ln_q" if route.startswith("ln_q") else route.rsplit("_", 1)[0] if route.startswith("gn") else route


# ================================================================================================ the case table
@dataclass(frozen=True)
class Case:
    op: str                 # gn_fwd, gn_bwd, ln_fwd, ln_bwd
    route: str              # gn_cluster_fwd | gn_pair_fwd | gn_cluster_bwd | gn_pair_bwd | ln_q_<W>_<Q> | ln_fallback | error
    N: int                  # images (GroupNorm) / 1 (LayerNorm)
    rows: int               # HW (GroupNorm) / M (LayerNorm)
    C: int
    G: int                  # groups (GroupNorm) / 0
    xd: torch.dtype
    od: torch.dtype         # y (forward) / dx (backward)
    gd: torch.dtype = None  # dy (backward)
    eps: float = 1e-5
    silu: bool = False
    acc: bool = False
    lp: bool = False
    cap: int = 0            # CB_GN_CTA_CAP(cap), forward
    junk: bool = False      # set the flag bits the entry ignores (1-7 and 24-31)
    rho: float = 1.0        # |mean| / std of every group / row
    values: str = "randn"   # randn | smallvar (std 1e-2) | const (every third group / row has std 0)
    shift: str = ""         # LayerNorm: this pointer is 8 bytes past a 16-byte boundary

    @property
    def id(self):
        s = f"{self.op}-{self.route}-N{self.N}x{self.rows}xC{self.C}"
        s += f"G{self.G}" if self.G else ""
        s += f"-{NAME[self.xd]}"
        s += f"-{NAME[self.gd]}" if self.gd is not None else ""
        s += f"-{NAME[self.od]}"
        for flag in ("silu", "acc", "lp", "junk"):
            s += f"-{flag}" if getattr(self, flag) else ""
        s += f"-cap{self.cap}" if self.cap else ""
        s += f"-eps{self.eps:g}" if self.eps != 1e-5 else ""
        s += f"-rho{self.rho:g}" if self.rho != 1.0 else ""
        s += f"-{self.values}" if self.values != "randn" else ""
        s += f"-{self.shift}+8" if self.shift else ""
        return s

    @property
    def family(self):
        return family(self.route)

    @property
    def groups(self):
        """(images, rows per image, groups): a LayerNorm row is one group of one image"""
        return (self.N, self.rows, self.G) if self.op.startswith("gn") else (self.rows, 1, 1)

    def row_type(self):
        return (self.op, self.route, self.xd, self.gd, self.od, self.silu, self.acc, self.lp)


def _cases():
    T = []
    gf = lambda route, N, HW, C, G, xd, yd, **kw: T.append(Case("gn_fwd", route, N, HW, C, G, xd, yd, **kw))
    gb = lambda route, N, HW, C, G, xd, gd, dd, **kw: T.append(Case("gn_bwd", route, N, HW, C, G, xd, dd, gd, **kw))
    lf = lambda route, M, C, xd, yd, **kw: T.append(Case("ln_fwd", route, 1, M, C, 0, xd, yd, **kw))
    lb = lambda route, M, C, gd, dd, xd=F32, **kw: T.append(Case("ln_bwd", route, 1, M, C, 0, xd, dd, gd, **kw))
    BWD = [(g, d) for g in DTYPES for d in ((F32,) if g == F32 else (F32, g))]      # (dy, dx) pairings
    # ---- GroupNorm forward: every (x, y) pairing, SiLU on and off, on both routes (G = 64 only the pair takes)
    for xd in DTYPES:
        for yd in DTYPES:
            for silu in (False, True):
                gf("gn_cluster_fwd", 1, 256, 320, 32, xd, yd, silu=silu)
                gf("gn_pair_fwd", 2, 300, 128, 64, xd, yd, silu=silu)
    # channels per group: 4-channel accesses straddle two groups for C/G in {2, 6, 10, 30}
    for C in (64, 192, 320, 960, 128, 640, 1280, 2560):
        gf("gn_cluster_fwd", 1, 64, C, 32, F32, F16, silu=True)
        gf("gn_cluster_fwd", 2, 40, C, 32, BF16, BF16)
    # other group counts: gpc 2 (G = 2), gpc 1 (G = 1, 3, 5), no slab fits (G = 10 with C/G = 2), G in (32, 64]
    gf("gn_cluster_fwd", 1, 96, 320, 16, F32, F16, silu=True)
    gf("gn_cluster_fwd", 1, 96, 320, 8, F16, F32)
    gf("gn_cluster_fwd", 1, 96, 64, 4, F32, BF16)
    gf("gn_cluster_fwd", 1, 96, 40, 2, F16, F16, silu=True)
    gf("gn_cluster_fwd", 1, 96, 64, 1, F32, F32)
    gf("gn_cluster_fwd", 2, 33, 48, 3, F32, F16)
    gf("gn_cluster_fwd", 1, 50, 40, 5, F16, BF16, silu=True)
    gf("gn_cluster_fwd", 3, 64, 24, 12, F32, F16)
    gf("gn_pair_fwd", 2, 70, 20, 10, F32, F16, silu=True)
    gf("gn_pair_fwd", 1, 200, 320, 40, BF16, F32)
    gf("gn_pair_fwd", 3, 90, 96, 48, F16, F16, silu=True)
    # slab widths 8, 16, 32 (many images of few rows)
    for N in (40, 70, 140):
        gf("gn_cluster_fwd", N, 4, 64, 32, F32, F16, silu=True)
        gf("gn_cluster_fwd", N, 3, 128, 32, F16, BF16)
    # rows: HW = 1, below S, CTAs with empty row ranges (17 and 100 rows over 16 CTAs), not a multiple of S, N
    for N, HW in ((1, 1), (2, 1), (1, 5), (1, 17), (1, 100), (1, 4097), (3, 64), (16, 256), (2, 777)):
        gf("gn_cluster_fwd", N, HW, 320, 32, F32, F16, silu=True)
        gf("gn_cluster_fwd", N, HW, 640, 32, BF16, BF16)
    for N, HW in ((1, 1), (3, 5), (16, 37), (1, 3000)):
        gf("gn_pair_fwd", N, HW, 128, 64, F32, F16, silu=True)
    # VAE-sized maps on the streaming pair; 66000 rows is no multiple of the 64 rows per TMA chunk
    gf("gn_pair_fwd", 1, 65536, 128, 32, F32, F16, silu=True, eps=1e-6)
    gf("gn_pair_fwd", 1, 66000, 256, 32, F16, F16, eps=1e-6)
    gf("gn_pair_fwd", 1, 65536, 256, 32, BF16, BF16, silu=True, eps=1e-6)
    # epsilon (std 1e-2: s2 ~ 1e-4) and constant groups, mean / spread ratios
    for route, N, HW, C, G in (("gn_cluster_fwd", 1, 256, 320, 32), ("gn_pair_fwd", 2, 300, 128, 64)):
        for eps in (1e-5, 1e-6):
            gf(route, N, HW, C, G, F32, F32, eps=eps, values="smallvar")
            gf(route, N, HW, C, G, F32, F16, eps=eps, values="const", silu=True)
            gf(route, N, HW, C, G, BF16, F32, eps=eps, values="const")
        for rho in (0.0, 8.0, 64.0, 256.0):
            gf(route, N, HW, C, G, F32, F32, rho=rho)
            gf(route, N, HW, C, G, F16, BF16, rho=rho, silu=True)
    # flag bits: the streaming pair's CTA cap, and the ignored bits on both routes
    for cap in (1, 7, 16):
        gf("gn_pair_fwd", 1, 3000, 128, 64, F32, F16, cap=cap, silu=True)
    gf("gn_pair_fwd", 1, 65536, 128, 32, F32, F16, cap=16, eps=1e-6)
    gf("gn_cluster_fwd", 1, 256, 320, 32, F32, F16, junk=True, silu=True)
    gf("gn_cluster_fwd", 1, 256, 320, 32, F32, F16, junk=True)
    gf("gn_pair_fwd", 2, 300, 128, 64, F16, F32, junk=True, cap=7)

    # ---- GroupNorm backward: every (x, dy, dx) triple x SiLU x accumulate x dx_lp on both routes
    for xd in DTYPES:
        for g, d in BWD:
            for silu in (False, True):
                for acc in (False, True):
                    for lp in (False, True):
                        gb("gn_cluster_bwd", 1, 256, 320, 32, xd, g, d, silu=silu, acc=acc, lp=lp)
                        gb("gn_pair_bwd", 2, 300, 128, 64, xd, g, d, silu=silu, acc=acc, lp=lp)
    for C in (64, 192, 320, 960, 128, 640, 1280, 2560):
        gb("gn_cluster_bwd", 1, 64, C, 32, F32, F16, F32, silu=True, acc=True)
        gb("gn_cluster_bwd", 2, 40, C, 32, BF16, BF16, BF16, lp=True)
    gb("gn_cluster_bwd", 1, 96, 40, 2, F16, F16, F32, silu=True)
    gb("gn_cluster_bwd", 1, 96, 64, 1, F32, F32, F32)
    gb("gn_cluster_bwd", 2, 33, 48, 3, F32, BF16, BF16, acc=True)
    gb("gn_pair_bwd", 2, 70, 20, 10, F32, F16, F32, silu=True)
    gb("gn_pair_bwd", 1, 200, 320, 40, BF16, BF16, F32, acc=True, lp=True)
    gb("gn_pair_bwd", 2, 30, 12, 6, F32, F16, F16, silu=True)            # C = 12: any even C/G on the backward
    for N in (40, 70, 140):
        gb("gn_cluster_bwd", N, 4, 64, 32, F32, F16, F32, silu=True, acc=True)
    for N, HW in ((1, 1), (2, 1), (1, 5), (1, 17), (1, 100), (1, 4097), (3, 64), (16, 256)):
        gb("gn_cluster_bwd", N, HW, 320, 32, F32, F16, F32, silu=True, acc=True)
        gb("gn_cluster_bwd", N, HW, 640, 32, BF16, BF16, BF16, lp=True)
    for N, HW in ((1, 1), (3, 5), (16, 37), (1, 3000)):
        gb("gn_pair_bwd", N, HW, 128, 64, F32, F16, F32, silu=True, acc=True, lp=True)
    gb("gn_pair_bwd", 1, 65536, 128, 32, F32, F16, F32, silu=True, acc=True, lp=True)
    gb("gn_pair_bwd", 1, 66000, 128, 32, F16, F16, F16, lp=True)
    for route, N, HW, C, G in (("gn_cluster_bwd", 1, 256, 320, 32), ("gn_pair_bwd", 2, 300, 128, 64)):
        for rho in (0.0, 8.0, 64.0, 256.0):
            gb(route, N, HW, C, G, F32, F16, F32, rho=rho, silu=True, acc=True)
            gb(route, N, HW, C, G, BF16, BF16, BF16, rho=rho, lp=True)
        gb(route, N, HW, C, G, F32, F16, F32, values="const", silu=True, eps=1e-6)
        gb(route, N, HW, C, G, F32, F16, F32, values="smallvar", silu=True, eps=1e-6)
        gb(route, N, HW, C, G, F32, F16, F32, junk=True, silu=True)

    # ---- LayerNorm forward: every y dtype on every quad plan; both sides of each ln_plan switch
    plans = ((1025, 320, "ln_q_1_3"), (1025, 640, "ln_q_1_10"), (77, 768, "ln_q_4_3"), (64, 2048, "ln_q_4_10"))
    for M, C, route in plans:
        for yd in DTYPES:
            lf(route, M, C, F32, yd)
    for M, C, route in ((256, 320, "ln_q_4_3"), (257, 320, "ln_q_1_3"), (1024, 640, "ln_q_4_3"),
                        (1025, 640, "ln_q_1_10"), (1024, 1280, "ln_q_4_3"), (1025, 1280, "ln_q_1_10"),
                        (1027, 512, "ln_q_1_10"), (4096, 320, "ln_q_1_3"), (1, 320, "ln_q_4_3")):
        lf(route, M, C, F32, F16)
    for C, route in ((64, "ln_q_1_3"), (320, "ln_q_1_3"), (384, "ln_q_1_3"), (388, "ln_q_1_10"), (640, "ln_q_4_3"),
                     (768, "ln_q_4_3"), (1280, "ln_q_4_3"), (1284, "ln_q_4_3"), (2048, "ln_q_4_10"),
                     (4100, "ln_q_4_10"), (5120, "ln_q_4_10")):
        lf(route, 300, C, F32, BF16)
    for C, route in ((1284, "ln_q_4_3"), (2048, "ln_q_4_10"), (5120, "ln_q_4_10")):
        lf(route, 2000, C, F32, F32)                  # one warp per row gives more than 10 quads: four warps per row
    # fallback: 16-bit x, a misaligned pointer, C % 4 == 2
    for xd in (F16, BF16):
        for yd in DTYPES:
            lf("ln_fallback", 100, 768, xd, yd)
    for yd, shift in ((F32, "x"), (F16, "y"), (BF16, "gamma"), (F16, "beta")):
        lf("ln_fallback", 70, 640, F32, yd, shift=shift)
    for C in (322, 770, 2046):
        lf("ln_fallback", 131, C, F32, F16)
    lf("ln_fallback", 9, 2048, BF16, F32)
    # errors: C beyond the quad plans' 5120, fallback C beyond 2048
    lf("error", 8, 5124, F32, F16)
    lf("error", 8, 2052, F16, F16)
    lf("error", 8, 2050, F32, F32)
    # epsilon, constant rows, mean / spread ratios on both routes
    for route, xd, C in (("ln_q_4_3", F32, 768), ("ln_fallback", F16, 768)):
        for eps in (1e-5, 1e-6):
            lf(route, 77, C, xd, F32, eps=eps, values="smallvar")
            lf(route, 77, C, xd, F16, eps=eps, values="const")
        for rho in (0.0, 8.0, 64.0, 256.0):
            lf(route, 77, C, xd, F32, rho=rho)

    # ---- LayerNorm backward: every (dy, dx) pairing x accumulate x dx_lp on every quad plan and on the fallback
    for M, C, route in plans:
        for g, d in BWD:
            for acc in (False, True):
                for lp in (False, True):
                    lb(route, M, C, g, d, acc=acc, lp=lp)
    for xd in (F16, BF16):
        for g, d in BWD:
            for acc in (False, True):
                for lp in (False, True):
                    lb("ln_fallback", 100, 768, g, d, xd=xd, acc=acc, lp=lp)
    for (g, d), shift in zip(BWD, ("x", "dy", "dx", "gamma", "dx_lp")):
        lb("ln_fallback", 70, 640, g, d, shift=shift, acc=True, lp=True)
    for M, C, route in ((256, 320, "ln_q_4_3"), (257, 320, "ln_q_1_3"), (1024, 1280, "ln_q_4_3"),
                        (1025, 1280, "ln_q_1_10"), (2000, 1284, "ln_q_4_3"), (300, 4100, "ln_q_4_10"),
                        (300, 5120, "ln_q_4_10"), (300, 64, "ln_q_1_3"), (300, 388, "ln_q_1_10")):
        lb(route, M, C, F16, F32, acc=True, lp=True)
    for C in (322, 770, 2046):
        lb("ln_fallback", 131, C, BF16, F32, acc=True, lp=True)
    lb("error", 8, 5124, F16, F32)
    lb("error", 8, 2052, F16, F32, xd=F16)
    lb("error", 8, 2050, F32, F32)
    for route, xd in (("ln_q_4_3", F32), ("ln_fallback", BF16)):
        for rho in (0.0, 8.0, 64.0, 256.0):
            lb(route, 77, 768, F16, F32, xd=xd, rho=rho, acc=True)
        lb(route, 77, 768, F32, F32, xd=xd, values="const", eps=1e-6)
        lb(route, 77, 768, F32, F32, xd=xd, values="smallvar", eps=1e-6)
    return T


CASES = list(dict.fromkeys(_cases()))
RUN_CASES = [c for c in CASES if c.route != "error"]
ERR_CASES = [c for c in CASES if c.route == "error"]
MAX_RHO = max(c.rho for c in CASES)


# ================================================================================================ values
def gen(name):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()))


def make_inputs(c):
    """host tensors: x (rows, C) in c.xd, gamma, beta (fp32), dy (backward), dx before (accumulate)"""
    g = gen(c.id)
    n_img, hw, G = c.groups
    cpg = c.C // G
    sd = torch.exp2(torch.empty(n_img, 1, G, 1).uniform_(-1, 1, generator=g).double())
    if c.values == "smallvar":
        sd = torch.full_like(sd, 1e-2)
    sign = torch.randint(0, 2, sd.shape, generator=g).double() * 2 - 1
    mu = c.rho * sd * sign
    z = torch.randn(n_img, hw, G, cpg, generator=g, dtype=F64)
    x = mu + sd * z
    if c.values == "const":
        x[:, :, ::3, :] = (mu + sd)[:, :, ::3, :]
    x = x.reshape(n_img * hw, c.C).to(c.xd)
    gamma = (1.0 + 0.5 * torch.randn(c.C, generator=g)).float()
    beta = (0.5 * torch.randn(c.C, generator=g)).float()
    out = {"x": x, "gamma": gamma, "beta": beta}
    if c.op.endswith("bwd"):
        out["dy"] = torch.randn(n_img * hw, c.C, generator=g).to(c.gd)
        mu64, var64, _ = stats_ref(x.double(), n_img, G)
        out["mean"] = mu64.reshape(-1).float()
        out["rstd"] = (1.0 / torch.sqrt(var64 + c.eps)).reshape(-1).float()
        if c.acc:
            out["prev"] = torch.randn(n_img * hw, c.C, generator=g).to(c.od)
    return out


# ================================================================================================ reference and bounds
def stats_ref(x, n_img, G):
    """fp64 (mean, variance, mean |x|) per (image, group) of x (n_img * hw, C), two-pass"""
    xg = x.reshape(n_img, -1, G, x.shape[-1] // G)
    mu = xg.mean(dim=(1, 3))
    var = ((xg - mu[:, None, :, None]) ** 2).mean(dim=(1, 3))
    return mu, var, xg.abs().mean(dim=(1, 3))


def per_elem(v, like):
    """(n_img, G) -> the shape (n_img * hw, C) of `like`"""
    (n_img, G), (rows, C) = v.shape, like.shape
    return v[:, None, :, None].expand(n_img, rows // n_img, G, C // G).reshape(rows, C)


def gmean(t, n_img, G):
    """per (image, group) mean of t (n_img * hw, C), broadcast back to t's shape"""
    C = t.shape[-1]
    m = t.reshape(n_img, -1, G, C // G).mean(dim=(1, 3))
    return m[:, None, :, None].expand(n_img, t.shape[0] // n_img, G, C // G).reshape(-1, C)


def half_ulp(a, dt):
    _, e = torch.frexp(a)
    return torch.ldexp(torch.ones_like(a), torch.clamp(e - 1, min=EMIN[dt]) - MANT[dt])


def ratio(d, scale):
    """d / scale, with 0 / 0 = 0 and d / 0 = inf"""
    return torch.where(scale > 0, d / torch.where(scale > 0, scale, 1.0), torch.where(d > 0, math.inf, 0.0))


def excess(out, ref, T):
    """(|out - ref| - half an ulp of out's dtype at the result) / (u T), >= 0"""
    o = out.double()
    d = (o - ref).abs() - half_ulp(torch.maximum(o.abs(), ref.abs()), out.dtype)
    return ratio(d.clamp_min(0), U * T)


def _worst(r):
    return r.max().item() if r.numel() else 0.0


def measure_fwd(c, inp, y, mean, rstd):
    """worst ratio per quantity of a forward's outputs"""
    n_img, _, G = c.groups
    x = inp["x"].to(y.device).double()
    g, b = inp["gamma"].to(y.device).double(), inp["beta"].to(y.device).double()
    mu, var, mabs = stats_ref(x, n_img, G)
    r = 1.0 / torch.sqrt(var + c.eps)
    cc = mu * mu / (var + c.eps) if c.op.startswith("gn") else torch.zeros_like(mu)
    res = {}
    for name, t in (("y", y), ("mean", mean), ("rstd", rstd)):
        if not torch.isfinite(t).all():
            return {name: math.inf}
    res["mean"] = _worst(ratio((mean.double().reshape(mu.shape) - mu).abs(), U * mabs))
    res["rstd"] = _worst(ratio((rstd.double().reshape(r.shape) - r).abs() / r, U * (1 + cc)))
    C = c.C
    xh = (x - per_elem(mu, x)) * per_elem(r, x)
    z = g * xh + b
    T = (g * xh).abs() * (1 + per_elem(cc, x)) + b.abs() + g.abs() * per_elem(r * mabs, x)
    if c.silu:
        s = torch.sigmoid(z)
        ref = z * s
        T = (s * (1 + z * (1 - s))).abs() * T + ref.abs() * (1 + z.abs())
    else:
        ref = z
    res["y"] = _worst(excess(y, ref, T))
    return res


def measure_bwd(c, inp, outs):
    """worst ratio of the backward's dx (and dx_lp): outs = [tensor, ...] holding the same result"""
    n_img, _, G = c.groups
    dev = outs[0].device
    x = inp["x"].to(dev).double()
    dy = inp["dy"].to(dev).double()
    g = inp["gamma"].to(dev).double()
    b = inp["beta"].to(dev).double()
    C = c.C
    m = per_elem(inp["mean"].to(dev).double().reshape(n_img, G), x)
    r = per_elem(inp["rstd"].to(dev).double().reshape(n_img, G), x)
    xh = (x - m) * r
    xa = (x.abs() + m.abs()) * r
    if c.silu:
        z = g * xh + b
        s = torch.sigmoid(z)
        dz = dy * s * (1 + z * (1 - s))
        tabs = (dy * g).abs() * (s + (z * s * (1 - s)).abs() + 0.5 * (g.abs() * xa + b.abs()))
    else:
        dz = dy
        tabs = (dy * g).abs()
    t = dz * g
    m1, m2 = gmean(t, n_img, G), gmean(t * xh, n_img, G)
    ref = r * (t - m1 - xh * m2)
    T = r * (tabs + gmean(tabs, n_img, G) + xh.abs() * gmean(tabs * xa, n_img, G) + xa * m2.abs())
    if c.acc:
        prev = inp["prev"].to(dev).double()
        ref = ref + prev
        T = T + prev.abs()
    worst = 0.0
    for o in outs:
        if not torch.isfinite(o).all():
            return {"dx": math.inf}
        worst = max(worst, _worst(excess(o, ref, T)))
    return {"dx": worst}


def verdict(c, res, record=True):
    """the quantities of res that exceed their K (recording the worst ratios when asked)"""
    bad = []
    for q, w in res.items():
        key = (q, c.family)
        dt = c.od if q in ("y", "dx") else F32
        if record:
            wk = (q, c.family, NAME[dt])
            WORST[wk] = max(WORST.get(wk, (0.0, "")), (w, c.id))
        if not w <= K[key]:
            bad.append(f"{q} {w:.3g} u > {K[key]}")
    return bad


# ================================================================================================ launching
class Buf:
    """a view of n elements (offset `extra` elements past a 16-byte boundary) in a NaN-filled allocation with GUARD
    elements before and after it"""

    def __init__(self, dtype, n, extra=0, fill=None):
        self.dtype = dtype
        self.buf = torch.full((n + 2 * GUARD + extra,), float("nan"), dtype=dtype, device="cuda")
        self.v = self.buf[GUARD + extra:GUARD + extra + n]
        if fill is not None:
            self.v.copy_(fill.reshape(-1))

    def ptr(self):
        return ctypes.c_void_p(self.v.data_ptr())

    def guards_intact(self):
        a = self.v.storage_offset()
        return bool(torch.isnan(self.buf[:a]).all() and torch.isnan(self.buf[a + self.v.numel():]).all())


def new_ws():
    ws = torch.empty(WS_BYTES // 8, dtype=F64, device="cuda")
    ws.view(torch.uint8).fill_(0xFF)
    return ws


def flags(c):
    f = (1 if c.silu else 0) | ((c.cap & 0xFFFF) << 8)
    if c.junk:
        f |= 0xFE | (0xFF << 24)
    return f - (1 << 32) if f >= 1 << 31 else f


def st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def shift_of(c, name):
    """8 bytes past a 16-byte boundary for the named pointer of a misaligned LayerNorm case"""
    if c.shift != name:
        return 0
    dt = {"x": c.xd, "y": c.od, "dx": c.od, "dy": c.gd, "dx_lp": c.gd}.get(name, F32)
    return 8 // esize(dt)


def launch(L, c, inp, ws=None, codes=None):
    """one call of the case's entry point on fresh poisoned buffers.  Returns (rc, outputs {name: Buf}, inputs)."""
    n_img, hw, G = c.groups
    nrow, C = n_img * hw, c.C
    codes = codes or {}
    x = Buf(c.xd, nrow * C, shift_of(c, "x"), inp["x"])
    gamma = Buf(F32, C, shift_of(c, "gamma"), inp["gamma"])
    beta = Buf(F32, C, shift_of(c, "beta"), inp["beta"])
    cx = codes.get("x", CODE[c.xd])
    ws = new_ws() if ws is None else ws
    if c.op.endswith("fwd"):
        y = Buf(c.od, nrow * C, shift_of(c, "y"))
        nst = n_img * G if c.op == "gn_fwd" else nrow
        mean, rstd = Buf(F32, nst), Buf(F32, nst)
        cy = codes.get("y", CODE[c.od])
        if c.op == "gn_fwd":
            rc = L.cb_groupnorm_fwd(x.ptr(), cx, y.ptr(), cy, gamma.ptr(), beta.ptr(), c.N, c.rows, C, c.G, c.eps,
                                    flags(c), mean.ptr(), rstd.ptr(), ctypes.c_void_p(ws.data_ptr()), st())
        else:
            rc = L.cb_layernorm_fwd(x.ptr(), cx, y.ptr(), cy, gamma.ptr(), beta.ptr(), c.rows, C, c.eps, mean.ptr(),
                                    rstd.ptr(), st())
        return rc, {"y": y, "mean": mean, "rstd": rstd}, [x, gamma, beta]
    dy = Buf(c.gd, nrow * C, shift_of(c, "dy"), inp["dy"])
    mean, rstd = Buf(F32, inp["mean"].numel(), 0, inp["mean"]), Buf(F32, inp["rstd"].numel(), 0, inp["rstd"])
    dx = Buf(c.od, nrow * C, shift_of(c, "dx"), inp.get("prev"))
    lp = Buf(c.gd, nrow * C, shift_of(c, "dx_lp")) if c.lp else None
    outs = {"dx": dx, **({"dx_lp": lp} if lp else {})}
    cg, cd = codes.get("dy", CODE[c.gd]), codes.get("dx", CODE[c.od])
    lpp = lp.ptr() if lp else None
    if c.op == "gn_bwd":
        rc = L.cb_groupnorm_bwd(dy.ptr(), cg, x.ptr(), cx, gamma.ptr(), beta.ptr(), mean.ptr(), rstd.ptr(), dx.ptr(), cd,
                                lpp, c.N, c.rows, C, c.G, flags(c), 1 if c.acc else 0, ctypes.c_void_p(ws.data_ptr()),
                                st())
    else:
        rc = L.cb_layernorm_bwd(dy.ptr(), cg, x.ptr(), cx, gamma.ptr(), mean.ptr(), rstd.ptr(), dx.ptr(), cd, lpp,
                                c.rows, C, 1 if c.acc else 0, st())
    return rc, outs, [x, gamma, beta, dy, mean, rstd]


def bits(t):
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def expected_kernels(c):
    """[(kernel, template arguments)] the case must launch, in order"""
    if c.route == "error":
        return []
    if c.op == "gn_fwd":
        if c.route == "gn_cluster_fwd":
            return [("gn_cluster_fwd_kernel", (c.xd, c.od))]
        return [("gn_stats_tma_kernel", (c.xd,)), ("gn_apply_tma_kernel", (c.xd, c.od))]
    if c.op == "gn_bwd":
        if c.route == "gn_cluster_bwd":
            return [("gn_cluster_bwd_kernel", (c.xd, c.gd, c.od))]
        return [("gn_bwd_stats_kernel", (c.xd, c.gd)), ("gn_bwd_apply_kernel", (c.xd, c.gd, c.od))]
    if c.route == "ln_fallback":
        return [("ln_fwd_kernel", (c.xd, c.od))] if c.op == "ln_fwd" else [("ln_bwd_kernel", (c.xd, c.gd, c.od))]
    w, q = (int(v) for v in c.route.split("_")[2:])
    return [("ln_fwd_q_kernel", (c.od, w, q))] if c.op == "ln_fwd" else [("ln_bwd_q_kernel", (c.gd, c.od, w, q))]


KERNEL_RE = re.compile(r"\b((?:gn|ln)_[a-z_]+_kernel)<([^<>]*)>")


def parse_kernel(name):
    m = KERNEL_RE.search(name)
    if m is None:
        return None
    args = []
    for a in m.group(2).split(","):
        a = re.sub(r"^\(\w+\)", "", a.strip())
        args.append(CTYPE[a] if a in CTYPE else int(a))
    return m.group(1), tuple(args)


# ================================================================================================ GPU tests
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from celebbasis_b200 import lib
    assert lib.load().cb_device_ok() == 1, "tests must run on an sm_90 device"
    yield torch.device("cuda:0")
    print()
    for (q, fam, dt), (w, what) in sorted(WORST.items()):
        print(f"[worst] {q:5s} {fam:12s} {dt:5s} {w:9.3f}  {what}")


def run_twice(L, c, inp):
    """two calls on fresh poisoned buffers: same bits, guards intact, every output element written"""
    rc1, o1, i1 = launch(L, c, inp)
    rc2, o2, _ = launch(L, c, inp)
    torch.cuda.synchronize()
    assert rc1 == 0 and rc2 == 0, f"{c.id}: rc={rc1}/{rc2}: {L.cb_last_error().decode()}"
    for k in o1:
        assert o1[k].guards_intact() and o2[k].guards_intact(), f"{c.id}: a write landed outside {k}"
        assert not torch.isnan(o1[k].v).any(), f"{c.id}: {int(torch.isnan(o1[k].v).sum())} elements of {k} unwritten"
        assert torch.equal(bits(o1[k].v), bits(o2[k].v)), f"{c.id}: two calls give different {k}"
    for b in i1:
        assert b.guards_intact()
    return o1


def check_case(L, c):
    inp = make_inputs(c)
    o = run_twice(L, c, inp)
    if c.op.endswith("fwd"):
        res = measure_fwd(c, inp, o["y"].v.view(-1, c.C), o["mean"].v, o["rstd"].v)
    else:
        res = measure_bwd(c, inp, [b.v.view(-1, c.C) for b in o.values()])
    bad = verdict(c, res)
    assert not bad, f"{c.id}: " + "; ".join(bad)
    return o


@pytest.mark.gpu
@pytest.mark.parametrize("c", RUN_CASES, ids=lambda c: c.id)
def test_case_within_fp64_bound(dev, c):
    from celebbasis_b200 import lib
    check_case(lib.load(), c)


@pytest.mark.gpu
@pytest.mark.parametrize("c", ERR_CASES, ids=lambda c: c.id)
def test_unsupported_shape_is_refused(dev, c):
    """C past the quad plans' 5120 (fp32) or the fallback's 2048 returns CB_ERR_ARG and launches nothing"""
    from celebbasis_b200 import lib
    L = lib.load()
    _refused(L, c, {})


def _refused(L, c, codes):
    c = replace(c, acc=False)                 # every output buffer starts as NaN
    inp = make_inputs(c)
    ws = new_ws()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        rc, outs, _ = launch(L, c, inp, ws=ws, codes=codes)
        torch.cuda.synchronize()
    assert rc == CB_ERR_ARG, f"{c.id} {codes}: rc={rc}"
    launched = [e.name for e in prof.events() if parse_kernel(e.name)]
    assert launched == [], f"{c.id} {codes}: launched {launched}"
    for k, b in outs.items():
        assert torch.isnan(b.buf).all(), f"{c.id} {codes}: {k} was written"
    assert bool((ws.view(torch.uint8) == 0xFF).all()), f"{c.id} {codes}: the workspace was written"


BAD_DTYPES = (3, 7, -1)


@pytest.mark.gpu
def test_invalid_dtype_launches_nothing(dev):
    """Every dtype argument outside {F16, BF16, F32} returns CB_ERR_ARG before any launch, on every route: buffers of
    the right size, no kernel in the profile, outputs and workspace untouched.  (The LayerNorm backward's quad route once
    took any dy dtype other than F32 / F16 for bf16 and launched; the GroupNorm forward's streaming pair launched its
    statistics kernel before it looked at the y dtype.)"""
    from celebbasis_b200 import lib
    L = lib.load()
    reps = {}
    for c in RUN_CASES:
        reps.setdefault((c.op, c.route, c.xd == F32), c)
    assert {r for _, r, _ in reps} == {c.route for c in RUN_CASES}
    for c in reps.values():
        args = ("x", "y") if c.op.endswith("fwd") else ("x", "dy", "dx")
        for a in args:
            for bad in BAD_DTYPES:
                _refused(L, c, {a: bad})
        if c.op.endswith("bwd"):
            _refused(L, replace(c, od=F32), {"dy": BAD_DTYPES[1]})       # dx fp32: only dy is wrong


@pytest.mark.gpu
def test_routes_match_the_table(dev):
    """The kernels each case launches (name and template arguments, read from the profiler) are the route and
    instantiation its table row states."""
    from celebbasis_b200 import lib
    L = lib.load()
    data = [(c, make_inputs(c)) for c in RUN_CASES]
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for c, inp in data:
            rc, _, _ = launch(L, c, inp)
            assert rc == 0, c.id
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if parse_kernel(e.name)), key=lambda e: e.time_range.start)
    got = [parse_kernel(e.name) for e in ev]
    want = [k for c, _ in data for k in expected_kernels(c)]
    assert len(got) == len(want), (len(got), len(want))
    i = 0
    for c, _ in data:
        n = len(expected_kernels(c))
        assert got[i:i + n] == expected_kernels(c), f"{c.id}: launched {got[i:i + n]}"
        i += n


@pytest.mark.gpu
def test_cta_caps_and_stale_workspace(dev):
    """CB_GN_CTA_CAP(n): each cap's streaming runs are bit-reproducible and within the bound.  A call with fewer CTAs
    on a workspace that a call with many CTAs just filled gives the same bits as on a NaN-filled workspace, so no stale
    partial is read."""
    from celebbasis_b200 import lib
    L = lib.load()
    base = Case("gn_fwd", "gn_pair_fwd", 1, 3000, 128, 64, F32, F16, silu=True)
    inp = make_inputs(base)
    for cap in (1, 7, 16):
        c = replace(base, cap=cap)
        check_case(L, c)
        ws = new_ws()
        rc, _, _ = launch(L, replace(base, cap=0), inp, ws=ws)          # every CTA publishes a partial
        assert rc == 0
        rc, o_stale, _ = launch(L, c, inp, ws=ws)
        rc2, o_fresh, _ = launch(L, c, inp)
        torch.cuda.synchronize()
        assert rc == 0 and rc2 == 0
        for k in o_fresh:
            assert torch.equal(bits(o_stale[k].v), bits(o_fresh[k].v)), f"cap {cap}: {k} depends on stale partials"
    bw = Case("gn_bwd", "gn_pair_bwd", 1, 3000, 128, 64, F32, F32, F16)
    ws = new_ws()
    big = Case("gn_bwd", "gn_pair_bwd", 1, 60000, 128, 64, F32, F32, F16)
    assert launch(L, big, make_inputs(big), ws=ws)[0] == 0
    inp = make_inputs(bw)
    rc, o_stale, _ = launch(L, bw, inp, ws=ws)
    rc2, o_fresh, _ = launch(L, bw, inp)
    torch.cuda.synchronize()
    assert rc == 0 and rc2 == 0 and torch.equal(bits(o_stale["dx"].v), bits(o_fresh["dx"].v))


@pytest.mark.gpu
def test_ignored_flag_bits(dev):
    """Bits 1-7 and 24-31 of the flag word change nothing: same bits as the call without them"""
    from celebbasis_b200 import lib
    L = lib.load()
    for c in [c for c in RUN_CASES if c.junk]:
        inp = make_inputs(c)
        _, a, _ = launch(L, c, inp)
        _, b, _ = launch(L, replace(c, junk=False), inp)
        torch.cuda.synchronize()
        for k in a:
            assert torch.equal(bits(a[k].v), bits(b[k].v)), f"{c.id}: {k}"


# ------------------------------------------------------------------------------------------------ the workload's calls
def _route_of_call(op, x, C, n, hw, G, dts, ptrs):
    if op.startswith("gn"):
        bpe = esize(x.dtype) + (esize(dts[0]) if op == "gn_bwd" else 0)
        return (f"gn_cluster_{op[3:]}" if gn_plan(n, hw, C, G, bpe) else f"gn_pair_{op[3:]}")
    plan = ln_plan(x.shape[0], C)
    aligned = all(p % 16 == 0 for p in ptrs if p)
    if x.dtype == F32 and aligned and plan:
        return f"ln_q_{plan[0]}_{plan[1]}"
    return "ln_fallback"


class _Recorder:
    """wraps ops.groupnorm / groupnorm_bwd / layernorm / layernorm_bwd: synchronizes, clones the inputs (and dx before
    an accumulate), calls the original and measures the result against the fp64 bounds"""

    def __init__(self, ops):
        self.ops = ops
        self.orig = {n: getattr(ops, n) for n in ("groupnorm", "groupnorm_bwd", "layernorm", "layernorm_bwd")}
        self.engine = None
        self.calls, self.bad, self.types, self.rho = 0, [], set(), {}

    def _record(self, c, res, x, n_img, G):
        self.calls += 1
        self.types.add(c.row_type())
        bad = verdict(c, res)
        if bad:
            self.bad.append(f"{self.engine}: {c.id}: " + "; ".join(bad))
        if c.op.endswith("fwd"):
            mu, var, _ = stats_ref(x.double(), n_img, G)
            rho = (mu.abs() / torch.sqrt(var + c.eps)).max().item()
            self.rho[self.engine] = max(self.rho.get(self.engine, 0.0), rho)

    def groupnorm(self, x, geo, gamma, beta, *, groups=32, eps=1e-5, silu=False, out_dtype=F16, want_stats=True):
        torch.cuda.synchronize()
        inp = {"x": x.clone(), "gamma": gamma.clone(), "beta": beta.clone()}
        y, stats = self.orig["groupnorm"](x, geo, gamma, beta, groups=groups, eps=eps, silu=silu, out_dtype=out_dtype,
                                          want_stats=want_stats)
        torch.cuda.synchronize()
        C = x.shape[1]
        route = _route_of_call("gn_fwd", x, C, geo.n, geo.hw, groups, (), ())
        c = Case("gn_fwd", route, geo.n, geo.hw, C, groups, x.dtype, out_dtype, eps=eps, silu=silu)
        self._record(c, measure_fwd(c, inp, y, stats.mean, stats.rstd), inp["x"], geo.n, groups)
        return y, stats

    def groupnorm_bwd(self, dy, x, geo, gamma, beta, stats, *, groups=32, silu=False, dx=None, accumulate=False,
                      dx_dtype=F32, dx_lp=None):
        torch.cuda.synchronize()
        acc = accumulate and dx is not None
        inp = {"x": x.clone(), "dy": dy.clone(), "gamma": gamma.clone(), "beta": beta.clone(),
               "mean": stats.mean.clone(), "rstd": stats.rstd.clone()}
        if acc:
            inp["prev"] = dx.clone()
        out = self.orig["groupnorm_bwd"](dy, x, geo, gamma, beta, stats, groups=groups, silu=silu, dx=dx,
                                         accumulate=accumulate, dx_dtype=dx_dtype, dx_lp=dx_lp)
        torch.cuda.synchronize()
        C = x.shape[1]
        route = _route_of_call("gn_bwd", x, C, geo.n, geo.hw, groups, (dy.dtype,), ())
        c = Case("gn_bwd", route, geo.n, geo.hw, C, groups, x.dtype, out.dtype, dy.dtype, silu=silu, acc=acc,
                 lp=dx_lp is not None)
        outs = [out.view(-1, C)] + ([dx_lp.view(-1, C)] if dx_lp is not None else [])
        self._record(c, measure_bwd(c, inp, outs), inp["x"], geo.n, groups)
        return out

    def layernorm(self, x, gamma, beta, *, eps=1e-5, out_dtype=F16):
        torch.cuda.synchronize()
        inp = {"x": x.clone(), "gamma": gamma.clone(), "beta": beta.clone()}
        y, stats = self.orig["layernorm"](x, gamma, beta, eps=eps, out_dtype=out_dtype)
        torch.cuda.synchronize()
        M, C = x.shape
        route = _route_of_call("ln_fwd", x, C, M, 1, 1, (), (x.data_ptr(), y.data_ptr(), gamma.data_ptr(),
                                                             beta.data_ptr()))
        c = Case("ln_fwd", route, 1, M, C, 0, x.dtype, out_dtype, eps=eps)
        self._record(c, measure_fwd(c, inp, y, stats.mean, stats.rstd), inp["x"], M, 1)
        return y, stats

    def layernorm_bwd(self, dy, x, gamma, stats, *, dx=None, accumulate=False, dx_dtype=F32, dx_lp=None):
        torch.cuda.synchronize()
        acc = accumulate and dx is not None
        inp = {"x": x.clone(), "dy": dy.clone(), "gamma": gamma.clone(), "beta": torch.zeros_like(gamma),
               "mean": stats.mean.clone(), "rstd": stats.rstd.clone()}
        if acc:
            inp["prev"] = dx.clone()
        out = self.orig["layernorm_bwd"](dy, x, gamma, stats, dx=dx, accumulate=accumulate, dx_dtype=dx_dtype,
                                         dx_lp=dx_lp)
        torch.cuda.synchronize()
        M, C = x.shape
        ptrs = (x.data_ptr(), dy.data_ptr(), out.data_ptr(), dx_lp.data_ptr() if dx_lp is not None else 0,
                gamma.data_ptr())
        route = _route_of_call("ln_bwd", x, C, M, 1, 1, (dy.dtype,), ptrs)
        c = Case("ln_bwd", route, 1, M, C, 0, x.dtype, out.dtype, dy.dtype, acc=acc, lp=dx_lp is not None)
        outs = [out.view(-1, C)] + ([dx_lp.view(-1, C)] if dx_lp is not None else [])
        self._record(c, measure_bwd(c, inp, outs), inp["x"], M, 1)
        return out

    def install(self, monkeypatch):
        for n in self.orig:
            monkeypatch.setattr(self.ops, n, getattr(self, n))


@pytest.mark.gpu
def test_workload_calls_within_bounds(dev, monkeypatch):
    """Every GroupNorm / LayerNorm call of eager engine runs -- the tiny and the full (SD-v1, 64x64 latent) UNet forward
    + backward, the CLIP text encoder forward + backward, the VAE encoder at 512x512 and the decoder from a 64x64
    latent, each in fp16 and bf16 -- is within the fp64 bounds above; every (route, dtypes, SiLU, accumulate, dx_lp)
    combination these calls make is a row type of CASES; and the largest mean / spread ratio |mu| / sqrt(s2 + eps) of
    their inputs is covered by CASES.  The weights are synthetic (synth.synth_state_dict): the ratios a trained
    checkpoint produces are not measured here."""
    from celebbasis_b200 import ops, synth, workload
    from celebbasis_b200.clip_engine import CLIPTextEngine
    from celebbasis_b200.unet_engine import UNetEngine
    from celebbasis_b200.vae_engine import VAEDecoderEngine, VAEEncoderEngine
    from oracle import torch_ref
    rec = _Recorder(ops)
    rec.install(monkeypatch)
    g = torch.Generator().manual_seed(5)
    for kind in ("tiny", "full"):
        params = workload.model_params(kind)
        om = torch_ref.OracleModel(params, clip_layers=workload.clip_layers(kind))
        sd = synth.synth_state_dict(om, seed=0)
        del om
        sub = lambda pre: {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}
        lat = params["image_size"]
        for dt in (F16, BF16):
            rec.engine = f"unet-{kind}-{NAME[dt]}"
            eng = UNetEngine(params["unet_config"]["params"], sub("model.diffusion_model."), dev, dtype=dt)
            x = torch.randn(1, 4, lat, lat, generator=g).to(dev)
            t = torch.tensor([371], device=dev)
            ctx = torch.randn(1, 77, 768, generator=g).to(dev)
            eps = eng.forward(x, t, ctx)
            eng.backward(torch.randn(eps.shape, generator=g).to(dev) * 1e-3)
            del eng
            rec.engine = f"clip-{kind}-{NAME[dt]}"
            clip = CLIPTextEngine(sub("cond_stage_model.transformer."), dev, dtype=dt)
            clip.forward(torch.randn(77, 768, generator=g).to(dev) * 0.5, 1)
            clip.backward(torch.randn(77, 768, generator=g).to(dev) * 1e-3)
            del clip
            if kind == "full":
                fs = params["first_stage_config"]["params"]
                rec.engine = f"vae-enc-{NAME[dt]}"
                enc = VAEEncoderEngine(fs["ddconfig"], fs["embed_dim"], sub("first_stage_model."), dev, dtype=dt)
                enc.encode_moments(torch.rand(1, 3, 512, 512, generator=g).to(dev) * 2 - 1)
                del enc
                rec.engine = f"vae-dec-{NAME[dt]}"
                dsd = synth.synth_state_dict(torch_ref.AutoencoderKLDecode(fs["ddconfig"], fs["embed_dim"]), seed=0,
                                             prefix="first_stage_model.")
                dec = VAEDecoderEngine(fs["ddconfig"], fs["embed_dim"], dsd, dev, dtype=dt)
                dec.decode(torch.randn(1, 4, 64, 64, generator=g).to(dev))
                del dec
            torch.cuda.empty_cache()
    for e, r in sorted(rec.rho.items()):
        print(f"[rho] {e:18s} {r:10.3f}")
    print(f"[workload] {rec.calls} norm calls, {len(rec.types)} row types")
    assert rec.calls > 100
    assert not rec.bad, "\n".join(rec.bad[:20])
    table = {c.row_type() for c in RUN_CASES}
    missing = sorted(str(t) for t in rec.types - table)
    assert not missing, "row types without a synthetic case:\n" + "\n".join(missing)
    assert max(rec.rho.values()) <= MAX_RHO, rec.rho


# ================================================================================================ CPU tests
def test_table_routes_follow_the_plans():
    """The route of every row is the one cb_groupnorm_cluster_plan / the ln_plan mirror give; the cluster rows reach
    every slab width the plan can pick, and some have CTAs with empty row ranges."""
    gpcs, empty_ctas = set(), 0
    for c in CASES:
        if c.op.startswith("gn"):
            bpe = esize(c.xd) + (esize(c.gd) if c.op == "gn_bwd" else 0)
            plan = gn_plan(c.N, c.rows, c.C, c.G, bpe)
            want = f"gn_{'cluster' if plan else 'pair'}_{c.op[3:]}"
            assert c.route == want, f"{c.id}: the plan gives {want}"
            if plan:
                S, gpc, rows, _ = plan
                gpcs.add(gpc)
                empty_ctas += S * rows - c.rows >= rows
            if c.op == "gn_fwd":
                assert c.C * esize(c.xd) % 16 == 0, c.id
        else:
            plan = ln_plan(c.rows, c.C)
            if c.xd == F32 and plan and not c.shift:
                want = f"ln_q_{plan[0]}_{plan[1]}"
            elif c.C <= 2048 and c.C % 2 == 0:
                want = "ln_fallback"
            else:
                want = "error"
            assert c.route == want, f"{c.id}: ln_plan gives {want}"
    assert gpcs == {1, 2, 4, 8, 16, 32}
    assert empty_ctas >= 2


def test_table_covers_the_edges():
    gn = [c for c in RUN_CASES if c.op.startswith("gn")]
    ln = [c for c in RUN_CASES if c.op.startswith("ln")]
    for op, route in (("gn_fwd", "gn_cluster_fwd"), ("gn_fwd", "gn_pair_fwd")):
        got = {(c.xd, c.od, c.silu) for c in gn if c.route == route}
        assert got == {(a, b, s) for a in DTYPES for b in DTYPES for s in (False, True)}, route
    for route in ("gn_cluster_bwd", "gn_pair_bwd"):
        got = {(c.xd, c.gd, c.od, c.silu, c.acc, c.lp) for c in gn if c.route == route}
        assert len(got) == 3 * 5 * 8, route
    assert {c.C // c.G for c in gn} >= {2, 6, 10, 30, 4, 20, 40, 80}
    assert {c.G for c in gn} >= {1, 2, 3, 4, 8, 16, 32, 64} and any(32 < c.G < 64 for c in gn)
    assert {c.N for c in gn} >= {1, 2, 3, 16} and min(c.rows for c in gn) == 1
    assert any(c.rows >= 65536 and c.route == "gn_pair_fwd" for c in gn)
    assert any(c.rows >= 65536 and c.route == "gn_pair_bwd" for c in gn)
    assert {c.cap for c in gn} >= {1, 7, 16}
    quad = {r for r in (c.route for c in ln) if r.startswith("ln_q")}
    assert quad == {"ln_q_1_3", "ln_q_1_10", "ln_q_4_3", "ln_q_4_10"}
    for r in quad:
        assert {c.od for c in ln if c.op == "ln_fwd" and c.route == r} == set(DTYPES), r
        assert len({(c.gd, c.od, c.acc, c.lp) for c in ln if c.op == "ln_bwd" and c.route == r}) == 20, r
    assert {c.C for c in ln} >= {64, 320, 384, 388, 640, 768, 1280, 1284, 2048, 4100, 5120}
    assert {c.rows for c in ln} >= {256, 257, 1024, 1025}
    assert {c.shift for c in ln} >= {"x", "y", "gamma", "beta", "dy", "dx", "dx_lp"}
    for op in ("gn", "ln"):
        cs = [c for c in RUN_CASES if c.op.startswith(op)]
        assert {c.rho for c in cs} >= {0.0, 1.0, 8.0, 64.0}
        assert {(c.eps, c.values) for c in cs} >= {(e, v) for e in (1e-5, 1e-6) for v in ("smallvar", "const")}


def _tool(name):
    found = shutil.which(name)
    if found:
        return found
    cand = os.path.join("/usr/local/cuda/bin", name)
    return cand if os.path.exists(cand) else None


@pytest.mark.parametrize("src", ["cb_norm.cu", "cb_layernorm.cu"])
def test_every_compiled_instantiation_has_cases(src, tmp_path):
    """Every gn_* / ln_* kernel instantiation in the compiled object is launched by at least one case, and every case's
    kernels are compiled."""
    from celebbasis_b200 import build
    cuobjdump, cufilt = _tool("cuobjdump"), _tool("cu++filt")
    if cuobjdump is None or cufilt is None:
        pytest.skip("cuobjdump / cu++filt not available")
    path = os.path.join(build.CSRC, src)
    obj = os.path.join(build.OBJ, src[:-3] + ".o")
    stamp = obj + ".sha1"
    if not (os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == build._digest(path)):
        nvcc = _tool("nvcc")
        if nvcc is None:
            pytest.skip(f"no up-to-date {src[:-3]}.o and no nvcc")
        obj = str(tmp_path / (src[:-3] + ".o"))
        r = subprocess.run([nvcc, *build.NVCC_FLAGS, "-c", path, "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-4000:]
    r = subprocess.run([cuobjdump, "-symbols", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    mangled = sorted(set(re.findall(r"\S*(?:gn|ln)_\w+_kernel\S*", r.stdout)))
    r = subprocess.run([cufilt], input="\n".join(mangled) + "\n", capture_output=True, text=True)
    mine = {parse_kernel(line) for line in r.stdout.splitlines()} - {None}
    assert mine, f"no gn_* / ln_* kernel in {src[:-3]}.o"
    cased = {k for c in RUN_CASES for k in expected_kernels(c)}
    prefix = ("gn_", "ln_bwd_kernel", "ln_fwd_kernel") if src == "cb_norm.cu" else ("ln_fwd_q", "ln_bwd_q")
    cased = {k for k in cased if k[0].startswith(prefix)}
    assert sorted(map(str, mine - cased)) == [], "instantiations without cases"
    assert sorted(map(str, cased - mine)) == [], "cases whose kernels are not compiled"


# ------------------------------------------------------------------------------------------------ bound tightness
MUTANTS = ("unbiased", "eps_sigma", "eps_swap", "straddle", "drop_slice", "twice_slice", "sq16", "silu_sigma",
           "no_xhat_term")
f32 = np.float32


def _slices(n, k):
    step = -(-n // k)
    return [(i, min(n, i + step)) for i in range(0, n, step)]


def _fp32_sums(a, b, n_img, G, mut, sq=False):
    """sums per (image, group) of a and of b (n_img, hw, C) float32: each CTA slice of the rows adds its rows one after
    the other in fp32 per channel, then its channels in fp32; the slices' partials are added in fp64"""
    hw, C = a.shape[1], a.shape[2]
    s1 = np.zeros((n_img, G))
    s2 = np.zeros((n_img, G))
    sl = _slices(hw, min(4, hw))
    for k, (r0, r1) in enumerate(sl):
        acc1 = np.zeros((n_img, C), f32)
        acc2 = np.zeros((n_img, C), np.float16 if (sq and mut == "sq16") else f32)
        for r in range(r0, r1):
            acc1 = (acc1 + a[:, r]).astype(f32)
            acc2 = (acc2.astype(f32) + b[:, r]).astype(acc2.dtype)
        p1 = acc1.reshape(n_img, G, -1).sum(-1, dtype=f32)
        p2 = acc2.astype(f32).reshape(n_img, G, -1).sum(-1, dtype=f32)
        if mut == "drop_slice" and k == len(sl) - 1 and len(sl) > 1:
            continue
        reps = 2 if mut == "twice_slice" and k == 0 else 1
        s1 += reps * p1.astype(np.float64)
        s2 += reps * p2.astype(np.float64)
    return s1, s2


def emulate_fwd(c, inp, mut=None):
    """an fp32 emulation of the forward kernels (one-pass statistics for GroupNorm, two-pass for LayerNorm)"""
    n_img, hw, G = c.groups
    C, cpg = c.C, c.C // G
    x = inp["x"].float().numpy().reshape(n_img, hw, C)
    gam, bet = inp["gamma"].numpy(), inp["beta"].numpy()
    eps = {1e-5: 1e-6, 1e-6: 1e-5}[c.eps] if mut == "eps_swap" else c.eps
    n = hw * cpg
    if c.op == "gn_fwd":
        s1, s2 = _fp32_sums(x, (x * x).astype(f32), n_img, G, mut, sq=True)
        m = s1 / n
        var = np.maximum(s2 / n - m * m, 0.0)
    else:
        xs = x.reshape(n_img, C)
        m32 = xs.sum(-1, dtype=f32, keepdims=True) / f32(C)
        if mut == "drop_slice":
            m32 = xs[:, :C - C // 4].sum(-1, dtype=f32, keepdims=True) / f32(C)
        d = (xs - m32).astype(f32)
        acc = (d * d).astype(np.float16 if mut == "sq16" else f32)
        var = acc.sum(-1, dtype=acc.dtype, keepdims=True).astype(f32) / f32(C)
        m, var = m32.astype(np.float64), var.astype(np.float64)
    if mut == "unbiased" and n > 1:
        var = var * n / (n - 1)
    if mut == "eps_sigma":
        rs = (1.0 / (np.sqrt(var) + eps)).astype(f32)
    elif c.op == "gn_fwd":
        rs = (1.0 / np.sqrt(var + eps)).astype(f32)
    else:
        rs = (f32(1) / np.sqrt((var.astype(f32) + f32(eps)).astype(f32))).astype(f32)
    m32 = m.astype(f32)
    ch = np.arange(C)
    gch = (4 * (ch // 4)) // cpg if mut == "straddle" else ch // cpg
    if c.op == "gn_fwd":
        ga = (gam * rs[:, gch]).astype(f32)
        be = (bet - (m32[:, gch] * ga).astype(f32)).astype(f32)
        y = ((x * ga[:, None]).astype(f32) + be[:, None]).astype(f32)
    else:
        xs = x.reshape(n_img, C)
        y = (((((xs - m32).astype(f32) * rs).astype(f32)) * gam).astype(f32) + bet).astype(f32)
    if c.silu:
        y = (y * (f32(1) / (f32(1) + np.exp(-y)).astype(f32))).astype(f32)
    y = torch.from_numpy(y.reshape(-1, C)).to(c.od)
    return y, torch.from_numpy(m32.reshape(-1)), torch.from_numpy(rs.reshape(-1))


def emulate_bwd(c, inp, mut=None):
    """an fp32 emulation of the backward kernels"""
    n_img, hw, G = c.groups
    C, cpg = c.C, c.C // G
    x = inp["x"].float().numpy().reshape(n_img, hw, C)
    dy = inp["dy"].float().numpy().reshape(n_img, hw, C)
    gam, bet = inp["gamma"].numpy(), inp["beta"].numpy()
    gch = np.arange(C) // cpg
    m = inp["mean"].numpy().reshape(n_img, G)[:, None, gch]
    r = inp["rstd"].numpy().reshape(n_img, G)[:, None, gch]
    xh = ((x - m).astype(f32) * r).astype(f32)
    d = dy
    if c.silu:
        z = ((xh * gam).astype(f32) + bet).astype(f32)
        s = (f32(1) / (f32(1) + np.exp(-z)).astype(f32)).astype(f32)
        sp = s if mut == "silu_sigma" else (s * (f32(1) + (z * (f32(1) - s)).astype(f32))).astype(f32)
        d = (dy * sp).astype(f32)
    t = (d * gam).astype(f32)
    s1, s2 = _fp32_sums(t, (t * xh).astype(f32), n_img, G, mut)
    n = hw * cpg
    m1 = (s1 / n).astype(f32)[:, None, gch]
    m2 = (s2 / n).astype(f32)[:, None, gch]
    if mut == "no_xhat_term":
        m2 = np.zeros_like(m2)
    o = (r * ((t - m1).astype(f32) - (xh * m2).astype(f32)).astype(f32)).astype(f32)
    if c.acc:
        o = (o + inp["prev"].float().numpy().reshape(o.shape)).astype(f32)
    return torch.from_numpy(o.reshape(-1, C)).to(c.od)


def _reduced(c):
    if c.op.startswith("gn"):
        return replace(c, N=min(c.N, 2), rows=min(c.rows, 37))
    return replace(c, rows=min(c.rows, 5))


EMU_CASES = sorted({_reduced(c) for c in RUN_CASES if not c.junk and not c.cap}, key=lambda c: c.id)


def _emu_fails(c, inp, mut):
    with np.errstate(over="ignore"):          # exp(-z) of very negative z, fp16 squares past 65504: inf as intended
        if c.op.endswith("fwd"):
            y, mean, rstd = emulate_fwd(c, inp, mut)
        else:
            dx = emulate_bwd(c, inp, mut)
    if c.op.endswith("fwd"):
        res = measure_fwd(c, inp, y, mean, rstd)
    else:
        outs = [dx]
        if c.lp:
            outs.append(outs[0].float().to(c.gd) if c.od != c.gd else outs[0])
        res = measure_bwd(c, inp, outs)
    return verdict(c, res, record=False)


def test_bounds_pass_an_fp32_emulation_and_fail_mutants():
    """An fp32 emulation of the kernels passes every case (at reduced size); each mutant -- unbiased variance, eps added
    to the spread or 1e-5 / 1e-6 swapped, a straddling quad normalised with one group's statistics, one CTA slice's
    partial dropped or added twice, squares summed in fp16, SiLU backward with sigma(z) for its derivative, a backward
    without the xhat * mean(dz g xhat) term -- fails at least one."""
    caught = {m: [] for m in MUTANTS}
    for c in EMU_CASES:
        inp = make_inputs(c)
        bad = _emu_fails(c, inp, None)
        assert not bad, f"faithful emulation, {c.id}: {bad}"
        for mut in MUTANTS:
            if _emu_fails(c, inp, mut):
                caught[mut].append(c.id)
    missed = [m for m, v in caught.items() if not v]
    assert not missed, f"mutants that pass every case: {missed}"
