"""Typed launchers over the C-ABI: torch tensors are only storage + stream plumbing here.

Layout conventions (see include/celebbasis_b200.h): activations are 2-D channels-last matrices
[rows][C] (rows = N*H*W pixels in raster order, or tokens).  All math happens inside the .so.
"""
import ctypes
import os

import torch

from . import lib as _lib
from .lib import (CB_ACT_GELU, CB_ACT_NONE, CB_ACT_PRELU, CB_ACT_QUICK_GELU, CB_ACT_SILU, CB_BF16, CB_F16, CB_F32,
                  CB_MAJOR_K, CB_MAJOR_MN, GemmDesc)

_DT = {torch.float16: CB_F16, torch.bfloat16: CB_BF16, torch.float32: CB_F32}


def _dt(t):
    return _DT[t.dtype]


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _L():
    return _lib.load()


GEMM_DEBUG_TIMELINE = None   # device int64 tensor (8 per CTA) to receive per-CTA timestamps (tools/gemm_timeline.py)
GEMM_RECORD = None   # when set to a list, every cb_gemm launch appends (bytes(GemmDesc), flops) -- bench.py roofline


SPLITK_WS_BYTES = 96 << 20
_splitk_ws = {}
_LANE = 0     # launches that share a workspace must be stream-ordered: a concurrent branch runs under `with lane(1)`


class lane:
    """Select the workspace set (split-K accumulators, GroupNorm slots) used by launches inside the block.  The two
    independent branches of the step (VAE encode | face net -> CLIP text) run on two streams; each gets its own lane."""

    def __init__(self, idx):
        self.idx = int(idx)

    def __enter__(self):
        global _LANE
        self.prev, _LANE = _LANE, self.idx

    def __exit__(self, *exc):
        global _LANE
        _LANE = self.prev


def _splitk_workspace(device):
    """One zero-initialised split-K workspace per (device, lane); stream-ordered cb_gemm launches share it."""
    ws = _splitk_ws.get((device, _LANE))
    if ws is None:
        ws = torch.zeros(SPLITK_WS_BYTES if _LANE == 0 else SPLITK_WS_BYTES // 4, dtype=torch.uint8, device=device)
        _splitk_ws[(device, _LANE)] = ws
    return ws


# ---- per-shape tile autotuner --------------------------------------------------------------------------------
# cb_gemm picks its tile width and split-K factor from a cost model; at bs=1 most launches are latency / L2-fabric
# bound and the model is off by up to 1.5x on some shapes, so the first (eager, un-captured) launch of every distinct
# shape times the candidates on the device (CUDA-graph replay of 8 launches each, output redirected to scratch) and
# later launches -- including the ones captured into the step graph -- pass the winner in desc.tile_n / desc.splits.
AUTOTUNE = os.environ.get("CB_GEMM_AUTOTUNE", "1") != "0"
# split-K slices as a thread-block cluster reducing through DSMEM (desc.splitk_cluster): an autotuner candidate on the lane-0
# stream (=1, default), on every lane (=2) or never (=0).  Lane 0 is the default because the lanes other than 0 were tuned
# and measured without cluster split-K; whether it helps beside concurrent streams has not been measured.
CLUSTER_SK = os.environ.get("CB_GEMM_CLUSTER_SK", "1") != "0"
CLUSTER_SK_ALL_LANES = os.environ.get("CB_GEMM_CLUSTER_SK", "1") == "2"   # A/B aid: also beside concurrent streams
# Front-end SM budget (CB_FE_CTAS = n > 0): the software-pipelined front end (VAE encode of the NEXT batch, lane 2) runs
# its large GEMMs as fixed 128 x (128 | 256) tiles without split-K (no autotuning) and its streaming GroupNorm on at most n
# CTAs, so the latency-bound chain of small launches that trains the CURRENT batch finds free SMs instead of queueing behind
# a wave of VAE CTAs (step_graph.py).  0 = every kernel sizes its grid for the whole device.
FE_CTAS = int(os.environ.get("CB_FE_CTAS", "0"))
FE_LANES = (2,)
_TUNE = {}
_TUNE_NC = {}
_tune_scratch = {}
_tune_stream = {}
TUNE_LOG = None     # set to a list to collect (key, table of candidate times)


def _tune_key(d):
    return (d.M, d.N, d.K, d.batch, d.batch_inner, d.ab_dtype, d.a_major, d.b_major, d.conv, d.img_n, d.img_h, d.img_w,
            d.out_h, d.out_w, d.kh, d.kw, d.stride, d.flip_taps, d.d_dtype, d.d_transposed, 1 if d.R else 0, d.r_dtype,
            1 if d.bias else 0, d.act, d.lda, d.ldb, d.ldd, (d.d2_dtype + 1) if d.D2 else 0, 1 if d.d2_scale else 0, d.glu,
            1 if d.D else 0)


def _set_out2(d, out2, out2_affine=None, act_param=None):
    if out2 is not None:
        assert out2.dim() == 2 and out2.stride(1) == 1
        d.D2, d.d2_dtype, d.ldd2 = out2.data_ptr(), _dt(out2), out2.stride(0)
        if out2_affine is not None:
            sc, sh = out2_affine
            assert sc.dtype == torch.float32 and sh.dtype == torch.float32 and sc.numel() >= d.N and sh.numel() >= d.N
            d.d2_scale, d.d2_shift = sc.data_ptr(), sh.data_ptr()
    if act_param is not None:
        assert act_param.dtype == torch.float32 and act_param.numel() >= d.N
        d.act_param = act_param.data_ptr()


def _autotune(d, key):
    dev = torch.cuda.current_device()
    M = d.img_n * d.out_h * d.out_w if d.conv else d.M
    taps = d.kh * d.kw if d.conv else 1
    kiters = taps * ((d.K + 63) // 64)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    bns = [64] if d.N <= 64 else ([64, 128] if d.b_major == CB_MAJOR_MN else [64, 128, 160])
    if d.N >= 256 and d.a_major != CB_MAJOR_MN and M >= 1024 and os.environ.get("CB_GEMM_TILE256", "1") != "0":
        bns = bns + [256]          # 128x256 tiles (4-stage ring, one CTA per SM): fewer operand bytes per flop for large GEMMs
    # Only knobs that leave the arithmetic unchanged are timed: tile width, ring depth and cluster vs workspace reduction
    # of the k-slices.  The split count stays the library's (a function of the shape), so every
    # candidate adds the same products in the same order and the winner of a noisy timing never changes the results.
    cands = [(0, 0, 0, 0, 0)]
    for bn in bns:
        tiles = ((d.N + bn - 1) // bn) * ((M + 127) // 128) * d.batch
        cands.append((bn, 0, 0, 0, 0))
        if tiles <= sms:
            cands.append((bn, 0, 3, 0, 0))          # 3-stage ring: leaves room for the next kernel's CTAs on the SM
        if CLUSTER_SK and not d.glu and kiters >= 8:
            cands.append((bn, 0, 0, 0, 1))          # k-slices (if the library splits this shape) reduced inside a cluster
    t = GemmDesc.from_buffer_copy(bytes(d))
    # scratch output large enough for any addressing the descriptor can produce
    inner = d.batch_inner if d.batch_inner > 0 else d.batch
    outer = max(1, d.batch // max(1, inner))
    span = (d.ldd * (d.N if d.d_transposed else M) + abs(d.d_batch_stride) * (inner - 1) +
            abs(d.d_batch_stride2) * (outer - 1) + max(M, d.N) + 64)
    nbytes = int(span) * (4 if d.d_dtype == CB_F32 else 2)
    sc = _tune_scratch.get(dev)
    if sc is None or sc.numel() < nbytes:
        sc = None
        _tune_scratch.pop(dev, None)
        sc = torch.empty(max(nbytes, 64 << 20), dtype=torch.uint8, device="cuda")
        _tune_scratch[dev] = sc
    t.D, t.R = (sc.data_ptr() if d.D else None), None
    if d.D2:
        off = (nbytes + 255) // 256 * 256
        n2 = int(d.ldd2 * M + d.N + 64) * (4 if d.d2_dtype == CB_F32 else 2)
        if sc.numel() < off + n2:
            sc = torch.empty(off + n2, dtype=torch.uint8, device="cuda")
            _tune_scratch[dev] = sc
            t.D = sc.data_ptr()
        t.D2 = sc.data_ptr() + off
    L = _L()
    times = {}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    cur = torch.cuda.current_stream()
    side = _tune_stream.get(dev)
    if side is None:
        side = _tune_stream[dev] = torch.cuda.Stream()
    side.wait_stream(cur)
    with torch.cuda.stream(side):
        sp_ = ctypes.c_void_p(side.cuda_stream)
        for bn, sp, stg, pair, cl in cands:
            t.tile_n, t.splits, t.stages, t.cta_pair, t.splitk_cluster = bn, sp, stg, pair, cl
            if L.cb_gemm(ctypes.byref(t), sp_) != 0:
                # a refused launch (e.g. a cluster this device cannot co-schedule) leaves its code in CUDA's last-error slot;
                # the library's own cudaGetLastError() check at the end of the next launch would report it for that launch.
                # Absorb it with one launch of the library's default configuration whose return code is ignored.
                t.tile_n, t.splits, t.stages, t.cta_pair, t.splitk_cluster = 0, 0, 0, 0, 0
                L.cb_gemm(ctypes.byref(t), sp_)
                continue
            g = torch.cuda.CUDAGraph()
            g.capture_begin()
            ok = True
            for _ in range(8):
                ok = ok and L.cb_gemm(ctypes.byref(t), sp_) == 0
            g.capture_end()
            if not ok:
                continue
            g.replay()
            best = 1e9
            for _ in range(3):
                e0.record(side)
                g.replay()
                e1.record(side)
                e1.synchronize()
                best = min(best, e0.elapsed_time(e1) * 125.0)     # us per launch
            times[(bn, sp, stg, pair, cl)] = best
            del g
    cur.wait_stream(side)
    base = times.get((0, 0, 0, 0, 0), 1e9)
    win = min(times, key=times.get) if times else (0, 0, 0, 0, 0)
    if times.get(win, 1e9) > 0.97 * base:     # keep the library's own choice unless the gain is real
        win = (0, 0, 0, 0, 0)
    _TUNE[key] = win
    # best configuration that does not launch a cluster of k-slices (see _gemm: lanes other than 0)
    nc = {k: v for k, v in times.items() if k[4] == 0}
    win_nc = min(nc, key=nc.get) if nc else (0, 0, 0, 0, 0)
    if nc.get(win_nc, 1e9) > 0.97 * base:
        win_nc = (0, 0, 0, 0, 0)
    _TUNE_NC[key] = win_nc
    if TUNE_LOG is not None:
        TUNE_LOG.append((key, {f"{k[0]}x{k[1]}s{k[2]}p{k[3]}c{k[4]}": round(v, 2) for k, v in times.items()}, win))
    log_path = os.environ.get("CB_GEMM_TUNE_LOG")
    if log_path:
        import json
        with open(log_path, "a") as f:
            f.write(json.dumps({"M": M, "N": d.N, "K": d.K, "batch": d.batch, "conv": d.conv, "kh": d.kh, "b_major": d.b_major,
                                "a_major": d.a_major, "d_dtype": d.d_dtype, "win": list(win),
                                "us": {f"{k[0]}x{k[1]}s{k[2]}p{k[3]}c{k[4]}": round(v, 2) for k, v in times.items()}}) + "\n")
    return win


def _gemm(d, what):
    ws = _splitk_workspace(torch.cuda.current_device())
    d.splitk_ws, d.splitk_ws_bytes = ws.data_ptr(), ws.numel()
    if GEMM_DEBUG_TIMELINE is not None:
        d.debug_timeline = GEMM_DEBUG_TIMELINE.data_ptr()
    if FE_CTAS > 0 and _LANE in FE_LANES and d.cta_pair == 0 and d.a_major != CB_MAJOR_MN and d.N >= 64 \
            and not d.d_transposed and (d.img_n * d.out_h * d.out_w if d.conv else d.M) >= 2048:
        d.cta_pair, d.tile_n, d.splits = FE_CTAS, (256 if d.N >= 256 else 128), 1
    if AUTOTUNE and d.tile_n == 0 and d.splits == 0 and d.stages == 0 and d.cta_pair == 0 and d.splitk_cluster == 0:
        key = _tune_key(d)
        win = _TUNE.get(key)
        if win is None and not torch.cuda.is_current_stream_capturing():
            win = _autotune(d, key)
        if win is not None:
            # Cluster split-K only on the lane-0 stream (see CLUSTER_SK): the other lanes keep the configuration they were
            # tuned and measured with, the best one without cluster split-K.
            if win[4] == 1 and _LANE != 0 and not CLUSTER_SK_ALL_LANES:
                win = _TUNE_NC.get(key, (0, 0, 0, 0, 0))
            d.tile_n, d.splits, d.stages, d.cta_pair, d.splitk_cluster = win
    if GEMM_RECORD is not None:
        taps = d.kh * d.kw if d.conv else 1
        M = d.img_n * d.out_h * d.out_w if d.conv else d.M
        GEMM_RECORD.append((bytes(d), 2.0 * M * d.N * d.K * taps * d.batch))
    _lib.check(_L().cb_gemm(ctypes.byref(d), _st()), what)


class Geo:
    """Image geometry of a channels-last activation matrix."""
    __slots__ = ("n", "h", "w")

    def __init__(self, n, h, w):
        self.n, self.h, self.w = int(n), int(h), int(w)

    @property
    def rows(self):
        return self.n * self.h * self.w

    @property
    def hw(self):
        return self.h * self.w


# ------------------------------------------------------------------------------------------------
# weight packing (host side, once per checkpoint load)
# ------------------------------------------------------------------------------------------------
def pack_conv_weight(w, dtype, cin_pad=None, cout_pad=None, out_scale=None, device=None):
    """[Cout][Cin][kh][kw] fp32 (host or device) -> [kh*kw][Cout_pad][Cin_pad] (tap-major, Cin contiguous) as one 2-D
    matrix on the device (cb_pack_conv_weight); out_scale [Cout] folds a following eval BatchNorm into the weights."""
    cout, cin, kh, kw = w.shape
    cin_pad = cin_pad or cin
    cout_pad = cout_pad or cout
    dev = torch.device(device) if device is not None else w.device
    w32 = w.detach().to(dev, torch.float32).contiguous()
    out = torch.empty(kh * kw * cout_pad, cin_pad, dtype=dtype, device=dev)
    sc = out_scale.detach().to(dev, torch.float32).contiguous() if out_scale is not None else None
    _lib.check(_L().cb_pack_conv_weight(_p(w32), _p(out), _dt(out), cout, cin, kh, kw, cout_pad, cin_pad, _p(sc), _st()),
               "cb_pack_conv_weight")
    return out


def to_device(t, device, dtype=torch.float32, scale=1.0):
    """Checkpoint tensor (host or device, any float dtype) -> contiguous device tensor of `dtype`; the conversion to a
    16-bit operand type is a cb kernel (cb_convert_f32), not a torch cast."""
    x = t.detach().to(device, torch.float32).contiguous()
    if dtype == torch.float32 and scale == 1.0:
        return x
    out = torch.empty(x.shape, dtype=dtype, device=x.device)
    if x.numel():
        _lib.check(_L().cb_convert_f32(_p(x), _p(out), _dt(out), x.numel(), float(scale), _st()), "cb_convert_f32")
    return out


# ------------------------------------------------------------------------------------------------
# GEMM family
# ------------------------------------------------------------------------------------------------
def gemm_raw(A, B, D, **kw):
    from . import raw
    return raw.gemm(A, B, D, **kw)


def linear(x, w, bias=None, *, out_dtype=None, out=None, act=CB_ACT_NONE, residual=None, alpha=1.0, out2=None):
    """y[M][N] = act(alpha * x[M][K] @ w[N][K]^T + bias) + residual."""
    M, K = x.shape
    N = w.shape[0]
    assert w.shape[1] == K and x.is_contiguous() and w.is_contiguous()
    if out is None:
        out = torch.empty(M, N, dtype=out_dtype or x.dtype, device=x.device)
    d = GemmDesc()
    d.M, d.N, d.K, d.batch, d.ab_dtype = M, N, K, 1, _dt(x)
    d.A, d.lda, d.a_major = x.data_ptr(), K, CB_MAJOR_K
    d.B, d.ldb, d.b_major = w.data_ptr(), K, CB_MAJOR_K
    d.D, d.d_dtype, d.ldd = out.data_ptr(), _dt(out), out.stride(0)
    if bias is not None:
        d.bias, d.bias_row_div, d.ldbias = bias.data_ptr(), 0, N
    if residual is not None:
        d.R, d.r_dtype, d.ldr = residual.data_ptr(), _dt(residual), residual.stride(0)
    d.alpha, d.act = alpha, act
    _set_out2(d, out2)
    _gemm(d, "cb_gemm(linear)")
    return out


def linear_dgrad(dy, w, *, out_dtype=None, out=None, residual=None, alpha=1.0):
    """dx[M][K] = alpha * dy[M][N] @ w[N][K] (+ residual): the forward weight is read MN-major."""
    M, N = dy.shape
    K = w.shape[1]
    assert w.shape[0] == N and dy.is_contiguous() and w.is_contiguous()
    if out is None:
        out = torch.empty(M, K, dtype=out_dtype or dy.dtype, device=dy.device)
    d = GemmDesc()
    d.M, d.N, d.K, d.batch, d.ab_dtype = M, K, N, 1, _dt(dy)
    d.A, d.lda, d.a_major = dy.data_ptr(), N, CB_MAJOR_K
    d.B, d.ldb, d.b_major = w.data_ptr(), K, CB_MAJOR_MN
    d.D, d.d_dtype, d.ldd = out.data_ptr(), _dt(out), out.stride(0)
    if residual is not None:
        d.R, d.r_dtype, d.ldr = residual.data_ptr(), _dt(residual), residual.stride(0)
    d.alpha = alpha
    _gemm(d, "cb_gemm(linear_dgrad)")
    return out


def conv2d(x, geo, wpack, cout, bias=None, *, ksize=3, stride=1, pad=(1, 1, 1, 1), out_dtype=None, out=None,
           residual=None, bias_per_image=False, ldbias=None, act=CB_ACT_NONE, cout_rows=None, out2=None, out2_affine=None,
           act_param=None):
    """Implicit-GEMM convolution on an NHWC activation matrix.

    x: [geo.rows][Cin]; wpack: [k*k*cout_rows][Cin] from pack_conv_weight; pad=(top,bottom,left,right).
    Returns (y [n*oh*ow][cout], Geo(n,oh,ow)).
    """
    cin = x.shape[1]
    assert x.shape[0] == geo.rows and x.is_contiguous()
    cout_rows = cout_rows or cout
    oh = (geo.h + pad[0] + pad[1] - ksize) // stride + 1
    ow = (geo.w + pad[2] + pad[3] - ksize) // stride + 1
    ogeo = Geo(geo.n, oh, ow)
    if out is None:
        out = torch.empty(ogeo.rows, cout, dtype=out_dtype or x.dtype, device=x.device)
    d = GemmDesc()
    d.M, d.N, d.K, d.batch, d.ab_dtype = ogeo.rows, cout, cin, 1, _dt(x)
    d.A, d.lda, d.a_major = x.data_ptr(), cin, CB_MAJOR_K
    d.B, d.ldb, d.b_major = wpack.data_ptr(), wpack.shape[1], CB_MAJOR_K
    d.conv = 1
    d.img_n, d.img_h, d.img_w, d.out_h, d.out_w = geo.n, geo.h, geo.w, oh, ow
    d.kh = d.kw = ksize
    d.stride, d.pad_top, d.pad_left = stride, pad[0], pad[2]
    d.b_tap_rows, d.flip_taps = cout_rows, 0
    d.D, d.d_dtype, d.ldd = out.data_ptr(), _dt(out), out.stride(0)
    if bias is not None:
        d.bias = bias.data_ptr()
        d.bias_row_div = oh * ow if bias_per_image else 0
        d.ldbias = ldbias if ldbias is not None else cout
    if residual is not None:
        d.R, d.r_dtype, d.ldr = residual.data_ptr(), _dt(residual), residual.stride(0)
    d.alpha, d.act = 1.0, act
    _set_out2(d, out2, out2_affine, act_param)
    _gemm(d, "cb_gemm(conv2d)")
    return out, ogeo


def conv2d_dgrad(dy, ogeo, wpack, cin, *, ksize=3, pad=(1, 1, 1, 1), out_dtype=None, out=None, residual=None,
                 cout_rows=None):
    """dx of a stride-1 convolution: taps flipped, forward weight pack read MN-major (K = Cout)."""
    cout = dy.shape[1]
    assert dy.shape[0] == ogeo.rows and dy.is_contiguous()
    cout_rows = cout_rows or cout
    # forward: oh = h + pt + pb - k + 1  =>  input size
    h = ogeo.h - pad[0] - pad[1] + ksize - 1
    w = ogeo.w - pad[2] - pad[3] + ksize - 1
    geo = Geo(ogeo.n, h, w)
    if out is None:
        out = torch.empty(geo.rows, cin, dtype=out_dtype or dy.dtype, device=dy.device)
    d = GemmDesc()
    d.M, d.N, d.K, d.batch, d.ab_dtype = geo.rows, cin, cout, 1, _dt(dy)
    d.A, d.lda, d.a_major = dy.data_ptr(), cout, CB_MAJOR_K
    d.B, d.ldb, d.b_major = wpack.data_ptr(), wpack.shape[1], CB_MAJOR_MN
    d.conv = 1
    d.img_n, d.img_h, d.img_w, d.out_h, d.out_w = ogeo.n, ogeo.h, ogeo.w, h, w
    d.kh = d.kw = ksize
    d.stride, d.pad_top, d.pad_left = 1, ksize - 1 - pad[0], ksize - 1 - pad[2]
    d.b_tap_rows, d.flip_taps = cout_rows, 1
    d.D, d.d_dtype, d.ldd = out.data_ptr(), _dt(out), out.stride(0)
    if residual is not None:
        d.R, d.r_dtype, d.ldr = residual.data_ptr(), _dt(residual), residual.stride(0)
    d.alpha = 1.0
    _gemm(d, "cb_gemm(conv2d_dgrad)")
    return out, geo


def bmm(A, B, D, *, M, N, K, heads, images=1, lda, ldb, ldd, a_hs, b_hs, d_hs, a_is=0, b_is=0, d_is=0,
        a_major=CB_MAJOR_K, b_major=CB_MAJOR_K, alpha=1.0):
    """Two-level batched GEMM over (image, head); *_hs = head stride, *_is = image stride (elements)."""
    d = GemmDesc()
    d.M, d.N, d.K, d.batch, d.ab_dtype = M, N, K, heads * images, _dt(A)
    d.batch_inner = heads
    d.A, d.lda, d.a_batch_stride, d.a_batch_stride2, d.a_major = A.data_ptr(), lda, a_hs, a_is, a_major
    d.B, d.ldb, d.b_batch_stride, d.b_batch_stride2, d.b_major = B.data_ptr(), ldb, b_hs, b_is, b_major
    d.D, d.d_dtype, d.ldd, d.d_batch_stride, d.d_batch_stride2 = D.data_ptr(), _dt(D), ldd, d_hs, d_is
    d.alpha = alpha
    _gemm(d, "cb_gemm(bmm)")
    return D


# ------------------------------------------------------------------------------------------------
# normalisation
# ------------------------------------------------------------------------------------------------
class NormStats:
    __slots__ = ("mean", "rstd")

    def __init__(self, mean, rstd):
        self.mean, self.rstd = mean, rstd


_ws_cache = {}
CB_GN_WS_BYTES = 131072


def _gn_workspace(device):
    """One GroupNorm workspace per device (calls are stream-ordered)."""
    ws = _ws_cache.get(("gn", device, _LANE))
    if ws is None:
        ws = torch.zeros(CB_GN_WS_BYTES // 8, dtype=torch.float64, device=device)
        _ws_cache[("gn", device, _LANE)] = ws
    return ws


def _gn_ws(device, n):
    key = (device, n)
    ws = _ws_cache.get(key)
    if ws is None:
        ws = torch.empty(n, dtype=torch.float64, device=device)
        _ws_cache[key] = ws
    return ws


def _gn_flags(silu):
    """bit 0: fused SiLU; bits 8..23 (CB_GN_CTA_CAP(n)): the front-end SM budget of the streaming GroupNorm pair."""
    cap = (FE_CTAS & 0xFFFF) << 8 if (FE_CTAS > 0 and _LANE in FE_LANES) else 0     # CB_GN_CTA_CAP(n)
    return (1 if silu else 0) | cap


def groupnorm(x, geo, gamma, beta, *, groups=32, eps=1e-5, silu=False, out_dtype=torch.float16, want_stats=True):
    C = x.shape[1]
    y = torch.empty(x.shape, dtype=out_dtype, device=x.device)
    mean = torch.empty(geo.n * groups, dtype=torch.float32, device=x.device)
    rstd = torch.empty_like(mean)
    ws = _gn_workspace(x.device)
    _lib.check(_L().cb_groupnorm_fwd(_p(x), _dt(x), _p(y), _dt(y), _p(gamma), _p(beta), geo.n, geo.hw, C, groups,
                                     eps, _gn_flags(silu), _p(mean), _p(rstd), _p(ws), _st()), "cb_groupnorm_fwd")
    return y, NormStats(mean, rstd)


def groupnorm_bwd(dy, x, geo, gamma, beta, stats, *, groups=32, silu=False, dx=None, accumulate=False,
                  dx_dtype=torch.float32, dx_lp=None):
    C = x.shape[1]
    if dx is None:
        dx = torch.empty(x.shape, dtype=dx_dtype, device=x.device)
        accumulate = False
    ws = _gn_workspace(x.device)
    _lib.check(_L().cb_groupnorm_bwd(_p(dy), _dt(dy), _p(x), _dt(x), _p(gamma), _p(beta), _p(stats.mean),
                                     _p(stats.rstd), _p(dx), _dt(dx), _p(dx_lp), geo.n, geo.hw, C, groups, _gn_flags(silu),
                                     1 if accumulate else 0, _p(ws), _st()), "cb_groupnorm_bwd")
    return dx


def layernorm(x, gamma, beta, *, eps=1e-5, out_dtype=torch.float16):
    M, C = x.shape
    y = torch.empty(M, C, dtype=out_dtype, device=x.device)
    mean = torch.empty(M, dtype=torch.float32, device=x.device)
    rstd = torch.empty_like(mean)
    _lib.check(_L().cb_layernorm_fwd(_p(x), _dt(x), _p(y), _dt(y), _p(gamma), _p(beta), M, C, eps, _p(mean),
                                     _p(rstd), _st()), "cb_layernorm_fwd")
    return y, NormStats(mean, rstd)


def layernorm_bwd(dy, x, gamma, stats, *, dx=None, accumulate=False, dx_dtype=torch.float32, dx_lp=None):
    M, C = x.shape
    if dx is None:
        dx = torch.empty(M, C, dtype=dx_dtype, device=x.device)
        accumulate = False
    _lib.check(_L().cb_layernorm_bwd(_p(dy), _dt(dy), _p(x), _dt(x), _p(gamma), _p(stats.mean), _p(stats.rstd),
                                     _p(dx), _dt(dx), _p(dx_lp), M, C, 1 if accumulate else 0, _st()), "cb_layernorm_bwd")
    return dx


# ------------------------------------------------------------------------------------------------
# parameter gradients (fine-tuning the UNet / CLIP weights): fp32 results, alpha = 1 / loss scale
# ------------------------------------------------------------------------------------------------
def conv2d_wgrad(x, geo, dy, *, ksize=3, stride=1, pad=1, alpha=1.0, out=None):
    """dW [cout][cin][k][k] fp32 of a k x k convolution (k = 1 or 3, symmetric padding `pad`) from its NHWC input
    x [geo.rows][cin] and output gradient dy [n*oh*ow][cout], both 16-bit (cb_conv_wgrad)."""
    assert x.stride(1) == 1 and dy.stride(1) == 1 and x.dtype == dy.dtype and x.shape[0] == geo.rows
    cin, cout = x.shape[1], dy.shape[1]
    L = _L()
    col_b, sk_b = ctypes.c_longlong(0), ctypes.c_longlong(0)
    _lib.check(L.cb_conv_wgrad_ws_bytes(geo.n, geo.h, geo.w, cin, cout, ksize, stride, pad, ctypes.byref(col_b),
                                        ctypes.byref(sk_b)), "cb_conv_wgrad_ws_bytes")
    col = torch.empty(col_b.value // 2, dtype=x.dtype, device=x.device) if col_b.value else None
    ws = _splitk_workspace(x.device)
    if out is None:
        out = torch.empty(cout, cin, ksize, ksize, dtype=torch.float32, device=x.device)
    assert out.dtype == torch.float32 and out.is_contiguous() and out.shape == (cout, cin, ksize, ksize)
    _lib.check(L.cb_conv_wgrad(_p(x), x.stride(0), _p(dy), dy.stride(0), _dt(x), geo.n, geo.h, geo.w, cin, cout, ksize,
                               stride, pad, float(alpha), _p(out), _p(col), _p(ws), ws.numel(), _st()), "cb_conv_wgrad")
    return out


def linear_wgrad(x, dy, *, alpha=1.0, out=None):
    """dW[N][K] = alpha * dy[M][N]^T @ x[M][K] in fp32: one cb_gemm with both operands read MN-major."""
    M, K = x.shape
    N = dy.shape[1]
    assert dy.shape[0] == M and x.stride(1) == 1 and dy.stride(1) == 1 and x.dtype == dy.dtype
    if out is None:
        out = torch.empty(N, K, dtype=torch.float32, device=x.device)
    assert out.dtype == torch.float32 and out.stride(1) == 1
    d = GemmDesc()
    d.M, d.N, d.K, d.batch, d.ab_dtype = N, K, M, 1, _dt(x)
    d.A, d.lda, d.a_major = dy.data_ptr(), dy.stride(0), CB_MAJOR_MN
    d.B, d.ldb, d.b_major = x.data_ptr(), x.stride(0), CB_MAJOR_MN
    d.D, d.d_dtype, d.ldd = out.data_ptr(), CB_F32, out.stride(0)
    d.alpha = alpha
    _gemm(d, "cb_gemm(linear_wgrad)")
    return out


def colsum(x, *, groups=1, alpha=1.0, out=None):
    """out[g][c] = alpha * sum of x's rows of group g (groups equal runs of rows), fp32 [groups][C] (cb_colsum)."""
    assert x.dim() == 2 and x.stride(1) == 1
    rows, C = x.shape
    if out is None:
        out = torch.empty(groups, C, dtype=torch.float32, device=x.device)
    assert out.dtype == torch.float32 and out.is_contiguous() and out.numel() == groups * C
    _lib.check(_L().cb_colsum(_p(x), _dt(x), x.stride(0), _p(out), rows, C, groups, float(alpha), _st()), "cb_colsum")
    return out


def groupnorm_affine_bwd(dy, x, geo, gamma, beta, stats, *, groups=32, silu=False, alpha=1.0):
    """(dgamma, dbeta) fp32 [C] of a GroupNorm (fused with SiLU when silu) from the forward's saved statistics."""
    C = x.shape[1]
    dg = torch.empty(C, dtype=torch.float32, device=x.device)
    db = torch.empty_like(dg)
    _lib.check(_L().cb_groupnorm_affine_bwd(_p(dy), _dt(dy), _p(x), _dt(x), _p(gamma), _p(beta), _p(stats.mean),
                                            _p(stats.rstd), _p(dg), _p(db), geo.n, geo.hw, C, groups, 1 if silu else 0,
                                            float(alpha), _st()), "cb_groupnorm_affine_bwd")
    return dg, db


def layernorm_affine_bwd(dy, x, stats, *, alpha=1.0):
    """(dgamma, dbeta) fp32 [C] of a LayerNorm from the forward's saved statistics."""
    M, C = x.shape
    dg = torch.empty(C, dtype=torch.float32, device=x.device)
    db = torch.empty_like(dg)
    _lib.check(_L().cb_layernorm_affine_bwd(_p(dy), _dt(dy), _p(x), _dt(x), _p(stats.mean), _p(stats.rstd), _p(dg),
                                            _p(db), M, C, float(alpha), _st()), "cb_layernorm_affine_bwd")
    return dg, db


# ------------------------------------------------------------------------------------------------
# pointwise
# ------------------------------------------------------------------------------------------------
def axpby(x, a=1.0, y=None, b=0.0, *, out=None, out_dtype=None):
    """out = a*x + b*y on 2-D (possibly row-strided) views; also the cast / strided-copy kernel."""
    assert x.dim() == 2 and x.stride(1) == 1
    rows, cols = x.shape
    if out is None:
        out = torch.empty(rows, cols, dtype=out_dtype or x.dtype, device=x.device)
    assert out.stride(1) == 1 and (y is None or y.stride(1) == 1)
    _lib.check(_L().cb_axpby2d(_p(x), _dt(x), x.stride(0), a, _p(y), _dt(y) if y is not None else 0,
                               y.stride(0) if y is not None else 0, b, _p(out), _dt(out), out.stride(0), rows, cols,
                               _st()), "cb_axpby2d")
    return out


def cast(x, dtype, scale=1.0):
    return axpby(x, scale, out_dtype=dtype)


def act_fwd(x, act, out_dtype=None):
    y = torch.empty(x.shape, dtype=out_dtype or x.dtype, device=x.device)
    _lib.check(_L().cb_act_fwd(_p(x), _dt(x), _p(y), _dt(y), x.numel(), act, _st()), "cb_act_fwd")
    return y


def act_bwd(dy, x, act, out_dtype=None):
    dx = torch.empty(x.shape, dtype=out_dtype or dy.dtype, device=x.device)
    _lib.check(_L().cb_act_bwd(_p(dy), _dt(dy), _p(x), _dt(x), _p(dx), _dt(dx), x.numel(), act, _st()), "cb_act_bwd")
    return dx


def geglu(x, interleaved=False):
    M, F2 = x.shape
    y = torch.empty(M, F2 // 2, dtype=x.dtype, device=x.device)
    _lib.check(_L().cb_geglu_fwd(_p(x), _p(y), _dt(x), M, F2 // 2, 1 if interleaved else 0, _st()), "cb_geglu_fwd")
    return y


def geglu_bwd(dy, x, interleaved=False):
    M, F2 = x.shape
    dx = torch.empty(M, F2, dtype=dy.dtype, device=x.device)
    _lib.check(_L().cb_geglu_bwd(_p(dy), _p(x), _p(dx), _dt(x), _dt(dy), M, F2 // 2, 1 if interleaved else 0, _st()),
               "cb_geglu_bwd")
    return dx


def glu_interleave_rows(w):
    """[2F][...] rows ordered [all values | all gates] -> 64-row groups of 32 value rows followed by their 32 gate rows
    (F % 32 == 0): the layout the GEGLU epilogue of cb_gemm expects for the FF-in projection (attention.py:37-45)."""
    F2 = w.shape[0]
    F = F2 // 2
    assert F % 32 == 0
    v = w[:F].reshape(F // 32, 32, *w.shape[1:])
    g = w[F:].reshape(F // 32, 32, *w.shape[1:])
    return torch.cat([v, g], dim=1).reshape(w.shape).contiguous()


def linear_geglu(x, w_il, bias_il, *, keep_preact=True):
    """u = (x W_v^T + b_v) * gelu(x W_g^T + b_g) with W = interleaved FF-in weight (glu_interleave_rows): ONE GEMM launch
    whose epilogue applies the GEGLU.  Returns (u [M][F], pre-activations [M][2F] in the interleaved layout or None)."""
    M, K = x.shape
    N = w_il.shape[0]
    assert w_il.shape[1] == K and N % 64 == 0 and x.is_contiguous()
    u = torch.empty(M, N // 2, dtype=x.dtype, device=x.device)
    g = torch.empty(M, N, dtype=x.dtype, device=x.device) if keep_preact else None
    d = GemmDesc()
    d.M, d.N, d.K, d.batch, d.ab_dtype = M, N, K, 1, _dt(x)
    d.A, d.lda, d.a_major = x.data_ptr(), K, CB_MAJOR_K
    d.B, d.ldb, d.b_major = w_il.data_ptr(), K, CB_MAJOR_K
    if g is not None:
        d.D, d.ldd = g.data_ptr(), N
    d.d_dtype = _dt(u)
    if bias_il is not None:
        d.bias, d.bias_row_div, d.ldbias = bias_il.data_ptr(), 0, N
    d.alpha, d.glu = 1.0, 1
    d.D2, d.d2_dtype, d.ldd2 = u.data_ptr(), _dt(u), N // 2
    _gemm(d, "cb_gemm(linear_geglu)")
    return u, g


def softmax_(s, rows, ncols, ld, causal_period=0):
    """In-place row softmax over the first ncols of each ld-wide row; pad columns are zeroed."""
    _lib.check(_L().cb_softmax_fwd(_p(s), _p(s), _dt(s), rows, ncols, ld, causal_period, _st()), "cb_softmax_fwd")
    return s


def softmax_bwd_(dp, p, rows, ncols, ld):
    """In-place: dp <- p * (dp - sum(dp*p))."""
    _lib.check(_L().cb_softmax_bwd(_p(dp), _p(p), _p(dp), _dt(p), _dt(dp), rows, ncols, ld, _st()), "cb_softmax_bwd")
    return dp


def upsample2x(x, geo):
    C = x.shape[1]
    y = torch.empty(4 * geo.rows, C, dtype=x.dtype, device=x.device)
    _lib.check(_L().cb_upsample2x_fwd(_p(x), _p(y), _dt(x), geo.n, geo.h, geo.w, C, _st()), "cb_upsample2x_fwd")
    return y, Geo(geo.n, 2 * geo.h, 2 * geo.w)


def upsample2x_bwd(dy, geo, *, dx=None, accumulate=False, dx_dtype=None):
    """geo = geometry of the (smaller) forward input."""
    C = dy.shape[1]
    if dx is None:
        dx = torch.empty(geo.rows, C, dtype=dx_dtype or dy.dtype, device=dy.device)
        accumulate = False
    _lib.check(_L().cb_upsample2x_bwd(_p(dy), _dt(dy), _p(dx), _dt(dx), geo.n, geo.h, geo.w, C,
                                      1 if accumulate else 0, _st()), "cb_upsample2x_bwd")
    return dx


def zero_insert2x(dy, geo):
    C = dy.shape[1]
    z = torch.empty(4 * geo.rows, C, dtype=dy.dtype, device=dy.device)
    _lib.check(_L().cb_zero_insert2x(_p(dy), _p(z), _dt(dy), geo.n, geo.h, geo.w, C, _st()), "cb_zero_insert2x")
    return z, Geo(geo.n, 2 * geo.h, 2 * geo.w)


def nchw_to_nhwc(x, cpad, dtype):
    n, c, h, w = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous()
    y = torch.empty(n * h * w, cpad, dtype=dtype, device=x.device)
    _lib.check(_L().cb_nchw_to_nhwc(_p(x), _p(y), _dt(y), n, c, h * w, cpad, _st()), "cb_nchw_to_nhwc")
    return y, Geo(n, h, w)


def nhwc_to_nchw(x, geo, c):
    y = torch.empty(geo.n, c, geo.h, geo.w, dtype=torch.float32, device=x.device)
    _lib.check(_L().cb_nhwc_to_nchw(_p(x), _dt(x), _p(y), geo.n, c, geo.hw, x.shape[1], _st()), "cb_nhwc_to_nchw")
    return y


def mse_fwd_bwd(pred, target, gscale=1.0, want_grad=True):
    """Returns (loss_simple [B], grad of mean_b(loss_simple) w.r.t. pred (scaled by gscale) or None)."""
    assert pred.dtype == torch.float32 and target.dtype == torch.float32
    B = pred.shape[0]
    loss = torch.empty(B, dtype=torch.float32, device=pred.device)
    grad = torch.empty_like(pred) if want_grad else None
    _lib.check(_L().cb_mse_fwd_bwd(_p(pred), _p(target), _p(loss), _p(grad), B, pred.numel() // B, gscale, _st()),
               "cb_mse_fwd_bwd")
    return loss, grad


def timestep_embedding(t, dim, dtype=torch.float16, max_period=10000.0):
    assert t.dtype == torch.int64
    out = torch.empty(t.shape[0], dim, dtype=dtype, device=t.device)
    _lib.check(_L().cb_timestep_embedding(_p(t), _p(out), _dt(out), t.shape[0], dim, max_period, _st()),
               "cb_timestep_embedding")
    return out


# ------------------------------------------------------------------------------------------------
# CosFace front end / celeb-basis embedding path / optimiser (fp32 side kernels)
# ------------------------------------------------------------------------------------------------
def channel_affine_act(x, scale=None, shift=None, slope=None, out=None, out_dtype=None):
    rows, C = x.shape
    y = out if out is not None else torch.empty(rows, C, dtype=out_dtype or x.dtype, device=x.device)
    _lib.check(_L().cb_channel_affine_act(_p(x), _dt(x), _p(y), _dt(y), _p(scale), _p(shift), _p(slope), rows, C,
                                          _st()), "cb_channel_affine_act")
    return y


def face_warp_resize(faces, n_chunks, affine6, out_hw=112, cpad=8, dtype=torch.float16):
    """faces: [B][H][W][3*n_chunks] fp32 -> ([n_chunks*B*out_hw*out_hw][cpad], Geo)."""
    B, H, W, C = faces.shape
    assert C == 3 * n_chunks and faces.dtype == torch.float32 and faces.is_contiguous()
    out = torch.empty(n_chunks * B * out_hw * out_hw, cpad, dtype=dtype, device=faces.device)
    arr = (ctypes.c_float * 6)(*[float(v) for v in affine6])
    _lib.check(_L().cb_face_warp_resize(_p(faces), _p(out), _dt(out), B, H, W, n_chunks, out_hw, cpad, arr, _st()),
               "cb_face_warp_resize")
    return out, Geo(n_chunks * B, out_hw, out_hw)


def l2norm_rows(x):
    y = torch.empty_like(x)
    _lib.check(_L().cb_l2norm_rows(_p(x), _p(y), x.shape[0], x.shape[1], _st()), "cb_l2norm_rows")
    return y


def ema_rows(table, idx, src, momentum):
    """table[idx[b]] = m*table[idx[b]] + (1-m)*src[b]; idx is a device int64 (B,) / (B,k) tensor (column 0 is used)."""
    B = src.shape[0]
    row = src[0].numel()
    assert idx.dtype == torch.int64 and table.dtype == torch.float32 and src.dtype == torch.float32
    assert table.is_contiguous() and src.is_contiguous() and table[0].numel() == row
    stride = idx.stride(0) if idx.dim() > 1 else 1
    _lib.check(_L().cb_ema_rows(_p(table), _p(idx), stride, _p(src), B, row, table.shape[0], float(momentum), _st()),
               "cb_ema_rows")


def ema_rows_sel(table, ids, slot, src_row, src, momentum):
    """For k in list order: table[ids.view(-1)[slot[k]]] = m*table[..] + (1-m)*src[src_row[k]]; slot[k] < 0 skips entry k
    (cb_ema_rows_sel).  ids: contiguous device int64; slot / src_row: device int32 (n,)."""
    n = slot.numel()
    row = src[0].numel()
    assert ids.dtype == torch.int64 and ids.is_contiguous() and slot.dtype == torch.int32 and src_row.dtype == torch.int32
    assert src_row.numel() == n and table.dtype == torch.float32 and src.dtype == torch.float32
    assert table.is_contiguous() and src.is_contiguous() and table[0].numel() == row
    _lib.check(_L().cb_ema_rows_sel(_p(table), _p(ids), _p(slot), _p(src_row), _p(src), n, row, table.shape[0],
                                    float(momentum), _st()), "cb_ema_rows_sel")


def embedding_gather(ids, table):
    n = ids.numel()
    out = torch.empty(n, table.shape[1], dtype=torch.float32, device=table.device)
    _lib.check(_L().cb_embedding_gather(_p(ids), _p(table), _p(out), n, table.shape[1], table.shape[0], _st()),
               "cb_embedding_gather")
    return out


def embedding_bwd(ids, dout, num_rows, *, alpha=1.0, out=None):
    """Gradient [num_rows][D] fp32 of embedding_gather: row v = alpha * the sum of dout's rows whose id is v, added in
    token order; rows no id selects are zero (cb_embedding_bwd)."""
    n, D = ids.numel(), dout.shape[1]
    assert dout.dtype == torch.float32 and dout.stride(1) == 1 and dout.shape[0] == n and ids.dtype == torch.int64
    if out is None:
        out = torch.zeros(num_rows, D, dtype=torch.float32, device=dout.device)
    assert out.dtype == torch.float32 and out.is_contiguous() and out.shape == (num_rows, D)
    _lib.check(_L().cb_embedding_bwd(_p(ids.contiguous()), _p(dout), dout.stride(0), _p(out), n, D, num_rows,
                                     float(alpha), _st()), "cb_embedding_bwd")
    return out


def celeb_mlp_fwd(v, W, b, es, slope=0.2):
    F_, in_dim = v.shape
    K = W.shape[0] // es
    pre = torch.empty(F_, es * K, dtype=torch.float32, device=v.device)
    coef = torch.empty(F_, es, K, dtype=torch.float32, device=v.device)
    nrm = torch.empty(F_ * es, dtype=torch.float32, device=v.device)
    _lib.check(_L().cb_celeb_mlp_fwd(_p(v), _p(W), _p(b), _p(pre), _p(coef), _p(nrm), F_, in_dim, K, es, slope, _st()),
               "cb_celeb_mlp_fwd")
    return pre, coef, nrm


def celeb_basis_fwd(coef, basis):
    F_, es, K = coef.shape
    D = basis.shape[2]
    z = torch.empty(F_, es, D, dtype=torch.float32, device=coef.device)
    _lib.check(_L().cb_celeb_basis_fwd(_p(coef), _p(basis), _p(z), F_, es, K, D, _st()), "cb_celeb_basis_fwd")
    return z


def celeb_basis_bwd(dz, basis):
    F_, es, D = dz.shape
    K = basis.shape[1] - 1
    dcoef = torch.empty(F_, es, K, dtype=torch.float32, device=dz.device)
    _lib.check(_L().cb_celeb_basis_bwd(_p(dz), _p(basis), _p(dcoef), F_, es, K, D, _st()), "cb_celeb_basis_bwd")
    return dcoef


def celeb_mlp_bwd(dcoef, coef, nrm, pre, v, dW, db, slope=0.2, gscale=1.0):
    F_, es, K = coef.shape
    ws = torch.empty(F_, es * K, dtype=torch.float32, device=v.device)
    _lib.check(_L().cb_celeb_mlp_bwd(_p(dcoef), _p(coef), _p(nrm), _p(pre), _p(v), _p(ws), _p(dW), _p(db), F_,
                                     v.shape[1], K, es, slope, gscale, _st()), "cb_celeb_mlp_bwd")
    return dW, db


def embed_inject_fwd(tok, z_rows, map_, pos, B, T):
    D = tok.shape[1]
    out = torch.empty(B * T, D, dtype=torch.float32, device=tok.device)
    _lib.check(_L().cb_embed_inject_fwd(_p(tok), _p(z_rows), _p(map_), _p(pos), _p(out), B, T, D, _st()),
               "cb_embed_inject_fwd")
    return out


def embed_inject_bwd(dout, map_, n_z_rows, B, T, out=None):
    """Gradient of the z rows (every row written; a row no prompt uses gets 0); `out` may be a (n_z_rows, D) view."""
    D = dout.shape[1]
    dz = torch.empty(n_z_rows, D, dtype=torch.float32, device=dout.device) if out is None else out
    assert dz.shape == (n_z_rows, D) and dz.is_contiguous()
    _lib.check(_L().cb_embed_inject_bwd(_p(dout), _p(map_), _p(dz), n_z_rows, B, T, D, _st()), "cb_embed_inject_bwd")
    return dz


def adamw_step(p, g, m, v, *, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=1e-2, step=0, step_dev=None):
    _lib.check(_L().cb_adamw_step(_p(p), _p(g), _p(m), _p(v), p.numel(), lr, beta1, beta2, eps, weight_decay, step,
                                  _p(step_dev), _st()), "cb_adamw_step")


def loss_mean(loss):
    """(B,) per-sample losses -> (1,) batch mean (cb_loss_mean)."""
    out = torch.empty(1, dtype=torch.float32, device=loss.device)
    _lib.check(_L().cb_loss_mean(_p(loss), _p(out), loss.shape[0], _st()), "cb_loss_mean")
    return out


def diffusion_loss_fwd_bwd(pred, target, t, logvar, lvlb_weights, l_simple_weight, original_elbo_weight, gscale=1.0,
                           want_grad=True):
    """p_losses with its loss weights (cb_diffusion_loss_fwd_bwd).  t: device int64 (B,); logvar / lvlb_weights: device
    fp32 (T,).  Returns (loss_simple [B], loss [1], loss_vlb [1], d loss / d pred * gscale or None)."""
    assert pred.dtype == torch.float32 and target.dtype == torch.float32 and t.dtype == torch.int64
    assert pred.shape == target.shape and pred.is_contiguous() and target.is_contiguous()
    B = pred.shape[0]
    assert t.shape == (B,) and t.is_contiguous()
    assert logvar.dtype == torch.float32 and lvlb_weights.dtype == torch.float32
    assert logvar.dim() == 1 and logvar.shape == lvlb_weights.shape and logvar.is_contiguous() and lvlb_weights.is_contiguous()
    # t is read on the device (a host check would sync): the tables must cover every timestep the schedule draws
    loss_simple = torch.empty(B, dtype=torch.float32, device=pred.device)
    out = torch.empty(2, dtype=torch.float32, device=pred.device)
    grad = torch.empty_like(pred) if want_grad else None
    _lib.check(_L().cb_diffusion_loss_fwd_bwd(_p(pred), _p(target), _p(t), _p(logvar), _p(lvlb_weights),
                                              float(l_simple_weight), float(original_elbo_weight), _p(loss_simple),
                                              _p(out[0:1]), _p(out[1:2]), _p(grad), B, pred.numel() // B, gscale, _st()),
               "cb_diffusion_loss_fwd_bwd")
    return loss_simple, out[0:1], out[1:2], grad


def ti_coarse_reg(rows, init_rows, grad, loss, n_init, weight):
    """loss += weight * mean((rows-init)(rows-init)^T / n_init); grad += its gradient (cb_ti_coarse_reg).  rows, init_rows
    and grad are (nv, D) fp32 views; loss a (1,) fp32 tensor."""
    assert rows.shape == init_rows.shape == grad.shape and rows.is_contiguous() and init_rows.is_contiguous()
    assert grad.is_contiguous() and loss.dtype == torch.float32
    nv, D = rows.shape
    _lib.check(_L().cb_ti_coarse_reg(_p(rows), _p(init_rows), _p(grad), _p(loss), nv, D, int(n_init), float(weight),
                                     _st()), "cb_ti_coarse_reg")


def posterior_sample(moments_nchw, eps, scale):
    N, C2, H, W = moments_nchw.shape
    z = torch.empty(N, C2 // 2, H, W, dtype=torch.float32, device=moments_nchw.device)
    _lib.check(_L().cb_posterior_sample(_p(moments_nchw), _p(eps), _p(z), N, C2 // 2, H * W, scale, _st()),
               "cb_posterior_sample")
    return z


def q_sample(x0, noise, t, sqrt_ac, sqrt_1mac):
    out = torch.empty_like(x0)
    B = x0.shape[0]
    _lib.check(_L().cb_q_sample(_p(x0), _p(noise), _p(t), _p(sqrt_ac), _p(sqrt_1mac), _p(out), B, x0.numel() // B,
                                _st()), "cb_q_sample")
    return out


def mask_strides(mask, shape):
    """(batch stride, channel stride) of an fp32 mask broadcast to `shape` = (B, C, h, w), 0 where it broadcasts.  The
    spatial dimensions must be dense (stride w and 1)."""
    B, C, h, w = shape
    sb, sc, sh, sw = mask.expand(B, C, h, w).stride()
    if (h > 1 and sh != w) or (w > 1 and sw != 1):
        raise ValueError(f"mask of shape {tuple(mask.shape)} / strides {tuple(mask.stride())}: spatial dims must be dense")
    return (sb if B > 1 else 0), (sc if C > 1 else 0)


def q_sample_masked(x0, noise, t, sqrt_ac, sqrt_1mac, mask, img, out=None):
    """out = q_sample(x0, t, noise) * mask + (1 - mask) * img (ddim.py:144-147) in one launch; `out` may be `img`."""
    B, C, h, w = img.shape
    assert x0.shape == noise.shape == img.shape and mask.dtype == torch.float32
    assert x0.is_contiguous() and noise.is_contiguous() and img.is_contiguous() and t.dtype == torch.long
    sb, sc = mask_strides(mask, (B, C, h, w))
    out = torch.empty_like(img) if out is None else out
    assert out.shape == img.shape and out.is_contiguous()
    _lib.check(_L().cb_q_sample_masked(_p(x0), _p(noise), _p(t), _p(sqrt_ac), _p(sqrt_1mac), _p(mask), sb, sc, _p(img),
                                       _p(out), B, C, h * w, _st()), "cb_q_sample_masked")
    return out


def p_sample(x, eps, noise, t, sqrt_recip_ac, sqrt_recipm1_ac, coef1, coef2, log_var, *, temperature=1.0,
             clip_denoised=False, out=None, want_x0=True):
    """One DDPM ancestral step (LatentDiffusion.p_sample, eps-parameterisation, ddpm.py:1149-1178) in one launch:
    returns (x_prev, x_recon or None).  `out` may be `x`; t is an int64 (B,) device tensor."""
    B = x.shape[0]
    assert x.dtype == eps.dtype == noise.dtype == torch.float32 and t.dtype == torch.long and t.shape == (B,)
    assert x.shape == eps.shape == noise.shape and x.is_contiguous() and eps.is_contiguous() and noise.is_contiguous()
    out = torch.empty_like(x) if out is None else out
    assert out.shape == x.shape and out.is_contiguous()
    x0 = torch.empty_like(x) if want_x0 else None
    _lib.check(_L().cb_p_sample(_p(x), _p(eps), _p(noise), _p(t), _p(sqrt_recip_ac), _p(sqrt_recipm1_ac), _p(coef1),
                                _p(coef2), _p(log_var), float(temperature), int(bool(clip_denoised)), _p(out), _p(x0),
                                B, x.numel() // B, _st()), "cb_p_sample")
    return out, x0


def ddim_step(x, e_uncond, e_cond, noise, *, scale, a_t, a_prev, sigma_t, sqrt_one_minus_at, want_x0=True):
    x_prev = torch.empty_like(x)
    pred_x0 = torch.empty_like(x) if want_x0 else None
    _lib.check(_L().cb_ddim_step(_p(x), _p(e_uncond), _p(e_cond), _p(noise), _p(x_prev), _p(pred_x0), x.numel(),
                                 scale, a_t, a_prev, sigma_t, sqrt_one_minus_at, _st()), "cb_ddim_step")
    return x_prev, pred_x0


def attention_fwd(q, k, v, out, *, images, heads, dh, nq, nk, scale, causal=False, want_p=False, want_lse=False):
    """Fused flash attention forward (cb_attention_fwd).  q/k/v/out are row-strided 2-D views whose head h lives in
    columns [h*dh, (h+1)*dh).  Returns (P or None, lse or None); P is [images*heads*nq][round_up(nk, 8)]."""
    P = lse = None
    ldp = 0
    if want_p:
        ldp = (nk + 7) // 8 * 8
        P = torch.empty(images * heads * nq, ldp, dtype=q.dtype, device=q.device)
    if want_lse:
        lse = torch.empty(images * heads * nq, dtype=torch.float32, device=q.device)
    _lib.check(_L().cb_attention_fwd(_p(q), q.stride(0), _p(k), k.stride(0), _p(v), v.stride(0), _p(out), out.stride(0),
                                     _p(lse), _p(P), ldp, _dt(q), images, heads, nq, nk, dh, scale, 1 if causal else 0,
                                     _st()), "cb_attention_fwd")
    return P, lse


def attention_bwd_dq(q, k, v, o, dO, lse, dq, dS, *, images, heads, dh, nq, nk, scale, causal=False):
    """Query-stationary half of the flash backward (cb_attention_bwd_dq): dq (or None) and, optionally, the scaled score
    gradient dS [images*heads*nq][ldds] for GEMM-based dK / dV (short key sequences)."""
    delta = torch.empty(images * heads * nq, dtype=torch.float32, device=q.device)
    _lib.check(_L().cb_attention_bwd_dq(_p(q), q.stride(0), _p(k), k.stride(0), _p(v), v.stride(0), _p(o), o.stride(0),
                                        _p(dO), dO.stride(0), _p(lse), _p(delta), _p(dq), dq.stride(0) if dq is not None else 0,
                                        _p(dS), dS.shape[1] if dS is not None else 0, _dt(q), images, heads, nq, nk, dh,
                                        scale, 1 if causal else 0, _st()), "cb_attention_bwd_dq")


def attention_bwd(q, k, v, o, dO, lse, dq, dk, dv, *, images, heads, dh, nq, nk, scale, causal=False):
    """Flash attention backward (cb_attention_bwd): dq/dk/dv from q, k, v, the forward output o, its gradient dO and the
    forward log-sum-exp; all operands are row-strided 2-D views with head h in columns [h*dh, (h+1)*dh)."""
    delta = torch.empty(images * heads * nq, dtype=torch.float32, device=q.device)
    _lib.check(_L().cb_attention_bwd(_p(q), q.stride(0), _p(k), k.stride(0), _p(v), v.stride(0), _p(o), o.stride(0),
                                     _p(dO), dO.stride(0), _p(lse), _p(delta), _p(dq), dq.stride(0), _p(dk),
                                     dk.stride(0), _p(dv), dv.stride(0), _dt(q), images, heads, nq, nk, dh, scale,
                                     1 if causal else 0, _st()), "cb_attention_bwd")
