"""ctypes binding of libcelebbasis_b200.so (the C-ABI in include/celebbasis_b200.h).

There is deliberately NO fallback: if the shared object is missing or the device is not sm_90
the product path raises.  (tests/ and bench.py's cpu_baseline are the only users of oracle/.)
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcelebbasis_b200.so")

CB_F16, CB_BF16, CB_F32 = 0, 1, 2
CB_ACT_NONE, CB_ACT_SILU, CB_ACT_GELU, CB_ACT_QUICK_GELU, CB_ACT_PRELU = 0, 1, 2, 3, 4
CB_MAJOR_K, CB_MAJOR_MN = 0, 1


class GemmDesc(ctypes.Structure):
    _fields_ = [
        ("M", ctypes.c_int32), ("N", ctypes.c_int32), ("K", ctypes.c_int32),
        ("batch", ctypes.c_int32), ("ab_dtype", ctypes.c_int32),
        ("A", ctypes.c_void_p), ("lda", ctypes.c_int64), ("a_batch_stride", ctypes.c_int64),
        ("a_major", ctypes.c_int32),
        ("B", ctypes.c_void_p), ("ldb", ctypes.c_int64), ("b_batch_stride", ctypes.c_int64),
        ("b_major", ctypes.c_int32),
        ("conv", ctypes.c_int32),
        ("img_n", ctypes.c_int32), ("img_h", ctypes.c_int32), ("img_w", ctypes.c_int32),
        ("out_h", ctypes.c_int32), ("out_w", ctypes.c_int32),
        ("kh", ctypes.c_int32), ("kw", ctypes.c_int32),
        ("stride", ctypes.c_int32), ("pad_top", ctypes.c_int32), ("pad_left", ctypes.c_int32),
        ("b_tap_rows", ctypes.c_int32), ("flip_taps", ctypes.c_int32),
        ("D", ctypes.c_void_p), ("d_dtype", ctypes.c_int32), ("ldd", ctypes.c_int64),
        ("d_batch_stride", ctypes.c_int64), ("d_transposed", ctypes.c_int32),
        ("bias", ctypes.c_void_p), ("bias_row_div", ctypes.c_int32), ("ldbias", ctypes.c_int64),
        ("R", ctypes.c_void_p), ("r_dtype", ctypes.c_int32), ("ldr", ctypes.c_int64),
        ("r_batch_stride", ctypes.c_int64),
        ("alpha", ctypes.c_float), ("act", ctypes.c_int32),
        ("batch_inner", ctypes.c_int32),
        ("a_batch_stride2", ctypes.c_int64), ("b_batch_stride2", ctypes.c_int64),
        ("d_batch_stride2", ctypes.c_int64), ("r_batch_stride2", ctypes.c_int64),
        ("splitk_ws", ctypes.c_void_p), ("splitk_ws_bytes", ctypes.c_int64),
        ("debug_timeline", ctypes.c_void_p),
        ("tile_n", ctypes.c_int32), ("splits", ctypes.c_int32), ("stages", ctypes.c_int32), ("cta_pair", ctypes.c_int32),
        ("D2", ctypes.c_void_p), ("ldd2", ctypes.c_int64), ("d2_dtype", ctypes.c_int32), ("glu", ctypes.c_int32),
        ("act_param", ctypes.c_void_p), ("d2_scale", ctypes.c_void_p), ("d2_shift", ctypes.c_void_p),
        ("splitk_cluster", ctypes.c_int32),
    ]


_lib = None


class CelebBasisB200Error(RuntimeError):
    pass


def load():
    """Load the shared object (building it in-tree if it is absent and nvcc is available)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        from . import build as _build
        _build.build()
    lib = ctypes.CDLL(LIB_PATH)
    lib.cb_last_error.restype = ctypes.c_char_p
    lib.cb_abi_version.restype = ctypes.c_int
    lib.cb_device_ok.restype = ctypes.c_int
    lib.cb_launch_count.restype = ctypes.c_ulonglong
    lib.cb_gemm.argtypes = [ctypes.POINTER(GemmDesc), ctypes.c_void_p]
    lib.cb_gemm.restype = ctypes.c_int
    _declare_rest(lib)
    _lib = lib
    return lib


def _declare_rest(lib):
    """argtypes for the non-GEMM entry points (filled in by ops modules as they are added)."""
    from . import _abi
    _abi.declare(lib)


def check(rc, what=""):
    if rc != 0:
        msg = load().cb_last_error().decode(errors="replace")
        raise CelebBasisB200Error(f"{what} failed rc={rc}: {msg}")


def last_error():
    return load().cb_last_error().decode(errors="replace")


def launch_count():
    return int(load().cb_launch_count())
