"""CPU: the C-ABI shared library loads without a GPU and exports every symbol include/celebbasis_b200.h declares."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "celebbasis_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(cb_[a-z0-9_]+)\s*\(", text)))


def test_library_loads_exports_header_symbols_and_abi_version():
    from celebbasis_b200 import lib
    L = lib.load()
    syms = _declared_symbols()
    assert len(syms) >= 35
    for s in syms:
        assert hasattr(L, s), f"symbol {s} declared in the header but not exported"
    assert L.cb_abi_version() == 6
    assert isinstance(lib.last_error(), str)


def test_ctypes_signatures_cover_header():
    from celebbasis_b200 import _abi
    declared = set(_declared_symbols()) - {"cb_abi_version", "cb_last_error", "cb_device_ok", "cb_gemm", "cb_launch_count"}
    assert declared == set(_abi.SIGS.keys())


def test_gemm_desc_layout_matches_header():
    """ctypes struct must mirror `struct cb_gemm_desc` field for field."""
    from celebbasis_b200.lib import GemmDesc
    text = open(os.path.join(ROOT, "include", "celebbasis_b200.h")).read()
    body = text[text.index("typedef struct cb_gemm_desc {") + len("typedef struct cb_gemm_desc {"): text.index("} cb_gemm_desc;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        m = re.match(r"(?:const\s+)?(?:int32_t|int64_t|float|void\*|float\*|void \*|const void\*|const float\*)\s*(.*)", decl)
        if not m:
            continue
        for name in m.group(1).split(","):
            name = name.strip().lstrip("*").strip()
            if name:
                fields.append(name)
    assert fields == [f[0] for f in GemmDesc._fields_]


def test_no_cpu_fallback_without_device():
    """Without an sm_90 device the product path must fail loudly (no oracle / CPU fallback)."""
    import pytest
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from celebbasis_b200 import lib
    assert lib.load().cb_device_ok() == 0
    from ldm.modules.attention import CrossAttention
    with pytest.raises(RuntimeError):
        CrossAttention(64, heads=2, dim_head=32)(torch.zeros(1, 4, 64))


def test_pointwise_entries_reject_bad_dtype_act_shape_and_alignment():
    """The pointwise entry points check dtype and activation codes, the interleaved GEGLU width and the alignment of
    the pointers their 8- / 16-byte vector accesses use before they launch anything.  Fake, never-dereferenced device
    addresses: a call that got past its checks would launch (or, without a device, return a CUDA error)."""
    import pytest
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: a call that slipped past its checks would launch on fake pointers")
    from celebbasis_b200 import lib
    L = lib.load()
    F16, BF16, F32, BAD = lib.CB_F16, lib.CB_BF16, lib.CB_F32, 7
    ARG, ALIGN = -1, -2
    A = 1 << 32                 # aligned for every vector access
    O2, O4 = A + 2, A + 4       # 2-byte (one fp16 element) and 4-byte offsets
    cases = [
        # unknown dtype / act codes
        (ARG, "cb_axpby2d", (A, BAD, 4, 1.0, None, 0, 0, 0.0, A, F32, 4, 1, 4, None)),
        (ARG, "cb_axpby2d", (A, F16, 4, 1.0, A, BAD, 4, 1.0, A, F32, 4, 1, 4, None)),
        (ARG, "cb_act_fwd", (A, BAD, A, F16, 8, lib.CB_ACT_SILU, None)),
        (ARG, "cb_act_fwd", (A, F16, A, -1, 8, lib.CB_ACT_SILU, None)),
        (ARG, "cb_act_fwd", (A, F16, A, F16, 8, lib.CB_ACT_PRELU, None)),
        (ARG, "cb_act_fwd", (A, F16, A, F16, 8, 9, None)),
        (ARG, "cb_act_bwd", (A, F16, A, 3, A, F16, 8, lib.CB_ACT_GELU, None)),
        (ARG, "cb_act_bwd", (A, F16, A, F16, A, F16, 8, lib.CB_ACT_PRELU, None)),
        (ARG, "cb_nchw_to_nhwc", (A, A, BAD, 1, 3, 16, 8, None)),
        (ARG, "cb_nhwc_to_nchw", (A, BAD, A, 1, 3, 16, 8, None)),
        (ARG, "cb_timestep_embedding", (A, A, BAD, 2, 320, 10000.0, None)),
        (ARG, "cb_face_warp_resize", (A, A, BAD, 1, 64, 64, 1, 112, 8, (ctypes.c_float * 6)(), None)),
        (ARG, "cb_convert_f32", (A, A, BAD, 100, 1.0, None)),
        (ARG, "cb_pack_conv_weight", (A, A, BAD, 8, 8, 3, 3, 8, 8, None, None)),
        (ARG, "cb_upsample2x_fwd", (A, A, BAD, 1, 4, 4, 8, None)),
        (ARG, "cb_channel_affine_act", (A, F16, A, F16, A, None, None, 4, 8, None)),   # scale without shift
        # interleaved GEGLU needs whole 64-column groups
        (ARG, "cb_geglu_fwd", (A, A, F16, 2, 36, 1, None)),
        (ARG, "cb_geglu_bwd", (A, A, A, BF16, F16, 2, 36, 1, None)),
        # vector accesses: every pointer aligned to 4 elements of its dtype
        (ALIGN, "cb_axpby2d", (O4, F32, 4, 1.0, None, 0, 0, 0.0, A, F32, 4, 1, 4, None)),
        (ALIGN, "cb_axpby2d", (A, F16, 4, 1.0, O2, F16, 4, 1.0, A, F16, 4, 1, 4, None)),
        (ALIGN, "cb_axpby2d", (A, F16, 4, 1.0, None, 0, 0, 0.0, A + 8, F32, 4, 1, 4, None)),
        (ALIGN, "cb_geglu_fwd", (O2, A, F16, 2, 32, 0, None)),
        (ALIGN, "cb_geglu_fwd", (A, O4, BF16, 2, 32, 1, None)),
        (ALIGN, "cb_geglu_bwd", (O2, A, A, F16, F16, 2, 32, 0, None)),
        (ALIGN, "cb_geglu_bwd", (A, A, O4, F16, BF16, 2, 32, 1, None)),
        (ALIGN, "cb_upsample2x_fwd", (O4, A, F16, 1, 3, 3, 4, None)),
        (ALIGN, "cb_upsample2x_bwd", (A, F16, A + 8, F32, 1, 3, 3, 4, 1, None)),
        (ALIGN, "cb_zero_insert2x", (A, O2, BF16, 1, 3, 3, 4, None)),
        (ALIGN, "cb_channel_affine_act", (O2, F16, A, F16, A, A, None, 4, 8, None)),
        (ALIGN, "cb_channel_affine_act", (A, F16, A + 8, F32, None, None, A, 4, 8, None)),
        (ALIGN, "cb_embedding_gather", (A, O4, A, 2, 8, 10, None)),
        (ALIGN, "cb_embedding_gather", (A, A, A + 8, 2, 8, 10, None)),
    ]
    n0 = L.cb_launch_count()
    for want, name, args in cases:
        rc = getattr(L, name)(*args)
        assert rc == want, f"{name}{args}: returned {rc} ({lib.last_error()}), expected {want}"
    assert L.cb_launch_count() == n0


def test_graft_entry_build():
    """The driver's build hook: compiles (cached) every CUDA source for sm_90a, loads the library, checks the ABI."""
    import __graft_entry__ as g
    g.build()
