"""CPU: the C-ABI shared library loads without a GPU and exports every symbol include/celebbasis_b200.h declares."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "celebbasis_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(cb_[a-z0-9_]+)\s*\(", text)))


def test_library_loads_and_exports_header_symbols():
    from celebbasis_b200 import lib
    L = lib.load()
    syms = _declared_symbols()
    assert len(syms) >= 35
    for s in syms:
        assert hasattr(L, s), f"symbol {s} declared in the header but not exported"
    assert L.cb_abi_version() == 5
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


def test_graft_entry_build():
    """The driver's build hook: compiles (cached) every CUDA source for sm_90a, loads the library, checks the ABI."""
    import __graft_entry__ as g
    g.build()
