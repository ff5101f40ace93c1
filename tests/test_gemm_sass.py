"""What ptxas made of the cb_gemm main loop (no GPU needed).

cb_gemm.cu is compiled for sm_90a with the library's own nvcc flags, and for every cb_gemm_kernel instantiation the
ptxas notes and the SASS are checked for the patterns that stall the wgmma pipeline:
- C7519 / C7520 / C7515: ptxas injected a warpgroup.arrive, or serialised the wgmma.mma_async instructions;
- a dummy `HGMMA.64x8x16.F16 RZ, gdesc[URZ]`, which is what a commit of MMAs spread over branches compiles to;
- an HGMMA that does not wait for its scoreboard (no gsb0) but is not directly followed by the next HGMMA of its
  batch, i.e. a batch broken up by a branch or a second WARPGROUP.ARRIVE;
- more WARPGROUP.ARRIVE than batches (HGMMAs with gsb0).
The compile takes a minute or two.
"""
import os
import re
import shutil
import subprocess

import pytest

from celebbasis_b200 import build

GEMM_KERNEL = "cb_gemm_kernel"
STALL_NOTES = ("C7519", "C7520", "C7515")
DUMMY_COMMIT = re.compile(r"HGMMA\.64x8x16\.F16 RZ, gdesc\[URZ\]")
BRANCH = re.compile(r"^(@!?U?P\w+\s+)?(BRA|BRX|JMP|JMX|CALL|RET|EXIT)\b")


def _tool(name):
    found = shutil.which(name)
    if found:
        return found
    cand = os.path.join("/usr/local/cuda/bin", name)
    return cand if os.path.exists(cand) else None


def ptxas_notes(log):
    """{function: [note codes]} of the ptxas info lines that name a function."""
    out = {}
    for m in re.finditer(r"\((C\d+)\)[^\n]*in function '([^']+)'", log):
        out.setdefault(m.group(2), []).append(m.group(1))
    return out


def spills(log):
    """{function: (spill store bytes, spill load bytes)} from ptxas -v."""
    return {m.group(1): (int(m.group(2)), int(m.group(3))) for m in re.finditer(
        r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)}


def sass_functions(sass):
    """{function: [instruction text]} from cuobjdump -sass, addresses and encodings stripped."""
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = out.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
        if cur is not None and m:
            cur.append(m.group(1))
    return out


def mainloop_violations(instrs):
    """Reasons why this kernel's wgmma batches are not one straight-line group each (empty list: none)."""
    bad = []
    if any(DUMMY_COMMIT.search(i) for i in instrs):
        bad.append("dummy HGMMA.64x8x16 commit")
    hgmma = [k for k, i in enumerate(instrs) if i.startswith("HGMMA")]
    if not hgmma:
        bad.append("no HGMMA")
    waits = sum(1 for k in hgmma if "gsb0" in instrs[k])
    for k in hgmma:
        if "gsb0" in instrs[k]:
            continue
        for nxt in instrs[k + 1:]:
            if nxt.startswith("HGMMA"):
                break
            if BRANCH.match(nxt) or nxt.startswith("WARPGROUP.ARRIVE"):
                bad.append(f"HGMMA without gsb0 followed by {nxt!r} before the next HGMMA")
                break
        else:
            bad.append("HGMMA without gsb0 is the last HGMMA")
    arrives = sum(1 for i in instrs if i.startswith("WARPGROUP.ARRIVE"))
    if arrives > waits:
        bad.append(f"{arrives} WARPGROUP.ARRIVE for {waits} HGMMA batches")
    return bad


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    nvcc, cuobjdump = _tool("nvcc"), _tool("cuobjdump")
    if nvcc is None or cuobjdump is None:
        pytest.skip("nvcc / cuobjdump not available")
    out = tmp_path_factory.mktemp("cb_gemm_sass")
    obj = str(out / "cb_gemm.o")
    r = subprocess.run([nvcc, *build.NVCC_FLAGS, "-c", os.path.join(build.CSRC, "cb_gemm.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    d = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True)
    assert d.returncode == 0, d.stderr[-4000:]
    kernels = {k: v for k, v in sass_functions(d.stdout).items() if GEMM_KERNEL in k}
    assert kernels, "no cb_gemm_kernel in the SASS"
    return r.stdout + r.stderr, kernels


def test_no_injected_arrive_or_serialisation(compiled):
    log, kernels = compiled
    notes = {f: [c for c in codes if c in STALL_NOTES] for f, codes in ptxas_notes(log).items() if GEMM_KERNEL in f}
    notes = {f: c for f, c in notes.items() if c}
    assert not notes, notes


def test_no_spills(compiled):
    log, kernels = compiled
    sp = {f: s for f, s in spills(log).items() if GEMM_KERNEL in f}
    assert set(sp) == set(kernels)
    assert all(s == (0, 0) for s in sp.values()), {f: s for f, s in sp.items() if s != (0, 0)}


def test_one_wgmma_batch_per_k_iteration(compiled):
    log, kernels = compiled
    bad = {f: v for f, v in ((f, mainloop_violations(i)) for f, i in kernels.items()) if v}
    assert not bad, {f: v[:3] for f, v in bad.items()}


def test_checker_catches_a_drained_batch():
    # the SASS pattern of a k16 loop whose MMAs sit in branches of their own, committed by a dummy MMA
    drained = ["WARPGROUP.ARRIVE", "HGMMA.64x128x16.F32 R24, gdesc[UR8], R24", "BRA 0x2370",
               "WARPGROUP.ARRIVE", "HGMMA.64x128x16.F32 R24, gdesc[UR8], R24",
               "HGMMA.64x8x16.F16 RZ, gdesc[URZ], RZ, !UPT, gsb0", "WARPGROUP.DEPBAR.LE gsb0, 0x1"]
    bad = mainloop_violations(drained)
    assert any("dummy" in b for b in bad)
    assert any("BRA" in b for b in bad)
    assert any("WARPGROUP.ARRIVE for" in b for b in bad)
    batched = ["WARPGROUP.ARRIVE"] + ["HGMMA.64x128x16.F32 R24, gdesc[UR8], R24"] * 3 + \
              ["HGMMA.64x128x16.F32 R24, gdesc[UR8], R24, gsb0", "BRA 0x2370", "WARPGROUP.DEPBAR.LE gsb0, 0x1"]
    assert mainloop_violations(batched) == []
