"""What ptxas made of the flash-attention kernels (no GPU needed).

cb_attention.cu is compiled for sm_90a with the library's own nvcc flags, and every cb_attention_fwd_kernel /
cb_attention_bwd_kernel instantiation is checked with the SASS parser, spill parser and batch checker of
test_gemm_sass.py (imported, so both tests read ptxas output the same way), plus checks of its own:
- no note that ptxas serialised the wgmma.mma_async instructions or injected a warpgroup.arrive: C7519 / C7520 /
  C7515 as for the GEMM, and C7512 (insufficient registers), C7514 (accumulator read in flight), C7518 (wait in a
  divergent path);
- no spill in any instantiation;
- no dummy `HGMMA.64x8x16` commit, no branch or second WARPGROUP.ARRIVE inside a batch, no more arrives than batches;
- the MMAs of a group stay one batch: no kernel has as many scoreboard waits (gsb0) as HGMMAs, and at k16 step counts
  above 1, where every group has at least two MMAs, no batch holds a single HGMMA.
"""
import os
import re
import subprocess

import pytest

from celebbasis_b200 import build
from test_gemm_sass import STALL_NOTES, _tool, mainloop_violations, sass_functions, spills

ATTN_KERNEL = re.compile(r"cb_attention_(fwd|bwd)_kernel")
ATTN_STALL_NOTES = STALL_NOTES + ("C7512", "C7514", "C7518")
KSTEPS = re.compile(r"cb_attention_(?:fwd|bwd)_kernelILi(\d+)E")


def ptxas_notes(log):
    """{function: [note codes]} of every ptxas info line that names a function.  The serialisation notes name it as
    "in the function '...'" (C7514, C7515, C7518) or "for the function '...'" (C7512), the injected-arrive note as
    "in function '...'" (C7519)."""
    out = {}
    for m in re.finditer(r"\((C\d+)\)[^\n]*?function '([^']+)'", log):
        out.setdefault(m.group(2), []).append(m.group(1))
    return out


def batch_sizes(instrs):
    """HGMMA count of every batch, a batch ending at the HGMMA that waits for its scoreboard (gsb0)."""
    sizes, n = [], 0
    for i in instrs:
        if i.startswith("HGMMA"):
            n += 1
            if "gsb0" in i:
                sizes.append(n)
                n = 0
    return sizes


def split_batch_violations(instrs, ksteps):
    """Reasons why the MMAs of a group were issued as several batches (empty list: none)."""
    bad = []
    hgmma = sum(1 for i in instrs if i.startswith("HGMMA"))
    sizes = batch_sizes(instrs)
    if hgmma and len(sizes) >= hgmma:
        bad.append(f"{len(sizes)} gsb0 waits for {hgmma} HGMMA: every MMA is a batch of its own")
    if ksteps > 1 and 1 in sizes:
        bad.append(f"batches of one HGMMA at {ksteps} k16 steps: {sizes}")
    return bad


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    nvcc, cuobjdump = _tool("nvcc"), _tool("cuobjdump")
    if nvcc is None or cuobjdump is None:
        pytest.skip("nvcc / cuobjdump not available")
    out = tmp_path_factory.mktemp("cb_attention_sass")
    obj = str(out / "cb_attention.o")
    r = subprocess.run([nvcc, *build.NVCC_FLAGS, "-c", os.path.join(build.CSRC, "cb_attention.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    d = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True)
    assert d.returncode == 0, d.stderr[-4000:]
    kernels = {k: v for k, v in sass_functions(d.stdout).items() if ATTN_KERNEL.search(k)}
    assert kernels, "no cb_attention kernel in the SASS"
    return r.stdout + r.stderr, kernels


def test_every_head_dim_step_count_instantiated(compiled):
    log, kernels = compiled
    assert len(kernels) == 8 * 3, sorted(kernels)     # k16 steps 1..8; forward, dQ and dK/dV


def test_no_injected_arrive_or_serialisation(compiled):
    log, kernels = compiled
    notes = {f: [c for c in codes if c in ATTN_STALL_NOTES] for f, codes in ptxas_notes(log).items()
             if ATTN_KERNEL.search(f)}
    notes = {f: c for f, c in notes.items() if c}
    assert not notes, notes


def test_no_spills(compiled):
    log, kernels = compiled
    sp = {f: s for f, s in spills(log).items() if ATTN_KERNEL.search(f)}
    assert set(sp) == set(kernels)
    assert all(s == (0, 0) for s in sp.values()), {f: s for f, s in sp.items() if s != (0, 0)}


def test_one_wgmma_batch_per_group(compiled):
    log, kernels = compiled
    bad = {}
    for f, instrs in kernels.items():
        v = mainloop_violations(instrs) + split_batch_violations(instrs, int(KSTEPS.search(f).group(1)))
        if v:
            bad[f] = v[:3]
    assert not bad, bad


def test_note_parser_reads_every_wording():
    log = ("ptxas info    : (C7512) Potential Performance Loss: wgmma.mma_async instructions are serialized due to "
           "insufficient register resources for the function 'kA'\n"
           "ptxas info    : (C7515) Potential Performance Loss: wgmma.mma_async instructions are serialized due to non "
           "wgmma instructions defining accumulator registers of a wgmma between start and end of the pipeline stage in "
           "the function 'kB'\n"
           "ptxas info    : (C7519) warpgroup.arrive is injected in around line 568 by compiler to allow use of "
           "registers in GMMA in function 'kC'\n")
    assert ptxas_notes(log) == {"kA": ["C7512"], "kB": ["C7515"], "kC": ["C7519"]}


def test_checker_catches_one_mma_batches():
    # every HGMMA waits for its own scoreboard: what ptxas emits when it serialises a group (C7512 and friends)
    serial = ["WARPGROUP.ARRIVE", "HGMMA.64x128x16.F32 R24, gdesc[UR8], R24, gsb0", "WARPGROUP.DEPBAR.LE gsb0, 0x0"] * 4
    assert mainloop_violations(serial) == []           # the GEMM checker alone accepts it
    assert any("batch of its own" in b for b in split_batch_violations(serial, 3))
    batched = ["WARPGROUP.ARRIVE"] + ["HGMMA.64x64x16.F32 R24, gdesc[UR8], R24"] * 2 + \
              ["HGMMA.64x64x16.F32 R24, gdesc[UR8], R24, gsb0", "WARPGROUP.DEPBAR.LE gsb0, 0x1"]
    assert split_batch_violations(batched, 3) == []
    assert any("batches of one" in b for b in split_batch_violations(batched + serial[:3], 3))
