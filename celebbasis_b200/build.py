"""In-tree build of libcelebbasis_b200.so (sm_90a only) with explicit nvcc commands.

The shared object is the C-ABI declared in include/celebbasis_b200.h.  It is built next to this file
so that the package is importable straight from the source tree (a JIT cache under ~/.cache would not be).
"""
import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "build")
LIB = os.path.join(HERE, "libcelebbasis_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _nvcc():
    nv = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nv):
        raise RuntimeError("nvcc not found; cannot build libcelebbasis_b200.so")
    return nv


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(path):
    h = hashlib.sha1()
    with open(path, "rb") as f:
        h.update(f.read())
    for dep in sorted(os.listdir(CSRC)):
        if dep.endswith((".cuh", ".h")):
            with open(os.path.join(CSRC, dep), "rb") as f:
                h.update(f.read())
    with open(os.path.join(HERE, "..", "include", "celebbasis_b200.h"), "rb") as f:
        h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _compile_one(nv, src, verbose):
    obj = os.path.join(OBJ, src[:-3] + ".o")
    stamp = obj + ".sha1"
    dig = _digest(os.path.join(CSRC, src))
    if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
        return obj, False, ""
    cmd = [nv, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(dig)
    return obj, True, r.stderr


def build(verbose=False, force=False):
    os.makedirs(OBJ, exist_ok=True)
    nv = _nvcc()
    if force:
        for f in os.listdir(OBJ):
            os.remove(os.path.join(OBJ, f))
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile_one(nv, s, verbose), srcs))
    objs = [r[0] for r in results]
    rebuilt = any(r[1] for r in results)
    if verbose:
        for r in results:
            if r[2]:
                sys.stderr.write(r[2])
    if rebuilt or not os.path.exists(LIB):
        cmd = [nv, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB, *objs, "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
