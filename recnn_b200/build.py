"""Build librecnn_b200.so in-tree with nvcc for sm_90a (H100).

No torch.utils.cpp_extension: the product boundary is a plain C ABI
(include/recnn_b200.h), so the library is a plain ``nvcc -shared`` of
recnn_b200/csrc/*.cu.  The .so lives at recnn_b200/lib/librecnn_b200.so (git-ignored;
``__graft_entry__.build()`` makes it).
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIBDIR = os.path.join(PKG, "lib")
OBJDIR = os.path.join(PKG, "build")
LIB = os.path.join(LIBDIR, "librecnn_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17", "--use_fast_math=false",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    "--expt-relaxed-constexpr",
]
# --use_fast_math must stay off: the parity bar needs IEEE div/sqrt and no FTZ.
NVCC_FLAGS = [f for f in NVCC_FLAGS if f != "--use_fast_math=false"]


def find_nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.isfile(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _fingerprint() -> str:
    h = hashlib.sha256()
    h.update(" ".join(NVCC_FLAGS).encode())
    paths = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))]
    paths.append(os.path.join(ROOT, "include", "recnn_b200.h"))
    for p in paths:
        if os.path.isfile(p):
            h.update(p.encode())
            with open(p, "rb") as fh:
                h.update(fh.read())
    return h.hexdigest()


def is_current() -> bool:
    stamp = LIB + ".stamp"
    if not (os.path.isfile(LIB) and os.path.isfile(stamp)):
        return False
    try:
        with open(stamp) as fh:
            return fh.read().strip() == _fingerprint()
    except OSError:
        return False


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every .cu for sm_90a and link the shared library.  Returns its path."""
    if not force and is_current():
        return LIB
    nvcc = find_nvcc()
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    srcs = _sources()

    def compile_one(src):
        obj = os.path.join(OBJDIR, os.path.basename(src)[:-3] + ".o")
        cmd = [nvcc] + NVCC_FLAGS + ["-I", os.path.join(ROOT, "include"), "-c", src, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        # C7510: ptxas serialised the wgmma pipeline (e.g. a function call inside the k-loop); the GEMM would still be
        # correct but lose the overlap it is built around, so such a build is refused rather than shipped.
        if "C7510" in r.stderr:
            raise RuntimeError("ptxas serialised wgmma instructions in %s:\n%s" % (src, r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    with open(LIB + ".stamp", "w") as fh:
        fh.write(_fingerprint())
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
