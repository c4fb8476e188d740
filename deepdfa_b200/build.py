"""In-tree build of libddfa_b200.so (nvcc, sm_90a only: NVIDIA H100).

The shared library is a plain C-ABI object (include/ddfa_b200.h): it does not link against
torch or Python.  It is built into ``deepdfa_b200/lib/`` (git-ignored), next to the package that loads it.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIBDIR = PKG / "lib"
LIB = LIBDIR / "libddfa_b200.so"
STAMP = LIBDIR / "libddfa_b200.stamp"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC,-O3,-Wall,-Wno-unused-function",
    "-Xptxas", "-v",
]


def sources():
    return sorted(CSRC.glob("*.cu"))


def _digest() -> str:
    h = hashlib.sha256()
    for p in sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "ddfa_b200.h"]):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found: cannot build libddfa_b200.so")


def cuda_tool(name: str) -> Path:
    """A CUDA toolkit binary (cuobjdump, ...) from the toolkit whose nvcc builds the library."""
    return Path(nvcc_path()).resolve().parent / name


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every .cu under csrc/ for sm_90a and link libddfa_b200.so. Idempotent."""
    LIBDIR.mkdir(exist_ok=True)
    digest = _digest()
    if not force and LIB.exists() and STAMP.exists() and STAMP.read_text().strip() == digest:
        return LIB
    nvcc = nvcc_path()
    objdir = LIBDIR / "obj"
    objdir.mkdir(exist_ok=True)
    procs = []
    for src in sources():
        obj = objdir / (src.stem + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    objs = []
    log = []
    for src, obj, p in procs:
        out, _ = p.communicate()
        log.append(f"==== {src.name}\n{out}")
        if p.returncode != 0:
            sys.stderr.write("\n".join(log))
            raise RuntimeError(f"nvcc failed on {src}")
        objs.append(str(obj))
    (LIBDIR / "build.log").write_text("\n".join(log))
    if verbose:
        print("\n".join(log))
    cmd = [nvcc, "-shared", "-o", str(LIB), *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "shared"]
    subprocess.run(cmd, check=True)
    STAMP.write_text(digest)
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(path)
