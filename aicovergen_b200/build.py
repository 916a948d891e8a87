"""In-tree build of libb200vc.so (sm_90a only).

`python -m aicovergen_b200.build` or `__graft_entry__.build()`.  nvcc
cross-compiles without a GPU; the resulting .so is git-ignored but travels with
the repo snapshot to the GPU box.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
OUT_DIR = PKG / "lib"
LIB = OUT_DIR / "libb200vc.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every .cu under csrc/ and link lib/libb200vc.so. Incremental by content hash."""
    OUT_DIR.mkdir(exist_ok=True)
    srcs = sorted(CSRC.glob("*.cu"))
    hdrs = sorted(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "b200vc.h"]
    stamp = OUT_DIR / "build.stamp"
    digest = _digest(srcs + hdrs)
    if not force and LIB.exists() and stamp.exists() and stamp.read_text() == digest:
        return LIB
    nvcc = _nvcc()
    hdr_digest = _digest(hdrs)

    def compile_one(src: Path) -> Path:
        obj = OUT_DIR / (src.stem + ".o")
        ostamp = OUT_DIR / (src.stem + ".stamp")
        d = hashlib.sha256((hdr_digest + hashlib.sha256(src.read_bytes()).hexdigest()).encode()).hexdigest()
        if not force and obj.exists() and ostamp.exists() and ostamp.read_text() == d:
            return obj
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
        ostamp.write_text(d)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    cmd = [nvcc, "-shared", "-o", str(LIB), *map(str, objs), "-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    stamp.write_text(digest)
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose=True)
    print(p)
