"""In-tree build of libpanacea_b200.so (hand-written CUDA for sm_90a + the C ABI).

nvcc cross-compiles without a GPU; the objects go to build/ and the .so lands next to this file (both git-ignored),
so the package imports from the source tree.
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
INCLUDE = PKG.parent / "include"
BUILD = PKG / "build"
LIB = PKG / "libpanacea_b200.so"

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-I", str(INCLUDE),
]


def _sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def _digest(src: Path) -> str:
    h = hashlib.sha256()
    h.update(" ".join(NVCC_FLAGS).encode())
    h.update(src.read_bytes())
    for hdr in sorted(list(CSRC.glob("*.cuh")) + list(INCLUDE.glob("*.h"))):
        h.update(hdr.read_bytes())
    return h.hexdigest()[:16]


def _compile_one(src: Path, verbose: bool) -> Path:
    obj = BUILD / f"{src.stem}.{_digest(src)}.o"
    if obj.exists():
        return obj
    for old in BUILD.glob(f"{src.stem}.*.o"):
        old.unlink()
    cmd = [NVCC, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
    if verbose:
        sys.stderr.write(r.stderr)
    return obj


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every csrc/*.cu for sm_90a and link libpanacea_b200.so. Idempotent (content-hashed)."""
    BUILD.mkdir(exist_ok=True)
    if force:
        for old in BUILD.glob("*.o"):
            old.unlink()
    srcs = _sources()
    if not srcs:
        raise RuntimeError(f"no CUDA sources under {CSRC}")
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile_one(s, verbose), srcs))
    stamp = BUILD / "link.stamp"
    key = " ".join(o.name for o in objs)
    if LIB.exists() and stamp.exists() and stamp.read_text() == key and not force:
        return LIB
    cmd = [NVCC, "-shared", "-o", str(LIB), *[str(o) for o in objs],
           "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC", "-cudart", "static"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    stamp.write_text(key)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
