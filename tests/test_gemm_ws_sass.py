"""Compile-time guard on gemm_ws_kernel, the persistent weight-stationary GEMM (no GPU needed, only nvcc).

Like gemm_tc_kernel (test_gemm_sass.py), the kernel only runs at speed if ptxas keeps its wgmma pipelined: no
serialisation warning (C7515 / C7516 / C7518), and the four HGMMAs of a k-block issue back to back, not split by a
`WARPGROUP.DEPBAR`. Its persistent loop keeps the 80-float accumulator live across row tiles, next to the epilogue's
addressing, so it must also compile without spills within the 168 registers per thread that its 384-thread CTA allows.
"""
import re
import subprocess
from pathlib import Path

import pytest

from panacea_b200 import build

SRC = build.CSRC / "gemm_ws.cu"
HGMMAS_PER_K_BLOCK = 64 // 16
SERIALISED = ("C7515", "C7516", "C7518")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    nvcc = Path(build.NVCC)
    cuobjdump = nvcc.with_name("cuobjdump")
    if not nvcc.exists() or not cuobjdump.exists():
        pytest.skip(f"no nvcc / cuobjdump at {nvcc.parent}")
    obj = tmp_path_factory.mktemp("gemm_ws_sass") / "gemm_ws.o"
    r = subprocess.run([str(nvcc), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(SRC), "-o", str(obj)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sass = subprocess.run([str(cuobjdump), "-sass", str(obj)], capture_output=True, text=True, check=True).stdout
    kernels = {}
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = chunk.split("\n", 1)
        if "gemm_ws_kernel" in name:
            kernels[name.strip()] = [m.group(1).strip() for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", body)]
    return r.stderr, kernels


def test_every_mode_is_compiled(compiled):
    _, kernels = compiled
    modes = {m.group(1) for m in (re.search(r"gemm_ws_kernelILi(\d)E", k) for k in kernels) if m}
    assert modes == {"0", "1", "2"}, sorted(kernels)


def test_ptxas_does_not_serialise_wgmma(compiled):
    log, _ = compiled
    bad = [line for line in log.splitlines() if any(code in line for code in SERIALISED)]
    assert not bad, "ptxas serialises wgmma:\n" + "\n".join(bad)


def test_k_block_hgmmas_are_not_split(compiled):
    _, kernels = compiled
    for name, ins in kernels.items():
        seq = [i for i in ins if "HGMMA" in i or i.startswith("WARPGROUP.")]
        runs, run = [], 0
        for i in seq:
            if "HGMMA" in i:
                run += 1
            elif run:
                runs.append(run)
                run = 0
        if run:
            runs.append(run)
        assert runs, f"{name}: no HGMMA"
        assert all(r % HGMMAS_PER_K_BLOCK == 0 for r in runs), f"{name}: a k-block's HGMMAs are split: {seq}"


def test_no_spills(compiled):
    log, kernels = compiled
    reports = re.findall(r"Function properties for (\w*gemm_ws_kernel\w*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", log)
    assert {r[0] for r in reports} == set(kernels), "ptxas -v did not report every mode"
    spilled = [r for r in reports if r[2] != "0" or r[3] != "0"]
    assert not spilled, f"ptxas spills (kernel, stack, spill stores, spill loads): {spilled}"
