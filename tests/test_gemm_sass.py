"""Compile-time guard on the wgmma main loop of gemm_tc_kernel (no GPU needed, only nvcc).

ptxas serialises wgmma instructions when it finds a non-wgmma definition of accumulator registers, or a thread-dependent
branch, between a group's issue and its wait (C7515 / C7516 / C7518): each HGMMA is then followed by a full
`WARPGROUP.DEPBAR.LE gsb0, 0x0` and the one-group-in-flight pipelining of the loop silently disappears. The kernel
still computes the same result, only slower, so only the compiler's output can show it. This test compiles
gemm_tc.cu with the build's flags and checks every instantiation: no serialisation warning, and in the SASS the
BK / 16 HGMMAs of a k-block issue back to back and the k-block's wait leaves one group in flight.
"""
import re
import subprocess
from pathlib import Path

import pytest

from panacea_b200 import build

SRC = build.CSRC / "gemm_tc.cu"
HGMMAS_PER_K_BLOCK = 64 // 16          # BK / k16
SERIALISED = ("C7515", "C7516", "C7518")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    nvcc = Path(build.NVCC)
    cuobjdump = nvcc.with_name("cuobjdump")
    if not nvcc.exists() or not cuobjdump.exists():
        pytest.skip(f"no nvcc / cuobjdump at {nvcc.parent}")
    obj = tmp_path_factory.mktemp("gemm_sass") / "gemm_tc.o"
    r = subprocess.run([str(nvcc), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(SRC), "-o", str(obj)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sass = subprocess.run([str(cuobjdump), "-sass", str(obj)], capture_output=True, text=True, check=True).stdout
    return r.stderr, _kernels(sass)


def _kernels(sass):
    """{mangled name: [instruction text]} for every gemm_tc_kernel instantiation."""
    out = {}
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = chunk.split("\n", 1)
        if "gemm_tc_kernel" not in name:
            continue
        out[name.strip()] = [m.group(1).strip() for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", body)]
    return out


def test_every_instantiation_is_compiled(compiled):
    _, kernels = compiled
    # gemm_tc_kernel<BN, STAGES, MODE>: every BN = 160 / 128 / 64 / 32 with every MODE = 0 / 1 / 2
    shapes = {m.groups() for m in (re.search(r"gemm_tc_kernelILi(\d+)ELi\d+ELi(\d)E", k) for k in kernels) if m}
    assert shapes == {(bn, mode) for bn in ("160", "128", "64", "32") for mode in "012"}, sorted(kernels)


def test_ptxas_does_not_serialise_wgmma(compiled):
    log, kernels = compiled
    bad = [line for line in log.splitlines() if any(code in line for code in SERIALISED)]
    assert not bad, "ptxas serialises wgmma:\n" + "\n".join(bad)


def test_k_block_hgmmas_issue_back_to_back(compiled):
    _, kernels = compiled
    for name, ins in kernels.items():
        seq = [i for i in ins if "HGMMA" in i or i.startswith("WARPGROUP.")]
        runs, i = [], 0
        while i < len(seq):
            if "HGMMA" not in seq[i]:
                i += 1
                continue
            j = i
            while j < len(seq) and "HGMMA" in seq[j]:
                j += 1
            runs.append((j - i, seq[j] if j < len(seq) else None))
            i = j
        assert runs, f"{name}: no HGMMA"
        for length, after in runs:
            # a WARPGROUP.DEPBAR between the HGMMAs of one k-block would split the run
            assert length % HGMMAS_PER_K_BLOCK == 0, f"{name}: a k-block's HGMMAs are split: {seq}"
            assert after is not None and re.fullmatch(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1", after), \
                f"{name}: the k-block's wait is {after!r}, not one group in flight: {seq}"
