"""Compile-time guards on the two wgmma GEMM kernels, gemm_tc_kernel (gemm_tc.cu) and the persistent gemm_ws_kernel
(gemm_ws.cu); no GPU needed, only nvcc. The kernels still compute the same results when any of these fails, only slower,
so only the compiler's output can show it.

- ptxas serialises wgmma instructions when it finds a non-wgmma definition of accumulator registers, or a
  thread-dependent branch, between a group's issue and its wait (C7515 / C7516 / C7518): each HGMMA is then followed by
  a full `WARPGROUP.DEPBAR.LE gsb0, 0x0`. So in the SASS of every instantiation the BK / 16 HGMMAs of a k-block must
  issue back to back, and in gemm_tc_kernel's main loop the k-block's wait must leave one group in flight.
- gemm_tc_kernel's epilogue: `out` may be `residual` (an in-place residual add), so the compiler may not move a global
  load above an earlier global store of the same thread, and an epilogue that interleaves them runs as one dependent
  memory round trip per 8-column block and row. The kernel walks the tile in chunks of 32 columns and issues all of a
  chunk's loads before its stores, so a load may follow a store at most (chunks - 1) times.
- Nothing spills: gemm_tc_kernel holds a chunk's loads in flight within the 128 registers of two CTAs per SM, and
  gemm_ws_kernel keeps its 80-float accumulator live across row tiles within the 168 registers of its 384-thread CTA.
"""
import re
import subprocess
from pathlib import Path

import pytest

from panacea_b200 import build

KERNELS = {"gemm_tc_kernel": "gemm_tc.cu", "gemm_ws_kernel": "gemm_ws.cu"}
HGMMAS_PER_K_BLOCK = 64 // 16          # BK / k16
SERIALISED = ("C7515", "C7516", "C7518")
CHUNK_COLUMNS = 32
MEM = re.compile(r"(?:@!?U?P\w+\s+)?(LDG|STG)\.")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """{kernel: (ptxas -v log, {mangled name: [instruction text]} of its instantiations)}"""
    nvcc = Path(build.NVCC)
    cuobjdump = nvcc.with_name("cuobjdump")
    if not nvcc.exists() or not cuobjdump.exists():
        pytest.skip(f"no nvcc / cuobjdump at {nvcc.parent}")
    out = tmp_path_factory.mktemp("gemm_sass")
    procs = {}
    for kernel, src in KERNELS.items():
        obj = out / f"{kernel}.o"
        procs[kernel] = (obj, subprocess.Popen([str(nvcc), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(build.CSRC / src),
                                                "-o", str(obj)], stderr=subprocess.PIPE, text=True))
    result = {}
    for kernel, (obj, proc) in procs.items():
        log = proc.communicate()[1]
        assert proc.returncode == 0, log
        sass = subprocess.run([str(cuobjdump), "-sass", str(obj)], capture_output=True, text=True, check=True).stdout
        result[kernel] = (log, _kernels(sass, kernel))
    return result


def _kernels(sass, kernel):
    """{mangled name: [instruction text]} for every instantiation of `kernel`"""
    out = {}
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = chunk.split("\n", 1)
        if kernel in name:
            out[name.strip()] = [m.group(1).strip() for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", body)]
    return out


def _hgmma_runs(ins):
    """[(length of a run of HGMMAs, the WARPGROUP instruction after it or None)] of one instantiation's SASS"""
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
    return runs


def _assert_k_blocks_not_split(name, runs):
    assert runs, f"{name}: no HGMMA"
    # a WARPGROUP.DEPBAR between the HGMMAs of one k-block would split the run
    assert all(length % HGMMAS_PER_K_BLOCK == 0 for length, _ in runs), f"{name}: a k-block's HGMMAs are split: {runs}"


def _assert_not_serialised(log):
    bad = [line for line in log.splitlines() if any(code in line for code in SERIALISED)]
    assert not bad, "ptxas serialises wgmma:\n" + "\n".join(bad)


def _assert_no_spills(log, kernels, kernel):
    reports = re.findall(rf"Function properties for (\w*{kernel}\w*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", log)
    assert {r[0] for r in reports} == set(kernels), "ptxas -v did not report every instantiation"
    spilled = [r for r in reports if r[2] != "0" or r[3] != "0"]
    assert not spilled, f"ptxas spills (kernel, stack, spill stores, spill loads): {spilled}"


def test_every_instantiation_is_compiled(compiled):
    _, kernels = compiled["gemm_tc_kernel"]
    # gemm_tc_kernel<BN, STAGES, MODE>: every BN = 160 / 128 / 64 / 32 with every MODE = 0 / 1 / 2
    shapes = {m.groups() for m in (re.search(r"gemm_tc_kernelILi(\d+)ELi\d+ELi(\d)E", k) for k in kernels) if m}
    assert shapes == {(bn, mode) for bn in ("160", "128", "64", "32") for mode in "012"}, sorted(kernels)


def test_every_mode_is_compiled(compiled):
    _, kernels = compiled["gemm_ws_kernel"]
    modes = {m.group(1) for m in (re.search(r"gemm_ws_kernelILi(\d)E", k) for k in kernels) if m}
    assert modes == {"0", "1", "2"}, sorted(kernels)


def test_ptxas_does_not_serialise_wgmma(compiled):
    _assert_not_serialised(compiled["gemm_tc_kernel"][0])


def test_ws_ptxas_does_not_serialise_wgmma(compiled):
    _assert_not_serialised(compiled["gemm_ws_kernel"][0])


def test_k_block_hgmmas_issue_back_to_back(compiled):
    _, kernels = compiled["gemm_tc_kernel"]
    for name, ins in kernels.items():
        runs = _hgmma_runs(ins)
        _assert_k_blocks_not_split(name, runs)
        for _, after in runs:
            assert after is not None and re.fullmatch(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1", after), \
                f"{name}: the k-block's wait is {after!r}, not one group in flight: {runs}"


def test_k_block_hgmmas_are_not_split(compiled):
    _, kernels = compiled["gemm_ws_kernel"]
    for name, ins in kernels.items():
        _assert_k_blocks_not_split(name, _hgmma_runs(ins))


def test_epilogue_loads_are_not_behind_its_stores(compiled):
    _, kernels = compiled["gemm_tc_kernel"]
    for name, ins in kernels.items():
        bn = int(re.search(r"gemm_tc_kernelILi(\d+)E", name).group(1))
        mem = [m.group(1) for m in map(MEM.match, ins) if m]
        assert "STG" in mem, f"{name}: no global store"
        load_after_store = sum(1 for a, b in zip(mem, mem[1:]) if (a, b) == ("STG", "LDG"))
        assert load_after_store <= bn // CHUNK_COLUMNS - 1, \
            f"{name}: a global load follows a global store {load_after_store} times (chunks of {CHUNK_COLUMNS} columns allow {bn // CHUNK_COLUMNS - 1})"


def test_tc_no_spills(compiled):
    _assert_no_spills(*compiled["gemm_tc_kernel"], "gemm_tc_kernel")


def test_ws_no_spills(compiled):
    _assert_no_spills(*compiled["gemm_ws_kernel"], "gemm_ws_kernel")
