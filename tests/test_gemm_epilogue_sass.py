"""Compile-time guard on the epilogue of gemm_tc_kernel (no GPU needed, only nvcc).

The epilogue adds bias, row vector and residuals to the accumulators and stores the tile. `out` may be `residual` (an
in-place residual add), so the compiler may not move a global load above an earlier global store of the same thread:
an epilogue that interleaves them runs as one dependent memory round trip per 8-column block and row. The kernel walks
the tile in chunks of 32 columns and issues all of a chunk's loads before its stores, so in the SASS of every
instantiation a load may follow a store at most (chunks - 1) times. Holding a chunk's loads in flight must not cost
spills either. Both are visible only in the compiler's output: the results stay the same, only slower.
"""
import re

from test_gemm_sass import _kernels, compiled  # noqa: F401  (the compiled fixture is reused, not redefined)

CHUNK_COLUMNS = 32
MEM = re.compile(r"(?:@!?U?P\w+\s+)?(LDG|STG)\.")


def test_epilogue_loads_are_not_behind_its_stores(compiled):
    _, kernels = compiled
    for name, ins in kernels.items():
        bn = int(re.search(r"gemm_tc_kernelILi(\d+)E", name).group(1))
        mem = [m.group(1) for m in map(MEM.match, ins) if m]
        assert "STG" in mem, f"{name}: no global store"
        load_after_store = sum(1 for a, b in zip(mem, mem[1:]) if (a, b) == ("STG", "LDG"))
        assert load_after_store <= bn // CHUNK_COLUMNS - 1, \
            f"{name}: a global load follows a global store {load_after_store} times (chunks of {CHUNK_COLUMNS} columns allow {bn // CHUNK_COLUMNS - 1})"


def test_no_spills(compiled):
    log, kernels = compiled
    reports = re.findall(r"Function properties for (\w*gemm_tc_kernel\w*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", log)
    assert {r[0] for r in reports} == set(kernels), "ptxas -v did not report every instantiation"
    spilled = [r for r in reports if r[2] != "0" or r[3] != "0"]
    assert not spilled, f"ptxas spills (kernel, stack, spill stores, spill loads): {spilled}"
