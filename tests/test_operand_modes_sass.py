"""Which operand modes (pn_operand_mode, include/panacea_b200.h) the operand-templated kernels are compiled for; no GPU
needed, only nvcc. Each entry point rejects the modes it does not accept before any work and instantiates its kernels for
exactly the modes it accepts, so the library holds no kernel that no call can launch.

The attentions serve bf16 on their tensor-core kernels (attn_fa.cu, attn_small.cu); attn_f32.cu holds only the two
parity-mode stores.
"""
import re
import subprocess
from pathlib import Path

import pytest

from panacea_b200 import build

BF16, SPLIT3, F32, SPLIT3_B = 0, 1, 2, 3
# kernel: (source, index of OP among its integer template arguments, the modes it is compiled for)
FAMILIES = {
    "gn_fused_kernel": ("norm.cu", 0, {BF16, SPLIT3, F32}),
    "gn_pixel_kernel": ("norm.cu", 1, {BF16, SPLIT3, F32}),
    "layernorm_kernel": ("norm.cu", 1, {BF16, SPLIT3, F32}),
    "upsample2x_kernel": ("elementwise.cu", 0, {BF16, SPLIT3, F32}),
    "geglu_operand_kernel": ("elementwise.cu", 0, {BF16, SPLIT3, F32}),
    "gelu_operand_kernel": ("elementwise.cu", 0, {BF16, SPLIT3, F32}),
    "cast_operand_kernel": ("elementwise.cu", 0, {BF16, SPLIT3, SPLIT3_B}),
    "im2col_s2_kernel": ("elementwise.cu", 0, {BF16, SPLIT3}),
    "softmax_rows_kernel": ("elementwise.cu", 0, {BF16, SPLIT3}),
    "attn_f32_view_kernel": ("attn_f32.cu", 1, {SPLIT3, F32}),
    "attn_f32_temporal_kernel": ("attn_f32.cu", 1, {SPLIT3, F32}),
    "attn_f32_causal_kernel": ("attn_f32.cu", 0, {SPLIT3, F32}),
}
INT_ARG = re.compile(r"Li(\d+)E")


@pytest.fixture(scope="module")
def kernels(tmp_path_factory):
    """the mangled names of the kernels compiled from each source"""
    nvcc = Path(build.NVCC)
    cuobjdump = nvcc.with_name("cuobjdump")
    if not nvcc.exists() or not cuobjdump.exists():
        pytest.skip(f"no nvcc / cuobjdump at {nvcc.parent}")
    out = tmp_path_factory.mktemp("operand_modes_sass")
    procs = {}
    for src in sorted({src for src, _, _ in FAMILIES.values()}):
        obj = out / f"{Path(src).stem}.o"
        procs[src] = (obj, subprocess.Popen([str(nvcc), *build.NVCC_FLAGS, "-c", str(build.CSRC / src), "-o", str(obj)],
                                            stderr=subprocess.PIPE, text=True))
    result = {}
    for src, (obj, proc) in procs.items():
        log = proc.communicate()[1]
        assert proc.returncode == 0, log
        sass = subprocess.run([str(cuobjdump), "-sass", str(obj)], capture_output=True, text=True, check=True).stdout
        result[src] = re.findall(r"Function : (\S+)", sass)
    return result


@pytest.mark.parametrize("kernel", sorted(FAMILIES))
def test_kernel_is_compiled_for_exactly_the_accepted_modes(kernels, kernel):
    src, op_index, modes = FAMILIES[kernel]
    # {the other template arguments: the modes compiled with them}
    shapes = {}
    for name in kernels[src]:
        m = re.match(rf"_ZN2pn{len(kernel)}{kernel}I(.*?)EEv", name)
        if m is None:
            continue
        args = INT_ARG.findall(m.group(1))
        op = int(args.pop(op_index))
        shapes.setdefault((tuple(args), INT_ARG.sub("", m.group(1))), set()).add(op)
    assert shapes, f"{kernel}: not compiled from {src}"
    wrong = {shape: ops for shape, ops in shapes.items() if ops != modes}
    assert not wrong, f"{kernel}: compiled for operand modes other than {sorted(modes)}: {wrong}"
