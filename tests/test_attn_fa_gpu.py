"""attn_fa_kernel (attn_fa.cu): key blocks sized to the real key count, row-major query tiles, and S of one key block
issued with P V of the previous one.

GPU tests compare against torch fp32 attention on the same bf16 inputs, at geometries that reach each path: query tiles of
128 row-major tokens that straddle view rows (w = 56, 24) next to rectangular tiles (w = 28, 14, 7); key blocks of 112 keys
(n112), of 96 keys, and of 28 keys on n32 whose last 4 columns are masked; 77 text keys on n80; head_dim 80; many key
blocks per query tile with a peaked softmax, so the running maximum moves from block to block.
The cross-view cases include view 5, whose only neighbour is view 4.

The CPU test reads the SASS of every instantiation: no serialised wgmma, no spills.
"""
import re
import subprocess
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

from panacea_b200 import build

torch.backends.cuda.matmul.allow_tf32 = False

NEIGH = ((5, 1), (0, 2), (1, 3), (2, 4), (3, 5), (4,))
WIDTHS = (16, 32, 48, 64, 80, 96, 112, 128)          # N of the S wgmma, one instantiation each per head_dim


@pytest.fixture(scope="module")
def ops():
    from panacea_b200.ops import NativeOps
    return NativeOps()


def _rand(shape, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(torch.bfloat16).cuda()


def _mha(q, k, v, heads):
    B, Nq, C = q.shape
    d = C // heads
    sp = lambda z: z.reshape(B, -1, heads, d).transpose(1, 2)
    return F.scaled_dot_product_attention(sp(q), sp(k), sp(v)).transpose(1, 2).reshape(B, Nq, C)


def _view_ref(qkv, heads, cross):
    Fr, H, V, w, C3 = qkv.shape
    C = C3 // 3
    q, k, v = qkv.float().split(C, dim=-1)
    out = torch.empty_like(q)
    for i in range(V):
        nb = NEIGH[i] if cross else (i,)
        ki = torch.cat([k[:, :, j] for j in nb], dim=2).reshape(Fr, -1, C)
        vi = torch.cat([v[:, :, j] for j in nb], dim=2).reshape(Fr, -1, C)
        out[:, :, i] = _mha(q[:, :, i].reshape(Fr, H * w, C), ki, vi, heads).reshape(Fr, H, w, C)
    return out


def _check(got, ref, name, tol=2e-2):
    got = got.float()
    assert torch.isfinite(got).all(), f"{name}: non-finite"
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item()
    rel_l2 = ((got - ref).norm() / ref.norm()).item()
    assert err <= tol * scale and rel_l2 <= 1e-2, f"{name}: max err {err:.3e} (scale {scale:.3e}), rel-L2 {rel_l2:.3e}"


# (F, H, w): query tiling / keys per block
VIEWS = [
    (1, 32, 56),     # row-major tiles (14 per view), n112
    (2, 3, 56),      # row-major: one full tile and one of 40 tokens; 56 keys (kh = 1) on n64
    (2, 16, 24),     # row-major (3 tiles of 128 instead of 4 rectangles of 120), n96
    (2, 12, 28),     # rectangles of 4 rows, n112
    (2, 8, 14),      # rectangles of 8 rows, n112
    (3, 4, 7),       # 28 keys on n32: 4 masked columns
    (1, 16, 7),      # 28 keys on n32, 4 key blocks per view
]


@pytest.mark.gpu
@pytest.mark.parametrize("d", [64, 80])
@pytest.mark.parametrize("cross", [False, True])
@pytest.mark.parametrize("Fr,H,w", VIEWS)
def test_attention_view_tiles(ops, Fr, H, w, cross, d):
    heads = 2
    qkv = _rand((Fr, H, 6, w, 3 * heads * d), 100 + H * w + d)
    out = ops.attention_view(qkv, heads, cross, NEIGH)
    torch.cuda.synchronize()
    _check(out, _view_ref(qkv, heads, cross), f"attention_view F={Fr} H={H} w={w} d={d} cross={cross}")


@pytest.mark.gpu
@pytest.mark.parametrize("w", [56, 28])
def test_attention_view_peaked_softmax(ops, w):
    """Logits of a few tens: each query's maximum sits in one of 16-32 key blocks, so O and the row sum are rescaled
    by a running maximum that changes across blocks."""
    Fr, H, heads = 1, 32, 2
    qkv = _rand((Fr, H, 6, w, 3 * heads * 64), 7, 3.0)
    out = ops.attention_view(qkv, heads, True, NEIGH)
    torch.cuda.synchronize()
    _check(out, _view_ref(qkv, heads, True), f"attention_view peaked w={w}", 3e-2)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [64, 80])
@pytest.mark.parametrize("Nq", [300, 1792])
def test_attention_text_77_keys(ops, d, Nq):
    b, heads, Nk = 2, 2, 77
    C = heads * d
    q = _rand((b, Nq, C), 30 + d)
    kv = _rand((b, Nk, 2 * C), 31 + d)
    out = ops.attention_text(q, kv, heads)
    torch.cuda.synchronize()
    _check(out, _mha(q.float(), kv.float()[..., :C], kv.float()[..., C:], heads), f"attention_text Nq={Nq} d={d}")


# ------------------------------------------------------------------------------------------------ SASS
def _functions(sass, kernel):
    out = {}
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = chunk.split("\n", 1)
        if kernel in name:
            out[name.strip()] = [m.group(1).strip() for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", body)]
    return out


def test_attn_fa_sass(tmp_path):
    """Every instantiation: ptxas reports no serialised wgmma (C7515/C7516/C7518) and no spills, the SASS has no local
    memory access, and the main loop issues S of the next block and all N / 16 P V steps of the current one as one
    unbroken run of HGMMAs ahead of its wait."""
    nvcc = Path(build.NVCC)
    cuobjdump = nvcc.with_name("cuobjdump")
    if not nvcc.exists() or not cuobjdump.exists():
        pytest.skip(f"no nvcc / cuobjdump at {nvcc.parent}")
    obj = tmp_path / "attn_fa.o"
    r = subprocess.run([str(nvcc), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(build.CSRC / "attn_fa.cu"), "-o", str(obj)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for code in ("C7515", "C7516", "C7518"):
        assert code not in r.stderr, r.stderr
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert spills and all(a == "0" and b == "0" for a, b in spills), r.stderr
    sass = subprocess.run([str(cuobjdump), "-sass", str(obj)], capture_output=True, text=True, check=True).stdout
    funcs = _functions(sass, "attn_fa_kernel")
    want = {(d, n) for d in (64, 80) for n in WIDTHS}
    got = {}
    for name, ins in funcs.items():
        m = re.search(r"attn_fa_kernelILi(\d+)ELi(\d+)E", name)
        assert m, name
        got[(int(m.group(1)), int(m.group(2)))] = ins
    assert set(got) == want
    for (d, n), ins in got.items():
        assert not any(re.match(r"(LDL|STL)\b", i) for i in ins), f"d={d} N={n}: local memory"
        seq = [i for i in ins if "HGMMA" in i or i.startswith("WARPGROUP.")]
        s_steps = 4 + (d == 80)
        pv_steps = (n // 16) * (2 if d == 80 else 1)
        loop_run = ["HGMMA"] * (s_steps + pv_steps) + ["WARPGROUP.DEPBAR.LE gsb0, 0x0"]
        flat = ["HGMMA" if "HGMMA" in i else i for i in seq]
        found = any(flat[i:i + len(loop_run)] == loop_run and (i == 0 or flat[i - 1] != "HGMMA") for i in range(len(flat)))
        assert found, f"d={d} N={n}: no run of {s_steps} + {pv_steps} HGMMAs ahead of a wait: {flat}"
