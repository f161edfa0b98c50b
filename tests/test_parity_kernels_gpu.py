"""GPU tests of the parity-mode building blocks (panacea_b200.ops.ParityOps) against float64 torch math:
split-bf16 operands through the wgmma GEMM / implicit conv, the fp32 attention kernels (head_dim 64 and 80), the
exact-erf GEGLU pass and the split stores of the normalisation kernels. Tolerances are fp32-class (1e-5 .. 1e-4)."""
import pytest
import torch
import torch.nn.functional as F

from op_check import _decode

pytestmark = pytest.mark.gpu

NEIGH = ((5, 1), (0, 2), (1, 3), (2, 4), (3, 5), (4,))


@pytest.fixture(scope="module")
def ops():
    from panacea_b200.ops import ParityOps
    return ParityOps()


def _rand(shape, seed, scale=1.0, shift=0.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale + shift).cuda()


def _rel(got, ref):
    return ((got.double() - ref.double()).norm() / ref.double().norm()).item()


@pytest.mark.parametrize("M,K,N", [(300, 320, 960), (4096, 1280, 320), (172032 // 8, 320, 2560), (77, 1024, 640)])
def test_split3_gemm_is_fp32_class(ops, M, K, N):
    from panacea_b200.ops import split3
    a = _rand((M, K), 1)
    w = _rand((N, K), 2, K ** -0.5)
    bias = _rand((N,), 3)
    res = _rand((M, N), 4)
    a_op = ops.cast_operand(a)
    assert a_op.shape == (M, 3 * K) and _rel(_decode(a_op, "split3"), a) < 1e-5
    y = ops.gemm(a_op, split3(w), bias=bias, residual=res)
    torch.cuda.synchronize()
    ref = a.double() @ w.double().t() + bias.double() + res.double()
    assert _rel(y, ref) < 2e-5, _rel(y, ref)


@pytest.mark.parametrize("NB,H,W,C,N,taps", [(2, 16, 48, 64, 160, (3, 3)), (4, 32, 56, 320, 320, (3, 3)), (2, 8, 96, 128, 128, (3, 1))])
def test_split3_implicit_conv_is_fp32_class(ops, NB, H, W, C, N, taps):
    from panacea_b200.ops import split3
    th, tw = taps
    x = _rand((NB, H, W, C), 5)
    w = _rand((N, th * tw * C), 6, (th * tw * C) ** -0.5)
    y = ops.gemm(ops.cast_operand(x), split3(w, th * tw), taps=taps)
    torch.cuda.synchronize()
    wk = w.double().reshape(N, th, tw, C).permute(0, 3, 1, 2)
    ref = F.conv2d(x.double().permute(0, 3, 1, 2), wk, padding=(th // 2, tw // 2)).permute(0, 2, 3, 1)
    assert _rel(y.reshape(ref.shape), ref) < 2e-5


def _mha64(q, k, v, heads):
    B, Nq, C = q.shape
    d = C // heads
    qh = q.double().reshape(B, Nq, heads, d).transpose(1, 2)
    kh = k.double().reshape(B, -1, heads, d).transpose(1, 2)
    vh = v.double().reshape(B, -1, heads, d).transpose(1, 2)
    s = (qh @ kh.transpose(-1, -2)) * (d ** -0.5)
    return (s.softmax(-1) @ vh).transpose(1, 2).reshape(B, Nq, C)


@pytest.mark.parametrize("d", [64, 80])
@pytest.mark.parametrize("cross", [False, True])
def test_attention_view_f32(ops, d, cross):
    Fr, H, V, w, heads = 2, 8, 6, 14, 2
    C = heads * d
    qkv = _rand((Fr, H, V, w, 3 * C), 7)
    out = _decode(ops.attention_view(qkv, heads, cross, NEIGH), "split3")
    torch.cuda.synchronize()
    q, k, v = qkv.split(C, dim=-1)
    for i in range(V):
        nb = NEIGH[i] if cross else (i,)
        ki = torch.cat([k[:, :, j] for j in nb], dim=2).reshape(Fr, -1, C)
        vi = torch.cat([v[:, :, j] for j in nb], dim=2).reshape(Fr, -1, C)
        ref = _mha64(q[:, :, i].reshape(Fr, H * w, C), ki, vi, heads).reshape(Fr, H, w, C)
        assert _rel(out[:, :, i], ref) < 1e-5


@pytest.mark.parametrize("d", [64, 80])
def test_attention_text_and_temporal_f32(ops, d):
    heads = 3
    C = heads * d
    q = _rand((2, 500, C), 8)
    kv = _rand((2, 77, 2 * C), 9)
    out = _decode(ops.attention_text(q, kv, heads), "split3")
    ref = _mha64(q, kv[..., :C], kv[..., C:], heads)
    assert _rel(out, ref) < 1e-5
    for T in (1, 4, 8, 16):
        b, P = 2, 37
        qkv = _rand((b, T, P, 3 * C), 10 + T)
        o = _decode(ops.attention_temporal(qkv, heads), "split3")
        qq, kk, vv = qkv.split(C, dim=-1)
        seq = lambda z: z.permute(0, 2, 1, 3).reshape(b * P, T, C)
        r = _mha64(seq(qq), seq(kk), seq(vv), heads).reshape(b, P, T, C).permute(0, 2, 1, 3)
        assert _rel(o, r) < 1e-5


def test_attention_entry_points_refuse_other_operand_modes(ops):
    """each attention entry point serves bf16, split3 and fp32; any other operand_mode, the weight form included, is
    refused with a message that names it"""
    import ctypes
    from panacea_b200.ops import OP_SPLIT3_B, _attn_args, _stream
    qkv = torch.zeros(1, 8, 3 * 64, device="cuda")
    out = torch.empty(1, 8, 3 * 64, device="cuda", dtype=torch.bfloat16)
    p, o, lib = qkv.data_ptr(), out.data_ptr(), ops.lib
    for mode in (OP_SPLIT3_B, 7):
        a = _attn_args(p, p, p, o, q_ld=192, kv_ld=192, F=1, H=1, V=1, W=8, Hk=1, Vk=1, Wk=8, heads=1, head_dim=64, views=[[0]])
        for call in (lambda: lib.pn_attention(ctypes.byref(a), mode, _stream()),
                     lambda: lib.pn_attention_temporal(p, p, p, o, 1, 8, 1, 1, 64, 192, 64, 0.125, mode, _stream()),
                     lambda: lib.pn_attention_causal(p, p, p, o, 1, 8, 1, 64, 192, 64, 0.125, mode, _stream())):
            assert call() == -1 and f"operand_mode {mode}".encode() in lib.pn_last_error()
    torch.cuda.synchronize()


# the operand modes each producer entry point accepts (include/panacea_b200.h pn_operand_mode)
PRODUCER_MODES = {
    "pn_groupnorm_silu": (0, 1, 2), "pn_groupnorm_pixel_silu": (0, 1, 2), "pn_layernorm": (0, 1, 2),
    "pn_upsample2x": (0, 1, 2), "pn_geglu_operand": (0, 1, 2), "pn_gelu_operand": (0, 1, 2),
    "pn_cast_operand": (0, 1, 3), "pn_im2col3x3_s2": (0, 1), "pn_softmax_rows_operand": (0, 1),
    "pn_attention": (0, 1, 2), "pn_attention_temporal": (0, 1, 2), "pn_attention_causal": (0, 1, 2),
}


@pytest.mark.parametrize("mode", [0, 1, 2, 3, 7])
@pytest.mark.parametrize("entry", sorted(PRODUCER_MODES))
def test_producers_accept_exactly_their_operand_modes(ops, entry, mode):
    """every producer entry point runs in the operand modes it accepts and refuses any other one, writing nothing, with a
    message that names it. The calls work on zero inputs of at most 64 rows of 64 channels, and the output buffer holds
    the widest layout, [64, 3 * 64] bf16, so every call stays in bounds whatever mode it runs in."""
    import ctypes
    from panacea_b200.ops import _attn_args, _stream
    lib = ops.lib
    x = torch.zeros(64 * 128, device="cuda")
    y = torch.full((64, 3 * 64), 7.0, device="cuda", dtype=torch.bfloat16)
    g, b = torch.ones(64, device="cuda"), torch.zeros(64, device="cuda")
    ws = torch.zeros(lib.pn_groupnorm_workspace_floats(2, 32, 64), device="cuda")
    X, Y, G, B, s = x.data_ptr(), y.data_ptr(), g.data_ptr(), b.data_ptr(), _stream()
    a = _attn_args(X, X, X, Y, q_ld=192, kv_ld=192, F=1, H=1, V=1, W=8, Hk=1, Vk=1, Wk=8, heads=1, head_dim=64, views=[[0]])
    calls = {
        "pn_groupnorm_silu": lambda: lib.pn_groupnorm_silu(X, G, B, Y, None, ws.data_ptr(), 2, 32, 64, 1e-5, 1, mode, s),
        "pn_groupnorm_pixel_silu": lambda: lib.pn_groupnorm_pixel_silu(X, G, B, Y, 1, 2, 32, 64, 1e-5, 1, mode, s),
        "pn_layernorm": lambda: lib.pn_layernorm(X, 0, G, B, Y, 64, 64, 1e-5, mode, s),
        "pn_upsample2x": lambda: lib.pn_upsample2x(X, Y, 1, 4, 4, 64, mode, s),
        "pn_geglu_operand": lambda: lib.pn_geglu_operand(X, Y, 64, 64, mode, s),
        "pn_gelu_operand": lambda: lib.pn_gelu_operand(X, Y, 64, 64, mode, s),
        "pn_cast_operand": lambda: lib.pn_cast_operand(X, Y, 64, 64, mode, s),
        "pn_im2col3x3_s2": lambda: lib.pn_im2col3x3_s2(X, Y, 1, 4, 4, 64, 1, mode, s),
        "pn_softmax_rows_operand": lambda: lib.pn_softmax_rows_operand(X, Y, 64, 64, 64, 3 * 64, 1.0, mode, s),
        "pn_attention": lambda: lib.pn_attention(ctypes.byref(a), mode, s),
        "pn_attention_temporal": lambda: lib.pn_attention_temporal(X, X, X, Y, 1, 8, 1, 1, 64, 192, 64, 0.125, mode, s),
        "pn_attention_causal": lambda: lib.pn_attention_causal(X, X, X, Y, 1, 8, 1, 64, 192, 64, 0.125, mode, s),
    }
    rc = calls[entry]()
    torch.cuda.synchronize()
    if mode in PRODUCER_MODES[entry]:
        assert rc == 0, lib.pn_last_error()
    else:
        assert rc == -1 and f"{entry}: operand_mode {mode}".encode() in lib.pn_last_error(), lib.pn_last_error()
        assert bool((y == 7.0).all()), "a refused call wrote its output"


def test_geglu_pass_uses_the_exact_erf(ops):
    from panacea_b200.ops import geglu_pack, split3
    M, K, inner = 1000, 320, 1280
    a = _rand((M, K), 20)
    w = _rand((2 * inner, K), 21, K ** -0.5)
    b = _rand((2 * inner,), 22)
    y = _decode(ops.gemm(ops.cast_operand(a), split3(geglu_pack(w)), bias=geglu_pack(b).contiguous(), geglu=True), "split3")
    torch.cuda.synchronize()
    h = a.double() @ w.double().t() + b.double()
    ref = h[:, :inner] * F.gelu(h[:, inner:])
    assert _rel(y, ref) < 2e-5


def test_norm_kernels_store_split_operands(ops):
    x = _rand((3, 700, 320), 30, 2.0, 0.5)
    g = _rand((320,), 31, 0.1, 1.0); b = _rand((320,), 32, 0.1)
    y, raw = ops.groupnorm(x, g, b, 1e-5, True, want_raw=True)
    ref = F.silu(F.group_norm(x.double().permute(0, 2, 1), 32, g.double(), b.double(), 1e-5)).permute(0, 2, 1)
    assert _rel(_decode(y, "split3"), ref) < 1e-5 and _rel(_decode(raw, "split3"), x) < 1e-5
    yf = ops.groupnorm(x, g, b, 1e-5, True, out_f32=True)
    assert yf.dtype == torch.float32 and _rel(yf, ref) < 1e-5
    xp = _rand((2, 8, 50, 640), 33, 1.5, -0.3)
    gp = _rand((640,), 34, 0.1, 1.0); bp = _rand((640,), 35, 0.1)
    yp = _decode(ops.groupnorm_pixel(xp, gp, bp, 1e-5, True), "split3")
    z = xp.double().permute(0, 2, 3, 1).reshape(100, 640, 8)
    rp = F.silu(F.group_norm(z, 32, gp.double(), bp.double(), 1e-5)).reshape(2, 50, 640, 8).permute(0, 3, 1, 2)
    assert _rel(yp, rp) < 1e-5
    xl = _rand((999, 1280), 36, 3.0, 1.0)
    gl = _rand((1280,), 37, 0.1, 1.0); bl = _rand((1280,), 38, 0.1)
    yl = _decode(ops.layernorm(xl, gl, bl), "split3")
    assert _rel(yl, F.layer_norm(xl.double(), (1280,), gl.double(), bl.double(), 1e-5)) < 1e-5
    xu = _rand((2, 4, 6, 64), 39)
    assert _rel(_decode(ops.upsample2x(xu), "split3"), xu.repeat_interleave(2, 1).repeat_interleave(2, 2)) < 1e-5
    cols, (Fr, Ho, Wo) = ops.im2col_s2(xu)
    assert cols.shape == (2 * 2 * 3, 9 * 3 * 64)


def test_groupnorm_two_phase_form_matches_the_fused_one():
    """PN_GN_TWO_PHASE=1 (devices that cannot hold the cooperative grid) must give the same bits as the fused launch."""
    import os, subprocess, sys
    code = ("import torch;from panacea_b200.ops import NativeOps;o=NativeOps();g=torch.Generator().manual_seed(0);"
            "x=torch.randn(4,3000,640,generator=g).cuda();w=torch.ones(640).cuda();b=torch.zeros(640).cuda();"
            "y=o.groupnorm(x,w,b,1e-5,True);torch.cuda.synchronize();print(float(y.float().double().sum()),float(y.float().abs().double().sum()))")
    outs = []
    for flag in ("0", "1"):
        env = dict(os.environ, PN_GN_TWO_PHASE=flag)
        outs.append(subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, check=True,
                                   cwd=str(__import__("pathlib").Path(__file__).resolve().parent.parent)).stdout.strip())
    assert outs[0] == outs[1], outs
