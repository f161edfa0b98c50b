"""GPU parity of the wgmma GEMM / implicit-conv kernel against torch fp32 math on the same bf16 inputs."""
import pytest
import torch
import torch.nn.functional as F

from gemm_cases import _check, _rand
from panacea_b200.ops import geglu_pack

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from panacea_b200.ops import NativeOps
    return NativeOps()


@pytest.mark.parametrize("M,N,K", [(128, 160, 64), (256, 160, 128), (1000, 320, 320), (777, 128, 192),
                                   (4096, 2560, 320), (130, 96, 64), (154, 640, 1024), (64, 8, 64), (16, 1280, 320)])
def test_plain_gemm(ops, M, N, K):
    a = _rand((M, K), 1)
    w = _rand((N, K), 2, K ** -0.5)
    out = ops.gemm(a, w)
    torch.cuda.synchronize()
    _check(out, a.float() @ w.float().t(), name=f"gemm {M}x{N}x{K}")


def test_gemm_bias_residual_inplace(ops):
    M, N, K = 3000, 320, 640
    a = _rand((M, K), 3); w = _rand((N, K), 4, K ** -0.5)
    bias = _rand((N,), 5, dtype=torch.float32)
    res = _rand((M, N), 6, dtype=torch.float32)
    ref = a.float() @ w.float().t() + bias + res
    out = ops.gemm(a, w, bias=bias, residual=res, out=res)  # aliasing allowed
    torch.cuda.synchronize()
    _check(out, ref, name="bias+residual")


def test_gemm_bf16_out_and_rowvec(ops):
    M, N, K = 2048, 640, 320
    a = _rand((M, K), 7); w = _rand((N, K), 8, K ** -0.5)
    rv = _rand((4, N), 9, dtype=torch.float32)
    out = ops.gemm(a, w, rowvec=rv, rows_per_group=256, n_groups=4, out_dtype=torch.bfloat16)
    torch.cuda.synchronize()
    grp = (torch.arange(M, device="cuda") // 256) % 4
    ref = a.float() @ w.float().t() + rv[grp]
    _check(out, ref, tol=1e-2, name="bf16 out + rowvec")


@pytest.mark.parametrize("M,N,K", [(3000, 320, 320), (2048, 640, 640), (1500, 1280, 1280), (172032 // 4, 320, 1280), (130, 320, 320)])
def test_gemm_bf16_token_stream_residual(ops, M, N, K):
    """bf16 output with a bf16 residual updated in place (the transformer blocks' token stream), in place and not,
    for K <= 640 and larger K."""
    a = _rand((M, K), 13); w = _rand((N, K), 14, K ** -0.5)
    bias = _rand((N,), 15, dtype=torch.float32)
    y = _rand((M, N), 16)
    ref = a.float() @ w.float().t() + bias + y.float()
    out = ops.gemm(a, w, bias=bias, residual=y, out=y, out_dtype=torch.bfloat16)
    torch.cuda.synchronize()
    assert out.data_ptr() == y.data_ptr()
    _check(out, ref, tol=1e-2, name="bf16 residual in place")
    y2 = _rand((M, N), 17)
    out2 = ops.gemm(a, w, residual=y2, out_dtype=torch.bfloat16)        # not in place
    torch.cuda.synchronize()
    _check(out2, a.float() @ w.float().t() + y2.float(), tol=1e-2, name="bf16 residual")


@pytest.mark.parametrize("M,C", [(3000, 320), (2500, 640), (172032 // 8, 320), (700, 128), (130, 512)])
def test_gemm_layernorm_fold(ops, M, C):
    """LayerNorm folded into the GEMMs around the bf16 token stream: (i) a producer (bf16 out + bf16 residual) emits
    per-row partial sums of the values it rounds and stores; (ii) a consumer (bf16 out) takes the un-normalised stream, W diag(gamma), the column sums and W beta, and must equal Linear(LayerNorm(stream))."""
    from panacea_b200.engine import Engine
    a = _rand((M, C), 30); wo = _rand((C, C), 31, C ** -0.5)
    y0 = _rand((M, C), 32, 2.0) + 0.7
    y, st = ops.gemm(a, wo, residual=y0.clone(), out_dtype=torch.bfloat16, ln_stats_out=True)
    torch.cuda.synchronize()
    assert st.shape == (M, 2 * (C // (160 if C % 160 == 0 else 128)), 2)
    yf = y.float()
    # the sums are taken from the fp32 values before their bf16 rounding: equal to the rounded rows' sums to ~2^-9 / sqrt(C)
    torch.testing.assert_close(st[..., 0].sum(1), yf.sum(1), rtol=5e-3, atol=0.5)
    torch.testing.assert_close(st[..., 1].sum(1), (yf * yf).sum(1), rtol=5e-3, atol=0.5)
    gamma = _rand((C,), 33, 0.2, dtype=torch.float32) + 1.0
    beta = _rand((C,), 34, 0.2, dtype=torch.float32)
    ln = F.layer_norm(yf, (C,), gamma, beta, 1e-5)
    # consumer 1: q|k|v projection, no bias
    wq = _rand((3 * C, C), 35, C ** -0.5, dtype=torch.float32)
    wp, s, t = Engine._ln_fold_pack(wq, None, gamma, beta)
    out = ops.gemm(y, wp, bias=t, out_dtype=torch.bfloat16, ln=(st, s, 1e-5))
    torch.cuda.synchronize()
    _check(out, ln @ wq.t(), tol=1.5e-2, name="LN fold -> linear")


def test_gemm_geglu(ops):
    M, C = 1500, 320
    a = _rand((M, C), 10)
    w = _rand((8 * C, C), 11, C ** -0.5)       # reference layout: rows [0,4C) value, [4C,8C) gate
    b = _rand((8 * C,), 12, dtype=torch.float32)
    wi, bi = geglu_pack(w), geglu_pack(b)
    out = ops.gemm(a, wi, bias=bi, geglu=True, out_dtype=torch.bfloat16)
    torch.cuda.synchronize()
    y = a.float() @ w.float().t() + b
    ref = y[:, :4 * C] * F.gelu(y[:, 4 * C:])
    _check(out, ref, tol=1e-2, name="geglu")


@pytest.mark.parametrize("kind", ["fp32_res", "bf16", "geglu", "fp32_wide"])
def test_gemm_weight_stationary_schedule(ops, kind):
    """K = 320 over many waves of row tiles (8 x 148 x 128 + 333 rows): the last 128-row tile is partial, and each
    epilogue (fp32 + residual, bf16, GEGLU) spans several 160-wide column tiles (N = 480, 960, 2560)."""
    M, K = 8 * 148 * 128 + 333, 320
    a = _rand((M, K), 40)
    if kind == "geglu":
        N = 2560
        w = _rand((N, K), 41, K ** -0.5)
        b = _rand((N,), 42, dtype=torch.float32)
        out = ops.gemm(a, geglu_pack(w), bias=geglu_pack(b), geglu=True, out_dtype=torch.bfloat16)
        torch.cuda.synchronize()
        y = a.float() @ w.float().t() + b
        _check(out, y[:, :N // 2] * F.gelu(y[:, N // 2:]), tol=1e-2, name="bstat geglu")
    elif kind == "bf16":
        N = 960
        w = _rand((N, K), 43, K ** -0.5)
        out = ops.gemm(a, w, out_dtype=torch.bfloat16)
        torch.cuda.synchronize()
        _check(out, a.float() @ w.float().t(), tol=1e-2, name="bstat bf16")
    else:
        N = 960 if kind == "fp32_wide" else 480
        w = _rand((N, K), 44, K ** -0.5)
        bias = _rand((N,), 45, dtype=torch.float32)
        res = _rand((M, N), 46, dtype=torch.float32)
        ref = a.float() @ w.float().t() + bias + res
        out = ops.gemm(a, w, bias=bias, residual=res)
        torch.cuda.synchronize()
        _check(out, ref, name="bstat fp32+res")


@pytest.mark.parametrize("M,N,K", [(3000, 320, 1280), (700, 1280, 5120)])
def test_gemm_bf16_out_with_fp32_residual(ops, M, N, K):
    """Last GEMM of a transformer block (ff2 + residual) emitting the bf16 operand of proj_out directly."""
    a = _rand((M, K), 50); w = _rand((N, K), 51, K ** -0.5)
    bias = _rand((N,), 52, dtype=torch.float32)
    res = _rand((M, N), 53, dtype=torch.float32)
    out = ops.gemm(a, w, bias=bias, residual=res, out_dtype=torch.bfloat16)
    torch.cuda.synchronize()
    assert out.dtype == torch.bfloat16
    _check(out, a.float() @ w.float().t() + bias + res, tol=1e-2, name="bf16 out + fp32 residual")


def test_gemm_strided_view(ops):
    M, C = 900, 320
    qkv = _rand((M, 3 * C), 13)
    w = _rand((C, C), 14, C ** -0.5)
    out = ops.gemm(qkv[:, C:2 * C], w)
    torch.cuda.synchronize()
    _check(out, qkv[:, C:2 * C].float() @ w.float().t(), name="strided A")


@pytest.mark.parametrize("NB,H,W,C,N", [(2, 8, 24, 64, 160), (3, 4, 42, 128, 320), (2, 32, 336, 320, 320),
                                        (4, 16, 168, 64, 64), (16, 4, 42, 64, 160),
                                        # narrow images: the 128-row tile is a box of several image rows, so the taps
                                        # read across its top, bottom and side edges
                                        (1, 16, 24, 64, 160), (2, 32, 40, 128, 320), (1, 48, 16, 64, 640), (3, 16, 168, 192, 640)])
def test_conv3x3(ops, NB, H, W, C, N):
    x = _rand((NB, H, W, C), 15)
    w = _rand((N, C, 3, 3), 16, (9 * C) ** -0.5)
    wp = w.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    bias = _rand((N,), 17, dtype=torch.float32)
    out = ops.gemm(x, wp, bias=bias, taps=(3, 3))
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1).permute(0, 2, 3, 1)
    _check(out.reshape(NB, H, W, N), ref, name=f"conv3x3 {NB}x{H}x{W}x{C}->{N}")


@pytest.mark.parametrize("b,T,P,C", [(2, 8, 300, 64), (1, 8, 2688, 320), (2, 4, 128, 128)])
def test_temporal_conv(ops, b, T, P, C):
    x = _rand((b, T, P, C), 18)
    w = _rand((C, C, 3), 19, (3 * C) ** -0.5)          # Conv1d weight [Cout, Cin, k]
    wp = w.permute(0, 2, 1).reshape(C, 3 * C).contiguous()
    res = _rand((b, T, P, C), 20, dtype=torch.float32)
    out = ops.gemm(x, wp, taps=(3, 1), residual=res)
    torch.cuda.synchronize()
    xin = x.float().permute(0, 2, 3, 1).reshape(b * P, C, T)
    ref = F.conv1d(xin, w.float(), padding=1).reshape(b, P, C, T).permute(0, 3, 1, 2) + res
    _check(out.reshape(b, T, P, C), ref, name="temporal conv")


@pytest.mark.parametrize("M,N,K,G", [(2048, 320, 320, 8), (1536, 640, 64, 3), (640, 128, 128, 5)])
def test_gemm_fp32_rowvec_residual_streaming_epilogue(ops, M, N, K, G):
    """fp32 output + per-row-group vector (time-emb / pos-emb, strided rows) + in-place residual."""
    a = _rand((M, K), 30); w = _rand((N, K), 31, K ** -0.5)
    bias = _rand((N,), 32, dtype=torch.float32)
    rv_full = _rand((G, N + 64), 33, dtype=torch.float32)
    rv = rv_full[:, 32:32 + N]                               # strided rows (slice of a wider matrix)
    res = _rand((M, N), 34, dtype=torch.float32)
    rpg = M // (2 * G)
    grp = (torch.arange(M, device="cuda") // rpg) % G
    ref = a.float() @ w.float().t() + bias + rv[grp] + res
    out = ops.gemm(a, w, bias=bias, rowvec=rv, rows_per_group=rpg, n_groups=G, residual=res, out=res)
    torch.cuda.synchronize()
    _check(out, ref, name="fp32 rowvec+residual")
