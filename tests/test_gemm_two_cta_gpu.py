"""GPU parity of the two-CTA-per-SM wgmma GEMM / implicit-conv kernel where its shallow shared-memory ring matters:
reductions with fewer k-blocks than ring stages and long ones, every column tile width (BN = 160 / 128 / 64 / 32 with
3 / 3 / 4 / 5 stages), every epilogue at the level-0 row count and at long reductions, 3x3 / 3x1 taps at the network's
channel counts. Same torch fp32 references and tolerances as test_gemm_gpu.py."""
import pytest
import torch
import torch.nn.functional as F

from panacea_b200.ops import geglu_pack
from test_gemm_gpu import _check, _rand, ops  # noqa: F401  (ops is the module-scoped NativeOps fixture)

pytestmark = pytest.mark.gpu

M0 = 172032          # level-0 rows of the benchmarked ε-evaluation: 16 frames x 32 x 336


def _rand_dev(shape, seed, scale=1.0, dtype=torch.bfloat16):
    """_rand drawn on the device: the level-0 operands have 10^8 elements."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(dtype)


@pytest.mark.parametrize("N", [320, 384, 64, 8])                   # BN = 160, 128, 64, 32
# 1..5 k-blocks: fewer than, as many as, more than the stages; 90 k-blocks: a long level-1 conv reduction
@pytest.mark.parametrize("K", [64, 128, 192, 256, 320, 5760])
def test_reduction_length_every_tile_width(ops, K, N):
    M = 1000                                                       # a partial last row tile
    a = _rand((M, K), 60)
    w = _rand((N, K), 61, K ** -0.5)
    bias = _rand((N,), 62, dtype=torch.float32)
    out = ops.gemm(a, w, bias=bias)
    torch.cuda.synchronize()
    _check(out, a.float() @ w.float().t() + bias, name=f"gemm {M}x{N}x{K}")


@pytest.mark.parametrize("kind", ["f32_res_res2", "bf16_res_f32", "bf16_res_bf16", "ln_stats", "ln_fold", "geglu", "rowvec"])
@pytest.mark.parametrize("K", [320, 1280])
def test_level0_epilogues(ops, K, kind):
    _epilogue_case(ops, M0, K, kind)


# 89 and 90 k-blocks: reductions as long as the level-1 3x3 convs, with a partial last k-block tap in the first case. A
# folded-LayerNorm consumer is left out: the host allows at most 64 partial sums per row, i.e. K <= 5,120.
@pytest.mark.parametrize("kind", ["f32_res_res2", "bf16_res_f32", "bf16_res_bf16", "ln_stats", "geglu", "rowvec"])
@pytest.mark.parametrize("K", [5696, 5760])
def test_long_reduction_epilogues(ops, K, kind):
    _epilogue_case(ops, 3000, K, kind)


def _epilogue_case(ops, M, K, kind):
    a = _rand_dev((M, K), 70)
    if kind == "geglu":
        N = 2560
        w = _rand_dev((N, K), 71, K ** -0.5)
        b = _rand_dev((N,), 72, dtype=torch.float32)
        out = ops.gemm(a, geglu_pack(w), bias=geglu_pack(b), geglu=True, out_dtype=torch.bfloat16)
        torch.cuda.synchronize()
        y = a.float() @ w.float().t() + b
        _check(out, y[:, :N // 2] * F.gelu(y[:, N // 2:]), tol=1e-2, name="geglu")
        return
    if kind in ("ln_stats", "ln_fold"):
        from panacea_b200.engine import Engine
        C = min(K, 1280)                # token-stream width: 320 at level 0, 1280 at level 2
        wo = _rand_dev((C, K), 73, K ** -0.5)
        y0 = _rand_dev((M, C), 74, 2.0) + 0.7
        y, st = ops.gemm(a, wo, residual=y0, out_dtype=torch.bfloat16, ln_stats_out=True)
        torch.cuda.synchronize()
        yf = y.float()
        if kind == "ln_stats":
            _check(y, a.float() @ wo.float().t() + y0.float(), tol=1e-2, name="ln producer output")
            torch.testing.assert_close(st[..., 0].sum(1), yf.sum(1), rtol=5e-3, atol=0.5)
            torch.testing.assert_close(st[..., 1].sum(1), (yf * yf).sum(1), rtol=5e-3, atol=0.5)
            return
        gamma = _rand_dev((C,), 75, 0.2, dtype=torch.float32) + 1.0
        beta = _rand_dev((C,), 76, 0.2, dtype=torch.float32)
        wq = _rand_dev((960, C), 77, C ** -0.5, dtype=torch.float32)
        wp, s, t = Engine._ln_fold_pack(wq, None, gamma, beta)
        out = ops.gemm(y, wp, bias=t, out_dtype=torch.bfloat16, ln=(st, s, 1e-5))
        torch.cuda.synchronize()
        _check(out, F.layer_norm(yf, (C,), gamma, beta, 1e-5) @ wq.t(), tol=1.5e-2, name="LN fold -> linear")
        return
    N = 320
    w = _rand_dev((N, K), 78, K ** -0.5)
    bias = _rand_dev((N,), 79, dtype=torch.float32)
    ref = a.float() @ w.float().t() + bias
    if kind == "f32_res_res2":
        r1 = _rand_dev((M, N), 80, dtype=torch.float32)
        r2 = _rand_dev((M, N), 81, dtype=torch.float32)
        out = ops.gemm(a, w, bias=bias, residual=r1, residual2=r2)
        ref += r1 + r2
        tol = 2e-3
    elif kind == "bf16_res_f32":
        r1 = _rand_dev((M, N), 82, dtype=torch.float32)
        out = ops.gemm(a, w, bias=bias, residual=r1, out_dtype=torch.bfloat16)
        ref += r1
        tol = 1e-2
    elif kind == "bf16_res_bf16":
        r1 = _rand_dev((M, N), 83)
        ref += r1.float()
        out = ops.gemm(a, w, bias=bias, residual=r1, out=r1, out_dtype=torch.bfloat16)      # in place, like the token stream
        tol = 1e-2
    else:
        G = 16
        rv = _rand_dev((G, N), 84, dtype=torch.float32)
        rpg = M // (2 * G)
        out = ops.gemm(a, w, bias=bias, rowvec=rv, rows_per_group=rpg, n_groups=G)
        ref += rv[(torch.arange(M, device="cuda") // rpg) % G]
        tol = 2e-3
    torch.cuda.synchronize()
    _check(out, ref, tol=tol, name=kind)


@pytest.mark.parametrize("NB,H,W,C,N", [(16, 32, 336, 64, 320),      # UNet/ControlNet stem (input channels padded to 64)
                                        (16, 32, 336, 320, 8),       # out head (output channels padded to 8): BN = 32
                                        (4, 16, 168, 128, 384),      # BN = 128
                                        (16, 4, 42, 1280, 1280)])    # level-3 conv: K = 11,520
def test_conv3x3_network_shapes(ops, NB, H, W, C, N):
    x = _rand_dev((NB, H, W, C), 90)
    w = _rand_dev((N, C, 3, 3), 91, (9 * C) ** -0.5)
    wp = w.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    bias = _rand_dev((N,), 92, dtype=torch.float32)
    out = ops.gemm(x, wp, bias=bias, taps=(3, 3))
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1).permute(0, 2, 3, 1)
    _check(out.reshape(NB, H, W, N), ref, name=f"conv3x3 {NB}x{H}x{W}x{C}->{N}")


@pytest.mark.parametrize("b,T,P,C", [(2, 8, 672, 640), (2, 8, 168, 1280)])     # levels 1 and 2: K = 1,920 and 3,840
def test_temporal_conv_network_shapes(ops, b, T, P, C):
    x = _rand_dev((b, T, P, C), 93)
    w = _rand_dev((C, C, 3), 94, (3 * C) ** -0.5)
    wp = w.permute(0, 2, 1).reshape(C, 3 * C).contiguous()
    res = _rand_dev((b, T, P, C), 95, dtype=torch.float32)
    out = ops.gemm(x, wp, taps=(3, 1), residual=res)
    torch.cuda.synchronize()
    xin = x.float().permute(0, 2, 3, 1).reshape(b * P, C, T)
    ref = F.conv1d(xin, w.float(), padding=1).reshape(b, P, C, T).permute(0, 3, 1, 2) + res
    _check(out.reshape(b, T, P, C), ref, name="temporal conv")
