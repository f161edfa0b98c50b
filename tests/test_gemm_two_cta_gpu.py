"""GPU parity of the wgmma GEMM / implicit-conv kernels where the two-CTA-per-SM kernel's shallow shared-memory ring
matters: reductions with fewer k-blocks than ring stages and long ones, every column tile width (BN = 160 / 128 / 64 / 32
with 3 / 3 / 4 / 5 stages), every epilogue at the level-0 row count and at long reductions, 3x3 / 3x1 taps at the
network's channel counts. Same torch fp32 references and tolerances as test_gemm_gpu.py. The level-0 epilogues at
K = 320 are the shapes pn_gemm runs on the persistent kernel (gemm_ws.cu); every other case runs on gemm_tc_kernel, and
the epilogue cases check which kernel ran."""
import pytest
import torch
import torch.nn.functional as F

from gemm_cases import _check, _rand, _rand_dev, check_case, epilogue_case, kernels_of
from test_gemm_gpu import ops  # noqa: F401  (the module-scoped NativeOps fixture)

pytestmark = pytest.mark.gpu

M0 = 172032          # level-0 rows of the benchmarked ε-evaluation: 16 frames x 32 x 336


def _epilogue(ops, M, K, kind, kernel):
    call, ref, tol = epilogue_case(ops, kind, M, K, seed=70)
    got, ran = kernels_of(lambda: call(M))
    assert ran and all(kernel in k for k in ran), ran
    check_case(kind, got, ref, tol, name=f"{kind} {M}x{K}")


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
    _epilogue(ops, M0, K, kind, "gemm_ws_kernel" if K == 320 else "gemm_tc_kernel")


# 89 and 90 k-blocks: reductions as long as the level-1 3x3 convs, with a partial last k-block tap in the first case. A
# folded-LayerNorm consumer is left out: the host allows at most 64 partial sums per row, i.e. K <= 5,120.
@pytest.mark.parametrize("kind", ["f32_res_res2", "bf16_res_f32", "bf16_res_bf16", "ln_stats", "geglu", "rowvec"])
@pytest.mark.parametrize("K", [5696, 5760])
def test_long_reduction_epilogues(ops, K, kind):
    _epilogue(ops, 3000, K, kind, "gemm_tc_kernel")


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
