"""GPU parity of the persistent weight-stationary GEMM (gemm_ws.cu), which pn_gemm runs for 1x1 GEMMs over at least
512 dense rows with C <= 320 and N % 160 == 0: partial and few row tiles, column-tile counts that leave SMs idle, every
epilogue, two calls on two streams. Each result is checked against torch fp32 math with test_gemm_gpu.py's tolerances,
against a rerun bit for bit, and against gemm_tc_kernel bit for bit: rows are independent, so the first 500 rows of a
call (below the row threshold, hence gemm_tc_kernel) must equal the same rows of the full call."""
import pytest
import torch

from gemm_cases import EPILOGUE_KINDS, _check, _rand_dev, check_case, epilogue_case, kernels_of
from test_gemm_gpu import ops  # noqa: F401  (the module-scoped NativeOps fixture)

pytestmark = pytest.mark.gpu

SMALL = 500          # below pn_gemm's row threshold for the persistent kernel


# 520 rows: 9 row tiles, fewer than the CTAs a full grid would have, the last one 8 rows deep; 8,447 rows: 132 row tiles,
# the last one partial; K = 64 and 192: one and three k-blocks
@pytest.mark.parametrize("M,K", [(520, 320), (8447, 320), (8447, 64), (3001, 192)])
@pytest.mark.parametrize("kind", EPILOGUE_KINDS)
def test_matches_torch_rerun_and_gemm_tc(ops, kind, M, K):
    call, ref, tol = epilogue_case(ops, kind, M, K, seed=100)
    got, ran = kernels_of(lambda: call(M))
    again = call(M)
    small, ran_small = kernels_of(lambda: call(SMALL))
    torch.cuda.synchronize()
    # the comparison with gemm_tc_kernel below means something only if each call ran the kernel it is meant to
    assert any("gemm_ws_kernel" in k for k in ran) and not any("gemm_tc_kernel" in k for k in ran), ran
    assert any("gemm_tc_kernel" in k for k in ran_small) and not any("gemm_ws_kernel" in k for k in ran_small), ran_small
    check_case(kind, got, ref, tol, name=f"{kind} {M}x{K}")
    for x, y in zip(got, again):
        assert torch.equal(x, y), f"{kind}: a rerun differs"
    for x, y in zip(got, small):
        assert torch.equal(x[:SMALL], y), f"{kind}: the persistent kernel and gemm_tc_kernel differ"


def test_two_streams_back_to_back(ops):
    """Two independent level-0-sized calls queued on two streams at once, the way the ControlNet and UNet branches of an
    ε-evaluation run: each must equal the same call run alone."""
    M, K, N = 43008, 320, 320
    a = [_rand_dev((M, K), 200 + i) for i in range(2)]
    w = [_rand_dev((N, K), 210 + i, K ** -0.5) for i in range(2)]
    r = [_rand_dev((M, N), 220 + i, dtype=torch.float32) for i in range(2)]
    alone = [ops.gemm(a[i], w[i], residual=r[i]) for i in range(2)]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(2)]
    outs = [None, None]
    for _ in range(3):
        for i, s in enumerate(streams):
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                outs[i] = ops.gemm(a[i], w[i], residual=r[i])
        for s in streams:
            torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        for i in range(2):
            assert torch.equal(outs[i], alone[i]), f"stream {i}: differs from the call run alone"
    _check(alone[0], a[0].float() @ w[0].float().t() + r[0], name="two streams")
