"""GPU parity of the persistent weight-stationary GEMM (gemm_ws.cu), which pn_gemm runs for 1x1 GEMMs over at least
512 dense rows with C <= 320 and N % 160 == 0: partial and few row tiles, column-tile counts that leave SMs idle, every
epilogue, two calls on two streams. Each result is checked against torch fp32 math with test_gemm_gpu.py's tolerances,
against a rerun bit for bit, and against gemm_tc_kernel bit for bit: rows are independent, so the first 500 rows of a
call (below the row threshold, hence gemm_tc_kernel) must equal the same rows of the full call."""
import pytest
import torch
import torch.nn.functional as F

from panacea_b200.ops import geglu_pack
from test_gemm_gpu import _check, ops  # noqa: F401  (ops is the module-scoped NativeOps fixture)

pytestmark = pytest.mark.gpu

SMALL = 500          # below pn_gemm's row threshold for the persistent kernel


def _rand_dev(shape, seed, scale=1.0, dtype=torch.bfloat16):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(dtype)


def _run(ops, kind, M, K, seed):
    """(call, fp32 reference, tolerance) for one epilogue; call(rows) runs the GEMM on the first `rows` rows and returns
    every output it wrote (fresh tensors, so an in-place residual starts from the same values each time)."""
    a = _rand_dev((M, K), seed)
    if kind == "geglu":
        N = 2560                                    # 16 column tiles: 128 of 132 SMs busy
        w = _rand_dev((N, K), seed + 1, K ** -0.5)
        b = _rand_dev((N,), seed + 2, dtype=torch.float32)
        y = a.float() @ w.float().t() + b
        return (lambda m: (ops.gemm(a[:m], geglu_pack(w), bias=geglu_pack(b), geglu=True, out_dtype=torch.bfloat16),),
                y[:, :N // 2] * F.gelu(y[:, N // 2:]), 1e-2)
    if kind in ("ln_stats", "ln_fold"):
        from panacea_b200.engine import Engine
        C = 320
        wo = _rand_dev((C, K), seed + 3, K ** -0.5)
        y0 = _rand_dev((M, C), seed + 4, 2.0) + 0.7
        if kind == "ln_stats":
            return (lambda m: ops.gemm(a[:m], wo, residual=y0[:m].clone(), out_dtype=torch.bfloat16, ln_stats_out=True),
                    a.float() @ wo.float().t() + y0.float(), 1e-2)
        y, st = ops.gemm(a, wo, residual=y0.clone(), out_dtype=torch.bfloat16, ln_stats_out=True)
        gamma = _rand_dev((C,), seed + 5, 0.2, dtype=torch.float32) + 1.0
        beta = _rand_dev((C,), seed + 6, 0.2, dtype=torch.float32)
        wq = _rand_dev((960, C), seed + 7, C ** -0.5, dtype=torch.float32)     # qkv: 6 column tiles
        wp, s, t = Engine._ln_fold_pack(wq, None, gamma, beta)
        return (lambda m: (ops.gemm(y[:m], wp, bias=t, out_dtype=torch.bfloat16, ln=(st[:m], s, 1e-5)),),
                F.layer_norm(y.float(), (C,), gamma, beta, 1e-5) @ wq.t(), 1.5e-2)
    N = 320
    w = _rand_dev((N, K), seed + 8, K ** -0.5)
    bias = _rand_dev((N,), seed + 9, dtype=torch.float32)
    ref = a.float() @ w.float().t() + bias
    if kind == "f32_res_res2":
        r1 = _rand_dev((M, N), seed + 10, dtype=torch.float32)
        r2 = _rand_dev((M, N), seed + 11, dtype=torch.float32)
        return lambda m: (ops.gemm(a[:m], w, bias=bias, residual=r1[:m], residual2=r2[:m]),), ref + r1 + r2, 2e-3
    if kind == "f32_res_inplace":
        r1 = _rand_dev((M, N), seed + 12, dtype=torch.float32)

        def call(m):
            r = r1[:m].clone()
            return (ops.gemm(a[:m], w, bias=bias, residual=r, out=r),)
        return call, ref + r1, 2e-3
    if kind == "bf16_res_f32":
        r1 = _rand_dev((M, N), seed + 13, dtype=torch.float32)
        return lambda m: (ops.gemm(a[:m], w, bias=bias, residual=r1[:m], out_dtype=torch.bfloat16),), ref + r1, 1e-2
    if kind == "bf16_res_bf16":
        r1 = _rand_dev((M, N), seed + 14)

        def call(m):
            r = r1[:m].clone()
            return (ops.gemm(a[:m], w, bias=bias, residual=r, out=r, out_dtype=torch.bfloat16),)
        return call, ref + r1.float(), 1e-2
    assert kind == "rowvec"
    G = 16
    rv = _rand_dev((G, N), seed + 15, dtype=torch.float32)
    rpg = 37
    rows = torch.arange(M, device="cuda")
    return (lambda m: (ops.gemm(a[:m], w, bias=bias, rowvec=rv, rows_per_group=rpg, n_groups=G),),
            ref + rv[(rows // rpg) % G], 2e-3)


def _kernels_of(fn):
    """fn()'s result and the names of the GEMM kernels it launched"""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, {e.name for e in prof.events() if "gemm" in e.name}


KINDS = ["f32_res_res2", "f32_res_inplace", "bf16_res_f32", "bf16_res_bf16", "ln_stats", "ln_fold", "geglu", "rowvec"]


# 520 rows: 9 row tiles, fewer than the CTAs a full grid would have, the last one 8 rows deep; 8,447 rows: 132 row tiles,
# the last one partial; K = 64 and 192: one and three k-blocks
@pytest.mark.parametrize("M,K", [(520, 320), (8447, 320), (8447, 64), (3001, 192)])
@pytest.mark.parametrize("kind", KINDS)
def test_matches_torch_rerun_and_gemm_tc(ops, kind, M, K):
    call, ref, tol = _run(ops, kind, M, K, seed=100)
    got, ran = _kernels_of(lambda: call(M))
    again = call(M)
    small, ran_small = _kernels_of(lambda: call(SMALL))
    torch.cuda.synchronize()
    # the comparison with gemm_tc_kernel below means something only if each call ran the kernel it is meant to
    assert any("gemm_ws_kernel" in k for k in ran) and not any("gemm_tc_kernel" in k for k in ran), ran
    assert any("gemm_tc_kernel" in k for k in ran_small) and not any("gemm_ws_kernel" in k for k in ran_small), ran_small
    _check(got[0], ref, tol=tol, name=f"{kind} {M}x{K}")
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
