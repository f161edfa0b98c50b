"""TEST INFRASTRUCTURE: random operands, the tolerance check and the epilogue cases shared by the GEMM GPU tests
(test_gemm_gpu.py, test_gemm_two_cta_gpu.py, test_gemm_ws_gpu.py). Each epilogue kind of pn_gemm is built here once, so
the two-CTA kernel and the persistent kernel are tested with the same calls and the same torch fp32 references."""
import torch
import torch.nn.functional as F

from panacea_b200.ops import geglu_pack

# the torch references must be true fp32 (cuDNN/cuBLAS default to TF32 for conv/matmul on this GPU)
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

EPILOGUE_KINDS = ["f32_res_res2", "f32_res_inplace", "bf16_res_f32", "bf16_res_bf16", "ln_stats", "ln_fold", "geglu",
                  "rowvec"]


def _rand(shape, seed, scale=1.0, dtype=torch.bfloat16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).cuda()


def _rand_dev(shape, seed, scale=1.0, dtype=torch.bfloat16):
    """_rand drawn on the device: the level-0 operands have 10^8 elements."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(dtype)


def _check(got, ref, tol=2e-3, name=""):
    got = got.float()
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item() + 1e-6
    assert torch.isfinite(got).all(), f"{name}: non-finite output"
    assert err <= tol * scale, f"{name}: max err {err:.4e} vs scale {scale:.3e}"


def epilogue_case(ops, kind, M, K, seed):
    """(call, fp32 reference, tolerance) of one epilogue kind over M rows and reduction length K. call(rows) runs the GEMM
    on the first `rows` rows and returns every output it wrote (fresh tensors, so an in-place residual starts from the
    same values each time); the reference covers all M rows."""
    a = _rand_dev((M, K), seed)
    if kind == "geglu":
        N = 2560                                    # 16 column tiles
        w = _rand_dev((N, K), seed + 1, K ** -0.5)
        b = _rand_dev((N,), seed + 2, dtype=torch.float32)
        y = a.float() @ w.float().t() + b
        return (lambda m: (ops.gemm(a[:m], geglu_pack(w), bias=geglu_pack(b), geglu=True, out_dtype=torch.bfloat16),),
                y[:, :N // 2] * F.gelu(y[:, N // 2:]), 1e-2)
    if kind in ("ln_stats", "ln_fold"):
        from panacea_b200.engine import Engine
        C = min(max(K, 320), 1280)                  # token-stream width: 320 at level 0, 1280 at level 2
        wo = _rand_dev((C, K), seed + 3, K ** -0.5)
        y0 = _rand_dev((M, C), seed + 4, 2.0) + 0.7
        if kind == "ln_stats":
            return (lambda m: ops.gemm(a[:m], wo, residual=y0[:m].clone(), out_dtype=torch.bfloat16, ln_stats_out=True),
                    a.float() @ wo.float().t() + y0.float(), 1e-2)
        y, st = ops.gemm(a, wo, residual=y0, out_dtype=torch.bfloat16, ln_stats_out=True)
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
    if kind == "bf16_res_f32":
        r1 = _rand_dev((M, N), seed + 12, dtype=torch.float32)
        return lambda m: (ops.gemm(a[:m], w, bias=bias, residual=r1[:m], out_dtype=torch.bfloat16),), ref + r1, 1e-2
    if kind == "bf16_res_bf16":
        r1 = _rand_dev((M, N), seed + 13)

        def call(m):                                # in place, like the token stream
            r = r1[:m].clone()
            return (ops.gemm(a[:m], w, bias=bias, residual=r, out=r, out_dtype=torch.bfloat16),)
        return call, ref + r1.float(), 1e-2
    if kind == "rowvec":
        G = 16
        rv = _rand_dev((G, N), seed + 14, dtype=torch.float32)
        rpg = 37                                    # a row tile spans several groups; the groups wrap around
        rows = torch.arange(M, device="cuda")
        return (lambda m: (ops.gemm(a[:m], w, bias=bias, rowvec=rv, rows_per_group=rpg, n_groups=G),),
                ref + rv[(rows // rpg) % G], 2e-3)
    assert kind == "f32_res_inplace", kind
    r1 = _rand_dev((M, N), seed + 15, dtype=torch.float32)

    def call(m):
        r = r1[:m].clone()
        return (ops.gemm(a[:m], w, bias=bias, residual=r, out=r),)
    return call, ref + r1, 2e-3


def check_case(kind, got, ref, tol, name):
    """Checks the outputs `got` of an epilogue_case call over all rows against its reference; a LayerNorm producer's
    row statistics must also sum to those of the output it stored."""
    _check(got[0], ref, tol=tol, name=name)
    if kind == "ln_stats":
        y, st = got
        yf = y.float()
        torch.testing.assert_close(st[..., 0].sum(1), yf.sum(1), rtol=5e-3, atol=0.5)
        torch.testing.assert_close(st[..., 1].sum(1), (yf * yf).sum(1), rtol=5e-3, atol=0.5)


def kernels_of(fn):
    """fn()'s result and the names of the GEMM kernels it launched"""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, {e.name for e in prof.events() if "gemm" in e.name}
