"""Per-kernel timing at the headline shapes (CFG batch 2 x 8 frames, 32x56 latent per view, 6 views).
Run on an H100:  python tools/bench_kernels.py [--json kernels.json] [--sampler-only]
CUDA-event timing on the launching stream, 3 warm-ups. The sampler-step section times CUDA-graph replays of launches that
cycle through a pool of inputs larger than the 50 MB L2, so its GB/s is HBM traffic and no host launch cost; it prints
the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from panacea_b200.ops import NativeOps  # noqa: E402

BF16, F32 = torch.bfloat16, torch.float32
NEIGH = ((5, 1), (0, 2), (1, 3), (2, 4), (3, 5), (4,))


def timeit(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default="")
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--sampler-only", action="store_true", help="only the pn_sampler_step section")
    a = ap.parse_args()
    ops = NativeOps()
    dev = "cuda"
    res = []

    def rec(name, secs, flops=0.0, bytes_=0.0):
        r = {"name": name, "us": secs * 1e6, "tflops": flops / secs / 1e12 if flops else None,
             "gbs": bytes_ / secs / 1e9 if bytes_ else None}
        res.append(r)
        print(f"{name:48s} {secs*1e6:10.1f} us  {r['tflops'] or 0:8.1f} TF/s  {r['gbs'] or 0:8.1f} GB/s", flush=True)

    if a.sampler_only:
        sampler_steps(ops, rec)
        if a.json:
            Path(a.json).parent.mkdir(parents=True, exist_ok=True)
            Path(a.json).write_text(json.dumps(res, indent=1))
        return
    BT, H, W = 16, 32, 336
    M0 = BT * H * W
    levels = [(M0, 320), (M0 // 4, 640), (M0 // 16, 1280)]
    for M, C in levels:
        x = torch.randn(M, C, device=dev).to(BF16)
        res32 = torch.randn(M, C, device=dev)
        w = (torch.randn(C, C, device=dev) * C ** -0.5).to(BF16)
        w3 = (torch.randn(3 * C, C, device=dev) * C ** -0.5).to(BF16)
        w8 = (torch.randn(8 * C, C, device=dev) * C ** -0.5).to(BF16)
        w4 = (torch.randn(C, 4 * C, device=dev) * (4 * C) ** -0.5).to(BF16)
        bias = torch.randn(C, device=dev)
        bias8 = torch.randn(8 * C, device=dev)
        t = timeit(lambda: ops.gemm(x, w, bias=bias, residual=res32, out=res32))
        rec(f"linear {M}x{C}->{C} +bias+res fp32", t, 2.0 * M * C * C, M * C * (2 + 4 + 4))
        t = timeit(lambda: ops.gemm(x, w3, out_dtype=BF16))
        rec(f"qkv    {M}x{C}->{3*C} bf16", t, 2.0 * M * C * 3 * C, M * C * 2 * 4)
        t = timeit(lambda: ops.gemm(x, w8, bias=bias8, geglu=True, out_dtype=BF16))
        rec(f"ff1    {M}x{C}->{8*C} geglu", t, 2.0 * M * C * 8 * C, M * C * 2 * 5)
        h = torch.randn(M, 4 * C, device=dev).to(BF16)
        t = timeit(lambda: ops.gemm(h, w4, bias=bias, residual=res32, out=res32))
        rec(f"ff2    {M}x{4*C}->{C} +res", t, 2.0 * M * 4 * C * C, M * C * (8 + 8))
        del h
        Hh, Ww = H // (1 if C == 320 else 2 if C == 640 else 4), W // (1 if C == 320 else 2 if C == 640 else 4)
        xi = x.reshape(BT, Hh, Ww, C)
        wc = (torch.randn(C, 9 * C, device=dev) * (9 * C) ** -0.5).to(BF16)
        t = timeit(lambda: ops.gemm(xi, wc, bias=bias, taps=(3, 3)))
        rec(f"conv3x3 [{BT},{Hh},{Ww},{C}]->{C}", t, 2.0 * M * 9 * C * C, M * C * 6)
        xt = x.reshape(2, 8, Hh * Ww, C)
        wt = (torch.randn(C, 3 * C, device=dev) * (3 * C) ** -0.5).to(BF16)
        t = timeit(lambda: ops.gemm(xt, wt, bias=bias, taps=(3, 1), residual=res32, out=res32))
        rec(f"conv1d-T [2,8,{Hh*Ww},{C}]->{C}", t, 2.0 * M * 3 * C * C, M * C * 10)
        # norms
        xf = res32.reshape(BT, Hh * Ww, C)
        g = torch.ones(C, device=dev); b = torch.zeros(C, device=dev)
        t = timeit(lambda: ops.groupnorm(xf, g, b, 1e-5, True))
        rec(f"groupnorm+silu [{BT},{Hh*Ww},{C}]", t, 0, M * C * (4 + 4 + 2))
        t = timeit(lambda: ops.groupnorm_pixel(res32.reshape(2, 8, Hh * Ww, C), g, b, 1e-5, True))
        rec(f"groupnorm_pixel [2,8,{Hh*Ww},{C}]", t, 0, M * C * 6)
        t = timeit(lambda: ops.layernorm(res32, g, b))
        rec(f"layernorm {M}x{C}", t, 0, M * C * 6)
        # attention
        heads = C // 64
        wv = Ww // 6
        qkv = torch.randn(BT, Hh, 6, wv, 3 * C, device=dev).to(BF16)
        n = Hh * wv
        t = timeit(lambda: ops.attention_view(qkv, heads, False, NEIGH))
        rec(f"attn intra  Nq={n} heads={heads}", t, 4.0 * BT * heads * 6 * n * n * 64, M * C * 2 * 4)
        t = timeit(lambda: ops.attention_view(qkv, heads, True, NEIGH))
        rec(f"attn cross  Nq={n}", t, 4.0 * BT * heads * (5 * 2 + 1) * n * n * 64, M * C * 2 * 4)
        t = timeit(lambda: ops.attention_temporal(qkv.reshape(2, 8, Hh * Ww, 3 * C), heads))
        rec(f"attn temporal T=8 P={Hh*Ww}", t, 4.0 * 2 * Hh * Ww * heads * 8 * 8 * 64, M * C * 2 * 4)
        q = x.reshape(2, 8 * Hh * Ww, C)
        kv = torch.randn(2, 77, 2 * C, device=dev).to(BF16)
        t = timeit(lambda: ops.attention_text(q, kv, heads))
        rec(f"attn text   Nq={8*Hh*Ww} Nk=77", t, 4.0 * M * heads * 77 * 64, M * C * 2 * 2)
        del qkv, x, res32
        torch.cuda.empty_cache()
        if a.quick:
            break
    # square GEMM for a cuBLAS-comparable number
    Mq = 8192
    xa = torch.randn(Mq, Mq, device=dev).to(BF16)
    wb = torch.randn(Mq, Mq, device=dev).to(BF16)
    t = timeit(lambda: ops.gemm(xa, wb, out_dtype=BF16), iters=5)
    rec("gemm 8192^3 bf16 (ours)", t, 2.0 * Mq ** 3)
    t = timeit(lambda: torch.matmul(xa, wb.t()), iters=5)
    rec("gemm 8192^3 bf16 (cuBLAS via torch)", t, 2.0 * Mq ** 3)
    del xa, wb
    torch.cuda.empty_cache()
    sampler_steps(ops, rec)
    if a.json:
        Path(a.json).parent.mkdir(parents=True, exist_ok=True)
        Path(a.json).write_text(json.dumps(res, indent=1))


def card():
    """(name, power limit) of the current card, read now."""
    import subprocess
    limit = "unknown"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        limit = r.stdout.strip() or limit
    except (OSError, subprocess.SubprocessError):
        pass
    return torch.cuda.get_device_name(), limit


# pn_sampler_step modes at the headline latent (8, 4, 32, 336): keyword arguments and the fp32 arrays of n elements
# the launch reads + writes (net and the next network input count twice with CFG)
SAMPLER_MODES = [
    ("euler (EulerEDM, Euler-a)", dict(mode=0, sigma=14.6, dt=-3.1), 6),
    ("euler + Philox noise", dict(mode=0, sigma=14.6, dt=-3.1, noise_amp=0.5), 6),
    ("euler + noise buffer", dict(mode=0, sigma=14.6, dt=-3.1, noise_amp=0.5, buffer_noise=True), 7),
    ("euler -> stage + d (Heun predictor)", dict(mode=0, sigma=14.6, dt=-3.1, out_stage=True, hist_write=0), 7),
    ("heun corrector", dict(mode=1, sigma=11.5, dt=-3.1, eval_stage=True, hist_read=(0,)), 8),
    ("lms order 4", dict(mode=2, sigma=9.2, coef=(-1.7, 0.9, -0.4, 0.1), hist_read=(2, 1, 0), hist_write=3), 10),
    ("dpm (2S midpoint / 2M first step)", dict(mode=3, coef=(0.8, -0.2), hist_write=0), 7),
    ("dpm_2m", dict(mode=4, coef=(0.8, -0.2, 1.5, 0.5), hist_read=(0,), hist_write=0), 8),
]


def sampler_steps(ops, rec):
    name, limit = card()
    print(f"pn_sampler_step on {name}, power limit {limit}; HBM3 data sheet 3.35 TB/s", flush=True)
    shape = (8, 4, 32, 336)
    n = 8 * 4 * 32 * 336
    pool = 8                                    # 8 sets of ~15 MB: > L2, every launch reads from HBM
    sets = [dict(x=torch.randn(shape, device="cuda"), net=torch.randn((16,) + shape[1:], device="cuda"),
                 stage=torch.randn(shape, device="cuda"), hist=torch.randn((4,) + shape, device="cuda"),
                 noise=torch.randn(shape, device="cuda"), x_in=torch.empty((16,) + shape[1:], device="cuda"))
            for _ in range(pool)]
    for label, spec, arrays in SAMPLER_MODES:
        spec = dict(spec)
        out_stage, eval_stage, buffer_noise = spec.pop("out_stage", False), spec.pop("eval_stage", False), spec.pop("buffer_noise", False)
        it = [0]

        def launch():
            b = sets[it[0] % pool]
            it[0] += 1
            ops.sampler_step(x=b["x"], net=b["net"], x_eval=b["stage"] if eval_stage else None, out=b["stage"] if out_stage else None,
                             hist=b["hist"], noise=b["noise"] if buffer_noise else None, x_in_next=b["x_in"], halves=2,
                             sigma_q=14.5, cfg_scale=5.0, c_in_next=0.07, seed=1, draw=it[0], **spec)
        # the Python/ctypes launch path costs more than the kernel: time replays of a graph of 2 * pool launches
        for _ in range(2 * pool):
            launch()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(2 * pool):
                launch()
        t = timeit(graph.replay, iters=20, warmup=3) / (2 * pool)
        rec(f"sampler_step {label}", t, 0, 4.0 * n * arrays)
        print(f"    {4.0 * n * arrays / 3.35e12 * 1e6:6.2f} us at 3.35 TB/s; {t * 1e3 / 416.0 * 100:.4f} % of a 416 ms evaluation",
              flush=True)


if __name__ == "__main__":
    main()
