"""Where the wgmma GEMM / implicit-conv and the view / text attention time goes, by launch shape, at the benchmark's
ε-evaluation.

Runs eager ε-evaluations of the full-size model at bench.py's shape (CFG batch 2 x 8 frames, 6 views of 32x56) on ONE
stream, with CUDA events around every `ops.gemm` call, the way `bench.py::profile_dominant_kernel` does, and groups the
launches by (M, N, K·taps, epilogue mode). Per class it prints launches, device time, TF/s, algorithmic bytes and the
roofline lower bound max(FLOP / 989 TF/s, bytes / 3.35 TB/s) (H100 SXM data sheet, dense bf16 and HBM3), naming the
bound that binds. Every `ops.attention_view` / `ops.attention_text` call (attn_fa_kernel) is timed the same way and listed
by kind and shape with its algorithmic TF/s (4 · queries · keys · channels FLOP). The card's name, power limit and SM
clock are read in the same run.

  python tools/gemm_classes.py [--repeats 3] [--json classes.json]

A class's time is the median over the repeats of the sum of its launches' event times. Each pass starts behind a device
sleep, so the host has queued its launches before the device reaches them and no event pair spans host issue time.
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from collections import defaultdict
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import bench  # noqa: E402
from tools.bench_kernels import card  # noqa: E402

PEAK_TFLOPS = 989.0       # H100 SXM data sheet, dense bf16 (700 W)
PEAK_TBS = 3.35           # H100 SXM data sheet, HBM3
HOST_HEAD_START_CYCLES = 1_000_000_000       # ~0.5 s at 2 GHz, more than the host needs to queue one evaluation


def record_launches(ops, run, repeats):
    """Calls run() `repeats` times with every ops.gemm and attention call timed; returns (gemm, attention) launch
    records, one list per repeat each."""
    # the timing wrapper and its byte count restate bench.py::profile_dominant_kernel (which keeps no shape per launch);
    # keep the two in step
    orig = ops.gemm
    orig_view, orig_text = ops.attention_view, ops.attention_text
    passes, attn = [], []

    def timed(a, w, **kw):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = orig(a, w, **kw)
        e.record()
        rows = a.numel() // a.shape[-1]
        geglu = bool(kw.get("geglu"))
        bf16_out = kw.get("out_dtype", torch.float32) == torch.bfloat16
        n_out = w.shape[0] // 2 if geglu else w.shape[0]
        abytes = 2.0 * rows * a.shape[-1] + 2.0 * w.numel() + (2 if bf16_out else 4) * rows * n_out
        for r in (kw.get("residual"), kw.get("residual2")):
            if r is not None:
                abytes += r.element_size() * rows * n_out
        mode = "geglu" if geglu else "bf16" if bf16_out else "f32"
        passes[-1].append(((rows, w.shape[0], w.shape[1], mode), 2.0 * rows * w.shape[0] * w.shape[1], abytes, s, e))
        return out

    def timed_view(qkv, heads, cross, neighbours):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = orig_view(qkv, heads, cross, neighbours)
        e.record()
        Fr, H, V, w, C3 = qkv.shape
        keys = sum(len(neighbours[v]) for v in range(V)) if cross else V
        attn[-1].append((("cross" if cross else "intra", f"{Fr}x{H}x{V}x{w} C={C3 // 3} h={heads}"),
                         4.0 * Fr * (H * w) ** 2 * keys * (C3 // 3), s, e))
        return out

    def timed_text(q, kv, heads):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = orig_text(q, kv, heads)
        e.record()
        b, Nq, C = q.shape
        attn[-1].append((("text", f"{b}x{Nq} Nk={kv.shape[1]} C={C} h={heads}"), 4.0 * b * Nq * kv.shape[1] * C, s, e))
        return out

    ops.gemm, ops.attention_view, ops.attention_text = timed, timed_view, timed_text
    try:
        for _ in range(repeats):
            passes.append([])
            attn.append([])
            # hold the device back until the host has queued the evaluation: otherwise an event pair around a short
            # launch also spans the host's time to issue it wherever the device has caught up with the host
            torch.cuda._sleep(HOST_HEAD_START_CYCLES)
            run()
            torch.cuda.synchronize()
    finally:
        ops.gemm, ops.attention_view, ops.attention_text = orig, orig_view, orig_text
    return passes, attn


def classify_attention(attn):
    per = defaultdict(lambda: {"launches": 0, "flop": 0.0, "secs": []})
    for i, recs in enumerate(attn):
        for key, flop, s, e in recs:
            c = per[key]
            if i == 0:
                c["launches"] += 1
                c["flop"] += flop
            if len(c["secs"]) <= i:
                c["secs"].append(0.0)
            c["secs"][i] += s.elapsed_time(e) * 1e-3
    rows = []
    for (kind, shape), c in per.items():
        secs = statistics.median(c["secs"])
        rows.append({"kind": kind, "shape": shape, "launches": c["launches"], "ms": secs * 1e3,
                     "ms_runs": [x * 1e3 for x in c["secs"]], "gflop": c["flop"] / 1e9, "tflops": c["flop"] / secs / 1e12})
    rows.sort(key=lambda r: -r["ms"])
    return rows


def classify(passes):
    per = defaultdict(lambda: {"launches": 0, "flop": 0.0, "bytes": 0.0, "secs": []})
    for i, recs in enumerate(passes):
        for key, flop, abytes, s, e in recs:
            c = per[key]
            if i == 0:
                c["launches"] += 1
                c["flop"] += flop
                c["bytes"] += abytes
            if len(c["secs"]) <= i:
                c["secs"].append(0.0)
            c["secs"][i] += s.elapsed_time(e) * 1e-3
    rows = []
    for (m, n, k, mode), c in per.items():
        secs = statistics.median(c["secs"])
        t_flop, t_bytes = c["flop"] / (PEAK_TFLOPS * 1e12), c["bytes"] / (PEAK_TBS * 1e12)
        bound = max(t_flop, t_bytes)
        rows.append({"M": m, "N": n, "K_taps": k, "mode": mode, "launches": c["launches"], "ms": secs * 1e3,
                     "ms_runs": [x * 1e3 for x in c["secs"]], "tflops": c["flop"] / secs / 1e12, "gflop": c["flop"] / 1e9,
                     "mbytes": c["bytes"] / 1e6, "bound_ms": bound * 1e3, "binds": "tensor" if t_flop >= t_bytes else "hbm",
                     "frac_of_bound": bound / secs})
    rows.sort(key=lambda r: -r["ms"])
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--repeats", type=int, default=3, help="timed ε-evaluations (median per class)")
    ap.add_argument("--json", default="", help="also write the table and the card's state to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gemm_classes.py: needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    seed = 3407
    torch.manual_seed(seed)
    pipe = bench.build_pipeline(dev, seed)
    pipe.wrapper.use_cuda_graph = False
    pipe.wrapper.hint_repeat = 2
    host = bench.synth_inputs_host(seed)
    cc = {"cond_feat": host["hint"].to(dev), "concat": torch.cat([host["concat"]] * 2).to(dev),
          "crossattn": torch.cat([host["uc_txt"], host["c_txt"]]).to(dev)}
    x_in = torch.randn(16, 4, bench.H, bench.VIEWS * bench.W_VIEW, device=dev)
    t = torch.full((16,), 999, dtype=torch.int64, device=dev)
    pipe.wrapper(x_in, t, cc)                      # conditioning, weight packing, module load
    eng = pipe.model.engine()
    eng.two_streams = False                        # an event pair must not span a launch queued behind the other branch
    concat = cc["concat"].float().contiguous()
    eng.eps(x_in, concat, t)                       # untimed single-stream pass: allocator warm-up
    torch.cuda.synchronize()

    clocks = bench.ClockSampler(0)
    clocks.start()
    passes, attn = record_launches(eng.ops, lambda: eng.eps(x_in, concat, t), args.repeats)
    clk = clocks.stop()
    name, limit = card()

    rows = classify(passes)
    total_ms = sum(r["ms"] for r in rows)
    total_flop = sum(r["gflop"] for r in rows) * 1e9
    print(f"{name}, power limit {limit}, SM clock median {clk.get('sm_mhz')} MHz (max {clk.get('sm_max_mhz')} MHz, "
          f"throttle reasons {clk.get('reasons')})")
    print(f"{len(passes[0])} pn_gemm launches per ε-evaluation, {total_ms:.1f} ms, {total_flop / total_ms / 1e9:.0f} TF/s "
          f"(median of {args.repeats} passes per class)")
    hdr = f"{'M':>7} {'N':>6} {'K*taps':>7} {'mode':>5} {'launch':>6} {'ms':>8} {'TF/s':>6} {'GFLOP':>8} {'MB':>8} {'bound ms':>8} {'binds':>6} {'of bound':>8}"
    print(hdr)
    for r in rows:
        print(f"{r['M']:>7} {r['N']:>6} {r['K_taps']:>7} {r['mode']:>5} {r['launches']:>6} {r['ms']:>8.3f} {r['tflops']:>6.0f} "
              f"{r['gflop']:>8.1f} {r['mbytes']:>8.1f} {r['bound_ms']:>8.3f} {r['binds']:>6} {r['frac_of_bound'] * 100:>7.0f}%")
    for lo, hi, label in ((0, 640, "K*taps <= 640"), (641, 1920, "641-1920"), (1921, 1 << 40, "> 1920")):
        sel = [r for r in rows if lo <= r["K_taps"] <= hi]
        ms = sum(r["ms"] for r in sel)
        gf = sum(r["gflop"] for r in sel)
        print(f"  {label:>14}: {sum(r['launches'] for r in sel):4d} launches {gf / 1e3:6.1f} TFLOP {ms:8.1f} ms "
              f"{(gf / ms if ms else 0):6.0f} TF/s")
    arows = classify_attention(attn)
    attn_ms = sum(r["ms"] for r in arows)
    print(f"{len(attn[0])} attention launches (attn_fa_kernel) per ε-evaluation, {attn_ms:.2f} ms, "
          f"{sum(r['gflop'] for r in arows) / attn_ms if attn_ms else 0:.0f} TF/s")
    print(f"{'kind':>6} {'shape':>32} {'launch':>6} {'ms':>8} {'TF/s':>6} {'GFLOP':>8}")
    for r in arows:
        print(f"{r['kind']:>6} {r['shape']:>32} {r['launches']:>6} {r['ms']:>8.3f} {r['tflops']:>6.0f} {r['gflop']:>8.1f}")
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps({"card": name, "power_limit": limit, "clocks": clk, "repeats": args.repeats,
                                               "launches": len(passes[0]), "total_ms": total_ms, "classes": rows,
                                               "attention_ms": attn_ms, "attention": arows}, indent=1))


if __name__ == "__main__":
    main()
