"""BASELINE.json configs[4]: attention-kernel roofline sweep — seq_len in {HW = 1792 (intra-view), 2 x 1792 keys
(cross-view), T in {4, 8, 16} (temporal)}, head_dim in {64, 80}, V = 6 views, bf16 N(0,1) inputs.

  python tools/attn_sweep.py --out gpurun_out/r02_attn_sweep.json                     # CUDA-event timings
  ncu --metrics sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active,dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum \
      --clock-control none --profile-from-start off -k regex:attn_ --csv --log-file gpurun_out/r02_attn_sweep_ncu.csv \
      python tools/attn_sweep.py --profile
  python tools/attn_sweep_report.py attn_sweep.json attn_sweep_ncu.csv > attn_sweep.md
"""
import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from panacea_b200.ops import NativeOps  # noqa: E402

NEIGH = ((5, 1), (0, 2), (1, 3), (2, 4), (3, 5), (4,))
BT, H, V, W = 16, 32, 6, 56          # CFG-doubled batch of one 8-frame sequence, 32x56 latent per view


def cases():
    for d in (64, 80):
        heads = 5
        C = heads * d
        yield dict(name=f"intra-view  Nq=Nk=1792 d={d}", kind="intra", d=d, heads=heads, C=C,
                   flops=4.0 * BT * V * heads * 1792 * 1792 * d, bytes=2.0 * d * BT * V * heads * (2 * 1792 + 2 * 1792))
        yield dict(name=f"cross-view  Nq=1792 Nk=3584 d={d}", kind="cross", d=d, heads=heads, C=C,
                   flops=4.0 * BT * heads * 1792 * d * (5 * 3584 + 1792), bytes=2.0 * d * BT * heads * (2 * 6 * 1792 + 2 * (5 * 3584 + 1792)))
        for T in (4, 8, 16):
            b = BT // 8                                  # 2 sequences; T frames each
            P = H * V * W
            yield dict(name=f"temporal    T={T} pixels={P} d={d}", kind="temporal", d=d, heads=heads, C=C, T=T, b=b, P=P,
                       flops=4.0 * b * P * heads * T * T * d, bytes=2.0 * b * T * P * 4 * C)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true", help="one launch per case inside a cudaProfilerStart/Stop range")
    a = ap.parse_args()
    ops = NativeOps()
    g = torch.Generator(device="cuda").manual_seed(0)
    res = []
    for c in cases():
        if c["kind"] == "temporal":
            qkv = torch.randn(c["b"], c["T"], c["P"], 3 * c["C"], device="cuda", generator=g).to(torch.bfloat16)
            fn = lambda: ops.attention_temporal(qkv, c["heads"])
        else:
            qkv = torch.randn(BT, H, V, W, 3 * c["C"], device="cuda", generator=g).to(torch.bfloat16)
            fn = lambda: ops.attention_view(qkv, c["heads"], c["kind"] == "cross", NEIGH)
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        if a.profile:
            torch.cuda.profiler.start()
            fn()
            torch.cuda.synchronize()
            torch.cuda.profiler.stop()
            continue
        flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        ts = []
        for _ in range(10):
            flush.zero_()                               # L2 flush between timed launches
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record(); fn(); e.record()
            torch.cuda.synchronize()
            ts.append(s.elapsed_time(e) * 1e-3)
        t = sorted(ts)[len(ts) // 2]
        rec = {k: v for k, v in c.items() if k in ("name", "kind", "d", "flops", "bytes")}
        rec.update(seconds=t, tflops=c["flops"] / t / 1e12, gbs=c["bytes"] / t / 1e9)
        print(f"{c['name']:40s} {t * 1e6:9.1f} us {rec['tflops']:8.1f} TF/s {rec['gbs']:8.1f} GB/s (algorithmic)", flush=True)
        res.append(rec)
        del qkv, flush
    if a.out:
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
