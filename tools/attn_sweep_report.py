"""Merge tools/attn_sweep.py's CUDA-event timings with the ncu metrics pass of the same launches into the markdown table
of the attention sweep report."""
import csv
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
ev = json.loads(Path(sys.argv[1]).read_text())
hdr, rows = None, {}
for r in csv.reader(open(sys.argv[2])):
    if r and r[0] == "ID":
        hdr = r
        continue
    if hdr and r and r[0].isdigit():
        d = rows.setdefault(int(r[0]), {"kernel": r[hdr.index("Kernel Name")].split("(")[0].replace("void ", "").replace("pn::", "")})
        unit, val = r[hdr.index("Metric Unit")], float(r[hdr.index("Metric Value")].replace(",", ""))
        scale = {"Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "us": 1e-6, "ms": 1e-3, "ns": 1e-9, "usecond": 1e-6, "msecond": 1e-3, "nsecond": 1e-9}.get(unit, 1.0)
        d[r[hdr.index("Metric Name")]] = val * scale
prof = [rows[k] for k in sorted(rows)]
peaks = {}
try:
    peaks = json.loads((ROOT / "MEASURED_PEAKS.json").read_text())
except (OSError, ValueError):
    pass
pk_tf, pk_bw = peaks.get("bf16_tflops", 1590.0), peaks.get("hbm_gbs", 6650.0)
print("| case | kernel | time (us, CUDA events, L2 flushed) | TF/s (algorithmic) | of bf16 burst peak | tensor-pipe active % (ncu) | DRAM traffic GB/s (ncu) | of HBM peak | DRAM MB read / written |")
print("|---|---|---|---|---|---|---|---|---|")
for i, e in enumerate(ev):
    p = prof[i] if i < len(prof) else {}
    dr, dw, tn = p.get("dram__bytes_read.sum", 0.0), p.get("dram__bytes_write.sum", 0.0), p.get("gpu__time_duration.sum", 0.0)
    tp = p.get("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active")
    gbs = (dr + dw) / tn / 1e9 if tn else float("nan")
    print(f"| {e['name']} | `{p.get('kernel', '?')}` | {e['seconds'] * 1e6:.1f} | {e['tflops']:.1f} | {e['tflops'] / pk_tf:.3f} | "
          f"{'-' if tp is None else f'{tp:.1f}'} | {gbs:.0f} | {gbs / pk_bw:.3f} | {dr / 1e6:.0f} / {dw / 1e6:.0f} |")
print(f"\nPeaks: MEASURED_PEAKS.json bf16 burst {pk_tf:.0f} TF/s, HBM copy {pk_bw:.0f} GB/s (of measured). FLOPs = 4 B heads Nq Nk d, "
      "bytes = 2 d B heads (2 Nq + 2 Nk) (SURVEY.md section 8d). The temporal kernel is the warp-level mma.sync kernel (T <= 16 rows cannot "
      "fill a wgmma tile): it is HBM-bound, its tensor-pipe figure is not a target.")
