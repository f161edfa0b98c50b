"""DRAM traffic per launch of the dominant kernel family, from an ncu metrics pass over ONE eager eps-evaluation:

  ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum --clock-control none \
      --profile-from-start off -k regex:gemm_tc --csv --log-file gpurun_out/r02_gemm_dram.csv python tools/profile_step.py
  python tools/ncu_traffic.py gemm_dram.csv profiles/gemm_traffic.json

The JSON is what bench.py reports as roofline.traffic (bytes per launch, averaged over the family's launches of one
eps-evaluation, like roofline.achieved)."""
import csv
import json
import re
import sys
from collections import defaultdict

src, dst = sys.argv[1], sys.argv[2]
hdr = None
per = defaultdict(dict)
names = {}
for r in csv.reader(open(src)):
    if r and r[0] == "ID":
        hdr = r
        continue
    if not r or not r[0].isdigit() or hdr is None:
        continue
    i = int(r[0])
    names[i] = re.sub(r"\(.*", "", r[hdr.index("Kernel Name")]).replace("void ", "").replace("pn::", "")
    unit, val = r[hdr.index("Metric Unit")], float(r[hdr.index("Metric Value")].replace(",", ""))
    scale = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1e-9, "us": 1e-6, "ms": 1e-3, "nsecond": 1e-9,
             "usecond": 1e-6, "msecond": 1e-3}.get(unit, 1.0)
    per[i][r[hdr.index("Metric Name")]] = val * scale
fam = defaultdict(lambda: {"launches": 0, "dram_read_bytes": 0.0, "dram_write_bytes": 0.0, "seconds": 0.0})
for i, m in per.items():
    f = fam[names[i]]
    f["launches"] += 1
    f["dram_read_bytes"] += m.get("dram__bytes_read.sum", 0.0)
    f["dram_write_bytes"] += m.get("dram__bytes_write.sum", 0.0)
    f["seconds"] += m.get("gpu__time_duration.sum", 0.0)
tot = {"launches": 0, "dram_read_bytes": 0.0, "dram_write_bytes": 0.0, "seconds": 0.0}
for f in fam.values():
    for k in tot:
        tot[k] += f[k]
out = {"source": src, "family": "gemm_tc_kernel (all instantiations, one eps-evaluation)", "launches": tot["launches"],
       "dram_bytes_total": tot["dram_read_bytes"] + tot["dram_write_bytes"],
       "dram_bytes_per_launch": (tot["dram_read_bytes"] + tot["dram_write_bytes"]) / max(tot["launches"], 1),
       "dram_read_bytes_total": tot["dram_read_bytes"], "dram_write_bytes_total": tot["dram_write_bytes"],
       "ncu_seconds_total": tot["seconds"],
       "per_instantiation": {k: {**v, "GBps": (v["dram_read_bytes"] + v["dram_write_bytes"]) / max(v["seconds"], 1e-12) / 1e9}
                             for k, v in sorted(fam.items(), key=lambda kv: -kv[1]["seconds"])}}
json.dump(out, open(dst, "w"), indent=1)
print(json.dumps({k: v for k, v in out.items() if k != "per_instantiation"}, indent=1))
