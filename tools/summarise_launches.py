"""Aggregate an ncu launch list (`--metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --csv`) of
tools/profile_c2.py into the per-kernel summary and the GEMM-family DRAM traffic per launch.

    python tools/summarise_launches.py launches.csv out_prefix

Keeps the LAST complete iteration (from the last-but-one vq_prep_kernel / vq_partial_kernel launch to the last one)."""
import csv
import json
import re
import sys
from collections import OrderedDict, defaultdict

src, out = sys.argv[1], sys.argv[2]
rows = OrderedDict()
with open(src) as f:
    lines = [l for l in f if l.startswith('"') or l[:1].isdigit()]
for r in csv.DictReader(lines, fieldnames=["ID", "pid", "pname", "host", "kernel", "ctx", "stream", "block", "grid", "dev", "cc",
                                           "section", "metric", "unit", "value"]):
    if r["ID"] == "ID":
        continue
    d = rows.setdefault(int(r["ID"]), {"kernel": r["kernel"], "grid": r["grid"], "block": r["block"]})
    d[r["metric"]] = float(r["value"].replace(",", ""))
ids = sorted(rows)
starts = [i for i in ids if "vq_partial_kernel" in rows[i]["kernel"] or "vq_prep_kernel" in rows[i]["kernel"]]
assert starts, "no iteration start (vq_prep_kernel / vq_partial_kernel) in the capture"
sel = [i for i in ids if starts[-2] <= i < starts[-1]] if len(starts) >= 2 else [i for i in ids if i >= starts[0]]


def short(name):
    m = re.search(r"([A-Za-z_0-9]+)(<[^(]*>)?\(", name)
    base = m.group(1) if m else name
    tmpl = m.group(2) if m and m.group(2) else ""
    return base + (tmpl if len(tmpl) < 60 else "")


agg = defaultdict(lambda: [0, 0.0, 0.0])
for i in sel:
    r = rows[i]
    a = agg[short(r["kernel"])]
    a[0] += 1
    a[1] += r.get("gpu__time_duration.sum", 0.0)
    a[2] += r.get("dram__bytes_read.sum", 0.0) + r.get("dram__bytes_write.sum", 0.0)
total = sum(a[1] for a in agg.values())
with open(out + "_iteration.csv", "w") as f:
    f.write("id,kernel,grid,block,ns,dram_read,dram_write\n")
    for i in sel:
        r = rows[i]
        f.write(f'{i},"{short(r["kernel"])}","{r["grid"]}","{r["block"]}",{r.get("gpu__time_duration.sum", 0):.0f},'
                f'{r.get("dram__bytes_read.sum", 0):.0f},{r.get("dram__bytes_write.sum", 0):.0f}\n')
with open(out + "_summary.txt", "w") as f:
    f.write(f"one config-2 iteration under ncu (cold-cache, serialised): {len(sel)} launches, {total / 1e6:.3f} ms of kernel time\n")
    f.write(f"{'kernel':70s} {'n':>5s} {'us':>10s} {'share':>7s} {'us each':>9s} {'MB/launch':>10s}\n")
    for k, a in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        f.write(f"{k[:70]:70s} {a[0]:5d} {a[1] / 1e3:10.1f} {a[1] / total:7.1%} {a[1] / 1e3 / a[0]:9.1f} {a[2] / a[0] / 1e6:10.2f}\n")
fam = [a for k, a in agg.items() if k.startswith(("gemm_tc", "attn_fwd", "attn_bwd"))]
n = sum(a[0] for a in fam)
json.dump({"source": f"ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum over one c2 iteration ({out}_iteration.csv)",
           "family": "gemm_tc*/gemm_tce*/attn_*", "gemm_launches": n, "gemm_time_ms": sum(a[1] for a in fam) / 1e6,
           "gemm_dram_bytes_per_launch": sum(a[2] for a in fam) / max(n, 1), "iteration_kernel_time_ms": total / 1e6},
          open(out.replace("ncu_launches_c2", "gemm_traffic") + ".json", "w"), indent=1)
print(open(out + "_summary.txt").read())
