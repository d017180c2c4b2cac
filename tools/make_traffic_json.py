#!/usr/bin/env python
"""ncu CSV (dram__bytes_read/write.sum per k_compute_items launch of one bench step) ->
profiles/roofline_traffic.json (not committed), the `traffic` field of bench.py's roofline object."""
import csv
import json
import sys

src, dst = sys.argv[1], sys.argv[2]
rows = list(csv.reader(open(src)))
hi = [i for i, r in enumerate(rows) if r and r[0] == "ID"][0]
hdr = rows[hi]
ki, mi, vi, ui = hdr.index("Kernel Name"), hdr.index("Metric Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
per = {}
for r in rows[hi + 1:]:
    if len(r) <= vi or "k_compute_items" not in r[ki]:
        continue
    v = float(r[vi].replace(",", ""))
    u = r[ui].lower()
    scale = {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9, "ns": 1, "us": 1e3, "ms": 1e6}.get(u, 1)
    per.setdefault(r[0], {})[r[mi]] = v * scale
n = len(per)
rd = sum(p.get("dram__bytes_read.sum", 0) for p in per.values())
wr = sum(p.get("dram__bytes_write.sum", 0) for p in per.values())
t = sum(p.get("gpu__time_duration.sum", 0) for p in per.values())
out = {"realdata_allpairs": {"kernel": "k_compute_items", "launches": n,
                             "dram_bytes_per_launch": (rd + wr) / max(n, 1),
                             "dram_read_per_launch": rd / max(n, 1), "dram_write_per_launch": wr / max(n, 1),
                             "ncu_ns_per_launch": t / max(n, 1),
                             "source": "ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum over the 9 "
                                       "k_compute_items launches of one bench.py step"}}
json.dump(out, open(dst, "w"), indent=1)
print(json.dumps(out))
