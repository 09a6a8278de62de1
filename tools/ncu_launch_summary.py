#!/usr/bin/env python
"""Condense an `ncu --csv` launch list (gpu__time_duration.sum, dram__bytes_read.sum, dram__bytes_write.sum per launch) of decode
steps into a per-kernel table and the per-launch DRAM traffic of the dominant kernel (roofline.traffic of bench.py).
    ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none \\
        -k regex:'gemv|attn|embedding|argmax' -c 400 --csv --log-file step_kernels.csv \\
        python bench.py --steps 1 --warmup 1 --no-cpu-baseline --ctx 2048
    python tools/ncu_launch_summary.py step_kernels.csv profiles/decode_step_kernels.csv profiles/roofline_traffic.json
"""
import collections
import csv
import json
import sys


def num(x):
    return float(x.replace(",", ""))


def main():
    src, out_csv, out_json = sys.argv[1:4]
    rows = list(csv.reader(open(src, errors="replace")))
    hi = next(i for i, r in enumerate(rows) if r and r[0] == "ID")
    h = rows[hi]
    iid, ik, im, iu, iv = h.index("ID"), h.index("Kernel Name"), h.index("Metric Name"), h.index("Metric Unit"), h.index("Metric Value")
    ig = h.index("Grid Size") if "Grid Size" in h else None
    launches = collections.OrderedDict()
    scale = {"ns": 1e-3, "us": 1.0, "ms": 1e3, "byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
    for r in rows[hi + 1:]:
        if len(r) <= iv:
            continue
        d = launches.setdefault(r[iid], {"name": r[ik].split("(")[0].split("::")[-1], "grid": r[ig] if ig is not None else ""})
        d[r[im]] = num(r[iv]) * scale.get(r[iu], 1.0)
    agg = collections.OrderedDict()
    for d in launches.values():
        a = agg.setdefault((d["name"], d["grid"]), {"n": 0, "us": 0.0, "rd": 0.0, "wr": 0.0})
        a["n"] += 1
        a["us"] += d.get("gpu__time_duration.sum", 0.0)
        a["rd"] += d.get("dram__bytes_read.sum", 0.0)
        a["wr"] += d.get("dram__bytes_write.sum", 0.0)
    total_us = sum(a["us"] for a in agg.values())
    with open(out_csv, "w") as f:
        f.write(f"# from {src}: per (kernel, grid) over {len(launches)} captured launches; times are ncu's cold-cache serialised durations (shares, not bench values)\n")
        w = csv.writer(f)
        w.writerow(["kernel", "grid", "launches", "mean_us", "share_of_captured_time", "mean_dram_read_bytes", "mean_dram_write_bytes"])
        for (name, grid), a in sorted(agg.items(), key=lambda kv: -kv[1]["us"]):
            w.writerow([name, grid, a["n"], round(a["us"] / a["n"], 3), round(a["us"] / total_us, 4), int(a["rd"] / a["n"]), int(a["wr"] / a["n"])])
    gem = [a for (name, _), a in agg.items() if "gemv" in name]
    n = sum(a["n"] for a in gem)
    traffic = {"kernel": "w4a16_gemv_kernel", "launches_captured": n, "dram_bytes_per_launch": (sum(a["rd"] + a["wr"] for a in gem) / n) if n else None,
               "share_of_step_time": (sum(a["us"] for a in gem) / total_us) if total_us else None, "source": out_csv}
    json.dump(traffic, open(out_json, "w"), indent=1)
    print(json.dumps(traffic))


if __name__ == "__main__":
    main()
