#!/usr/bin/env python
"""Per-solve kernel time and DRAM traffic of the solve pipeline, measured with ncu (run on the GPU box).

    python tools/ncu_traffic.py cfg2-mod cfg2-random ... > gpurun_out/r2f_dram_traffic.json

For every workload: `ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum` over
tools/one_solve.py, once with ncu's default cache control (every kernel starts COLD: all caches flushed) and once
with --cache-control none (WARM: caches as the previous kernel left them, which is how the timed loop runs).  The
last solve's kernels (from its k_cls_insert to the next lease-maintenance kernel) are summed.  Also writes the
per-launch list of the last solve to gpurun_out/r2f_launches_<workload>.csv.
"""
import csv
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
OUT = ROOT / "gpurun_out"
METRICS = "gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum"


def run(workload: str, warm: bool):
    log = OUT / f"ncu_{workload}_{'warm' if warm else 'cold'}.csv"
    cmd = ["ncu", "--metrics", METRICS, "--clock-control", "none", "--csv", "--log-file", str(log)]
    if warm:
        cmd += ["--cache-control", "none"]
    cmd += [sys.executable, str(ROOT / "tools" / "one_solve.py"), workload, "3"]
    subprocess.run(cmd, check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL, timeout=900)
    rows = [r for r in csv.reader(open(log)) if len(r) > 5 and r[0].isdigit()]
    # one row per (launch, metric): ID, ..., Kernel Name(4), ..., Block Size(7), Grid Size(8), ..., Metric Name(12), Unit(13), Value(14)
    launches: dict[int, dict] = {}
    for r in rows:
        d = launches.setdefault(int(r[0]), {"name": r[4].split("(")[0], "grid": r[8], "block": r[7]})
        d[r[12]] = float(r[14].replace(",", ""))
        d[r[12] + ".unit"] = r[13]
    seq = [launches[k] for k in sorted(launches)]
    # a solve starts with the fused front kernel, or (kernel-by-kernel pipeline) with k_cls_insert
    start = max(i for i, d in enumerate(seq) if d["name"].endswith("k_cls_insert") or d["name"].endswith("k_fused_front"))
    solve = []
    for d in seq[start:]:
        if any(x in d["name"] for x in ("k_free", "k_tick", "k_keep_alive")):
            break
        solve.append(d)

    def to_bytes(d, key):
        v, u = d.get(key, 0.0), d.get(key + ".unit", "byte").lower()
        return v * {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9}.get(u, 1)

    def to_us(d):
        v, u = d.get("gpu__time_duration.sum", 0.0), d.get("gpu__time_duration.sum.unit", "ns").lower()
        return v * {"ns": 1e-3, "us": 1.0, "usecond": 1.0, "ms": 1e3, "nsecond": 1e-3, "msecond": 1e3}.get(u, 1e-3)

    per = [{"kernel": d["name"].split("::")[-1], "grid": d["grid"], "block": d["block"], "us": round(to_us(d), 2),
            "dram_read": int(to_bytes(d, "dram__bytes_read.sum")), "dram_write": int(to_bytes(d, "dram__bytes_write.sum"))} for d in solve]
    return per


def main():
    OUT.mkdir(exist_ok=True)
    res = {"how": "ncu gpu__time_duration / dram__bytes_read / dram__bytes_write over tools/one_solve.py; kernels of the LAST solve; "
                  "cold = ncu's default cache control (all caches flushed before every kernel), warm = --cache-control none",
           "workloads": {}}
    for w in sys.argv[1:]:
        cold, warm = run(w, False), run(w, True)
        res["workloads"][w] = {
            "kernels": len(cold),
            "cold_bytes": sum(k["dram_read"] + k["dram_write"] for k in cold),
            "warm_bytes": sum(k["dram_read"] + k["dram_write"] for k in warm),
            "sum_kernel_us": round(sum(k["us"] for k in warm), 1),
            "sum_kernel_us_cold": round(sum(k["us"] for k in cold), 1),
            "source": "tools/ncu_traffic.py",
            "launches_warm": warm, "launches_cold": cold,
        }
        with open(OUT / f"r2f_launches_{w}.csv", "w") as f:
            f.write("kernel,grid,block,us_warm,dram_read_warm,dram_write_warm,us_cold,dram_read_cold,dram_write_cold\n")
            for a, b in zip(warm, cold):
                f.write(f"{a['kernel']},\"{a['grid']}\",\"{a['block']}\",{a['us']},{a['dram_read']},{a['dram_write']},{b['us']},{b['dram_read']},{b['dram_write']}\n")
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
