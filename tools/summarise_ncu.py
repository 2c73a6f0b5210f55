"""Turn Nsight Compute outputs (a --csv launch list, or a --set full report) into small summaries.
  python tools/summarise_ncu.py launches launches.csv launches_summary.csv
  python tools/summarise_ncu.py full decode_layer.ncu-rep decode_layer_ncu.json"""
import csv
import io
import json
import subprocess
import sys
from collections import OrderedDict

mode, src, dst = sys.argv[1:4]
if mode == "launches":
    rows = [r for r in csv.reader(l for l in open(src) if l.startswith('"'))]
    hdr = rows[0]
    ik, iv, iu = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    agg = OrderedDict()
    for r in rows[1:]:
        v = float(r[iv].replace(",", ""))
        us = v / 1e3 if r[iu] in ("ns", "nsecond") else v
        a = agg.setdefault(r[ik][:80], [0, 0.0]); a[0] += 1; a[1] += us
    tot = sum(a[1] for a in agg.values()); n = sum(a[0] for a in agg.values())
    with open(dst, "w") as f:
        f.write("# ncu launch list of `python bench.py --steps 2 --warmup 3 --no-prefill --no-cpu-baseline --no-graph` "
                "(timed region only; cold-cache, serialised: compare SHARES)\n")
        f.write(f"# {n} launches, {tot:.1f} us total = {tot / 2:.1f} us per step\n")
        f.write("kernel,launches,total_us,share\n")
        for k, (c, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write(f"\"{k}\",{c},{us:.1f},{us / tot:.3f}\n")
    print(open(dst).read())
else:
    out = subprocess.run(["ncu", "-i", src, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr = rows[0]
    keep = ["Kernel Name", "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "launch__grid_size",
            "launch__cluster_size", "launch__registers_per_thread", "launch__occupancy_limit_registers",
            "launch__occupancy_limit_shared_mem", "sm__warps_active.avg.pct_of_peak_sustained_active",
            "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
            "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
            "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum"]
    idx = [(k, hdr.index(k)) for k in keep if k in hdr]
    units = rows[1]
    res = []
    for r in rows[2:]:
        if "q4_gemv" not in r[hdr.index("Kernel Name")] and "decode_attn" not in r[hdr.index("Kernel Name")]:
            continue
        res.append({k: (r[i] + (" " + units[i] if units[i] and k != "Kernel Name" else "")) for k, i in idx})
    json.dump(res, open(dst, "w"), indent=1)
    for r in res:
        print(r["Kernel Name"][:50], r.get("gpu__time_duration.sum"), r.get("dram__bytes_read.sum"), r.get("dram__bytes_write.sum"))
