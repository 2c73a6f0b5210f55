#!/usr/bin/env python
"""Compile and run hbm_read.cu: the HBM read rate of one CTA per SM streaming a buffer of Llama-7B q4 layers (4.2 GB at 40
layers) with each load mechanism -- contiguous 8 / 16 KB bulk copies (a, d), the same under grid barriers with a release or a
relaxed arrival (b), the decode step's tensor-map weight units over the real stream-K ranges with and without evict-first (c),
ops of 2 or 4 K stages (d), plain ld.global.nc loads (e) and four-tile units with 2 KB runs (f).  Writes one JSON document with
the card's name and power limit.
    python tools/micro/hbm_read.py [--out profiles/hbm_read_h100.json] [--layers 40] [--reps 3]"""
import argparse, json, os, subprocess, tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

ap = argparse.ArgumentParser()
ap.add_argument("--out", default=None); ap.add_argument("--layers", type=int, default=40); ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--rounds", type=int, default=400); ap.add_argument("--spin-ns", type=int, default=10500)
args = ap.parse_args()
with tempfile.TemporaryDirectory() as tmp:
    exe = os.path.join(tmp, "hbm_read")
    subprocess.check_call([NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", os.path.join(HERE, "hbm_read.cu"), "-o", exe])
    out = subprocess.run([exe, str(args.layers), str(args.reps), str(args.rounds), str(args.spin_ns)], check=True, capture_output=True,
                         text=True, timeout=600).stdout
rows = json.loads(out)
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.max.mem", "--format=csv,noheader,nounits"],
                   capture_output=True, text=True).stdout.strip().splitlines()[0]
name, plim, sm_max, mem_max = [s.strip() for s in q.split(",")]
doc = {"gpu": name, "power_limit_w": float(plim), "sm_max_mhz": float(sm_max), "mem_max_mhz": float(mem_max),
       "tool": "tools/micro/hbm_read.py", "layers": args.layers, "reps": args.reps,
       "rate": "bytes landed / (last landing - first issue) over all CTAs, median of reps", "rows": rows}
text = json.dumps(doc, indent=1)
print(text)
if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(text + "\n")
