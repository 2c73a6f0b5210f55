#!/usr/bin/env python
"""Compile and run fence_load.cu: grid-barrier fence and round-trip time under a streaming load (bulk copies into shared
memory with 0-128 KB in flight per SM, or 32 KB in flight behind an L2 prefetch lookahead of 4-32 MB chip-wide), and the
HBM rate that load reached.  Writes one JSON document with the card's name and power limit.
    python tools/micro/fence_load.py [--out profiles/fence_load_h100.json] [--rounds 2000] [--spin-ns 3000]"""
import argparse, json, os, subprocess, tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

ap = argparse.ArgumentParser()
ap.add_argument("--out", default=None); ap.add_argument("--rounds", type=int, default=2000)
ap.add_argument("--spin-ns", type=int, default=3000); ap.add_argument("--buf-mb", type=int, default=2048)
args = ap.parse_args()
with tempfile.TemporaryDirectory() as tmp:
    exe = os.path.join(tmp, "fence_load")
    subprocess.check_call([NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", os.path.join(HERE, "fence_load.cu"), "-o", exe])
    out = subprocess.run([exe, str(args.buf_mb), str(args.rounds), str(args.spin_ns)], check=True, capture_output=True, text=True, timeout=600).stdout
rows = json.loads(out)
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True).stdout.strip().splitlines()[0]
name, plim = [s.strip() for s in q.split(",")]
doc = {"gpu": name, "power_limit_w": float(plim), "tool": "tools/micro/fence_load.py", "rows": rows}
text = json.dumps(doc, indent=1)
print(text)
if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(text + "\n")
