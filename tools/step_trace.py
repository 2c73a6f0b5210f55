#!/usr/bin/env python
"""Phase timeline of the persistent decode kernel (EXL_DS_TRACE): per phase, how long the prologue, the streaming loop and
the grid barrier take (median / max over CTAs), for layer 2 of a 6-layer stack (SHAPES or GQA_SHAPES names, e.g. 70b).
    EXL_DS_TRACE=1 python tools/step_trace.py [--ctx 1920] [--model 7b] [--seq 2048]"""
import argparse, json, os, sys
os.environ.setdefault("EXL_DS_TRACE", "1")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from exllama_b200.stack import GQA_SHAPES, SHAPES, DecodeStack

ap = argparse.ArgumentParser()
ap.add_argument("--model", default="7b"); ap.add_argument("--ctx", type=int, default=1920); ap.add_argument("--layers", type=int, default=6)
ap.add_argument("--groupsize", type=int, default=128); ap.add_argument("--seq", type=int, default=2048)
args = ap.parse_args()
shape = {**SHAPES, **GQA_SHAPES}[args.model]
st = DecodeStack(shape, groupsize=args.groupsize, device="cuda:0", max_seq=args.seq, layers=args.layers)
for kc, vc in zip(st.key_cache, st.value_cache):
    kc.normal_(0, 0.5); vc.normal_(0, 0.5)
st.make_plan()
x = (torch.randn((1, 1, shape.hidden), device="cuda") * 0.5).half()
for _ in range(5):
    st.decode_step_fused(x, args.ctx)
torch.cuda.synchronize()
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
a.record()
for _ in range(10): st.decode_step_fused(x, args.ctx)
b.record(); torch.cuda.synchronize()
ms = a.elapsed_time(b) / 10
tr = st.dplan.trace().astype(np.int64)          # [G, 4, 16]
L = 2
t = tr[:, L, :15] - tr[:, L, 0].min()
names = ["QKV pro", "QKV gemv", "B1", "ATT", "B2", "O pro", "O gemv", "B3", "GU pro", "GU gemv", "B4", "DOWN pro", "DOWN gemv", "B5"]
rows = []
for i, n in enumerate(names):
    d = (t[:, i + 1] - t[:, i]) / 1e3
    rows.append({"seg": n, "med_us": round(float(np.median(d)), 2), "min_us": round(float(d.min()), 2), "max_us": round(float(d.max()), 2),
                 "end_med_us": round(float(np.median(t[:, i + 1])) / 1e3, 2)})
qkv_resnorm = float(np.median(tr[:, L, 15] - tr[:, L, 0])) / 1e3
layer_us = float(np.median(tr[:, L, 14] - tr[:, L, 0])) / 1e3
print(json.dumps({"model": args.model, "gpu": torch.cuda.get_device_name(0), "debug": os.environ.get("EXL_DS_DEBUG"), "nst": os.environ.get("EXL_DS_DEPTH"), "ctx": args.ctx, "layers": args.layers,
                  "ms_per_step": round(ms, 4), "layer_us": round(layer_us, 2), "qkv_pro_residual_norm_us": round(qkv_resnorm, 2), "plan": st.dplan.info()}))
for r in rows:
    print(json.dumps(r))
