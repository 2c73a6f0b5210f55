#!/usr/bin/env python
"""Prefill q4_matmul sweep: wgmma fused-dequant GEMM (path 2) vs reconstruct + cuBLAS (path 3, the reference's algorithm)
and, with --ref, the reference's own q4_matmul_recons_cuda compiled for sm_90a.  CUDA-event timing over a rotating pool."""
import argparse, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from exllama_b200 import capi
from exllama_b200.stack import synth_q4_device

ap = argparse.ArgumentParser()
ap.add_argument("--m", type=int, nargs="+", default=[128, 512, 1920])
ap.add_argument("--shapes", type=int, nargs="+", default=[4096, 4096, 4096, 11008, 11008, 4096])
ap.add_argument("--gs", type=int, default=128)
ap.add_argument("--ref", action="store_true")
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--act", action="store_true")
ap.add_argument("--paths", type=int, nargs="+", default=[2, 3])
args = ap.parse_args()
dev = torch.device("cuda:0")
gen = torch.Generator(device=dev); gen.manual_seed(0)
peak = 1692.1
p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
if os.path.exists(p): peak = json.load(open(p)).get("bf16_tflops", peak)
ref = None
if args.ref:
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    from helpers import RefLib
    ref = RefLib(); ref.prepare_buffers(inter=11008, max_rows=2048, dq_numel=4096 * 11008)
tdq = torch.zeros((1, 4096 * 11008), dtype=torch.float16, device=dev)
tst = torch.zeros((2048, 11008), dtype=torch.float16, device=dev)
capi.prepare_buffers(0, tst, torch.zeros((4, 11008), dtype=torch.float16, device=dev), torch.zeros((1, 65536), dtype=torch.float32, device=dev), tdq)
shapes = [(args.shapes[i], args.shapes[i + 1]) for i in range(0, len(args.shapes), 2)]
for (K, N) in shapes:
    pool = [synth_q4_device(K, N, args.gs, dev, gen, act_order=args.act) for _ in range(4)]
    q4s = [capi.Q4(a, b, c, g) for (a, b, c, g) in pool]
    rh = [ref.make_q4(a.clone(), b, c, None) for (a, b, c, g) in pool] if ref and not args.act else None
    for M in args.m:
        x = (torch.randn((M, K), device=dev) * 0.5).half()
        out = torch.empty((M, N), dtype=torch.float16, device=dev)
        row = {"K": K, "N": N, "M": M, "gs": args.gs, "act": args.act}
        for path in args.paths:
            def f():
                for q in q4s: capi.q4_matmul(x, q, out=out, force_path=path)
            f(); torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.reps): f()
            b.record(); torch.cuda.synchronize()
            us = a.elapsed_time(b) * 1e3 / (args.reps * len(q4s))
            tf = 2.0 * M * K * N / us / 1e6
            row[f"path{path}_us"] = round(us, 2); row[f"path{path}_TF"] = round(tf, 1); row[f"path{path}_frac"] = round(tf / peak, 3)
        if rh:
            def g():
                for h in rh: ref.lib.ref_q4_matmul(x.data_ptr(), M, h, out.data_ptr(), 0, 1)
            torch.cuda.synchronize(); g(); ref.sync()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            import time; t0 = time.perf_counter()
            for _ in range(args.reps): g()
            ref.sync(); us = (time.perf_counter() - t0) * 1e6 / (args.reps * len(rh))
            row["ref_us"] = round(us, 2); row["ref_TF"] = round(2.0 * M * K * N / us / 1e6, 1)
        print(json.dumps(row), flush=True)
