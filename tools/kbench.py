#!/usr/bin/env python
"""Kernel-level sweep of q4_matmul (decode shapes): achieved HBM GB/s of our kernel and, when
oracle/_ref/libexllama_ref.so is present, of the reference's kernel compiled for sm_90a, on a rotating pool of
distinct weight sets (>= 1 GB, defeats the 50 MB L2).  CUDA-event timing, never under a profiler.
    python tools/kbench.py [--m 1] [--shapes 7b] [--ref] [--json out.json]"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from exllama_b200 import capi  # noqa: E402
from exllama_b200.stack import synth_q4_device  # noqa: E402

SHAPES = {
    "7b": [(4096, 4096, 128), (4096, 11008, 128), (11008, 4096, 128)],
    "13b": [(5120, 5120, 128), (5120, 13824, 128), (13824, 5120, 128)],
    "33b": [(6656, 6656, 128), (6656, 17920, 128), (17920, 6656, 128), (6656, 17920, 32)],
    "65b": [(8192, 8192, 128), (8192, 22016, 128), (22016, 8192, 128)],
}


def q4_bytes(K, N, gs, M=1):
    return K * N // 2 + 2 * (K // gs) * N + 4 * (K // gs) * (N // 8) + 2 * M * K + 2 * M * N


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, nargs="+", default=[1])
    ap.add_argument("--shapes", nargs="+", default=["7b"])
    ap.add_argument("--ref", action="store_true")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default=None)
    ap.add_argument("--pool-gb", type=float, default=1.0)
    ap.add_argument("--only", type=int, nargs=3, default=None, help="K N groupsize")
    args = ap.parse_args()
    peak = 6571.6
    p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
    if os.path.exists(p):
        peak = json.load(open(p)).get("hbm_gbs", peak)
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev); gen.manual_seed(0)
    ref = None
    if args.ref:
        sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
        from helpers import RefLib
        ref = RefLib(); ref.prepare_buffers(inter=22016, max_rows=16)
    rows = []
    fams = {"only": [tuple(args.only)]} if args.only else {f: SHAPES[f] for f in args.shapes}
    for fam in fams:
        for (K, N, gs) in fams[fam]:
            by1 = q4_bytes(K, N, gs)
            pool_n = max(2, int(args.pool_gb * 1e9 / by1) + 1)
            pool = [synth_q4_device(K, N, gs, dev, gen) for _ in range(pool_n)]
            q4s = [capi.Q4(a, b, c, None) for (a, b, c, _) in pool]
            rh = [ref.make_q4(a, b, c, None) for (a, b, c, _) in pool] if ref else None
            for M in args.m:
                x = (torch.randn((M, K), device=dev) * 0.5).half()
                out = torch.empty((M, N), dtype=torch.float16, device=dev)
                def ours():
                    for q in q4s:
                        capi.q4_matmul(x, q, out=out)
                res = {}
                # ours: whole pool pass captured in a CUDA graph (no host overhead in the timed region)
                ours(); torch.cuda.synchronize()
                side = torch.cuda.Stream(); side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    ours()
                torch.cuda.current_stream().wait_stream(side); torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    ours()
                g.replay(); torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.reps):
                    g.replay()
                b.record(); torch.cuda.synchronize()
                res["ours"] = a.elapsed_time(b) * 1e3 / (args.reps * pool_n)
                if ref:
                    import ctypes as C
                    arr = (C.c_void_p * pool_n)(*rh)
                    ref.lib.ref_bench_q4_pool.restype = C.c_float
                    ref.lib.ref_bench_q4_pool.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int]
                    torch.cuda.synchronize()
                    res["ref"] = float(ref.lib.ref_bench_q4_pool(x.data_ptr(), M, arr, pool_n, out.data_ptr(), args.reps, 0))
                by = q4_bytes(K, N, gs, M)
                row = {"K": K, "N": N, "gs": gs, "M": M, "bytes": by, "us": round(res["ours"], 3),
                       "GBps": round(by / res["ours"] / 1e3, 1), "frac": round(by / res["ours"] / 1e3 / peak, 4)}
                if ref:
                    row.update({"ref_us": round(res["ref"], 3), "ref_GBps": round(by / res["ref"] / 1e3, 1),
                                "speedup": round(res["ref"] / res["ours"], 2)})
                rows.append(row)
                print(json.dumps(row), flush=True)
            del pool, q4s
            capi.lib().exl_cleanup()
            torch.cuda.empty_cache()
    if args.json:
        json.dump({"peak_GBps": peak, "rows": rows}, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
