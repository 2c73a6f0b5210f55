#!/usr/bin/env python
"""Time csrc/prefill_attn.cu (exl_prefill_attn) against the program the reference runs for a prompt chunk, and prefill tok/s of a
2-layer stack in chunks against one prefill.  One JSON line per case, each naming the card and its power limit.

Kernel rows: 7B (32 / 32 heads) and 70B (64 / 8), q_len 512 and 1920, past_len 0, 512 and 1536 in a cache of max_seq 4096, bsz 1.
  reference at past > 0: repeat_kv of the cache rows + SDPA with model.py's additive fp16 mask [1, 1, q_len, past + q_len] (the mask
                         is built once per forward by model.py, so it is built outside the timed region here too)
  reference at past 0:   repeat_kv + SDPA(is_causal=True) (what DecodeStack.prefill runs)
  Each timed launch reads a different (q, cache) set; together the sets exceed L2.  CUDA events around `iters` launches, median
  of `reps` windows.  TFLOP/s counts the causal work, 4 * 128 * heads * sum_t (past_len + t + 1).
Stack rows: 2 layers of 7B / 70B, T = 1920: four chunks of 512 (past 0, 512, 1024, 1536) against one 1920-token prefill, tok/s.
    python tools/prefill_attn_bench.py [--reps 5] [--iters 10] [--no-stack]"""
import argparse, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from bench import power_limit
from exllama_b200 import cuda_ext
from exllama_b200.shapes import GQA_SHAPES, SHAPES
from exllama_b200.stack import DecodeStack, repeat_kv

HD = 128
MAX_SEQ = 4096
L2_BYTES = 50 * 2**20
ext = cuda_ext.exllama_ext


def _time(fn, n_sets, reps, iters):
    """median ms per call over reps windows of iters calls, call i on set i % n_sets"""
    for i in range(3):
        fn(i % n_sets)
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for i in range(iters):
            fn(i % n_sets)
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / iters)
    return sorted(ts)[len(ts) // 2]


def kernel_rows(card, reps, iters):
    for name, heads, kvh in (("7b", 32, 32), ("70b", 64, 8)):
        set_bytes = 2 * kvh * MAX_SEQ * HD * 2
        n_sets = max(2, -(-3 * L2_BYTES // set_bytes))             # the sets together exceed L2 at least 3x
        g = torch.Generator(device="cuda"); g.manual_seed(1)
        kcs = [torch.randn((1, kvh, MAX_SEQ, HD), device="cuda", generator=g).half() for _ in range(n_sets)]
        vcs = [torch.randn((1, kvh, MAX_SEQ, HD), device="cuda", generator=g).half() for _ in range(n_sets)]
        for q_len in (512, 1920):
            qs = [torch.randn((1, q_len, heads, HD), device="cuda", generator=g).half() for _ in range(n_sets)]
            out = torch.empty((1, q_len, heads * HD), dtype=torch.float16, device="cuda")
            for past in (0, 512, 1536):
                if past + q_len > MAX_SEQ:
                    continue
                n = past + q_len
                mask = None
                if past > 0:
                    mask = torch.zeros((1, 1, q_len, n), dtype=torch.float16, device="cuda")
                    mask[:, :, :q_len - 1, past + 1:] = torch.triu(torch.full((q_len - 1, q_len - 1), -65504.0, device="cuda")).half()

                def ours(i):
                    ext.prefill_attn(qs[i], kcs[i], vcs[i], out, heads, kvh, HD, past, MAX_SEQ)

                def reference(i):
                    keys = repeat_kv(kcs[i][:, :, :n], heads // kvh)
                    values = repeat_kv(vcs[i][:, :, :n], heads // kvh)
                    q = qs[i].transpose(1, 2)
                    if mask is None:
                        o = torch.nn.functional.scaled_dot_product_attention(q, keys, values, attn_mask=None, is_causal=True)
                    else:
                        o = torch.nn.functional.scaled_dot_product_attention(q, keys, values, attn_mask=mask, is_causal=False)
                    return o.transpose(1, 2).reshape(1, q_len, heads * HD)

                ms_ours = _time(ours, n_sets, reps, iters)
                ms_ref = _time(reference, n_sets, reps, iters)
                flops = 4 * HD * heads * (q_len * past + q_len * (q_len + 1) // 2)
                yield {"case": "kernel", "model": name, "heads": heads, "kv_heads": kvh, "q_len": q_len, "past_len": past,
                       "max_seq": MAX_SEQ, "ms_prefill_attn": round(ms_ours, 4), "ms_reference": round(ms_ref, 4),
                       "reference": "repeat_kv + SDPA(is_causal=True)" if past == 0 else "repeat_kv + SDPA(additive fp16 mask)",
                       "speedup": round(ms_ref / ms_ours, 3), "tflops_prefill_attn": round(flops / ms_ours / 1e9, 1),
                       "tflops_reference": round(flops / ms_ref / 1e9, 1), "distinct_sets": n_sets, **card}
            del qs, out
        del kcs, vcs
        torch.cuda.empty_cache()


def stack_rows(card, reps):
    T, C = 1920, 512
    for name in ("7b", "70b"):
        s = {**SHAPES, **GQA_SHAPES}[name]
        st = DecodeStack(s, groupsize=128, device="cuda:0", max_seq=2048, layers=2, seed=0)
        x = (torch.randn((1, T, s.hidden), device="cuda") * 0.5).half()
        chunks = [x[:, c:c + C].contiguous() for c in range(0, T, C)]

        def single(_):
            st.prefill(x)

        def chunked(_):
            for j, xc in enumerate(chunks):
                st.prefill(xc, j * C)

        ms_single = _time(single, 1, reps, 3)
        ms_chunked = _time(chunked, 1, reps, 3)
        st.close()
        del st
        torch.cuda.empty_cache()
        yield {"case": "stack", "model": name, "layers": 2, "heads": s.heads, "kv_heads": s.kv_heads, "groupsize": 128, "T": T,
               "chunk": C, "ms_single": round(ms_single, 3), "ms_chunked": round(ms_chunked, 3),
               "tok_s_single": round(T / ms_single * 1e3, 1), "tok_s_chunked": round(T / ms_chunked * 1e3, 1), **card}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--no-stack", action="store_true")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit(0)}
    for row in kernel_rows(card, args.reps, args.iters):
        print(json.dumps(row), flush=True)
    if not args.no_stack:
        for row in stack_rows(card, args.reps):
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
