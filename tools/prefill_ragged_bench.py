#!/usr/bin/env python
"""Time ragged prefill (exl_prefill_attn_ragged, DecodeStack.prefill_ragged) against one call per sequence and against the program
the reference runs for prompts of different lengths.  One JSON line per case, each naming the card and its power limit.

Kernel rows, 7B (32 / 32 heads) and 70B (64 / 8), caches of max_seq 4096, three mixes:
  a  8 prompts at past 0, q_len 17 .. 1920
  b  8 follow-up turns, q_len 32 .. 256 at past_len 512 .. 1536
  c  4 x 512 at past 512 (uniform: ragged and exl_prefill_attn launch the same tiles)
  arms  ragged: one exl_prefill_attn_ragged launch;  loop: one exl_prefill_attn per sequence;  uniform (mix c only): one
        exl_prefill_attn launch of the whole batch;  reference: the batch left-padded to the longest sequence (model.py's
        input_mask), repeat_kv, the additive fp16 mask of input_mask and the causal triangle, SDPA over [n, heads, longest q_len,
        longest past_len + q_len] (the mask is built once per forward, outside the timed region)
  TFLOP/s counts useful work only, 4 * 128 * heads * sum_i (q_len_i * past_len_i + q_len_i (q_len_i + 1) / 2).
Stack rows, 2 layers of 7B / 70B g128: prefill_ragged of n prompts at past 0 against a loop of prefill(x_i, 0, seq=i), tok/s:
  16 x 64, 8 x 256, and six prompts of 17 .. 789 tokens (1920 in all).
Arms alternate inside each repetition (one window of `iters` calls per arm per repetition, CUDA events); every shape is warmed up
first.  Each row gives the median and the range over the repetitions.
    python tools/prefill_ragged_bench.py [--reps 7] [--iters 10] [--no-stack]"""
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
ext = cuda_ext.exllama_ext

MIXES = {
    "a": ([17, 64, 150, 300, 600, 1000, 1500, 1920], [0] * 8),
    "b": ([32, 64, 96, 128, 160, 192, 224, 256], [512, 1536, 1024, 768, 1280, 640, 1408, 896]),
    "c": ([512] * 4, [512] * 4),
}
STACK_MIXES = {"16x64": [64] * 16, "8x256": [256] * 8, "mixed1920": [17, 64, 150, 300, 600, 789]}


def _time_arms(arms, reps, iters):
    """{arm: [ms per call of each repetition]}; the arms alternate inside every repetition"""
    for fn in arms.values():
        for _ in range(2):
            fn()
    torch.cuda.synchronize()
    ts = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                fn()
            b.record()
            b.synchronize()
            ts[k].append(a.elapsed_time(b) / iters)
    return ts


def _stats(v):
    v = sorted(v)
    return {"median": round(v[len(v) // 2], 4), "min": round(v[0], 4), "max": round(v[-1], 4)}


def kernel_rows(card, reps, iters):
    for name, heads, kvh in (("7b", 32, 32), ("70b", 64, 8)):
        for mix, (q_lens, past_lens) in MIXES.items():
            n, T = len(q_lens), sum(q_lens)
            seqs = list(range(n))
            g = torch.Generator(device="cuda"); g.manual_seed(1)
            kc = torch.randn((n, kvh, MAX_SEQ, HD), device="cuda", generator=g).half()
            vc = torch.randn((n, kvh, MAX_SEQ, HD), device="cuda", generator=g).half()
            q = torch.randn((T, heads, HD), device="cuda", generator=g).half()
            out = torch.empty((T, heads * HD), dtype=torch.float16, device="cuda")
            offs = [sum(q_lens[:i]) for i in range(n)]
            # the reference: left-padded to Q new tokens and N keys; input_mask marks each sequence's real keys, right-aligned
            Q, N = max(q_lens), max(p + l for p, l in zip(past_lens, q_lens))
            qp = torch.randn((n, heads, Q, HD), device="cuda", generator=g).half()
            mask = torch.zeros((n, 1, Q, N), dtype=torch.float16, device="cuda")
            for i, (l, p) in enumerate(zip(q_lens, past_lens)):
                mask[i, :, :, :N - (p + l)] = -65504.0                          # input_mask: left padding of the keys
            mask[:, :, :, N - Q:] += torch.triu(torch.full((Q, Q), -65504.0, device="cuda"), diagonal=1).half()

            def ragged():
                ext.prefill_attn_ragged(q, kc, vc, out, q_lens, past_lens, seqs, heads, kvh, HD, MAX_SEQ)

            def loop():
                for i in range(n):
                    ql = q_lens[i]
                    ext.prefill_attn(q[offs[i]:offs[i] + ql].view(1, ql, heads, HD), kc[i:i + 1], vc[i:i + 1], out[offs[i]:offs[i] + ql],
                                     heads, kvh, HD, past_lens[i], MAX_SEQ)

            def reference():
                keys = repeat_kv(kc[:, :, :N], heads // kvh)
                values = repeat_kv(vc[:, :, :N], heads // kvh)
                o = torch.nn.functional.scaled_dot_product_attention(qp, keys, values, attn_mask=mask, is_causal=False)
                return o.transpose(1, 2).reshape(n, Q, heads * HD)

            arms = {"ragged": ragged, "loop": loop, "reference": reference}
            if len(set(q_lens)) == 1 and len(set(past_lens)) == 1:
                def uniform():
                    ext.prefill_attn(q.view(n, q_lens[0], heads, HD), kc, vc, out, heads, kvh, HD, past_lens[0], MAX_SEQ)
                arms["uniform"] = uniform
            ts = _time_arms(arms, reps, iters)
            flops = 4 * HD * heads * sum(l * p + l * (l + 1) // 2 for l, p in zip(q_lens, past_lens))
            st = {k: _stats(v) for k, v in ts.items()}
            yield {"case": "kernel", "model": name, "heads": heads, "kv_heads": kvh, "mix": mix, "q_lens": q_lens, "past_lens": past_lens,
                   "max_seq": MAX_SEQ, "ms": st, "tflops_useful": {k: round(flops / v["median"] / 1e9, 1) for k, v in st.items()},
                   "speedup_vs_loop": round(st["loop"]["median"] / st["ragged"]["median"], 3),
                   "speedup_vs_reference": round(st["reference"]["median"] / st["ragged"]["median"], 3),
                   "reps": reps, "iters": iters, **card}
            del kc, vc, q, out, qp, mask
            torch.cuda.empty_cache()


def stack_rows(card, reps):
    for name in ("7b", "70b"):
        s = {**SHAPES, **GQA_SHAPES}[name]
        st = DecodeStack(s, groupsize=128, device="cuda:0", max_seq=2048, layers=2, seed=0, batch=max(len(v) for v in STACK_MIXES.values()))
        for mix, q_lens in STACK_MIXES.items():
            n, T = len(q_lens), sum(q_lens)
            x = (torch.randn((T, s.hidden), device="cuda") * 0.5).half()
            offs = [sum(q_lens[:i]) for i in range(n)]
            xs = [x[offs[i]:offs[i] + q_lens[i]].view(1, q_lens[i], s.hidden).contiguous() for i in range(n)]

            def ragged():
                st.prefill_ragged(x, q_lens, [0] * n)

            def loop():
                for i in range(n):
                    st.prefill(xs[i], 0, seq=i)

            ts = _time_arms({"ragged": ragged, "loop": loop}, reps, 3)
            ms = {k: _stats(v) for k, v in ts.items()}
            yield {"case": "stack", "model": name, "layers": 2, "heads": s.heads, "kv_heads": s.kv_heads, "groupsize": 128, "mix": mix,
                   "q_lens": q_lens, "T": T, "ms": ms, "tok_s": {k: round(T / v["median"] * 1e3, 1) for k, v in ms.items()},
                   "speedup_vs_loop": round(ms["loop"]["median"] / ms["ragged"]["median"], 3), "reps": reps, **card}
        st.close()
        del st
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
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
