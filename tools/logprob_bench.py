#!/usr/bin/env python
"""Time exl_token_logprobs (csrc/logprob.cu, scoring.token_logprobs) against the program the reference runs for the same answer, and
perplexity through a stack.  One JSON line per case, each naming the card and its power limit.

Kernel rows: the 7B head (H 4096, V 32000) and the 70B head (8192 x 32000) at T 512, 1920 and 4096, and a 128256-id vocabulary
(4096 x 128256) at T 512 and 1920.
  arms  fused: scoring.token_logprobs with its outputs and work buffer allocated once, outside the timed region;  torch: the
        reference's program, torch.matmul(hn, lm_head.t()).float() -> log_softmax -> gather (model.py:1077-1080, perplexity.py:118-121)
  TFLOP/s counts the GEMM, 2 T H V, and is given as a share of the data sheet's 989 dense fp16 TFLOP/s.
  extra_mb: torch.cuda.max_memory_allocated above what was allocated before one call of the arm (fused: outputs + work).
Stack row: perplexity over 16 chunks of 512 tokens on a 2-layer 7B g128 stack (batch 16): scoring.perplexity packed (one
prefill_ragged call), one chunk per call, and the reference's loop (prefill(last_only=False) per chunk, log_softmax, gather, .item()).
Arms alternate inside each repetition (CUDA events around `iters` calls); every shape is warmed up first.  Each row gives the
median and the range over the repetitions.
    python tools/logprob_bench.py [--reps 7] [--iters 10] [--no-stack]"""
import argparse, json, math, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from bench import power_limit
from exllama_b200 import scoring
from exllama_b200.shapes import SHAPES
from exllama_b200.stack import DecodeStack
from oracle.logprob_oracle import torch_program

PEAK_TFLOPS = 989.0
CASES = [("7b", 4096, 32000, [512, 1920, 4096]), ("70b", 8192, 32000, [512, 1920, 4096]), ("v128k", 4096, 128256, [512, 1920])]


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


def _extra_mb(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    r = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    del r
    return round((peak - base) / 2 ** 20, 2)


def kernel_rows(card, reps, iters):
    for name, H, V, Ts in CASES:
        g = torch.Generator(device="cuda"); g.manual_seed(1)
        lm = (torch.randn((V, H), device="cuda", generator=g) * 0.02).half()
        for T in Ts:
            hn = torch.randn((T, H), device="cuda", generator=g).half()
            y = torch.randint(0, V, (T,), device="cuda", generator=g)
            extra = {"fused": _extra_mb(lambda: scoring.token_logprobs(hn, lm, y)), "torch": _extra_mb(lambda: torch_program(hn, lm, y))}
            out = (torch.empty(T, device="cuda"), torch.empty(T, dtype=torch.int64, device="cuda"))
            work = torch.empty(scoring.work_size(T, V, 0), dtype=torch.uint8, device="cuda")
            arms = {"fused": lambda: scoring.token_logprobs(hn, lm, y, out=out, work=work), "torch": lambda: torch_program(hn, lm, y)}
            ts = _time_arms(arms, reps, iters)
            ms = {k: _stats(v) for k, v in ts.items()}
            flops = 2.0 * T * H * V
            tf = {k: round(flops / v["median"] / 1e9, 1) for k, v in ms.items()}
            lp_f = scoring.token_logprobs(hn, lm, y)[0].double()
            lp_t = torch_program(hn, lm, y).double()
            yield {"case": "kernel", "head": name, "T": T, "H": H, "V": V, "ms": ms, "tflops": tf,
                   "share_of_989": {k: round(v / PEAK_TFLOPS, 3) for k, v in tf.items()},
                   "speedup_vs_torch": round(ms["torch"]["median"] / ms["fused"]["median"], 3), "extra_mb": extra,
                   "max_abs_diff_vs_torch": round(float((lp_f - lp_t).abs().max()), 6), "work_bytes": work.numel(),
                   "reps": reps, "iters": iters, **card}
            del hn, y, out, work
        del lm
        torch.cuda.empty_cache()


def stack_row(card, reps):
    s = SHAPES["7b"]
    n, L = 16, 512
    st = DecodeStack(s, groupsize=128, device="cuda:0", max_seq=L, layers=2, seed=0, batch=n)
    g = torch.Generator(device="cuda"); g.manual_seed(2)
    embed = (torch.randn((s.vocab, s.hidden), device="cuda", generator=g) * 0.5).half()
    chunks = [torch.randint(0, s.vocab, (L,), device="cuda", generator=g) for _ in range(n)]

    def reference():
        tot, cnt = 0.0, 0
        for c in chunks:
            logits = st.prefill(embed[c[:-1]].view(1, L - 1, -1), 0, last_only=False)
            lp = torch.nn.functional.log_softmax(logits, dim=-1).gather(-1, c[1:].view(-1, 1)).view(-1)
            tot += lp.sum().item(); cnt += L - 1
        return math.exp(-tot / cnt)

    vals = {}
    arms = {"packed": lambda: vals.__setitem__("packed", scoring.perplexity(st, embed, chunks)),
            "per_chunk": lambda: vals.__setitem__("per_chunk", scoring.perplexity(st, embed, chunks, per_call=1)),
            "reference": lambda: vals.__setitem__("reference", reference())}
    ts = _time_arms(arms, reps, 1)
    ms = {k: _stats(v) for k, v in ts.items()}
    tokens = n * (L - 1)
    row = {"case": "stack_perplexity", "model": "7b", "layers": 2, "groupsize": 128, "chunks": n, "chunk_len": L, "ms": ms,
           "tok_s": {k: round(tokens / v["median"] * 1e3, 1) for k, v in ms.items()},
           "speedup_vs_reference": round(ms["reference"]["median"] / ms["packed"]["median"], 3),
           "perplexity": {k: round(v, 6) for k, v in vals.items()}, "reps": reps, **card}
    st.close()
    return row


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
        print(json.dumps(stack_row(card, args.reps)), flush=True)


if __name__ == "__main__":
    main()
