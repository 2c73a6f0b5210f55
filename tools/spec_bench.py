#!/usr/bin/env python
"""Measure speculative sampling (exl_spec_verify, exllama_b200.speculative) on one GPU and write one JSON file (default
profiles/spec_h100.json) naming the GPU and its power limit.  Everything is measured in one process:

  verify      CUDA-event time per exl_spec_verify call (ten replays of a CUDA graph of 100 calls), vocab 32000, k 1 / 2 / 3, the
              generator's defaults with a 1920-token history, next to exl_sample of k + 1 rows with the same settings
  loop        the 7B synthetic target at ctx 1920 emits --tokens tokens through SpeculativeGenerator, k 1 / 2 / 3, with the defaults
              and with greedy (top_k 1); the draft is an early exit of the target (its first --draft-layers layers, same seed, the
              target's final norm and lm_head).  tok/s, mean tokens per round, acceptance rate
  breakdown   per round, the CUDA-event time of the draft steps, the draft samplers, the target's multi-token step and the verify
              call, and the rest of the round's wall time (launch overhead and the one host synchronisation)
  baseline    sample_bench's loop on the same target: fused one-token step -> exl_sample -> embedding gather, --tokens tokens

The synthetic weights say nothing about how often a real draft model is accepted.  With an acceptance rate a, a round emits
(1 - a^(k+1)) / (1 - a) tokens on average; the breakdown gives a round's cost, so tok/s can be worked out for any a.

    python tools/spec_bench.py [--out profiles/spec_h100.json] [--tokens 128] [--draft-layers 2] [--layers N]"""
import argparse, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from bench import power_limit
from exllama_b200 import sampling, speculative
from exllama_b200.stack import SHAPES, DecodeStack

VOCAB = 32000
CTX = 1920
C_EMB = 25.0            # tied embeddings x = c * lm_head[token] (rows of rms ~ 0.5), as the tests tie them


def greedy():
    s = sampling.Settings()
    s.top_k = 1
    return s


def graph_us(fn, reps=100, replays=10):
    """CUDA-event time per call of fn, captured 100 times in one graph and replayed ten times."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        g.replay()
    e1.record(); torch.cuda.synchronize()
    return round(e0.elapsed_time(e1) * 1000 / (reps * replays), 2)


def verify_times(gen):
    out = {}
    s = sampling.Settings()
    hist = torch.randint(0, VOCAB, (CTX,), device="cuda", generator=gen)
    for k in (1, 2, 3):
        logits = torch.randn((k + 1, VOCAB), device="cuda", generator=gen) * 2.5
        draft = logits[:k] + torch.randn((k, VOCAB), device="cuda", generator=gen)
        q = torch.empty((k, VOCAB), device="cuda")
        d, _ = sampling.sample(draft, s, dist=q, generator=gen)
        u = torch.rand(k + 1, device="cuda", generator=gen)
        h2 = hist.view(1, -1).expand(k + 1, -1).contiguous()
        out[f"k{k}"] = {
            "verify_us": graph_us(lambda: speculative.verify(logits, d, q, s, history=hist, u=u, bos_token_id=1)),
            "sample_k_plus_1_rows_us": graph_us(lambda: sampling.sample(logits, s, history=h2, u=u, bos_token_id=1)),
        }
        print(f"verify k {k}: {out[f'k{k}']}", flush=True)
    return out


class Parts:
    """CUDA events around every call of the wrapped functions, summed per part after a synchronise."""

    def __init__(self):
        self.events = {}

    def wrap(self, name, fn):
        def timed(*a, **kw):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = fn(*a, **kw)
            e1.record()
            self.events.setdefault(name, []).append((e0, e1))
            return r
        return timed

    def totals_ms(self):
        torch.cuda.synchronize()
        return {k: sum(a.elapsed_time(b) for a, b in v) for k, v in self.events.items()}


def loop(target, draft, emb, prompt, s, k, tokens, gen, breakdown=False):
    g = speculative.SpeculativeGenerator(target, draft, emb, emb, k=k, settings=s, bos_token_id=1, generator=gen)
    g.begin(prompt)
    parts = Parts()
    saved = (speculative.sampling.sample, speculative.verify)
    if breakdown:
        draft.decode_step_fused_multi = parts.wrap("draft_steps", draft.decode_step_fused_multi)
        target.decode_step_fused_multi = parts.wrap("target_multi_step", target.decode_step_fused_multi)
        speculative.sampling.sample = parts.wrap("draft_samplers", sampling.sample)
        speculative.verify = parts.wrap("verify", speculative.verify)
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        start, accepted = g.n, []
        while g.n - start < tokens:
            accepted.append(g.round())
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    finally:
        if breakdown:
            del draft.decode_step_fused_multi, target.decode_step_fused_multi  # back to the class methods
            speculative.sampling.sample, speculative.verify = saved
    emitted = g.n - start
    res = {"tok_s": round(emitted / dt, 1), "tokens": emitted, "rounds": len(accepted),
           "tokens_per_round": round(emitted / len(accepted), 3), "acceptance_rate": round(sum(accepted) / (k * len(accepted)), 4)}
    if breakdown:
        n = len(accepted)
        per = {k2: round(v * 1000 / n, 1) for k2, v in parts.totals_ms().items()}
        per["round_wall_us"] = round(dt * 1e6 / n, 1)
        per["sync_and_launch_us"] = round(per["round_wall_us"] - sum(v for k2, v in per.items() if k2 != "round_wall_us"), 1)
        res = {"us_per_round": per, "rounds": n}
    return res


def baseline(target, emb, prompt, tokens, gen):
    """Fused one-token step -> exl_sample -> embedding gather, as tools/sample_bench.py's loop."""
    s = sampling.Settings()
    ids = torch.tensor(prompt, device="cuda")
    L = len(prompt)
    hist = torch.zeros(L + tokens + 1, dtype=torch.int64, device="cuda")
    hist[:L] = ids
    lg = target.prefill(emb[ids].view(1, L, -1), 0)
    hist[L:L + 1], _ = sampling.sample(lg, s, history=hist.view(1, -1), hist_lens=[L], generator=gen, bos_token_id=1)
    target.make_plan()
    best = 0.0
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(tokens):
            x = emb.index_select(0, hist[L + i:L + i + 1]).view(1, 1, -1)
            logits = target.decode_step_fused(x, L + i)
            hist[L + i + 1:L + i + 2], _ = sampling.sample(logits, s, history=hist.view(1, -1), hist_lens=[L + i + 1], generator=gen,
                                                          bos_token_id=1)
        torch.cuda.synchronize()
        best = max(best, tokens / (time.perf_counter() - t0))
    target.dplan.close(); target.dplan = None
    return round(best, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "spec_h100.json"))
    ap.add_argument("--tokens", type=int, default=128)
    ap.add_argument("--draft-layers", type=int, default=2)
    ap.add_argument("--layers", type=int, default=None, help="target layers (default all 32)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("spec_bench needs a GPU")
    torch.cuda.set_device(0)
    gen = torch.Generator(device="cuda"); gen.manual_seed(2026)
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit(0), "vocab": VOCAB,
           "note": "acceptance rates of synthetic weights say nothing about real checkpoints; a round emits (1 - a^(k+1)) / (1 - a) "
                   "tokens at acceptance rate a, and us_per_round gives its cost",
           "verify_us_per_call_defaults_hist1920": verify_times(gen)}
    shape = SHAPES["7b"]
    max_seq = CTX + args.tokens + 16
    target = DecodeStack(shape, groupsize=128, device="cuda:0", max_seq=max_seq, layers=args.layers, seed=0)
    draft = DecodeStack(shape, groupsize=128, device="cuda:0", max_seq=max_seq, layers=args.draft_layers, seed=0)
    draft.norm, draft.lm_head = target.norm, target.lm_head
    emb = (target.lm_head.float() * C_EMB).half().contiguous()
    prompt = torch.randint(0, VOCAB, (CTX,), generator=torch.Generator().manual_seed(5)).tolist()
    res["model"] = {"target": f"7B g128, {target.n_layers} layers", "draft": f"7B g128, first {args.draft_layers} layers + the target's head",
                    "ctx": CTX, "tokens": args.tokens}
    res["baseline_fused_step_sample_tok_s"] = baseline(target, emb, prompt, args.tokens, gen)
    print(f"baseline: {res['baseline_fused_step_sample_tok_s']} tok/s", flush=True)
    loops, breakdown = {}, {}
    for sname, s in (("defaults", sampling.Settings()), ("greedy", greedy())):
        for k in (1, 2, 3):
            loop(target, draft, emb, prompt, s, k, 16, gen)                  # warm-up: plans, graphs of the allocator, modules
            runs = [loop(target, draft, emb, prompt, s, k, args.tokens, gen) for _ in range(2)]
            loops[f"{sname}/k{k}"] = max(runs, key=lambda r: r["tok_s"])
            loops[f"{sname}/k{k}"]["tok_s_runs"] = [r["tok_s"] for r in runs]
            breakdown[f"{sname}/k{k}"] = loop(target, draft, emb, prompt, s, k, args.tokens, gen, breakdown=True)
            print(f"loop {sname} k {k}: {loops[f'{sname}/k{k}']} | {breakdown[f'{sname}/k{k}']}", flush=True)
    res["loop_7b_ctx1920"] = loops
    res["round_breakdown"] = breakdown
    for st in (draft, target):
        st.close()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
