#!/usr/bin/env python
"""Measure batched generation (exllama_b200.generate: exl_sample_rows and exl_gen_advance over the batched decode step) on one GPU
and write one JSON file (default profiles/generate_h100.json) naming the GPU and its power limit.  Synthetic 7B (32 layers, g128),
caches for 4 sequences, max_seq 2048, random N(0, 0.25) embeddings, sampler defaults.  Traffic: 16 requests with seeded prompt
lengths in 16 .. 1536 and max_new_tokens in {32, 64, 128, 256}, arriving all at step 0 ("burst") or two every 8 steps
("staggered").  The batch and static4 arms alternate; each arm runs twice and keeps the better run:

  batch       BatchGenerator: emitted tok/s, time to first token (median, max), per step the CUDA-event time of the step, the
              sampler and the advance, and the host gap (wall time per step minus the three)
  static4     static batches of 4: submit four, run them to completion, then the next four (the burst pattern only)
  single      one request at a time through BatchGenerator on a batch-1 stack (the fused single-sequence step), run last because
              closing the batch-4 stack first frees its q4 handles
  steady      the decode loop with 4 live requests at contexts 1024 .. 1027 (+64 tokens) against bare decode_step_fused_batch at the
              same contexts: their tok/s and the ratio
  sampler     exl_sample_rows with four different settings against exl_sample at bsz 4, vocab 32000 (CUDA events, 1000 calls)

    python tools/generate_bench.py [--out profiles/generate_h100.json] [--layers N]"""
import argparse, json, os, statistics, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from bench import power_limit
from exllama_b200 import generate, sampling
from exllama_b200.stack import SHAPES, DecodeStack

MAX_SEQ = 2048


def traffic(vocab, seed=7):
    rng = np.random.default_rng(seed)
    lens = rng.integers(16, 1537, 16)
    news = rng.choice([32, 64, 128, 256], 16)
    return [(rng.integers(0, vocab, int(L)).tolist(), int(n), 100 + i) for i, (L, n) in enumerate(zip(lens, news))]


def run_batch(st, emb, reqs, stagger=0):
    gen = generate.BatchGenerator(st, emb)
    gen.timings = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ids, pending, k, step_wall = [], list(reqs), 0, []
    while True:
        if pending and (stagger == 0 or k % stagger == 0):
            for p, n, seed in pending[:len(pending) if stagger == 0 else 2]:
                ids.append(gen.submit(generate.Request(p, n, seed=seed)))
            pending = [] if stagger == 0 else pending[2:]
        ts = time.perf_counter()
        more = gen.step()
        step_wall.append(time.perf_counter() - ts)
        k += 1
        if not more and not pending:
            break
    res = gen.run()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    toks = sum(len(r.tokens) for r in res.values())
    ttft = [r.t_first for r in res.values()]
    parts = {"step_ms": [], "sample_ms": [], "advance_ms": []}
    for ev, n in gen.timings:
        for name, (a, b) in zip(parts, ((0, 1), (1, 2), (2, 3))):
            parts[name].append(ev[a].elapsed_time(ev[b]))
    dev_ms = [sum(x) for x in zip(*parts.values())]
    return {"tok_s": toks / dt, "tokens": toks, "seconds": dt, "steps": len(gen.timings),
            "ttft_median_s": statistics.median(ttft), "ttft_max_s": max(ttft),
            **{k: statistics.median(v) for k, v in parts.items()},
            "host_gap_ms_median": statistics.median([1e3 * w - d for w, d in zip(step_wall, dev_ms)]) if dev_ms else None}


def run_static4(st, emb, reqs):
    t0 = time.perf_counter()
    toks, ttft = 0, []
    for i in range(0, len(reqs), 4):
        gen = generate.BatchGenerator(st, emb)
        tb = time.perf_counter()
        for p, n, seed in reqs[i:i + 4]:
            gen.submit(generate.Request(p, n, seed=seed))
        res = gen.run()
        toks += sum(len(r.tokens) for r in res.values())
        ttft += [r.t_first + (tb - t0) for r in res.values()]
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return {"tok_s": toks / dt, "tokens": toks, "seconds": dt, "ttft_median_s": statistics.median(ttft), "ttft_max_s": max(ttft)}


def run_single(st1, emb, reqs):
    t0 = time.perf_counter()
    toks, ttft = 0, []
    gen = generate.BatchGenerator(st1, emb)
    for p, n, seed in reqs:
        tb = time.perf_counter()
        rid = gen.submit(generate.Request(p, n, seed=seed))
        r = gen.run()[rid]
        toks += len(r.tokens)
        ttft.append(r.t_first + (tb - t0))
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return {"tok_s": toks / dt, "tokens": toks, "seconds": dt, "ttft_median_s": statistics.median(ttft), "ttft_max_s": max(ttft)}


def steady(st, emb, vocab, n_tok=64):
    rng = np.random.default_rng(3)
    prompts = [rng.integers(0, vocab, 1024 + b).tolist() for b in range(4)]
    gen = generate.BatchGenerator(st, emb)
    for b, p in enumerate(prompts):              # one admission each (an admission takes at most max_seq prompt tokens)
        gen.submit(generate.Request(p, n_tok + 8, seed=b))
        gen.step()
    gen.step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n_tok - 1):
        gen.step()
    torch.cuda.synchronize()
    loop = 4 * (n_tok - 1) / (time.perf_counter() - t0)
    gen.run()
    x = emb[torch.tensor([p[-1] for p in prompts], device="cuda")].view(4, 1, -1).contiguous()
    for i in range(3):
        st.decode_step_fused_batch(x, [1024 + b + i for b in range(4)])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n_tok - 1):
        st.decode_step_fused_batch(x, [1025 + b + i for b in range(4)])
    torch.cuda.synchronize()
    bare = 4 * (n_tok - 1) / (time.perf_counter() - t0)
    return {"loop_tok_s": loop, "bare_step_tok_s": bare, "ratio": loop / bare}


def sampler_rows_vs_one(vocab=32000, calls=1000):
    g = torch.Generator(device="cuda"); g.manual_seed(1)
    logits = torch.randn((4, vocab), device="cuda", generator=g) * 3
    hist = torch.randint(0, vocab, (4, 2048), device="cuda", generator=g)
    u = torch.rand(4, device="cuda", generator=g)
    s0 = sampling.Settings()
    rows = [sampling.Settings() for _ in range(4)]
    rows[1].top_k, rows[1].top_p = 0, 0.9
    rows[2].top_k, rows[2].top_p, rows[2].typical = 0, 0.0, 0.2
    rows[3].top_k, rows[3].token_repetition_penalty_max = 1, 1.0
    out = {}
    for name, s in (("exl_sample_defaults", s0), ("exl_sample_rows_4_settings", rows), ("exl_sample_rows_4x_defaults", [s0] * 4)):
        for _ in range(10):
            sampling.sample(logits, s, history=hist, hist_lens=[1920] * 4, u=u)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(calls):
            sampling.sample(logits, s, history=hist, hist_lens=[1920] * 4, u=u)
        b.record()
        torch.cuda.synchronize()
        out[name + "_us"] = 1e3 * a.elapsed_time(b) / calls
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "generate_h100.json"))
    ap.add_argument("--layers", type=int, default=None, help="layers (default all 32)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("generate_bench needs a GPU")
    torch.cuda.set_device(0)
    shape = SHAPES["7b"]
    st = DecodeStack(shape, groupsize=128, device="cuda:0", max_seq=MAX_SEQ, layers=args.layers, seed=0, batch=4)
    emb = (torch.randn((shape.vocab, shape.hidden), device="cuda", generator=torch.Generator(device="cuda").manual_seed(11)) * 0.5).half()
    reqs = traffic(shape.vocab)
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit(0),
           "model": f"7B g128, {st.n_layers} layers, batch-4 caches, max_seq {MAX_SEQ}",
           "traffic": {"prompt_lens": [len(p) for p, _, _ in reqs], "max_new_tokens": [n for _, n, _ in reqs]},
           "settings": "sampling.Settings() defaults (temperature 0.95, top_k 40, top_p 0.65, penalty 1.15 / 256 / 128)", "arms": {}}
    run_batch(st, emb, [(p[:32], 4, s) for p, _, s in reqs[:6]])            # warm-up: plan, modules, allocator
    runs = {"batch/burst": [], "batch/staggered": [], "static4/burst": [], "single/burst": []}
    for _ in range(2):
        runs["batch/burst"].append(run_batch(st, emb, reqs))
        runs["batch/staggered"].append(run_batch(st, emb, reqs, stagger=8))
        runs["static4/burst"].append(run_static4(st, emb, reqs))
    res["steady_4_live"] = steady(st, emb, shape.vocab)
    print("steady", res["steady_4_live"], flush=True)
    res["sampler_bsz4"] = sampler_rows_vs_one()
    print("sampler", res["sampler_bsz4"], flush=True)
    st.close()                                   # before the batch-1 stack: closing a stack frees every q4 handle on the device
    st1 = DecodeStack(shape, groupsize=128, device="cuda:0", max_seq=MAX_SEQ, layers=args.layers, seed=0, batch=1)
    for _ in range(2):
        runs["single/burst"].append(run_single(st1, emb, reqs))
    st1.close()
    for k, v in runs.items():
        line = max(v, key=lambda r: r["tok_s"])
        line["tok_s_runs"] = [r["tok_s"] for r in v]
        res["arms"][k] = line
        print(k, line, flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
