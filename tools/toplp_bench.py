#!/usr/bin/env python
"""Measure the log-probabilities of generated tokens (exl_top_logprobs, Request(logprobs=) in exllama_b200.generate) on one GPU and
write one JSON file (default profiles/toplp_h100.json) naming the GPU and its power limit, both read in the same run.

  kernel   exl_top_logprobs in us per call (CUDA events, 200 calls per run, median of 5 alternating runs) at bsz 1, 4, 16, 64, vocab
           32000 and 128256, N 0, 5, 20, with each row's token given, against the torch program it replaces: log_softmax in fp32,
           gather of the tokens, topk of N (N 0: log_softmax and gather only)
  loop     BatchGenerator on tools/generate_bench.py's traffic (16 requests arriving at step 0, synthetic 7B g128, batch-4 caches,
           max_seq 2048, sampler defaults) with logprobs=5 on every request against none; the arms alternate, three runs each;
           medians of tok/s and of the per-step CUDA-event time of the sampler span (which holds exl_top_logprobs when a row asks)
  steady   the decode loop with 4 live requests at contexts 1024 .. 1027 (+64 tokens), with logprobs=5 against none, alternating,
           three runs each: median tok/s and the ratio

    python tools/toplp_bench.py [--out profiles/toplp_h100.json] [--layers N]"""
import argparse, json, os, statistics, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
import torch
from bench import power_limit
from exllama_b200 import generate, sampling
from exllama_b200.stack import SHAPES, DecodeStack
from generate_bench import traffic

MAX_SEQ = 2048
N_LOOP = 5


def kernel_times(calls=200, runs=5):
    out = {}
    g = torch.Generator(device="cuda"); g.manual_seed(3)
    for vocab in (32000, 128256):
        for bsz in (1, 4, 16, 64):
            logits = torch.randn((bsz, vocab), device="cuda", generator=g) * 3
            tok = torch.randint(0, vocab, (bsz,), device="cuda", generator=g)
            for n in (0, 5, 20):
                def torch_arm():
                    l = torch.log_softmax(logits, -1)
                    lp = l.gather(1, tok.view(-1, 1))
                    if n:
                        torch.topk(l, n, dim=-1)
                    return lp
                arms = {"exl_top_logprobs": lambda: sampling.top_logprobs(logits, n, tok), "torch_log_softmax_gather_topk": torch_arm}
                res = {k: [] for k in arms}
                for fn in arms.values():
                    for _ in range(10):
                        fn()
                for _ in range(runs):
                    for k, fn in arms.items():
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        for _ in range(calls):
                            fn()
                        e1.record()
                        e1.synchronize()
                        res[k].append(1e3 * e0.elapsed_time(e1) / calls)
                key = f"vocab{vocab}/bsz{bsz}/n{n}"
                out[key] = {k: statistics.median(v) for k, v in res.items()}
                out[key]["ratio"] = out[key]["exl_top_logprobs"] / out[key]["torch_log_softmax_gather_topk"]
                print(key, out[key], flush=True)
    return out


def run_loop(st, emb, reqs, logprobs):
    gen = generate.BatchGenerator(st, emb)
    gen.timings = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for p, n, seed in reqs:
        gen.submit(generate.Request(p, n, seed=seed, logprobs=logprobs))
    res = gen.run()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    toks = sum(len(r.tokens) for r in res.values())
    assert all((r.logprobs is not None) == bool(logprobs) for r in res.values())
    return {"tok_s": toks / dt, "tokens": toks, "steps": len(gen.timings),
            "sampler_span_ms": statistics.median(ev[1].elapsed_time(ev[2]) for ev, _ in gen.timings)}


def steady(st, emb, vocab, logprobs, n_tok=64):
    rng = np.random.default_rng(3)
    prompts = [rng.integers(0, vocab, 1024 + b).tolist() for b in range(4)]
    gen = generate.BatchGenerator(st, emb)
    for b, p in enumerate(prompts):
        gen.submit(generate.Request(p, n_tok + 8, seed=b, logprobs=logprobs))
        gen.step()
    gen.step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n_tok - 1):
        gen.step()
    torch.cuda.synchronize()
    loop = 4 * (n_tok - 1) / (time.perf_counter() - t0)
    gen.run()
    return loop


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "toplp_h100.json"))
    ap.add_argument("--layers", type=int, default=None, help="layers (default all 32)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("toplp_bench needs a GPU")
    torch.cuda.set_device(0)
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit(0)}
    res["kernel_us"] = kernel_times()
    shape = SHAPES["7b"]
    st = DecodeStack(shape, groupsize=128, device="cuda:0", max_seq=MAX_SEQ, layers=args.layers, seed=0, batch=4)
    emb = (torch.randn((shape.vocab, shape.hidden), device="cuda", generator=torch.Generator(device="cuda").manual_seed(11)) * 0.5).half()
    reqs = traffic(shape.vocab)
    res["model"] = f"7B g128, {st.n_layers} layers, batch-4 caches, max_seq {MAX_SEQ}"
    res["settings"] = "sampling.Settings() defaults; logprobs=5 on every request in the 'on' arms"
    run_loop(st, emb, [(p[:32], 4, s) for p, _, s in reqs[:6]], N_LOOP)     # warm-up: plan, modules, allocator
    loops = {"off": [], "on": []}
    stead = {"off": [], "on": []}
    for _ in range(3):
        for arm, n in (("off", 0), ("on", N_LOOP)):
            loops[arm].append(run_loop(st, emb, reqs, n))
            stead[arm].append(steady(st, emb, shape.vocab, n))
            print(arm, loops[arm][-1], stead[arm][-1], flush=True)
    res["loop"] = {arm: {"tok_s_median": statistics.median(r["tok_s"] for r in v), "tok_s_runs": [r["tok_s"] for r in v],
                         "sampler_span_ms_median": statistics.median(r["sampler_span_ms"] for r in v)} for arm, v in loops.items()}
    res["loop"]["ratio"] = res["loop"]["on"]["tok_s_median"] / res["loop"]["off"]["tok_s_median"]
    res["steady_4_live"] = {arm: {"tok_s_median": statistics.median(v), "tok_s_runs": v} for arm, v in stead.items()}
    res["steady_4_live"]["ratio"] = res["steady_4_live"]["on"]["tok_s_median"] / res["steady_4_live"]["off"]["tok_s_median"]
    st.close()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
