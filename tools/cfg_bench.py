#!/usr/bin/env python
"""Measure classifier-free guidance (exl_cfg_mix, guided requests in exllama_b200.generate) on one GPU and write one JSON file
(default profiles/cfg_h100.json) naming the GPU and its power limit, both read in the same run.

  kernel      exl_cfg_mix in us per call (CUDA events, 200 calls, best of 3) at vocab 32000 and 128256 for 1, 2 and 32 pairs, with the default
              penalty (1.15 / 256 / 128) on a 1920-token history and with none, against the torch device program the reference runs
              after its penalty (log_softmax of every row, then (1 - alpha) * l_a + alpha * l_b); the two arms alternate
  generation  synthetic 7B (32 layers, g128), caches for 4 sequences, max_seq 2048, random N(0, 0.25) embeddings, sampler defaults;
              two guided requests (alpha 1.5) with prompts of 1500 / 1400 and 1900 / 1700 tokens, 128 tokens each:
                guided     BatchGenerator: emitted tok/s and the median per-step CUDA-event split (step, mix, sampler, advance)
                reference  example_cfg.py's loop restated on the same stack, one pair at a time: a batch-2 fused step, the logits to
                           the host, exl_apply_rep_penalty per row, torch log_softmax and the mix, and tools/sample_bench.py's host
                           sampler; per-part wall times
                unguided   the two prompts as plain requests through BatchGenerator
              the arms alternate; each runs twice and keeps the better run

    python tools/cfg_bench.py [--out profiles/cfg_h100.json] [--layers N]"""
import argparse, ctypes as C, json, os, statistics, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
import torch
from bench import power_limit
from exllama_b200 import capi, cfg, generate, sampling
from exllama_b200.stack import SHAPES, DecodeStack
from sample_bench import host_sample

MAX_SEQ = 2048
ALPHA = 1.5


def kernel_times(calls=200):
    out = {}
    g = torch.Generator(device="cuda"); g.manual_seed(3)
    for vocab in (32000, 128256):
        for n_pairs in (1, 2, 32):
            rows = 2 * n_pairs
            logits = torch.randn((rows, vocab), device="cuda", generator=g) * 3
            hist = torch.randint(0, vocab, (rows, 1920), device="cuda", generator=g)
            pairs = [(2 * k, 2 * k + 1) for k in range(n_pairs)]
            for pen_name, pen in (("penalty_1920", (1.15, 256, 128)), ("no_penalty", (1.0, -1, 0))):
                s = sampling.Settings()
                s.token_repetition_penalty_max, s.token_repetition_penalty_sustain, s.token_repetition_penalty_decay = pen
                # in place, so the kernel arm mixes its own output again: alpha 0.5 keeps those rows bounded (|w_a| + |w_b| = 1),
                # where a larger |w_a| + |w_b| would grow them call after call until exp underflows; the work does not depend on alpha
                arms = {
                    "exl_cfg_mix": lambda: cfg.mix(logits, pairs, [0.5] * n_pairs, s, history=hist, hist_lens=[1920] * rows),
                    "torch_log_softmax_mix": lambda: (1 - ALPHA) * torch.log_softmax(logits[0::2], -1) + ALPHA * torch.log_softmax(logits[1::2], -1),
                }
                res = {k: [] for k in arms}
                for k, fn in arms.items():
                    for _ in range(10):
                        fn()
                for rep in range(3):
                    for k, fn in arms.items():
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        for _ in range(calls):
                            fn()
                        e1.record()
                        e1.synchronize()
                        res[k].append(1e3 * e0.elapsed_time(e1) / calls)
                key = f"vocab{vocab}/pairs{n_pairs}/{pen_name}"
                out[key] = {k: min(v) for k, v in res.items()}
                if pen_name == "penalty_1920":
                    out[key]["torch_log_softmax_mix"] = None      # the torch arm has no penalty: compared on the no-penalty line
                print(key, out[key], flush=True)
    return out


def prompts(vocab, seed=5):
    rng = np.random.default_rng(seed)
    return [(rng.integers(0, vocab, a).tolist(), rng.integers(0, vocab, b).tolist()) for a, b in ((1500, 1400), (1900, 1700))]


def run_generator(st, emb, pairs, guided, n_tok=128):
    gen = generate.BatchGenerator(st, emb)
    gen.timings = []
    mix_ev = []
    orig = gen.dev._mix

    def timed_mix(*a):
        e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        e[0].record()
        r = orig(*a)
        e[1].record()
        mix_ev.append(e)
        return r

    gen.dev._mix = timed_mix
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i, (p, q) in enumerate(pairs):
        gen.submit(generate.Request(p, n_tok, seed=i, cfg_prompt=q if guided else None, cfg_alpha=ALPHA))
    res = gen.run()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    toks = sum(len(r.tokens) for r in res.values())
    assert all(len(r.tokens) == n_tok for r in res.values()), [r.finish for r in res.values()]
    # the step's events: start, after the step, after mix + sampler, after the advance; the mix's own pair is inside the second span
    n_adm = len(mix_ev) - len(gen.timings)
    split = {"step_ms": [], "mix_ms": [], "sampler_ms": [], "advance_ms": []}
    for (ev, _), me in zip(gen.timings, mix_ev[n_adm:] if n_adm >= 0 else mix_ev):
        m = me[0].elapsed_time(me[1])
        split["step_ms"].append(ev[0].elapsed_time(ev[1]))
        split["mix_ms"].append(m)
        split["sampler_ms"].append(ev[1].elapsed_time(ev[2]) - m)
        split["advance_ms"].append(ev[2].elapsed_time(ev[3]))
    return {"tok_s": toks / dt, "tokens": toks, "seconds": dt, "steps": len(gen.timings),
            **{k: statistics.median(v) for k, v in split.items()}}


def run_reference(st, emb, pairs, n_tok=128):
    """example_cfg.generate_cfg restated: per pair, both prompts prefilled into cache sequences 0 and 1, then per token a batch-2
    fused step, the logits to the host, the penalty per row, log_softmax and the mix in torch on the host, the host sampler."""
    lib = capi.lib()
    s = sampling.Settings()
    V = st.shape.vocab
    parts = {"step": 0.0, "d2h": 0.0, "rep_penalty": 0.0, "log_softmax_mix": 0.0, "sample": 0.0}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    toks = 0
    for p, q in pairs:
        hist = [np.array(p, np.int64), np.array(q, np.int64)]
        # one prefill per prompt: the prefill's scratch holds max_seq rows
        logits = torch.cat([st.prefill_ragged(emb[torch.tensor(x, device="cuda")], [len(x)], [0], seqs=[r], last_only=True)
                            for r, x in enumerate((p, q))])
        for j in range(n_tok):
            ta = time.perf_counter()
            lg = logits.cpu()
            tb = time.perf_counter()
            for r in range(2):
                capi.check(lib.exl_apply_rep_penalty(V, hist[r].ctypes.data, s.token_repetition_penalty_max, s.token_repetition_penalty_sustain,
                                                     s.token_repetition_penalty_decay, len(hist[r]), C.c_void_p(lg[r].data_ptr())))
            tc = time.perf_counter()
            ls = torch.log_softmax(lg, dim=-1)
            mixed = (1 - ALPHA) * ls[0] + ALPHA * ls[1]
            td = time.perf_counter()
            t = int(host_sample(mixed, s)[0])
            te = time.perf_counter()
            toks += 1
            for r in range(2):
                hist[r] = np.append(hist[r], t)
            if j + 1 < n_tok:
                x = emb[torch.tensor([t, t], device="cuda")].view(2, 1, -1)
                logits = st.decode_step_fused_batch(x, [len(hist[0]) - 1, len(hist[1]) - 1])
                torch.cuda.synchronize()
            tf = time.perf_counter()
            for k, v in zip(parts, (tf - te, tb - ta, tc - tb, td - tc, te - td)):
                parts[k] += v
    dt = time.perf_counter() - t0
    return {"tok_s": toks / dt, "tokens": toks, "seconds": dt, **{k + "_ms_per_token": 1e3 * v / toks for k, v in parts.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "cfg_h100.json"))
    ap.add_argument("--layers", type=int, default=None, help="layers (default all 32)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("cfg_bench needs a GPU")
    torch.cuda.set_device(0)
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit(0), "alpha": ALPHA}
    res["kernel_us"] = kernel_times()
    shape = SHAPES["7b"]
    st = DecodeStack(shape, groupsize=128, device="cuda:0", max_seq=MAX_SEQ, layers=args.layers, seed=0, batch=4)
    st.make_plan()
    emb = (torch.randn((shape.vocab, shape.hidden), device="cuda", generator=torch.Generator(device="cuda").manual_seed(11)) * 0.5).half()
    pairs = prompts(shape.vocab)
    res["model"] = f"7B g128, {st.n_layers} layers, batch-4 caches, max_seq {MAX_SEQ}"
    res["requests"] = {"prompt_lens": [[len(p), len(q)] for p, q in pairs], "new_tokens": 128,
                       "settings": "sampling.Settings() defaults (temperature 0.95, top_k 40, top_p 0.65, penalty 1.15 / 256 / 128)"}
    short = [(p[:64], q[:48]) for p, q in pairs]
    run_generator(st, emb, short, True, 8); run_reference(st, emb, short[:1], 4); run_generator(st, emb, short, False, 8)   # warm-up
    runs = {"guided": [], "reference": [], "unguided": []}
    for _ in range(2):
        runs["guided"].append(run_generator(st, emb, pairs, True))
        runs["reference"].append(run_reference(st, emb, pairs))
        runs["unguided"].append(run_generator(st, emb, pairs, False))
    res["arms"] = {}
    for k, v in runs.items():
        line = max(v, key=lambda r: r["tok_s"])
        line["tok_s_runs"] = [r["tok_s"] for r in v]
        res["arms"][k] = line
        print(k, line, flush=True)
    st.close()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
