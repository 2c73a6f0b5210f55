#!/usr/bin/env python
"""Measure beam search (exllama_b200.beam: exl_beam_select, exl_kv_copy_rows over the batched decode step) on one GPU and write one
JSON file (default profiles/beam_h100.json) naming the GPU and its power limit.  Everything is measured in one process, on the
synthetic 7B (32 layers, g128) with a --ctx-token prompt and --tokens emitted tokens, for beams 1 / 2 / 4 x beam_length 1 / 4 / 8:

  device      BeamSearch.generate: emitted tok/s; per expansion the CUDA-event time of the step, the sampler, the selection, the host
              read and host bookkeeping (the device idles between the selection and the copies), and the copies with the history
              updates; the host clock time spent in the selection read (it includes waiting for the expansion's device work); the
              mean number of live beams; and the prompt copy of begin() (exl_kv_copy_rows of rows [0, ctx) to beams - 1 sequences,
              CUDA events over five calls)
  reference   the reference's loop restated on the same stack: per expansion one per-op decode_step(seq=b) per beam, the logits to
              the host, the host penalty and the reference's torch sampler on the CPU, torch sorting for the selection and one torch
              copy per layer, K and V for each cloned beam's window rows
The two arms alternate (device, reference, device, reference) and each line keeps the better of its two runs.  The embeddings are
random N(0, 0.25): tied ones make the synthetic stack repeat its input token with one-token kept sets, and beams would never branch.

    python tools/beam_bench.py [--out profiles/beam_h100.json] [--tokens 128] [--ctx 1920] [--layers N]"""
import argparse, json, math, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import torch.nn.functional as F
from bench import power_limit
from exllama_b200 import beam, cuda_ext, sampling
from exllama_b200.stack import SHAPES, DecodeStack


def device_arm(st, emb, prompt, beams, beam_length, tokens, gen):
    bs = beam.BeamSearch(st, emb, beams, beam_length, settings=sampling.Settings(), bos_token_id=1, generator=gen)
    bs.begin(prompt)
    bs.timings = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    bs.generate(tokens)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    parts = {"step": 0.0, "sample": 0.0, "select": 0.0, "host_read_and_bookkeeping": 0.0, "copy_and_history": 0.0}
    read, live = 0.0, 0
    for ev, t_read, nb in bs.timings:
        for name, (a, b) in zip(parts, ((0, 1), (1, 2), (2, 3), (3, 4), (4, 5))):
            parts[name] += ev[a].elapsed_time(ev[b]) * 1000
        read += t_read * 1e6
        live += nb
    n = max(len(bs.timings), 1)
    out = {"tok_s": round(tokens / dt, 1), "expansions": len(bs.timings), "mean_live_beams": round(live / n, 2),
           "us_per_expansion": {k: round(v / n, 1) for k, v in parts.items()}, "read_wait_us": round(read / n, 1)}
    bs.end()
    return out


def prompt_copy_us(st, beams, L):
    if beams < 2:
        return None
    pairs = [(0, j, 0, L) for j in range(1, beams)]
    beam.copy_cache_rows(st, pairs)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        beam.copy_cache_rows(st, pairs)
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1000 / 5
    nbytes = 2 * st.n_layers * st.key_cache[0].shape[1] * L * st.shape.head_dim * 2 * (beams - 1) * 2   # read + write
    return {"us": round(us, 1), "GB_s": round(nbytes / us / 1e3, 1)}


def host_sample(logits, s, num):
    """generator.py:91-170 on the host (float32 torch on the CPU): the reference's sampler."""
    logits = logits / s.temperature + 1e-8
    probs = torch.softmax(logits, dim=-1)
    if s.top_k == 0:
        top_probs, top_indices = torch.sort(probs, descending=True)
    else:
        top_probs, top_indices = torch.topk(probs, s.top_k)
        top_probs = F.normalize(top_probs, p=1, dim=-1)
    if s.top_p > 0.0:
        n, cum = 0, top_probs[0].item()
        while True:
            n += 1
            if n == top_probs.shape[-1] or top_probs[n].item() < s.min_p:
                break
            cum += top_probs[n].item()
            if cum > s.top_p:
                break
        top_probs = F.normalize(top_probs[:n], p=1, dim=-1)
        top_indices = top_indices[:n]
    ind = torch.multinomial(top_probs, top_probs.shape[-1] if num == -1 else min(num, top_probs.shape[-1]))
    toks, ps = top_indices[ind], top_probs[ind]
    toks, o = toks.sort()
    return toks, ps[o]


def reference_arm(st, emb, prompt, beams, beam_length, tokens):
    """The reference's loop, restated: per-op steps one beam at a time, host sampling, torch selection and torch cache copies."""
    s = sampling.Settings()
    L = len(prompt)
    ids = torch.tensor(prompt, device="cuda")
    logits = st.prefill(emb[ids].view(1, L, -1), 0, seq=0)
    seq = list(prompt)
    mbl = min(st.max_seq - beam_length, beam_length)

    def penalised(lg, toks):
        x = lg.float().cpu()
        cuda_ext.ext_apply_rep_penalty_mask_cpu(torch.tensor([toks]), s.token_repetition_penalty_max, s.token_repetition_penalty_sustain,
                                                s.token_repetition_penalty_decay, x)
        return x.view(-1)

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    toks, ps = host_sample(penalised(logits, seq), s, beams)
    bl = [([int(t)], [float(p)], j) for j, (t, p) in enumerate(zip(toks.tolist(), ps.tolist()))]
    for j in range(1, len(bl)):
        for c in st.key_cache + st.value_cache:
            c[j, :, :L].copy_(c[0, :, :L])
    emitted = 0
    while emitted < tokens:
        while len(bl[0][0]) < mbl:
            n, m = len(seq), len(bl[0][0])
            pos = n + m - 1
            t_all, p_all, c_all, b_all = [], [], [], []
            for i, (w, pr, slot) in enumerate(bl):
                full = seq + w
                lg = st.decode_step(emb[full[-1]].view(1, 1, -1).clone(), pos, seq=slot)
                tk, pk = host_sample(penalised(lg, full), s, -1)
                t_all.append(tk); p_all.append(pk)
                c_all.append(torch.log(pk) + sum(math.log(x) for x in pr)); b_all.append(torch.full((tk.shape[0],), i))
            t_all, p_all, c_all, b_all = (torch.cat(x) for x in (t_all, p_all, c_all, b_all))
            c_all, o = c_all.sort(descending=True)
            t_all, p_all, b_all = (x[o][:beams] for x in (t_all, p_all, b_all))
            b_all, o = b_all.sort()
            t_all, p_all = t_all[o], p_all[o]
            used, new = set(), []
            free = [j for j in range(beams) if j not in {bl[int(b)][2] for b in b_all}]
            for t, p, b in zip(t_all.tolist(), p_all.tolist(), b_all.tolist()):
                w, pr, slot = bl[b]
                if slot not in used:
                    used.add(slot)
                    new.append((w + [t], pr + [p], slot))
                    continue
                d = free.pop(0)
                for c in st.key_cache + st.value_cache:
                    c[d, :, n:pos + 1].copy_(c[slot, :, n:pos + 1])
                new.append((w + [t], pr + [p], d))
            bl = new
        sc = [sum(math.log(x) for x in pr) for _, pr, _ in bl]
        best = max(range(len(bl)), key=lambda i: (sc[i], -i))
        t = bl[best][0][0]
        seq.append(t)
        emitted += 1
        bl = [bl[best]] + [b for i, b in enumerate(bl) if i != best and b[0][0] == t]
        bl = [(w[1:], pr[1:], slot) for w, pr, slot in bl]
    torch.cuda.synchronize()
    return {"tok_s": round(tokens / (time.perf_counter() - t0), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "beam_h100.json"))
    ap.add_argument("--tokens", type=int, default=128)
    ap.add_argument("--ctx", type=int, default=1920)
    ap.add_argument("--layers", type=int, default=None, help="layers (default all 32)")
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("beam_bench needs a GPU")
    torch.cuda.set_device(0)
    shape = SHAPES["7b"]
    st = DecodeStack(shape, groupsize=128, device="cuda:0", max_seq=args.ctx + args.tokens + 16, layers=args.layers, seed=0, batch=4)
    emb = (torch.randn((shape.vocab, shape.hidden), device="cuda", generator=torch.Generator(device="cuda").manual_seed(11)) * 0.5).half()
    prompt = torch.randint(0, shape.vocab, (args.ctx,), generator=torch.Generator().manual_seed(5)).tolist()
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit(0),
           "model": f"7B g128, {st.n_layers} layers, batch-4 caches", "ctx": args.ctx, "tokens": args.tokens,
           "settings": "sampling.Settings() defaults (temperature 0.95, top_k 40, top_p 0.65, penalty 1.15 / 256 / 128), bos 1",
           "lines": {}}
    gen = torch.Generator(device="cuda"); gen.manual_seed(2026)
    device_arm(st, emb, prompt[:64], 2, 2, 4, gen)                          # warm-up: plan, modules, allocator
    for beams in (1, 2, 4):
        for bl in (1, 4, 8):
            runs_d, runs_r = [], []
            for _ in range(2):
                runs_d.append(device_arm(st, emb, prompt, beams, bl, args.tokens, gen))
                if not args.no_reference:
                    runs_r.append(reference_arm(st, emb, prompt, beams, bl, args.tokens))
            line = max(runs_d, key=lambda r: r["tok_s"])
            line["tok_s_runs"] = [r["tok_s"] for r in runs_d]
            line["prompt_copy"] = prompt_copy_us(st, beams, args.ctx)
            if runs_r:
                line["reference_loop_tok_s"] = max(r["tok_s"] for r in runs_r)
                line["reference_loop_tok_s_runs"] = [r["tok_s"] for r in runs_r]
            res["lines"][f"beams{beams}/len{bl}"] = line
            print(f"beams {beams} beam_length {bl}: {line}", flush=True)
    st.close()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
