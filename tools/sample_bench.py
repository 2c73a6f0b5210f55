#!/usr/bin/env python
"""Time exl_sample (csrc/sample.cu) against the host path a reference generator takes per token, and a generation loop on the 7B
synthetic stack with either sampler.  Writes one JSON file (default profiles/sample_h100.json) naming the GPU and its power limit.

  kernel      CUDA-event time per call, 1000 calls (ten replays of a CUDA graph of 100), vocab 32000, bsz 1 / 4 / 16 / 64, for the
              generator's defaults with a 1920-token history, top_k 0 + top_p 0.9, and top_k 0 + typical 0.2
  host        wall time per token of the reference's host path: logits D2H, exl_apply_rep_penalty per row, the bos logit, and a
              torch-CPU restatement of ExLlamaGenerator.sample per row (the reference itself is not needed)
  loop        7B at ctx 1920, +128 tokens, batch 1 and 4: fused step -> sample -> embedding gather -> next step, with the GPU sampler
              and with the host path, against the bare fused step

    python tools/sample_bench.py [--out profiles/sample_h100.json] [--layers N] [--tokens 128]"""
import argparse, ctypes as C, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import torch.nn.functional as F
from bench import power_limit
from exllama_b200 import capi, sampling
from exllama_b200.stack import SHAPES, DecodeStack

VOCAB = 32000
CONFIGS = {
    "defaults_hist1920": dict(temperature=0.95, top_k=40, top_p=0.65, min_p=0.0, typical=0.0, penalty=(1.15, 256, 128), hist=1920),
    "topk0_topp0.9": dict(temperature=0.95, top_k=0, top_p=0.9, min_p=0.0, typical=0.0, penalty=(1.0, -1, 0), hist=0),
    "topk0_typical0.2": dict(temperature=0.95, top_k=0, top_p=0.0, min_p=0.0, typical=0.2, penalty=(1.0, -1, 0), hist=0),
}


def settings(cfg):
    s = sampling.Settings()
    s.temperature, s.top_k, s.top_p, s.min_p, s.typical = (cfg[k] for k in ("temperature", "top_k", "top_p", "min_p", "typical"))
    (s.token_repetition_penalty_max, s.token_repetition_penalty_sustain, s.token_repetition_penalty_decay) = cfg["penalty"]
    return s


def host_sample(logits, s):
    """ExLlamaGenerator.sample restated in torch on the CPU for one row: softmax, a sort or topk, the top-p and typical loops
    with .item() sums, and one multinomial draw."""
    logits = logits / s.temperature + 1e-8
    probs = torch.softmax(logits, dim=-1)
    if s.top_k == 0:
        top_probs, top_ids = torch.sort(probs, descending=True)
    else:
        top_probs, top_ids = torch.topk(probs, s.top_k)
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
        top_probs, top_ids = F.normalize(top_probs[:n], p=1, dim=-1), top_ids[:n]
    if s.typical > 0.0:
        lp = (top_probs + 1e-10).log()
        dev = ((top_probs * lp).sum() - lp).abs()
        order = torch.sort(dev).indices
        top_probs, top_ids = top_probs[order], top_ids[order]
        n, cum = 0, top_probs[0].item()
        while True:
            n += 1
            if n == top_probs.shape[-1]:
                break
            cum += top_probs[n].item()
            if cum > s.typical:
                break
        top_probs, top_ids = F.normalize(top_probs[:n], p=1, dim=-1), top_ids[:n]
    i = torch.multinomial(top_probs, 1)
    return top_ids[i], top_probs[i]


def host_path(logits_dev, s, hist_np, bos, parts):
    """One token per row the reference's way; adds the wall time of each part to parts."""
    lib = capi.lib()
    t0 = time.perf_counter()
    lg = logits_dev.cpu()
    t1 = time.perf_counter()
    pm, sus, dec = s.token_repetition_penalty_max, s.token_repetition_penalty_sustain, s.token_repetition_penalty_decay
    if hist_np is not None:
        for b in range(lg.shape[0]):
            row = lg[b]
            capi.check(lib.exl_apply_rep_penalty(VOCAB, hist_np[b].ctypes.data, pm, sus, dec, hist_np.shape[1], C.c_void_p(row.data_ptr())))
    t2 = time.perf_counter()
    lg[:, bos] = -10000.0
    t3 = time.perf_counter()
    toks = torch.cat([host_sample(lg[b], s)[0] for b in range(lg.shape[0])])
    t4 = time.perf_counter()
    for k, v in zip(("d2h", "rep_penalty", "bos", "sample"), (t1 - t0, t2 - t1, t3 - t2, t4 - t3)):
        parts[k] = parts.get(k, 0.0) + v
    return toks


def kernel_times(gen):
    out = {}
    for name, cfg in CONFIGS.items():
        for bsz in (1, 4, 16, 64):
            s = settings(cfg)
            logits = torch.randn((bsz, VOCAB), device="cuda", generator=gen) * 2.5
            hist = torch.randint(0, VOCAB, (bsz, max(cfg["hist"], 1)), device="cuda", generator=gen) if cfg["hist"] else None
            u = torch.rand(bsz, device="cuda", generator=gen)
            for _ in range(3):
                sampling.sample(logits, s, history=hist, u=u, bos_token_id=1)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for _ in range(100):
                    sampling.sample(logits, s, history=hist, u=u, bos_token_id=1)
            g.replay(); torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                g.replay()
            e1.record(); torch.cuda.synchronize()
            out[f"{name}/bsz{bsz}"] = round(e0.elapsed_time(e1) * 1000 / 1000, 2)      # us per call
            print(f"kernel {name} bsz {bsz}: {out[f'{name}/bsz{bsz}']} us", flush=True)
    return out


def host_times(gen):
    out = {}
    s = settings(CONFIGS["defaults_hist1920"])
    for bsz in (1, 4, 16, 64):
        logits = torch.randn((bsz, VOCAB), device="cuda", generator=gen) * 2.5
        hist = np.random.default_rng(bsz).integers(0, VOCAB, size=(bsz, 1920)).astype(np.int64)
        iters = max(10, 400 // bsz)
        host_path(logits, s, hist, 1, {})
        parts = {}
        torch.cuda.synchronize()
        for _ in range(iters):
            host_path(logits, s, hist, 1, parts)
        out[f"bsz{bsz}"] = {k: round(v / iters * 1e6, 1) for k, v in parts.items()}
        out[f"bsz{bsz}"]["total"] = round(sum(parts.values()) / iters * 1e6, 1)
        print(f"host bsz {bsz}: {out[f'bsz{bsz}']} us per token step", flush=True)
    return out


def loop_times(args, gen):
    shape = SHAPES["7b"]
    out = {}
    s = sampling.Settings()
    ctx = 1920
    emb = (torch.randn((VOCAB, shape.hidden), device="cuda", generator=gen) * 0.5).half()
    for bsz in (1, 4):
        st = DecodeStack(shape, groupsize=128, device="cuda:0", max_seq=ctx + args.tokens + 8, layers=args.layers, batch=bsz)
        for kc, vc in zip(st.key_cache, st.value_cache):
            kc.normal_(0, 0.5, generator=gen); vc.normal_(0, 0.5, generator=gen)
        st.make_plan()
        hist = torch.randint(0, VOCAB, (bsz, ctx + args.tokens), device="cuda", generator=gen)
        step = (lambda x, p: st.decode_step_fused(x, p[0]).view(1, -1)) if bsz == 1 else st.decode_step_fused_batch
        x0 = emb[hist[:, ctx - 1]].view(bsz, 1, shape.hidden)
        rng_u = torch.Generator(device="cuda"); rng_u.manual_seed(5)

        def run(mode):
            x = x0.clone()
            h_np = hist.cpu().numpy()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(args.tokens):
                past = ctx + i
                logits = step(x, [past] * bsz)
                if mode == "bare":
                    continue
                if mode == "gpu":
                    tok, _ = sampling.sample(logits, s, history=hist, hist_lens=[past] * bsz, generator=rng_u, bos_token_id=1)
                else:
                    tok = host_path(logits, s, h_np[:, :past], 1, {}).to("cuda")
                hist[:, past] = tok
                x = emb.index_select(0, tok).view(bsz, 1, shape.hidden)
            torch.cuda.synchronize()
            return (time.perf_counter() - t0)

        for mode in ("bare", "gpu", "host"):
            run(mode)                                        # warm-up
        res = {}
        for mode in ("bare", "gpu", "host", "bare", "gpu", "host"):
            dt = run(mode)
            res.setdefault(mode, []).append(bsz * args.tokens / dt)
        out[f"batch{bsz}"] = {m: round(max(v), 1) for m, v in res.items()}
        out[f"batch{bsz}"]["gpu_vs_bare"] = round(out[f"batch{bsz}"]["gpu"] / out[f"batch{bsz}"]["bare"], 4)
        out[f"batch{bsz}"]["host_vs_bare"] = round(out[f"batch{bsz}"]["host"] / out[f"batch{bsz}"]["bare"], 4)
        print(f"loop batch {bsz}: {out[f'batch{bsz}']} tok/s", flush=True)
        st.dplan.close(); st.close()
        del st
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "sample_h100.json"))
    ap.add_argument("--layers", type=int, default=None, help="7B stack layers (default all 32)")
    ap.add_argument("--tokens", type=int, default=128)
    ap.add_argument("--skip-loop", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sample_bench needs a GPU")
    torch.cuda.set_device(0)
    gen = torch.Generator(device="cuda"); gen.manual_seed(2026)
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit(0), "vocab": VOCAB,
           "kernel_us_per_call": kernel_times(gen), "host_path_us_per_step": host_times(gen),
           "torch_threads": torch.get_num_threads()}
    if not args.skip_loop:
        res["loop_7b_ctx1920_plus%d_tok_s" % args.tokens] = loop_times(args, gen)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
