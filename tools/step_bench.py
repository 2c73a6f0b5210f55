#!/usr/bin/env python
"""Time the whole-token persistent kernel (csrc/decode_step.cu) next to the per-op path on the synthetic stack.
Accepts the SHAPES names and the grouped-query attention ones (GQA_SHAPES, e.g. 70b); the line records the GPU and its power limit.
--batch N times one launch for N sequences, all at --ctx (aggregate tok/s = N tokens per launch; bytes = weights + head + N x K/V);
the per-op arm then times sequence 0 alone.
--tokens K[,K...] times the multi-token step (K consecutive tokens of one sequence per launch, token t at --ctx + t) against one
fused step, K fused steps, the batch-K launch (where the model allows it) and DecodeStack.prefill of K tokens at past_len --ctx, the
arms alternating in rounds; one line per K.
--lora-rank R attaches a synthetic LoRA adapter of rank R (DecodeStack.add_lora) to q and v (--lora-targets qv) or to all seven
projections (all); both arms then run it.
    python tools/step_bench.py [--model 7b] [--ctx 1920] [--seq 2048] [--groupsize 128] [--act-order] [--layers N] [--reps 20] [--batch N]
                               [--lora-rank R] [--lora-targets qv|all] [--tokens 1,2,3,4]"""
import argparse, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from bench import power_limit
from exllama_b200.stack import GQA_SHAPES, SHAPES, DecodeStack, _Arena

MIN_WINDOW_S = 1.2          # timed window per arm


def device_bytes(shape, layers, groupsize, seq, batch=1):
    """What DecodeStack allocates on the device, roughly: q4 tensors, lm_head, KV caches, prepare_buffers scratch."""
    h, hq, hkv, i = shape.hidden, shape.heads * shape.head_dim, shape.kv_heads * shape.head_dim, shape.inter
    per_layer = (_Arena.q4_bytes(h, hq, groupsize) + 2 * _Arena.q4_bytes(h, hkv, groupsize) + _Arena.q4_bytes(hq, h, groupsize) +
                 2 * _Arena.q4_bytes(h, i, groupsize) + _Arena.q4_bytes(i, h, groupsize))
    kv = 2 * layers * seq * hkv * 2 * batch
    scratch = seq * i * 2 + h * i * 2 + (1 << 20)
    return per_layer * layers + shape.vocab * h * 2 + kv + scratch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="7b"); ap.add_argument("--ctx", type=int, default=1920); ap.add_argument("--seq", type=int, default=2048)
    ap.add_argument("--groupsize", type=int, default=128); ap.add_argument("--layers", type=int, default=None)
    ap.add_argument("--act-order", action="store_true", help="act-order (g_idx) matrices")
    ap.add_argument("--reps", type=int, default=20, help="minimum timed steps per arm (more if the window would be under 1.2 s)")
    ap.add_argument("--no-per-op", action="store_true")
    ap.add_argument("--batch", type=int, default=1, help="sequences per launch (1..4, as far as the model fits)")
    ap.add_argument("--lora-rank", type=int, default=0, help="rank of a synthetic LoRA adapter (0: none)")
    ap.add_argument("--lora-targets", choices=["qv", "all"], default="qv", help="projections the adapter covers")
    ap.add_argument("--tokens", default=None, help="comma-separated token counts of the multi-token step (1..4)")
    args = ap.parse_args()
    shapes = {**SHAPES, **GQA_SHAPES}
    if args.model not in shapes:
        sys.exit(f"unknown model {args.model!r}; one of {sorted(shapes)}")
    shape = shapes[args.model]
    layers = args.layers if args.layers is not None else shape.layers
    if args.tokens:
        args.batch = max(int(k) for k in args.tokens.split(","))          # the batch-K arm's caches
    need = device_bytes(shape, layers, args.groupsize, args.seq, args.batch)
    free, total = torch.cuda.mem_get_info()
    if need > free * 0.95:
        sys.exit(f"{args.model}: about {need / 1e9:.1f} GB needed, {free / 1e9:.1f} GB of {total / 1e9:.1f} GB free on this GPU; use --layers")
    st = DecodeStack(shape, groupsize=args.groupsize, act_order=args.act_order, device="cuda:0", max_seq=args.seq, layers=args.layers,
                     batch=args.batch)
    for kc, vc in zip(st.key_cache, st.value_cache):
        kc.normal_(0, 0.5); vc.normal_(0, 0.5)
    if args.lora_rank:
        st.add_lora(args.lora_rank, targets=("q", "v") if args.lora_targets == "qv" else "all")
    if args.tokens:
        return multi_tokens(args, st, shape)
    st.make_plan()
    nb = args.batch
    xb = (torch.randn((nb, 1, shape.hidden), device="cuda") * 0.5).half()
    x = xb[:1]

    def timed(fn):
        for _ in range(3): fn()
        torch.cuda.synchronize()
        side = torch.cuda.Stream(); side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side): fn()
        torch.cuda.current_stream().wait_stream(side); torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g): fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(3): g.replay()
        b.record(); torch.cuda.synchronize()
        reps = max(args.reps, int(MIN_WINDOW_S * 1000 / (a.elapsed_time(b) / 3)) + 1)
        a.record()
        for _ in range(reps): g.replay()
        b.record(); torch.cuda.synchronize()
        return a.elapsed_time(b) / reps, reps
    res = {"tool": "tools/step_bench.py", "model": args.model, "ctx": args.ctx, "seq": args.seq, "groupsize": args.groupsize,
           "act_order": args.act_order, "layers": len(st.layers), "heads": shape.heads, "kv_heads": shape.kv_heads,
           "gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit(torch.cuda.current_device()), "plan": st.dplan.info(),
           "lora_rank": args.lora_rank, "lora_targets": args.lora_targets if args.lora_rank else None}
    if nb > 1:
        res["batch"] = nb
        ms, reps = timed(lambda: st.decode_step_fused_batch(xb, [args.ctx] * nb))
    else:
        ms, reps = timed(lambda: st.decode_step_fused(x, args.ctx))
    wbytes = st.q4_weight_bytes_per_token() + shape.vocab * shape.hidden * 2
    kv = nb * 2 * len(st.layers) * args.ctx * shape.kv_heads * shape.head_dim * 2     # K and V rows read once per KV head and sequence
    res["fused_ms"] = round(ms, 4); res["fused_tok_s"] = round(nb * 1000 / ms, 1); res["fused_reps"] = reps; res["bytes"] = wbytes + kv
    res["kv_bytes"] = kv; res["fused_GBps"] = round((wbytes + kv) / ms / 1e6, 1)
    lf = st._plan_logits[:1].clone()
    if not args.no_per_op:
        h = x.clone()
        def per_op():
            h.copy_(x); return st.decode_step(h, args.ctx)
        ms2, reps2 = timed(per_op)
        res["per_op_ms"] = round(ms2, 4); res["per_op_tok_s"] = round(1000 / ms2, 1); res["per_op_reps"] = reps2
        lp = per_op()
        d = (lf - lp).abs().max().item(); r = lp.pow(2).mean().sqrt().item()
        res["max_abs_diff_vs_per_op"] = d; res["logit_rms"] = r
    print(json.dumps(res))


def multi_tokens(args, st, shape):
    """One line per K: the K-token launch and its alternatives, timed from CUDA graphs (prefill: eagerly) in alternating rounds."""
    from exllama_b200 import capi
    ks = [int(k) for k in args.tokens.split(",")]
    H, ctx = shape.hidden, args.ctx
    xs = (torch.randn((max(ks), 1, H), device="cuda") * 0.5).half()
    st.batch = 1
    p1 = st.make_plan(); x1, l1 = st._plan_xout, st._plan_logits
    for k in ks:
        plans = []
        arms = {"one_step": lambda: p1.step(xs[:1], ctx, x_out=x1, logits=l1),
                "k_steps": lambda: [p1.step(xs[t:t + 1], ctx + t, x_out=x1, logits=l1) for t in range(k)]}
        st.batch = k
        batch_ok = k > 1
        if batch_ok:
            try:
                pb = st.make_plan(); plans.append(pb); xb, lb = st._plan_xout, st._plan_logits
                arms["batch_k"] = lambda: pb.step_batch(xs[:k], [ctx] * k, x_out=xb, logits=lb)
            except capi.ExlError:
                batch_ok = False
        pm = st.make_plan(max_tokens=k); plans.append(pm); xm, lm = st._plan_xout, st._plan_logits
        arms["multi"] = lambda: pm.step_multi(xs[:k], ctx, x_out=xm, logits=lm)
        graphs = {}
        for name, fn in arms.items():
            for _ in range(3): fn()
            torch.cuda.synchronize()
            side = torch.cuda.Stream(); side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side): fn()
            torch.cuda.current_stream().wait_stream(side); torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g): fn()
            graphs[name] = g.replay
        hp = xs[:k].view(1, k, H).clone()
        graphs["prefill"] = lambda: st.prefill(hp, ctx, last_only=False)
        for _ in range(3): graphs["prefill"]()
        times = {n: [] for n in graphs}
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = max(args.reps, 20)
        for _ in range(5):                                           # rounds, the arms alternating
            for n, fn in graphs.items():
                a.record()
                for _ in range(reps): fn()
                b.record(); torch.cuda.synchronize()
                times[n].append(a.elapsed_time(b) / reps)
        med = {n: sorted(v)[len(v) // 2] for n, v in times.items()}
        toks = {"one_step": 1, "k_steps": k, "batch_k": k, "multi": k, "prefill": k}
        res = {"tool": "tools/step_bench.py", "mode": "tokens", "model": args.model, "ctx": ctx, "tokens": k, "groupsize": args.groupsize,
               "layers": len(st.layers), "heads": shape.heads, "kv_heads": shape.kv_heads, "gpu": torch.cuda.get_device_name(0),
               "power_limit_w": power_limit(torch.cuda.current_device()), "plan": pm.info(), "rounds": 5, "reps_per_round": reps,
               "batch_k_fits": batch_ok}
        for n, ms in med.items():
            res[f"{n}_ms"] = round(ms, 4); res[f"{n}_tok_s"] = round(toks[n] * 1000 / ms, 1)
        res["multi_vs_one_step"] = round(med["multi"] / med["one_step"], 3)
        res["multi_vs_k_steps"] = round(med["multi"] / med["k_steps"], 3)
        res["multi_vs_prefill"] = round(med["multi"] / med["prefill"], 3)
        if batch_ok:
            res["multi_vs_batch_k"] = round(med["multi"] / med["batch_k"], 3)
        print(json.dumps(res), flush=True)
        for p in plans:
            p.close()
    p1.close()


if __name__ == "__main__":
    main()
