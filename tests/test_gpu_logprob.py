"""Token log-probabilities on the GPU (exl_token_logprobs, scoring.py, DecodeStack.prefill(targets=)).

Kernel: against the float64 oracle (oracle/logprob_oracle.py) at Llama head shapes, every T / H / V edge in at least one case, with
planted duplicate lm_head rows (the tie rule), a dominant id at V - 1 and at the first id of the last vocab tile (the tail mask);
RMS error no larger than the reference's fp16 matmul -> float -> log_softmax -> gather program; undefined rows; sentinels past T;
bitwise reproducibility and CUDA-graph replay; every argument error.
Stack: prefill(targets=) bitwise equal to token_logprobs of the final normed hidden state (skinny and wgmma routes, MHA / GQA,
past_len 0 and > 0, a batch of two), prefill_ragged(targets=) per sequence against prefill(targets=), cache rows unchanged by the
head, and perplexity() against the reference's program, one chunk per call and packed.
"""
import math

import pytest

from stack_harness import lib_state, restore, snapshot, stacks  # noqa: F401

pytestmark = pytest.mark.gpu


def _inputs(T, H, V, seed, plant=True):
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    hn = torch.randn((T, H), device="cuda", generator=g).half()
    lm = (torch.randn((V, H), device="cuda", generator=g) * 0.02).half()
    y = torch.randint(0, V, (T,), device="cuda", generator=g)
    planted = {}
    if plant:
        last_tile = (V - 1) // 256 * 256                # == V - 1 when the last tile holds one id: row 2 is then not planted
        rows = [(0, [3, 300, V - 2] if V > 300 else [0, V - 1]), (1, [V - 1]), (2, [last_tile])]
        used = set()
        for t, ids in rows:
            if t >= T or used & set(ids):
                continue
            used |= set(ids)
            for i in ids:
                lm[i] = (hn[t].float() * 0.01).half()
            planted[t] = min(ids)
            y[t] = ids[-1]
    return hn, lm, y, planted


def _run(hn, lm, y):
    from exllama_b200 import scoring
    return scoring.token_logprobs(hn, lm, y)


def _check_vs_oracle(hn, lm, y, lp, gr, what):
    import torch
    from oracle.logprob_oracle import logprobs64
    o = logprobs64(hn, lm, y)
    lp64 = lp.double()
    err = (lp64 - o["logprob"]).abs()
    tol = o["bound"] + 1e-6 * o["lse"].abs()
    worst = int(torch.argmax(err / tol))
    assert bool((err <= tol).all()), f"{what}: row {worst} err {float(err[worst]):.3e} bound {float(tol[worst]):.3e}"
    sure = o["margin"] > o["gbound"]
    assert bool((gr[sure] == o["greedy"][sure]).all()), f"{what}: greedy differs where the margin exceeds the bound"
    return o, err


# (T, H, V): every T of {1, 2, 63, 64, 65, 127, 128, 129, 257, 1920}, H of {4096, 5120, 6656, 8192}, V of {32000, 32001, 32016,
# 128256} appears at least once
CASES = [(1, 4096, 32000), (2, 5120, 32001), (63, 6656, 32016), (64, 8192, 128256), (65, 4096, 32001), (127, 5120, 32016),
         (128, 6656, 32000), (129, 8192, 32001), (257, 4096, 128256), (1920, 5120, 32000), (1920, 8192, 32016)]


@pytest.mark.parametrize("T,H,V", CASES)
def test_kernel_vs_oracle(T, H, V):
    import torch
    from oracle.logprob_oracle import torch_program
    hn, lm, y, planted = _inputs(T, H, V, seed=T * 7 + H + V)
    lp, gr = _run(hn, lm, y)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(lp).all())
    o, err = _check_vs_oracle(hn, lm, y, lp, gr, f"T {T} H {H} V {V}")
    for t, gid in planted.items():                 # duplicate rows: the lowest id; dominant ids at the tail of the vocabulary
        assert int(gr[t]) == gid == int(o["greedy"][t]), (t, int(gr[t]), gid)
    ref = torch_program(hn, lm, y).double()
    rms = lambda e: float(e.pow(2).mean().sqrt())
    assert rms(err) <= rms(ref - o["logprob"]), f"RMS error {rms(err):.3e} above the torch program's {rms(ref - o['logprob']):.3e}"


def test_undefined_rows_and_sentinels():
    import torch
    from exllama_b200 import scoring
    T, H, V = 70, 4096, 32001
    hn, lm, y, _ = _inputs(T, H, V, seed=11, plant=False)
    clean_lp, clean_gr = _run(hn, lm, y)
    bad_y = y.clone(); bad_y[3], bad_y[40], bad_y[69] = -1, V, 1 << 40
    bad_h = hn.clone(); bad_h[5, 17] = float("nan"); bad_h[6, 0] = float("inf"); bad_h[64, 4095] = float("-inf")
    need = scoring.work_size(T, V, 0)
    lp_buf = torch.full((T + 9,), 12345.0, device="cuda")
    gr_buf = torch.full((T + 9,), 777, dtype=torch.int64, device="cuda")
    work = torch.full((need + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    lp, gr = scoring.token_logprobs(bad_h, lm, bad_y, out=(lp_buf[:T], gr_buf[:T]), work=work)
    torch.cuda.synchronize()
    undefined_lp = {3, 40, 69, 5, 6, 64}
    undefined_gr = {5, 6, 64}
    for t in range(T):
        if t in undefined_lp:
            assert bool(torch.isnan(lp[t])), t
        else:
            assert lp[t].view(torch.int32) == clean_lp[t].view(torch.int32), t
        if t in undefined_gr:
            assert int(gr[t]) == -1, t
        else:
            assert int(gr[t]) == int(clean_gr[t]), t
    assert bool((lp_buf[T:] == 12345.0).all()) and bool((gr_buf[T:] == 777).all())
    assert bool((work[need:] == 0xA5).all())


def test_bitwise_repeat_and_graph_replay():
    import torch
    from exllama_b200 import scoring
    T, H, V = 600, 4096, 32000
    hn, lm, y, _ = _inputs(T, H, V, seed=5)
    work = torch.empty(scoring.work_size(T, V, 0), dtype=torch.uint8, device="cuda")
    out = (torch.empty(T, device="cuda"), torch.empty(T, dtype=torch.int64, device="cuda"))
    a = [t.clone() for t in scoring.token_logprobs(hn, lm, y, out=out, work=work)]
    b = [t.clone() for t in scoring.token_logprobs(hn, lm, y, out=out, work=work)]
    assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32)) and torch.equal(a[1], b[1])
    out[0].fill_(0); out[1].fill_(0)
    side = torch.cuda.Stream(); side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        scoring.token_logprobs(hn, lm, y, out=out, work=work)
    torch.cuda.current_stream().wait_stream(side); torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        scoring.token_logprobs(hn, lm, y, out=out, work=work)
    out[0].fill_(0); out[1].fill_(0)
    gr.replay(); gr.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0].view(torch.int32), a[0].view(torch.int32)) and torch.equal(out[1], a[1])


def test_argument_errors():
    import ctypes as C
    import torch
    from exllama_b200 import capi, scoring
    lib = capi.lib()
    T, H, V = 8, 128, 1000
    hn, lm, y, _ = _inputs(T, H, V, seed=2, plant=False)
    lp = torch.empty(T + 4, device="cuda"); gr = torch.empty(T + 2, dtype=torch.int64, device="cuda")
    need = scoring.work_size(T, V, 0)
    work = torch.empty(need + 16, dtype=torch.uint8, device="cuda")
    n = C.c_int64()
    assert lib.exl_token_logprobs_work_size(T, V, 0, C.byref(n)) == 0 and n.value == need
    P = lambda t: C.c_void_p(t.data_ptr())
    base = dict(hn=P(hn), T=T, H=H, lm=P(lm), V=V, y=P(y), lp=P(lp), g=P(gr), w=P(work), wb=need)
    call = lambda **kw: lib.exl_token_logprobs(*[{**base, **kw}[k] for k in ("hn", "T", "H", "lm", "V", "y", "lp", "g", "w", "wb")],
                                               capi._stream())
    assert call() == 0
    odd = lambda t, b: C.c_void_p(t.data_ptr() + b)
    host = torch.zeros(T, dtype=torch.int64)
    cases = [dict(T=0), dict(V=0), dict(H=100), dict(H=0), dict(wb=need - 1), dict(y=P(host)),
             dict(hn=odd(hn, 2)), dict(lm=odd(lm, 8)), dict(y=odd(y, 8)), dict(lp=odd(lp, 4)), dict(g=odd(gr, 8)), dict(w=odd(work, 8))]
    cases += [{k: None} for k in ("hn", "lm", "y", "lp", "g", "w")]
    for bad in cases:
        assert call(**bad) == 1, (bad, lib.exl_last_error())
    with pytest.raises(ValueError):
        scoring.token_logprobs(hn.float(), lm, y)
    with pytest.raises(ValueError):
        scoring.token_logprobs(hn, lm[:, :64].contiguous(), y)
    with pytest.raises(ValueError):
        scoring.token_logprobs(hn, lm, y.int())


# ---- through the stack --------------------------------------------------------------------------------------------------------

def _final_hidden(st, fn):
    """The stack's final hidden state of fn() (the same call with the head detached)."""
    head, st.lm_head = st.lm_head, None
    try:
        return fn()
    finally:
        st.lm_head = head


@pytest.mark.parametrize("kv_heads,bsz,q_len,past", [(None, 1, 5, 0), (None, 1, 100, 0), (None, 1, 37, 40), (2, 1, 100, 17),
                                                      (2, 2, 1, 30), (None, 2, 70, 0)])
def test_prefill_targets_bitwise(stacks, kv_heads, bsz, q_len, past):
    import torch
    from exllama_b200 import cuda_ext, scoring
    st = stacks(kv_heads=kv_heads, batch=2, vocab=2048 + 37)
    g = torch.Generator(device="cuda"); g.manual_seed(q_len + past)
    h = (torch.randn((bsz, q_len, st.shape.hidden), device="cuda", generator=g) * 0.5).half()
    y = torch.randint(0, st.shape.vocab, (bsz, q_len), device="cuda", generator=g)
    snap = snapshot(st)
    st.prefill(h.clone(), past, seq=0)
    plain = [(kc.clone(), vc.clone()) for kc, vc in zip(st.key_cache, st.value_cache)]
    restore(st, snap)
    lp, gr = st.prefill(h.clone(), past, seq=0, targets=y)
    for (kc, vc), (k0, v0) in zip(zip(st.key_cache, st.value_cache), plain):
        assert torch.equal(kc, k0) and torch.equal(vc, v0)
    restore(st, snap)
    x = _final_hidden(st, lambda: st.prefill(h.clone(), past, seq=0))
    want_lp, want_gr = scoring.token_logprobs(cuda_ext.ext_rms_norm(x, st.norm, st.shape.eps).view(-1, st.shape.hidden), st.lm_head,
                                              y.reshape(-1))
    torch.cuda.synchronize()
    assert lp.shape == (bsz * q_len,) and torch.equal(lp.view(torch.int32), want_lp.view(torch.int32)) and torch.equal(gr, want_gr)
    # and the head against the logits prefill returns without targets
    restore(st, snap)
    logits = st.prefill(h.clone(), past, seq=0, last_only=False).double()
    ref = torch.log_softmax(logits, -1).gather(1, y.reshape(-1, 1))[:, 0]
    assert float((lp.double() - ref).abs().max()) < 2e-2


@pytest.mark.parametrize("kv_heads", [None, 2])
def test_prefill_ragged_targets(stacks, kv_heads):
    import torch
    st = stacks(kv_heads=kv_heads, batch=3)
    q_lens, past_lens = [9, 1, 66], [0, 20, 3]
    T = sum(q_lens)
    g = torch.Generator(device="cuda"); g.manual_seed(7)
    h = (torch.randn((T, st.shape.hidden), device="cuda", generator=g) * 0.5).half()
    y = torch.randint(0, st.shape.vocab, (T,), device="cuda", generator=g)
    snap = snapshot(st)
    st.prefill_ragged(h.clone(), q_lens, past_lens)
    plain = [(kc.clone(), vc.clone()) for kc, vc in zip(st.key_cache, st.value_cache)]
    restore(st, snap)
    lp, gr = st.prefill_ragged(h.clone(), q_lens, past_lens, targets=y)
    for (kc, vc), (k0, v0) in zip(zip(st.key_cache, st.value_cache), plain):
        assert torch.equal(kc, k0) and torch.equal(vc, v0)
    off = 0
    for i, (ql, pl) in enumerate(zip(q_lens, past_lens)):
        restore(st, snap)
        one_lp, one_gr = st.prefill(h[off:off + ql].clone().view(1, ql, -1), pl, seq=i, targets=y[off:off + ql])
        torch.cuda.synchronize()
        # the GEMM route differs (M = T against M = q_len): a few 1e-3 of the logits' scale through two layers
        assert float((lp[off:off + ql] - one_lp).abs().max()) < 2e-2, i
        off += ql


def test_perplexity_matches_the_reference_program(stacks):
    import torch
    from exllama_b200 import scoring
    st = stacks(batch=4, max_seq=256)
    g = torch.Generator(device="cuda"); g.manual_seed(3)
    embed = (torch.randn((st.shape.vocab, st.shape.hidden), device="cuda", generator=g) * 0.5).half()
    lens = [65, 2, 130, 33, 200, 17]
    chunks = [torch.randint(0, st.shape.vocab, (n,), device="cuda", generator=g) for n in lens]
    # the reference: per chunk from an empty cache, log_softmax of prefill(last_only=False) logits, fp32 sums added on the host
    s, count = 0.0, 0
    for c in chunks:
        logits = st.prefill(embed[c[:-1]].view(1, c.numel() - 1, -1), 0, last_only=False)
        lp = torch.nn.functional.log_softmax(logits, dim=-1).gather(-1, c[1:].view(-1, 1)).view(-1)
        s += lp.sum().item(); count += c.numel() - 1
    want = math.exp(-s / count)
    packed = scoring.perplexity(st, embed, chunks)
    single = scoring.perplexity(st, embed, chunks, per_call=1)
    # logits rounded to fp16 by the reference (2^-11 relative) against fp32 sums here
    assert abs(packed - want) <= 2e-3 * want, (packed, want)
    assert abs(single - packed) <= 2e-3 * want, (single, packed)
