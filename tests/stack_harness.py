"""Synthetic decode stacks for the GPU tests (test infrastructure): the stack factory, cache snapshots, the fixtures that free the
library's state, and the checks every decode-step plan kind shares -- the fused step against the whole-token oracle and the per-op
path, consecutive tokens with CUDA-graph replay, and short contexts after a long one.

torch is imported inside the functions, so that collection works without a GPU.  conftest.py does not load this module: a test file
that wants the fixtures imports them by name (`from stack_harness import lib_state, stacks  # fixtures`)."""
import numpy as np
import pytest

from helpers import assert_close_ref64, assert_within_any, att_needs_reset, head_expectation, oracle_decode_step


def _np(t):
    return t.cpu().numpy()


def sincos(max_seq, hd):
    """The rope tables [max_seq, hd] fp16 of DecodeStack (base 10000), computed in float64."""
    inv = 1.0 / (10000 ** (np.arange(0, hd, 2, dtype=np.float64) / hd))
    ang = np.outer(np.arange(max_seq), inv)
    emb = np.concatenate([ang, ang], -1)
    return np.sin(emb).astype(np.float16), np.cos(emb).astype(np.float16)


def make_stack(shape=None, *, hidden=1024, inter=2816, layers=2, heads=8, kv_heads=None, vocab=2048, gs=128, act=False, max_seq=256,
               batch=1, seed=3):
    """A DecodeStack of `layers` layers whose KV caches hold N(0, 0.25) fp16 values (a CUDA generator seeded seed + 100, k then v of
    each layer), so that a stray write or read shows.  shape: a LlamaShape to take the dimensions and eps from; without one the
    dimensions given here make one (eps 1e-6, kv_heads None = heads).  gs None: one quantisation group per matrix."""
    import torch
    from exllama_b200.stack import DecodeStack, LlamaShape
    if shape is None:
        shape = LlamaShape("synthetic", hidden, inter, layers, heads, vocab=vocab, kv_heads=kv_heads)
    st = DecodeStack(shape, groupsize=gs, act_order=act, device="cuda:0", max_seq=max_seq, layers=layers, seed=seed, batch=batch)
    g = torch.Generator(device="cuda"); g.manual_seed(seed + 100)
    for kc, vc in zip(st.key_cache, st.value_cache):
        kc.copy_((torch.randn(kc.shape, device="cuda", generator=g) * 0.5).half())
        vc.copy_((torch.randn(vc.shape, device="cuda", generator=g) * 0.5).half())
    return st


def snapshot(st):
    return [(kc.clone(), vc.clone()) for kc, vc in zip(st.key_cache, st.value_cache)]


def restore(st, snap):
    for (kc, vc), (k0, v0) in zip(zip(st.key_cache, st.value_cache), snap):
        kc.copy_(k0); vc.copy_(v0)


@pytest.fixture
def lib_state():
    """A library without q4 handles or borrowed buffers at the start of the test, and again at its end, pass or fail: exl_cleanup
    frees every q4 handle on the device and resets temp_state, which a stack an earlier test failed to close would leave pointing at
    freed memory that the act-order gather writes through."""
    import torch
    from exllama_b200 import capi
    capi.check(capi.lib().exl_cleanup())
    yield capi
    torch.cuda.synchronize()
    capi.check(capi.lib().exl_cleanup())


@pytest.fixture
def stacks(lib_state):
    """make_stack as a fixture: every stack made, and the plan it holds at the end of the test (DecodeStack.close), is closed at
    teardown, pass or fail."""
    made = []

    def make(shape=None, **kw):
        made.append(make_stack(shape, **kw))
        return made[-1]
    yield make
    for st in made:
        st.close()


def fused_step(st, xs, pasts):
    """The fused step of xs [bsz, 1, hidden] at contexts pasts: decode_step_fused (exl_decode_step) on a single-sequence stack,
    decode_step_fused_batch (exl_decode_step_batch) on a batched one.  Returns the logits [bsz, vocab]."""
    if st.batch > 1:
        return st.decode_step_fused_batch(xs, pasts)
    return st.decode_step_fused(xs, pasts[0]).view(1, -1)


def per_op(st, snap, xs, pasts):
    """The per-op path, one sequence at a time on its own cache sequence: logits [1, vocab] and the new (k, v) rows of every layer
    per sequence; the caches are restored to snap afterwards."""
    logits, rows = [], []
    for b, past in enumerate(pasts):
        logits.append(st.decode_step(xs[b:b + 1].clone(), past, seq=b).clone())
        rows.append([(kc[b, :, past].clone(), vc[b, :, past].clone()) for kc, vc in zip(st.key_cache, st.value_cache)])
    restore(st, snap)
    return logits, rows


def untouched_except(st, snap, pasts):
    """No cache row of any sequence but row pasts[b] of sequences b < bsz was written."""
    import torch
    for i, (kc, vc) in enumerate(zip(st.key_cache, st.value_cache)):
        for b in range(kc.shape[0]):
            mask = np.ones(st.max_seq, bool)
            if b < len(pasts):
                mask[pasts[b]] = False
            assert torch.equal(kc[b][:, mask], snap[i][0][b][:, mask]) and torch.equal(vc[b][:, mask], snap[i][1][b][:, mask]), (i, b)


def check_head(st, logits, x_out, what):
    """The HEAD phase on the kernel's own final hidden state: logits [vocab] within head_expectation's fp32-summation bound of
    rms_norm(x_out, norm) . lm_head^T (one of the three fp16 row factors), about 1e-4 of their rms."""
    return assert_within_any(np.asarray(logits, np.float64).reshape(-1),
                             head_expectation(x_out, _np(st.norm), _np(st.lm_head), st.shape.eps), f"{what} HEAD")


def check_fused_step(oracle, st, xs, pasts, what):
    """The fused step (st's plan) on xs [bsz, 1, hidden] at contexts pasts against the per-op path, run sequence by sequence from the
    same caches, and -- unless oracle is None -- against oracle_decode_step: for every sequence the final hidden state, the logits
    and the new k and v rows, and no cache row written but pasts[b] of sequence b.  With oracle None: the logits against the per-op
    path only.  Either way the logits against the kernel's own final hidden state (check_head).  Returns (logits [bsz, vocab], per-op logits, oracle logits or None) as numpy arrays per sequence."""
    import torch
    bsz = len(pasts)
    snap = snapshot(st)
    ref_logits, ref_rows = per_op(st, snap, xs, pasts)
    got = fused_step(st, xs, pasts)
    torch.cuda.synchronize()
    assert torch.isfinite(got).all()
    logits = _np(got)
    ref_logits = [_np(r).reshape(-1) for r in ref_logits]
    want_logits = None
    got_x = _np(st._plan_xout.view(-1, st.shape.hidden)[:bsz])
    for b in range(bsz):
        check_head(st, logits[b], got_x[b], f"{what} seq {b} (ctx {pasts[b]})")
    if oracle is None:
        for b in range(bsz):
            assert_close_ref64(logits[b], ref_logits[b].astype(np.float64), rel=1.5e-2, rms=1.5e-2, what=f"{what} seq {b} logits")
        return logits, ref_logits, want_logits
    want_logits = []
    for b in range(bsz):
        want_x, want, rows = oracle_decode_step(oracle, st, snap, _np(xs[b]), pasts[b], b)
        want_logits.append(want.reshape(-1))
        w = f"{what} seq {b} (ctx {pasts[b]})"
        # three matmuls deep per layer with fp16 rounding points in between: a few 1e-3 of the rms per layer
        assert_close_ref64(got_x[b], want_x.reshape(-1).astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} final hidden vs oracle")
        assert_close_ref64(logits[b], want_logits[b], rel=1.5e-2, rms=1.5e-2, what=f"{w} logits vs oracle")
        assert_close_ref64(logits[b], ref_logits[b].astype(np.float64), rel=1.5e-2, rms=1.5e-2, what=f"{w} logits vs per-op")
        for i, (kc, vc) in enumerate(zip(st.key_cache, st.value_cache)):
            k_new, v_new = _np(kc[b, :, pasts[b]]), _np(vc[b, :, pasts[b]])
            assert_close_ref64(k_new, rows[i][0].astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} layer {i} new k vs oracle")
            assert_close_ref64(v_new, rows[i][1].astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} layer {i} new v vs oracle")
            assert_close_ref64(k_new, _np(ref_rows[b][i][0]).astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} layer {i} new k vs per-op")
            assert_close_ref64(v_new, _np(ref_rows[b][i][1]).astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} layer {i} new v vs per-op")
    untouched_except(st, snap, pasts)
    return logits, ref_logits, want_logits


def check_sequence_and_graph(st, xs, starts, replay_tol=2e-3):
    """Consecutive tokens xs[t] [bsz, 1, hidden], sequence b at context starts[b] + t (barrier generation, accumulator clean-up and
    the cache rows carry over between launches), against the per-op path token by token and sequence by sequence; then the last
    launch replayed from a CUDA graph.  fp32 atomics make bit-identical results across launches not required: the logits agree, and
    the replay's logits are held to check_head on the replay's own final hidden state."""
    import torch
    bsz = len(starts)
    snap = snapshot(st)
    ref = [[st.decode_step(x[b:b + 1].clone(), starts[b] + t, seq=b).clone() for b in range(bsz)] for t, x in enumerate(xs)]
    restore(st, snap)
    got = [fused_step(st, x, [p + t for p in starts]).clone() for t, x in enumerate(xs)]
    torch.cuda.synchronize()
    for t in range(len(xs)):
        for b in range(bsz):
            assert_close_ref64(_np(got[t][b]), _np(ref[t][b]).reshape(-1).astype(np.float64), rel=2e-2, rms=2e-2, what=f"token {t} seq {b}")
    x, last = xs[-1], [p + len(xs) - 1 for p in starts]
    side = torch.cuda.Stream(); side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fused_step(st, x, last)
    torch.cuda.current_stream().wait_stream(side); torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        fused_step(st, x, last)
    for _ in range(3):
        gr.replay()
    torch.cuda.synchronize()
    assert_close_ref64(_np(st._plan_logits)[:bsz], _np(got[-1]).astype(np.float64), rel=replay_tol, rms=replay_tol, what="graph replay")
    xo = _np(st._plan_xout.view(-1, st.shape.hidden)[:bsz]); lg = _np(st._plan_logits.view(-1, st.shape.vocab)[:bsz])
    for b in range(bsz):
        check_head(st, lg[b], xo[b], f"graph replay seq {b}")


def check_reset_after_long_context(st, xs, contexts, check_untouched=False):
    """ONE plan stepped at each of `contexts` (lists of past_lens, a long one first: every slot of the attention-partial table gets
    written) on xs[j] [bsz, 1, hidden].  Where short contexts leave CTAs inside a head's CTA range without an attention unit, the
    partials of the long context must not leak into the softmax combine: the table reset launches exactly where att_needs_reset
    (longest context) says, and every sequence matches the per-op path.  check_untouched: also no cache row but pasts[b] of
    sequence b written.  Returns the set of reset decisions seen."""
    import torch
    from exllama_b200 import capi
    grid = st.dplan.info()["grid"]
    s = st.shape
    snap = snapshot(st)
    seen = set()
    for x, pasts in zip(xs, contexts):
        ref, _ = per_op(st, snap, x, pasts)
        n0 = capi.launch_count()
        got = fused_step(st, x, pasts).clone()
        torch.cuda.synchronize()
        reset = att_needs_reset(s.heads, s.kv_heads, max(pasts), grid, len(pasts))
        seen.add(reset)
        assert capi.launch_count() - n0 == 1 + int(reset), (pasts, capi.launch_count() - n0)
        if check_untouched:
            untouched_except(st, snap, pasts)
        restore(st, snap)
        for b in range(len(pasts)):
            assert_close_ref64(_np(got[b]), _np(ref[b]).reshape(-1).astype(np.float64), rel=1.5e-2, rms=1.5e-2, what=f"ctx {pasts} seq {b}")
    return seen
