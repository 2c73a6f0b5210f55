"""Multi-token steps on the persistent decode step: up to four consecutive tokens of one sequence per launch (exl_decode_step_multi).

Token t of a launch sits at position past_len + t, attends the sequence's rows [0, past_len) and the launch's own tokens 0..t, and writes
row past_len + t: what DecodeStack.prefill(hidden, past_len, seq=seq, last_only=False) computes.  Every row of every launch is checked
against the float64 oracle composition of that prefill (tests/prefill_oracle.py) and against the per-op prefill itself, on the seeded
synthetic stacks of tests/stack_harness.py, with the tolerances of check_fused_step.  Also: one token against decode_step_fused, stale rows
at and past past_len are never read, one cache sequence only is written, consecutive steps with rewinding and CUDA-graph replay, short
contexts after a long one, the 7B and 13B shapes, every argument the C ABI rejects, and a greedy speculative loop whose tokens equal
single-step greedy decoding.
"""
import ctypes as C

import numpy as np
import pytest

from helpers import assert_close_ref64
from prefill_oracle import oracle_prefill
from stack_harness import check_head, lib_state, restore, snapshot, stacks  # noqa: F401

pytestmark = pytest.mark.gpu

PASTS = [0, 1, 15, 16, 37, 200]


def _np(t):
    return t.cpu().numpy()


def cta_of(u, U, G):
    return ((u + 1) * G - 1) // U


def att_needs_reset_multi(kv_heads, past, grid):
    """decode_step_sched.h: att_needs_reset_multi -- a KV head's CTA range holds an idle CTA at this context."""
    nph = max(1, (past + 15) // 16)
    U, G = kv_heads * nph, min(grid, 16 * kv_heads)
    if U >= G or nph < 2:
        return False
    return any(cta_of((h + 1) * nph - 1, U, G) - cta_of(h * nph, U, G) + 1 > nph for h in range(kv_heads))


def multi(st, xs, past, seq=0):
    """The multi-token step on xs [n, 1, hidden]: (logits [n, vocab], final hidden [n, hidden]) as cloned tensors."""
    lg = st.decode_step_fused_multi(xs, past, seq=seq).clone()
    return lg, st._plan_xout[:xs.shape[0]].clone()


def per_op(st, xs, past, seq=0):
    """DecodeStack.prefill of xs at past_len on cache sequence seq: (logits [n, vocab], final hidden [n, hidden]); leaves its rows written."""
    n, H = xs.shape[0], st.shape.hidden
    snap = snapshot(st)
    head = st.lm_head
    st.lm_head = None
    hid = st.prefill(xs.reshape(1, n, H).clone(), past, last_only=False, seq=seq).reshape(n, H).clone()
    st.lm_head = head
    restore(st, snap)
    lg = st.prefill(xs.reshape(1, n, H).clone(), past, last_only=False, seq=seq).clone()
    return lg, hid


def untouched_except(st, snap, seq, lo, hi):
    """No cache row but rows [lo, hi) of sequence seq was written."""
    import torch
    for i, (kc, vc) in enumerate(zip(st.key_cache, st.value_cache)):
        for b in range(kc.shape[0]):
            mask = np.ones(st.max_seq, bool)
            if b == seq:
                mask[lo:hi] = False
            assert torch.equal(kc[b][:, mask], snap[i][0][b][:, mask]) and torch.equal(vc[b][:, mask], snap[i][1][b][:, mask]), (i, b)


def check_multi_step(oracle, st, xs, past, seq, what):
    """Every row of one multi-token launch against the oracle and the per-op prefill: logits, final hidden state, new k / v rows; the
    logits against the kernel's own hidden state; no cache row written outside [past, past + n) of sequence seq."""
    import torch
    n = xs.shape[0]
    snap = snapshot(st)
    ref_lg, ref_x = per_op(st, xs, past, seq)
    ref_rows = [(kc[seq, :, past:past + n].clone(), vc[seq, :, past:past + n].clone()) for kc, vc in zip(st.key_cache, st.value_cache)]
    restore(st, snap)
    lg, x = multi(st, xs, past, seq)
    torch.cuda.synchronize()
    assert torch.isfinite(lg).all() and torch.isfinite(x).all()
    untouched_except(st, snap, seq, past, past + n)
    want, rows = oracle_prefill(oracle, st, list(zip(st.key_cache, st.value_cache)), _np(xs.reshape(n, -1)), past, seq, n)
    lg, x, ref_lg, ref_x = _np(lg), _np(x), _np(ref_lg), _np(ref_x)
    for t in range(n):
        w = f"{what} past {past} token {t}/{n}"
        check_head(st, lg[t], x[t], w)
        assert_close_ref64(x[t], ref_x[t].astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} final hidden vs per-op")
        assert_close_ref64(lg[t], want[t], rel=1.5e-2, rms=1.5e-2, what=f"{w} logits vs oracle")
        assert_close_ref64(lg[t], ref_lg[t].astype(np.float64), rel=1.5e-2, rms=1.5e-2, what=f"{w} logits vs per-op")
        for i, (kc, vc) in enumerate(zip(st.key_cache, st.value_cache)):
            k_new, v_new = _np(kc[seq, :, past + t]), _np(vc[seq, :, past + t])
            assert_close_ref64(k_new, rows[i][0][:, t].astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} layer {i} new k vs oracle")
            assert_close_ref64(v_new, rows[i][1][:, t].astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} layer {i} new v vs oracle")
            assert_close_ref64(k_new, _np(ref_rows[i][0][:, t]).astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} layer {i} new k vs per-op")
            assert_close_ref64(v_new, _np(ref_rows[i][1][:, t]).astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} layer {i} new v vs per-op")
    restore(st, snap)
    return lg, x


def rand_x(n, seed, H=1024):
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    return (torch.randn((n, 1, H), device="cuda", generator=g) * 0.5).half()


@pytest.mark.parametrize("gs", [128, 32])
@pytest.mark.parametrize("kv", [8, 2])
def test_every_position_vs_oracle_and_prefill(oracle, stacks, kv, gs):
    st = stacks(kv_heads=kv, gs=gs, seed=3 + kv + gs)
    st.make_plan(max_tokens=4)
    info = st.dplan.info()
    assert info["grid"] >= 100 and info["ring_stages"] >= 8, info
    for k in (1, 2, 3, 4):
        for past in PASTS:
            check_multi_step(oracle, st, rand_x(k, 100 * k + past + kv + gs), past, 0, f"kv {kv} g{gs} k {k}")


@pytest.mark.parametrize("kv", [8, 2])
def test_one_token_is_the_fused_step(stacks, kv):
    """n = 1 on a multi-token plan: the single-sequence fused step's logits, hidden state and new rows."""
    import torch
    st = stacks(kv_heads=kv, seed=21)
    x = rand_x(1, 7)
    snap = snapshot(st)
    st.make_plan()
    for past in (0, 37, 200):
        want = st.decode_step_fused(x, past).clone(); want_x = st._plan_xout.clone()
        want_rows = [(kc[0, :, past].clone(), vc[0, :, past].clone()) for kc, vc in zip(st.key_cache, st.value_cache)]
        restore(st, snap)
        st.dplan.close()
        st.make_plan(max_tokens=2)
        lg, xo = multi(st, x, past)
        torch.cuda.synchronize()
        assert_close_ref64(_np(lg[0]), _np(want[0]).astype(np.float64), rel=2e-3, rms=2e-3, what=f"past {past} logits")
        assert_close_ref64(_np(xo[0]), _np(want_x.view(-1)).astype(np.float64), rel=2e-3, rms=2e-3, what=f"past {past} hidden")
        for i, (kc, vc) in enumerate(zip(st.key_cache, st.value_cache)):      # fp32 atomics: not bit-identical across plans
            assert_close_ref64(_np(kc[0, :, past]), _np(want_rows[i][0]).astype(np.float64), rel=2e-3, rms=2e-3, what=f"past {past} layer {i} k")
            assert_close_ref64(_np(vc[0, :, past]), _np(want_rows[i][1]).astype(np.float64), rel=2e-3, rms=2e-3, what=f"past {past} layer {i} v")
        restore(st, snap)
        st.dplan.close()
        st.make_plan()


@pytest.mark.parametrize("kv", [8, 2])
def test_stale_rows_are_never_read(stacks, kv):
    """NaN in rows [past_len, max_seq) of the sequence: the outputs are finite and equal to the clean run's, and the rows past the launch's
    own are still NaN afterwards -- a speculative caller may leave rejected rows there."""
    import torch
    st = stacks(kv_heads=kv, seed=31)
    st.make_plan(max_tokens=4)
    snap = snapshot(st)
    for k, past in ((4, 0), (3, 16), (4, 37), (2, 200)):
        xs = rand_x(k, 50 + k + past)
        clean, clean_x = multi(st, xs, past)
        restore(st, snap)
        for kc, vc in zip(st.key_cache, st.value_cache):
            kc[0, :, past:] = float("nan"); vc[0, :, past:] = float("nan")
        lg, x = multi(st, xs, past)
        torch.cuda.synchronize()
        assert torch.isfinite(lg).all() and torch.isfinite(x).all(), (k, past)
        assert_close_ref64(_np(lg), _np(clean).astype(np.float64), rel=2e-3, rms=2e-3, what=f"k {k} past {past} logits")
        assert_close_ref64(_np(x), _np(clean_x).astype(np.float64), rel=2e-3, rms=2e-3, what=f"k {k} past {past} hidden")
        for kc, vc in zip(st.key_cache, st.value_cache):
            assert torch.isfinite(kc[0, :, past:past + k]).all() and torch.isfinite(vc[0, :, past:past + k]).all()
            assert torch.isnan(kc[0, :, past + k:]).all() and torch.isnan(vc[0, :, past + k:]).all()
        restore(st, snap)


def test_one_sequence_of_a_batched_cache(oracle, stacks):
    """A step on sequence 2 of a four-sequence cache reads and writes that sequence only."""
    st = stacks(kv_heads=2, batch=4, seed=41)
    st.make_plan(max_tokens=4)
    for seq, k, past in ((2, 4, 37), (3, 2, 0), (0, 3, 130)):
        check_multi_step(oracle, st, rand_x(k, seq + k + past), past, seq, f"seq {seq}")


def test_consecutive_steps_rewinding_and_graph(stacks):
    """Steps one after another, some keeping fewer tokens than they carried, so that the next step starts inside the rows the previous
    one wrote; against the same calls on the per-op prefill.  Then the last launch replayed from a CUDA graph."""
    import torch
    st = stacks(layers=3, kv_heads=2, seed=5)
    st.make_plan(max_tokens=4)
    snap = snapshot(st)
    plan = [(4, 40, 1), (3, None, 2), (4, None, 0), (2, None, 1), (1, None, 0), (4, None, 3)]     # (n, past or continue, accepted)
    calls, past = [], None
    for j, (n, p0, acc) in enumerate(plan):
        past = p0 if p0 is not None else past
        calls.append((rand_x(n, 300 + j), past))
        past += acc + 1
    ref = [per_op(st, xs, p)[0] for xs, p in calls]        # prefill leaves its rows written: the same cache history as the fused steps
    restore(st, snap)
    got = [multi(st, xs, p)[0] for xs, p in calls]
    torch.cuda.synchronize()
    for j, (g, r) in enumerate(zip(got, ref)):
        assert_close_ref64(_np(g), _np(r).astype(np.float64), rel=2e-2, rms=2e-2, what=f"step {j} (n {calls[j][0].shape[0]}, past {calls[j][1]})")
    xs, p = calls[-1]
    side = torch.cuda.Stream(); side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        st.decode_step_fused_multi(xs, p)
    torch.cuda.current_stream().wait_stream(side); torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        st.decode_step_fused_multi(xs, p)
    for _ in range(3):
        gr.replay()
    torch.cuda.synchronize()
    n = xs.shape[0]
    lg = _np(st._plan_logits[:n]); xo = _np(st._plan_xout[:n])
    assert_close_ref64(lg, _np(got[-1]).astype(np.float64), rel=2e-3, rms=2e-3, what="graph replay")
    for t in range(n):
        check_head(st, lg[t], xo[t], f"graph replay token {t}")


@pytest.mark.parametrize("kv", [8, 2])
def test_short_contexts_after_a_long_one(stacks, kv):
    """ONE plan: a long context first (every partial slot written), then short ones; the table reset launches exactly where
    att_needs_reset_multi says, and every row matches the per-op prefill."""
    import torch
    from exllama_b200 import capi
    st = stacks(kv_heads=kv, max_seq=1280, seed=17)
    st.make_plan(max_tokens=4)
    grid = st.dplan.info()["grid"]
    snap = snapshot(st)
    seen = set()
    for j, past in enumerate([1200, 0, 1, 15, 16, 37, 49, 100, 130, 200, 240, 300]):
        k = 1 + j % 4
        xs = rand_x(k, 700 + j)
        ref = per_op(st, xs, past)[0]
        restore(st, snap)
        n0 = capi.launch_count()
        got = st.decode_step_fused_multi(xs, past).clone()
        torch.cuda.synchronize()
        reset = att_needs_reset_multi(kv, past, grid)
        seen.add(reset)
        assert capi.launch_count() - n0 == 1 + int(reset), (past, capi.launch_count() - n0)
        untouched_except(st, snap, 0, past, past + k)
        restore(st, snap)
        assert_close_ref64(_np(got), _np(ref).astype(np.float64), rel=1.5e-2, rms=1.5e-2, what=f"past {past} k {k}")
    assert seen == {True, False}


@pytest.mark.parametrize("name,k", [("7b", 4), ("13b", 4)])
def test_full_size_shapes(stacks, name, k):
    """Two layers of the 7B and 13B shapes at their largest token count, context 1920, against the per-op prefill."""
    import torch
    from exllama_b200.shapes import SHAPES
    s = SHAPES[name]
    st = stacks(s, layers=2, max_seq=2048, seed=9)
    st.make_plan(max_tokens=k)
    xs = rand_x(k, 77, s.hidden)
    snap = snapshot(st)
    ref_lg, ref_x = per_op(st, xs, 1920)
    restore(st, snap)
    lg, x = multi(st, xs, 1920)
    torch.cuda.synchronize()
    untouched_except(st, snap, 0, 1920, 1920 + k)
    for t in range(k):
        assert_close_ref64(_np(lg[t]), _np(ref_lg[t]).astype(np.float64), rel=1.5e-2, rms=1.5e-2, what=f"{name} token {t} logits")
        assert_close_ref64(_np(x[t]), _np(ref_x[t]).astype(np.float64), rel=1e-2, rms=1e-2, what=f"{name} token {t} hidden")


def test_rejected_arguments(stacks):
    import torch
    from exllama_b200 import capi
    from exllama_b200.shapes import GQA_SHAPES
    st = stacks(kv_heads=2, batch=2, seed=1)

    def rejects(match, fn):
        with pytest.raises(capi.ExlError, match=match):
            fn()
    rejects(r"max_tokens 0 outside 1\.\.4", lambda: st.make_plan(max_tokens=0))
    rejects(r"max_tokens 5 outside 1\.\.4", lambda: st.make_plan(max_tokens=5))
    hs = [[L.q.q4, L.k.q4, L.v.q4, L.o.q4, L.gate.q4, L.up.q4, L.down.q4] for L in st.layers]
    args = (hs, [L.ln1 for L in st.layers], [L.ln2 for L in st.layers])
    tail = (st.sin, st.cos, st.local_heads, 128, st.max_seq, st.shape.eps)
    rejects(r"tensor parallelism .* exl_decode_step per token or prefill",
            lambda: capi.DecodePlan(*args, st.key_cache, st.value_cache, *tail, tp_world=2, num_kv_heads=2, max_tokens=2))
    empty = [torch.zeros((0, 2, st.max_seq, 128), dtype=torch.float16, device="cuda") for _ in st.layers]
    rejects(r"cache_seqs 0", lambda: capi.DecodePlan(*args, empty, empty, *tail, num_kv_heads=2, max_tokens=2))
    # a batch plan refuses exl_decode_step_multi, a multi-token plan the one-token calls
    st.make_plan()
    rejects(r"not a multi-token plan.*exl_decode_plan_create_multi", lambda: st.dplan.step_multi(rand_x(2, 1), 5))
    st.dplan.close()
    st.make_plan(max_tokens=2)
    x = rand_x(3, 2)
    rejects(r"exl_decode_step_multi", lambda: st.dplan.step(x[:1], 5, logits=st._plan_logits))
    rejects(r"exl_decode_step_multi", lambda: st.dplan.step_batch(x[:2], [5, 6], logits=st._plan_logits))
    rejects(r"n 3 outside 1\.\.2", lambda: st.dplan.step_multi(x, 5))
    rejects(r"seq 2 outside .*\[0, 2\)", lambda: st.dplan.step_multi(x[:2], 5, seq=2))
    rejects(r"seq -1 outside", lambda: st.dplan.step_multi(x[:2], 5, seq=-1))
    rejects(r"past_len -1", lambda: st.dplan.step_multi(x[:2], -1))
    rejects(r"past_len 255 \+ n 2 outside the cache \(max_seq 256\)", lambda: st.dplan.step_multi(x[:2], 255))
    lib, s = capi.lib(), capi._stream()
    rejects(r"x_in is NULL", lambda: capi.check(lib.exl_decode_step_multi(st.dplan.handle, None, 1, 0, 0, None, capi._ptr(st._plan_logits), s)))
    rejects(r"logits must be given", lambda: capi.check(lib.exl_decode_step_multi(st.dplan.handle, capi._ptr(x), 1, 0, 0, None, None, s)))
    st.dplan.close(); st.dplan = None
    act = stacks(act=True, seed=2)
    rejects(r"act-order", lambda: act.make_plan(max_tokens=2))
    big = stacks(GQA_SHAPES["70b"], layers=1, max_seq=64, seed=4)
    rejects(r"max_tokens 2 does not fit .* the largest is 1", lambda: big.make_plan(max_tokens=2))
    big.make_plan(max_tokens=1)


def test_greedy_speculative_loop(stacks):
    """Speculative decoding with tied embeddings (x = c * lm_head[token]): each launch carries the last token and three drafts taken from
    the single-step greedy continuation, every third draft corrupted; a draft is accepted while it equals the argmax after its
    predecessor, and the step after the first rejection starts over the rejected rows.  The emitted tokens equal single-step greedy
    decoding up to the first position where the single step's top-2 logit gap is within tolerance."""
    import torch
    st = stacks(kv_heads=2, seed=61)
    c = 25.0                                            # lm_head entries ~ N(0, 0.02^2): rows of rms ~ 0.5, like the other inputs
    emb = lambda toks: (st.lm_head[torch.tensor(toks, device="cuda")].float() * c).half().view(len(toks), 1, -1).contiguous()
    past0, n_ref = 37, 56
    snap = snapshot(st)
    st.make_plan()
    ref, gaps, tok = [], [], 5
    for i in range(n_ref):
        lg = st.decode_step_fused(emb([tok]), past0 + i)[0].clone().double()
        top = torch.topk(lg, 2).values
        gaps.append(float(top[0] - top[1]) / float(lg.pow(2).mean().sqrt()))
        tok = int(lg.argmax()); ref.append(tok)
    st.dplan.close()
    restore(st, snap)
    st.make_plan(max_tokens=4)
    out, cur, past, drafted, launches = [], 5, past0, 0, 0
    while len(out) < n_ref - 4:
        drafts = []
        for j in range(3):
            d = ref[len(out) + j]
            if drafted % 3 == 2:
                d = (d + 1) % st.shape.vocab            # corrupted draft: rejected, and the rows behind it rewound
            drafts.append(d); drafted += 1
        lg = st.decode_step_fused_multi(emb([cur] + drafts), past).argmax(-1).tolist()
        a = 0
        while a < 3 and lg[a] == drafts[a]:
            a += 1
        out += drafts[:a] + [lg[a]]
        cur, past, launches = lg[a], past + a + 1, launches + 1
    first_close = next((i for i, g in enumerate(gaps) if g < 5e-3), n_ref)
    m = min(first_close, len(out))
    assert m >= 16, (first_close, len(out))
    assert out[:m] == ref[:m], (out[:m], ref[:m])
    assert launches < len(out)                          # drafts were accepted: fewer launches than tokens
