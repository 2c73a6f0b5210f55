"""Batched decode on the persistent decode step: up to four sequences per launch, each at its own context.

Every sequence of a batch is checked against the float64 oracle composition for that sequence (its own cache rows, its own context)
and against the per-op path run sequence by sequence on the same seeded synthetic stack; the new K/V rows land in that sequence's
cache and nowhere else.  Also: permuting the batch permutes the outputs, consecutive tokens and CUDA-graph replay, short contexts
after a long one (the partial table is reset exactly where att_needs_reset over the virtual heads says), the 7B and 70B shapes, and
every argument the C ABI rejects.  Tolerances are those of tests/test_gpu_decode_step.py.
"""
import numpy as np
import pytest

from helpers import assert_close_ref64

pytestmark = pytest.mark.gpu


def _mk_stack(hidden, inter, layers, heads, kv_heads, gs, max_seq, batch, vocab=2048, seed=3, act=False):
    import torch
    from exllama_b200.stack import DecodeStack, LlamaShape
    shape = LlamaShape("synthetic-batch", hidden, inter, layers, heads, vocab=vocab, kv_heads=kv_heads)
    st = DecodeStack(shape, groupsize=gs, act_order=act, device="cuda:0", max_seq=max_seq, seed=seed, batch=batch)
    g = torch.Generator(device="cuda"); g.manual_seed(seed + 100)
    for kc, vc in zip(st.key_cache, st.value_cache):
        kc.copy_((torch.randn(kc.shape, device="cuda", generator=g) * 0.5).half())
        vc.copy_((torch.randn(vc.shape, device="cuda", generator=g) * 0.5).half())
    return st


def _snap(st):
    return [(kc.clone(), vc.clone()) for kc, vc in zip(st.key_cache, st.value_cache)]


def _restore(st, snap):
    for (kc, vc), (k0, v0) in zip(zip(st.key_cache, st.value_cache), snap):
        kc.copy_(k0); vc.copy_(v0)


def _oracle_step(oracle, st, snap, x, past, seq):
    """float64/fp16 restatement of one decode token of cache sequence `seq`: (final hidden fp16, logits float64, new k/v rows per layer)."""
    s = st.shape
    hd, heads, kvh = s.head_dim, s.heads, s.kv_heads
    sin = st.sin.view(-1, hd).cpu().numpy(); cos = st.cos.view(-1, hd).cpu().numpy()
    x = x.reshape(1, s.hidden).copy()
    rows = []

    def mm(xin, lin, acc=None):
        return oracle.q4_matmul_f64(xin, lin.qweight.cpu().numpy(), lin.qzeros.cpu().numpy(), lin.scales.cpu().numpy(), None, acc)
    for i, L in enumerate(st.layers):
        xn, _ = oracle.rms_norm(x, L.ln1.cpu().numpy(), s.eps)
        q = mm(xn, L.q).astype(np.float16); k = mm(xn, L.k).astype(np.float16); v = mm(xn, L.v).astype(np.float16)
        q = oracle.rope(q.reshape(1, heads, hd), sin, cos, 1, heads, hd, heads, past).reshape(-1)
        k = oracle.rope(k.reshape(1, kvh, hd), sin, cos, 1, kvh, hd, kvh, past).reshape(kvh, hd)
        kc = snap[i][0][seq].cpu().numpy().copy(); vc = snap[i][1][seq].cpu().numpy().copy()
        kc[:, past] = k; vc[:, past] = v.reshape(kvh, hd)
        rows.append((k.copy(), v.reshape(kvh, hd).copy()))
        attn = oracle.decode_attn_f64(q, kc, vc, heads, kvh, hd, past + 1, st.max_seq).astype(np.float16).reshape(1, -1)
        x = mm(attn, L.o, acc=x).astype(np.float16)
        xn, _ = oracle.rms_norm(x, L.ln2.cpu().numpy(), s.eps)
        act = oracle.silu_mul(mm(xn, L.gate).astype(np.float16), mm(xn, L.up).astype(np.float16))
        x = mm(act, L.down, acc=x).astype(np.float16)
    hn, _ = oracle.rms_norm(x, st.norm.cpu().numpy(), s.eps)
    logits = hn.astype(np.float64) @ st.lm_head.cpu().numpy().astype(np.float64).T
    return x, logits, rows


def _per_op(st, snap, xs, pasts):
    """The per-op path, one sequence at a time on its own cache sequence: logits [bsz, vocab] and the new rows; caches restored."""
    logits, rows = [], []
    for b, past in enumerate(pasts):
        logits.append(st.decode_step(xs[b:b + 1].clone(), past, seq=b).clone())
        rows.append([(kc[b, :, past].clone(), vc[b, :, past].clone()) for kc, vc in zip(st.key_cache, st.value_cache)])
    _restore(st, snap)
    return logits, rows


def _untouched_except(st, snap, pasts):
    """No cache row of any sequence but row pasts[b] of sequences b < bsz was written."""
    for i, (kc, vc) in enumerate(zip(st.key_cache, st.value_cache)):
        for b in range(kc.shape[0]):
            mask = np.ones(st.max_seq, bool)
            if b < len(pasts):
                mask[pasts[b]] = False
            assert torch_equal(kc[b][:, mask], snap[i][0][b][:, mask]) and torch_equal(vc[b][:, mask], snap[i][1][b][:, mask]), (i, b)


def torch_equal(a, b):
    import torch
    return torch.equal(a, b)


PAST_SETS = {"uniform": lambda bsz: [37] * bsz, "ragged": lambda bsz: [0, 200, 16, 1][:bsz]}


@pytest.mark.parametrize("pasts", list(PAST_SETS))
@pytest.mark.parametrize("bsz", [2, 3, 4])
@pytest.mark.parametrize("gs", [128, 32])
@pytest.mark.parametrize("kv", [8, 2])
def test_batched_step_vs_oracle_and_per_op_path(oracle, kv, gs, bsz, pasts):
    import torch
    past = PAST_SETS[pasts](bsz)
    st = _mk_stack(1024, 2816, 2, 8, kv, gs, 256, batch=4, seed=3 + kv + gs)
    st.make_plan()
    info = st.dplan.info()
    assert info["grid"] >= 100 and info["ring_stages"] >= 8, info
    g = torch.Generator(device="cuda"); g.manual_seed(11 * bsz + gs + kv)
    xs = (torch.randn((bsz, 1, 1024), device="cuda", generator=g) * 0.5).half()
    snap = _snap(st)
    ref_logits, ref_rows = _per_op(st, snap, xs, past)
    logits = st.decode_step_fused_batch(xs, past).cpu().numpy()
    torch.cuda.synchronize()
    got_x = st._plan_xout[:bsz].cpu().numpy()
    assert logits.shape == (bsz, 2048)
    for b in range(bsz):
        want_x, want_logits, rows = _oracle_step(oracle, st, snap, xs[b].cpu().numpy(), past[b], b)
        w = f"seq {b} (ctx {past[b]})"
        assert_close_ref64(got_x[b], want_x.reshape(-1).astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} final hidden vs oracle")
        assert_close_ref64(logits[b], want_logits.reshape(-1), rel=1.5e-2, rms=1.5e-2, what=f"{w} logits vs oracle")
        assert_close_ref64(logits[b], ref_logits[b].cpu().numpy().reshape(-1).astype(np.float64), rel=1.5e-2, rms=1.5e-2, what=f"{w} logits vs per-op")
        for i, (kc, vc) in enumerate(zip(st.key_cache, st.value_cache)):
            k_new = kc[b, :, past[b]].cpu().numpy(); v_new = vc[b, :, past[b]].cpu().numpy()
            assert_close_ref64(k_new, rows[i][0].astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} layer {i} new k vs oracle")
            assert_close_ref64(v_new, rows[i][1].astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} layer {i} new v vs oracle")
            assert_close_ref64(k_new, ref_rows[b][i][0].cpu().numpy().astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} layer {i} new k vs per-op")
            assert_close_ref64(v_new, ref_rows[b][i][1].cpu().numpy().astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} layer {i} new v vs per-op")
    _untouched_except(st, snap, past)
    st.dplan.close(); st.close()


@pytest.mark.parametrize("kv", [8, 2])
def test_permuting_the_batch_permutes_the_outputs(oracle, kv):
    """Sequence j of a permuted batch is sequence perm[j] of the original (its x, context and cache): same logits, hidden state and
    new rows.  A lane / sequence mix-up in the GEMV, attention or head would break this."""
    import torch
    st = _mk_stack(1024, 2816, 2, 8, kv, 128, 256, batch=4, seed=13)
    st.make_plan()
    g = torch.Generator(device="cuda"); g.manual_seed(5)
    xs = (torch.randn((4, 1, 1024), device="cuda", generator=g) * 0.5).half()
    past = [5, 130, 64, 17]
    snap = _snap(st)
    base = st.decode_step_fused_batch(xs, past).clone(); base_x = st._plan_xout.clone()
    base_rows = [(kc.clone(), vc.clone()) for kc, vc in zip(st.key_cache, st.value_cache)]
    torch.cuda.synchronize()
    for perm in ([3, 2, 1, 0], [1, 3, 0, 2], [2, 0, 3, 1]):
        for (kc, vc), (k0, v0) in zip(zip(st.key_cache, st.value_cache), snap):
            kc.copy_(k0[perm]); vc.copy_(v0[perm])
        got = st.decode_step_fused_batch(xs[perm].contiguous(), [past[p] for p in perm]).clone()
        torch.cuda.synchronize()
        for j, p in enumerate(perm):
            assert_close_ref64(got[j].cpu().numpy(), base[p].cpu().numpy().astype(np.float64), rel=2e-3, rms=2e-3, what=f"perm {perm} logits {j}")
            assert_close_ref64(st._plan_xout[j].cpu().numpy(), base_x[p].cpu().numpy().astype(np.float64), rel=2e-3, rms=2e-3, what=f"perm {perm} hidden {j}")
            for i, (kc, vc) in enumerate(zip(st.key_cache, st.value_cache)):
                assert_close_ref64(kc[j, :, past[p]].cpu().numpy(), base_rows[i][0][p, :, past[p]].cpu().numpy().astype(np.float64), rel=2e-3, rms=2e-3, what=f"perm {perm} layer {i} k row {j}")
                assert_close_ref64(vc[j, :, past[p]].cpu().numpy(), base_rows[i][1][p, :, past[p]].cpu().numpy().astype(np.float64), rel=2e-3, rms=2e-3, what=f"perm {perm} layer {i} v row {j}")
    st.dplan.close(); st.close()


def test_batched_sequence_and_graph(oracle):
    """Five consecutive tokens for four sequences at different contexts, then CUDA-graph replay of the last launch."""
    import torch
    st = _mk_stack(1024, 2816, 3, 8, 2, 128, 128, batch=4, seed=5)
    st.make_plan()
    g = torch.Generator(device="cuda"); g.manual_seed(9)
    xs = [(torch.randn((4, 1, 1024), device="cuda", generator=g) * 0.5).half() for _ in range(5)]
    starts = [40, 3, 90, 17]
    snap = _snap(st)
    ref = []
    for t, x in enumerate(xs):                        # the per-op path, token by token, sequence by sequence
        ref.append([st.decode_step(x[b:b + 1].clone(), starts[b] + t, seq=b).clone() for b in range(4)])
    _restore(st, snap)
    got = [st.decode_step_fused_batch(x, [p + t for p in starts]).clone() for t, x in enumerate(xs)]
    torch.cuda.synchronize()
    for t in range(5):
        for b in range(4):
            assert_close_ref64(got[t][b].cpu().numpy(), ref[t][b].cpu().numpy().reshape(-1).astype(np.float64), rel=2e-2, rms=2e-2, what=f"token {t} seq {b}")
    x, last = xs[-1], [p + 4 for p in starts]
    side = torch.cuda.Stream(); side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        st.decode_step_fused_batch(x, last)
    torch.cuda.current_stream().wait_stream(side); torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        st.decode_step_fused_batch(x, last)
    for _ in range(3):
        gr.replay()
    torch.cuda.synchronize()
    assert_close_ref64(st._plan_logits.cpu().numpy(), got[-1].cpu().numpy().astype(np.float64), rel=2e-3, rms=2e-3, what="graph replay")
    st.dplan.close(); st.close()


def _needs_reset(heads, kv, bsz, longest, grid):
    """decode_step_sched.h att_needs_reset over virtual heads (tests/test_batch_schedule.py proves where it is needed)."""
    nph = max(1, (longest + 15) // 16)
    cap = 16 if kv < heads else 7
    return nph >= 2 and bsz * kv * nph < min(grid, bsz * kv * cap)


@pytest.mark.parametrize("kv", [8, 2])
def test_short_contexts_after_a_long_one(oracle, kv):
    """ONE batched plan: long contexts first (every partial slot written), then short and mixed ones; the reset launches exactly
    where att_needs_reset(longest context) says, and every sequence matches the per-op path."""
    import torch
    from exllama_b200 import capi
    st = _mk_stack(1024, 2816, 2, 8, kv, 128, 512, batch=3, seed=7)
    st.make_plan()
    grid = st.dplan.info()["grid"]
    g = torch.Generator(device="cuda"); g.manual_seed(21)
    snap = _snap(st)
    sets = [[400, 400, 400], [37, 17, 3], [17, 0, 16], [200, 241, 3], [2, 1], [96, 1, 2], [0, 5, 400], [300]]
    seen = set()
    for past in sets:
        x = (torch.randn((len(past), 1, 1024), device="cuda", generator=g) * 0.5).half()
        ref, _ = _per_op(st, snap, x, past)
        n0 = capi.launch_count()
        got = st.decode_step_fused_batch(x, past).clone()
        torch.cuda.synchronize()
        reset = _needs_reset(8, kv, len(past), max(past), grid)
        seen.add(reset)
        assert capi.launch_count() - n0 == 1 + int(reset), (past, capi.launch_count() - n0)
        _untouched_except(st, snap, past)
        _restore(st, snap)
        for b in range(len(past)):
            assert_close_ref64(got[b].cpu().numpy(), ref[b].cpu().numpy().reshape(-1).astype(np.float64), rel=1.5e-2, rms=1.5e-2, what=f"ctx {past} seq {b}")
    assert seen == {True, False}
    st.dplan.close(); st.close()


@pytest.mark.parametrize("name,bsz,ctx,max_seq", [("7b", 4, 1920, 2048), ("70b", 2, 1920, 2048)])
def test_full_shapes_vs_per_op(oracle, name, bsz, ctx, max_seq):
    """Llama 7B (batch 4) and Llama-2 70B (batch 2, 64 heads over 8 KV heads) shapes, 2 layers, against the per-op path."""
    import torch
    from exllama_b200.shapes import GQA_SHAPES, SHAPES
    s = {**SHAPES, **GQA_SHAPES}[name]
    st = _mk_stack(s.hidden, s.inter, 2, s.heads, s.kv_heads, 128, max_seq, batch=bsz, vocab=s.vocab, seed=17)
    st.make_plan()
    assert st.dplan.info()["ring_stages"] >= 8
    g = torch.Generator(device="cuda"); g.manual_seed(23)
    xs = (torch.randn((bsz, 1, s.hidden), device="cuda", generator=g) * 0.5).half()
    past = [ctx - 37 * b for b in range(bsz)]
    snap = _snap(st)
    ref, _ = _per_op(st, snap, xs, past)
    got = st.decode_step_fused_batch(xs, past)
    torch.cuda.synchronize()
    assert torch.isfinite(got).all()
    for b in range(bsz):
        assert_close_ref64(got[b].cpu().numpy(), ref[b].cpu().numpy().reshape(-1).astype(np.float64), rel=1.5e-2, rms=1.5e-2, what=f"{name} seq {b} logits")
    _untouched_except(st, snap, past)
    st.dplan.close(); st.close()


def test_rejected_arguments(oracle):
    """Every EXL_ERR_ARG case of the batched entry points, each with a message that says what to use instead."""
    import torch
    from exllama_b200 import capi
    st = _mk_stack(1024, 2816, 1, 8, 8, 128, 64, batch=2)
    hs = [[L.q.q4, L.k.q4, L.v.q4, L.o.q4, L.gate.q4, L.up.q4, L.down.q4] for L in st.layers]
    args = (hs, [L.ln1 for L in st.layers], [L.ln2 for L in st.layers], st.key_cache, st.value_cache, st.sin, st.cos, 8, 128, st.max_seq, 1e-6)
    for mb in (0, 5):
        with pytest.raises(capi.ExlError, match=r"error 1: .*max_batch %d outside 1\.\.4.*per-op" % mb):
            capi.DecodePlan(*args, max_batch=mb)
    with pytest.raises(capi.ExlError, match=r"error 1: .*tensor parallelism.*max_batch 1 or the per-op path"):
        capi.DecodePlan(*args, tp_rank=0, tp_world=2, max_batch=2)
    plan = capi.DecodePlan(*args, max_batch=2)
    x = torch.zeros((4, 1024), dtype=torch.float16, device="cuda")
    lg = torch.zeros((4, 2048), dtype=torch.float32, device="cuda")
    with pytest.raises(capi.ExlError, match=r"error 1: .*bsz 3 outside 1\.\.2.*exl_decode_plan_create_batch"):
        plan.step_batch(x, [1, 2, 3], logits=lg)
    with pytest.raises(capi.ExlError, match=r"error 1: .*bsz 0 outside 1\.\.2"):
        plan.step_batch(x, [], logits=lg)
    with pytest.raises(capi.ExlError, match=r"error 1: .*past_len\[1\] = 64 outside the cache \(max_seq 64\)"):
        plan.step_batch(x, [3, 64], logits=lg)
    with pytest.raises(capi.ExlError, match=r"error 1: .*past_len\[0\] = -1 outside the cache"):
        plan.step_batch(x, [-1, 3], logits=lg)
    plan.close()
    one = capi.DecodePlan(*args)                                     # a single-sequence plan takes bsz 1 only
    with pytest.raises(capi.ExlError, match=r"error 1: .*bsz 2 outside 1\.\.1"):
        one.step_batch(x, [1, 2], logits=lg)
    one.close(); st.close()
    # act-order matrices with a batch
    sa = _mk_stack(1024, 2816, 1, 8, 8, 128, 64, batch=2, act=True)
    with pytest.raises(capi.ExlError, match=r"error 1: .*act-order.*max_batch 1 or the per-op path"):
        sa.make_plan()
    sa.close()
    # more than fits: 13B's 40 heads take at most 3 sequences on 132 SMs
    from exllama_b200.shapes import SHAPES
    s = SHAPES["13b"]
    big = _mk_stack(s.hidden, s.inter, 1, s.heads, s.heads, 128, 64, batch=4, vocab=512)
    with pytest.raises(capi.ExlError, match=r"error 1: .*max_batch 4 does not fit.*the largest batch is [0-3]$"):
        big.make_plan()
    big.close()


def test_single_sequence_plan_unchanged(oracle):
    """exl_decode_plan_create is exl_decode_plan_create_batch(.., 1, ..): the same plan info, and exl_decode_step is a batch of one."""
    import torch
    st = _mk_stack(1024, 2816, 2, 8, 2, 128, 128, batch=1, seed=31)
    st.make_plan()
    info1 = st.dplan.info()
    x = (torch.randn((1, 1, 1024), device="cuda") * 0.5).half()
    snap = _snap(st)
    a = st.decode_step_fused(x, 50).clone()
    _restore(st, snap)
    b = st.dplan.step_batch(x, [50], x_out=st._plan_xout).clone()
    torch.cuda.synchronize()
    assert_close_ref64(b.cpu().numpy(), a.cpu().numpy().astype(np.float64), rel=2e-3, rms=2e-3, what="step_batch(bsz 1) vs step")
    st.dplan.close(); st.close()
    sb = _mk_stack(1024, 2816, 2, 8, 2, 128, 128, batch=4, seed=31)
    sb.make_plan()
    assert sb.dplan.info()["barriers_per_step"] == info1["barriers_per_step"] and sb.dplan.info()["grid"] == info1["grid"]
    sb.dplan.close(); sb.close()
