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
from stack_harness import (check_fused_step, check_reset_after_long_context, check_sequence_and_graph, lib_state,  # noqa: F401
                           restore, snapshot, stacks, untouched_except)

pytestmark = pytest.mark.gpu


PAST_SETS = {"uniform": lambda bsz: [37] * bsz, "ragged": lambda bsz: [0, 200, 16, 1][:bsz]}


@pytest.mark.parametrize("pasts", list(PAST_SETS))
@pytest.mark.parametrize("bsz", [2, 3, 4])
@pytest.mark.parametrize("gs", [128, 32])
@pytest.mark.parametrize("kv", [8, 2])
def test_batched_step_vs_oracle_and_per_op_path(oracle, stacks, kv, gs, bsz, pasts):
    import torch
    past = PAST_SETS[pasts](bsz)
    st = stacks(kv_heads=kv, gs=gs, batch=4, seed=3 + kv + gs)
    st.make_plan()
    info = st.dplan.info()
    assert info["grid"] >= 100 and info["ring_stages"] >= 8, info
    g = torch.Generator(device="cuda"); g.manual_seed(11 * bsz + gs + kv)
    xs = (torch.randn((bsz, 1, 1024), device="cuda", generator=g) * 0.5).half()
    logits, _, _ = check_fused_step(oracle, st, xs, past, f"kv {kv} g{gs}")
    assert logits.shape == (bsz, 2048)


@pytest.mark.parametrize("kv", [8, 2])
def test_permuting_the_batch_permutes_the_outputs(oracle, stacks, kv):
    """Sequence j of a permuted batch is sequence perm[j] of the original (its x, context and cache): same logits, hidden state and
    new rows.  A lane / sequence mix-up in the GEMV, attention or head would break this."""
    import torch
    st = stacks(kv_heads=kv, batch=4, seed=13)
    st.make_plan()
    g = torch.Generator(device="cuda"); g.manual_seed(5)
    xs = (torch.randn((4, 1, 1024), device="cuda", generator=g) * 0.5).half()
    past = [5, 130, 64, 17]
    snap = snapshot(st)
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


def test_batched_sequence_and_graph(oracle, stacks):
    """Five consecutive tokens for four sequences at different contexts, then CUDA-graph replay of the last launch."""
    import torch
    st = stacks(layers=3, kv_heads=2, max_seq=128, batch=4, seed=5)
    st.make_plan()
    g = torch.Generator(device="cuda"); g.manual_seed(9)
    xs = [(torch.randn((4, 1, 1024), device="cuda", generator=g) * 0.5).half() for _ in range(5)]
    check_sequence_and_graph(st, xs, [40, 3, 90, 17])


@pytest.mark.parametrize("kv", [8, 2])
def test_short_contexts_after_a_long_one(oracle, stacks, kv):
    """ONE batched plan: long contexts first (every partial slot written), then short and mixed ones; the reset launches exactly
    where att_needs_reset(longest context) says, and every sequence matches the per-op path."""
    import torch
    st = stacks(kv_heads=kv, max_seq=512, batch=3, seed=7)
    st.make_plan()
    g = torch.Generator(device="cuda"); g.manual_seed(21)
    sets = [[400, 400, 400], [37, 17, 3], [17, 0, 16], [200, 241, 3], [2, 1], [96, 1, 2], [0, 5, 400], [300]]
    xs = [(torch.randn((len(past), 1, 1024), device="cuda", generator=g) * 0.5).half() for past in sets]
    assert check_reset_after_long_context(st, xs, sets, check_untouched=True) == {True, False}


@pytest.mark.parametrize("name,bsz,ctx,max_seq", [("7b", 4, 1920, 2048), ("70b", 2, 1920, 2048)])
def test_full_shapes_vs_per_op(oracle, stacks, name, bsz, ctx, max_seq):
    """Llama 7B (batch 4) and Llama-2 70B (batch 2, 64 heads over 8 KV heads) shapes, 2 layers, against the per-op path."""
    import torch
    from exllama_b200.shapes import GQA_SHAPES, SHAPES
    s = {**SHAPES, **GQA_SHAPES}[name]
    st = stacks(hidden=s.hidden, inter=s.inter, heads=s.heads, kv_heads=s.kv_heads, max_seq=max_seq, batch=bsz, vocab=s.vocab, seed=17)
    st.make_plan()
    assert st.dplan.info()["ring_stages"] >= 8
    g = torch.Generator(device="cuda"); g.manual_seed(23)
    xs = (torch.randn((bsz, 1, s.hidden), device="cuda", generator=g) * 0.5).half()
    past = [ctx - 37 * b for b in range(bsz)]
    snap = snapshot(st)
    check_fused_step(None, st, xs, past, name)
    untouched_except(st, snap, past)


def test_rejected_arguments(oracle, stacks):
    """Every EXL_ERR_ARG case of the batched entry points, each with a message that says what to use instead."""
    import torch
    from exllama_b200 import capi
    st = stacks(layers=1, kv_heads=8, max_seq=64, batch=2)
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
    one.close()
    # act-order matrices with a batch
    sa = stacks(layers=1, kv_heads=8, max_seq=64, batch=2, act=True)
    with pytest.raises(capi.ExlError, match=r"error 1: .*act-order.*max_batch 1 or the per-op path"):
        sa.make_plan()
    # more than fits: 13B's 40 heads take at most 3 sequences on 132 SMs
    from exllama_b200.shapes import SHAPES
    s = SHAPES["13b"]
    big = stacks(hidden=s.hidden, inter=s.inter, layers=1, heads=s.heads, kv_heads=s.heads, max_seq=64, batch=4, vocab=512)
    with pytest.raises(capi.ExlError, match=r"error 1: .*max_batch 4 does not fit.*the largest batch is [0-3]$"):
        big.make_plan()


def test_single_sequence_plan_unchanged(oracle, stacks):
    """exl_decode_plan_create is exl_decode_plan_create_batch(.., 1, ..): the same plan info, and exl_decode_step is a batch of one."""
    import torch
    st = stacks(kv_heads=2, max_seq=128, batch=1, seed=31)
    st.make_plan()
    info1 = st.dplan.info()
    x = (torch.randn((1, 1, 1024), device="cuda") * 0.5).half()
    snap = snapshot(st)
    a = st.decode_step_fused(x, 50).clone()
    restore(st, snap)
    b = st.dplan.step_batch(x, [50], x_out=st._plan_xout).clone()
    torch.cuda.synchronize()
    assert_close_ref64(b.cpu().numpy(), a.cpu().numpy().astype(np.float64), rel=2e-3, rms=2e-3, what="step_batch(bsz 1) vs step")
    st.dplan.close(); st.close()
    sb = stacks(kv_heads=2, max_seq=128, batch=4, seed=31)
    sb.make_plan()
    assert sb.dplan.info()["barriers_per_step"] == info1["barriers_per_step"] and sb.dplan.info()["grid"] == info1["grid"]
