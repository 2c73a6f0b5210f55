"""Grouped-query attention (kv_heads < heads, Llama-2 70B's 64 query heads over 8 KV heads) on the GPU.

(a) exl_q4_attn with kv_heads < heads -- the single-launch path (q/k/v share one x order) and the general path (act-order: three
    distinct x_maps) -- against the oracle composition and, where the reference can run it, the reference's own q4_attn (its H100
    outputs in tests/golden/ref_gpu_gqa.npz, written by oracle/gen_golden_ref_gpu_gqa.py).  The reference's cache update writes
    BLOCKSIZE_Z = 4 KV heads per thread (q4_attn.cu:17,50-71), so it needs kv_heads % 4 == 0: with 1 or 2 KV heads it writes
    past the end of the cache, and those cases are pinned to the oracle only.
(b) The persistent decode step on a GQA plan against the float64 oracle composition (decode_attn_f64 with kv_heads) and against
    the per-op path, on the same seeded synthetic stack: consecutive tokens, CUDA-graph replay, short contexts after a long one,
    the 70B shape.
Tolerances are those of tests/test_gpu_decode_step.py and tests/test_gpu_ref_pin.py.
"""
import os

import numpy as np
import pytest

from helpers import GOLDEN, close_to_reference, to_cuda
from stack_harness import (check_fused_step, check_reset_after_long_context, check_sequence_and_graph, lib_state,  # noqa: F401
                           sincos, stacks)

pytestmark = pytest.mark.gpu

SMS = 132


@pytest.fixture(scope="module")
def golden_gqa():
    return np.load(os.path.join(GOLDEN, "ref_gpu_gqa.npz"))


# ------------------------------------------------------------------------------------------------- (a) per-op q4_attn
Q4_ATTN_CASES = [(h, kv, q_len, past, act) for (h, kv) in [(8, 2), (8, 1), (16, 2), (8, 4), (16, 4)] for q_len in (1, 2)
                 for past in (0, 37) for act in (False, True)]
REF_CASES = [c for c in Q4_ATTN_CASES if c[1] % 4 == 0]          # what the reference's update_cache_kernel can do
MAX_SEQ_OP = 64


def q4_attn_inputs(oracle, heads, kv, q_len, act):
    """Seeded inputs of one q4_attn call: hidden = heads * 128, k / v projections kv * 128 wide, groupsize 128."""
    hd, hidden = 128, heads * 128
    seed = 500 + 10 * heads + kv
    t = {n: oracle.synth_q4(hidden, N, 128, act_order=act, seed=seed + i) for i, (n, N) in enumerate([("q", hidden), ("k", kv * hd), ("v", kv * hd)])}
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((1, q_len, hidden)).astype(np.float16)
    w = (1 + 0.1 * rng.standard_normal(hidden)).astype(np.float16)
    return t, x, w


def q4_attn_key(heads, kv, q_len, past, act):
    return f"q4_attn_{heads}_{kv}_{q_len}_{past}_{int(act)}"


@pytest.mark.parametrize("heads,kv,q_len,past,act", Q4_ATTN_CASES)
def test_q4_attn_gqa_vs_reference_and_oracle(oracle, golden_gqa, heads, kv, q_len, past, act):
    import torch
    from exllama_b200 import capi
    hd = 128
    hidden = heads * hd
    t, x, w = q4_attn_inputs(oracle, heads, kv, q_len, act)
    sin, cos = sincos(MAX_SEQ_OP, hd)
    ts, tc, tw = to_cuda(sin, cos, w)
    mats = [capi.Q4(*to_cuda(qw.copy(), qz, sc), None if g is None else torch.from_numpy(g)) for (qw, qz, sc, g) in (t["q"], t["k"], t["v"])]
    tx = to_cuda(x.copy())
    q = torch.zeros((1, q_len, hidden), dtype=torch.float16, device="cuda")
    k = torch.zeros((1, q_len, kv * hd), dtype=torch.float16, device="cuda"); v = torch.zeros_like(k)
    kc = torch.zeros((1, kv, MAX_SEQ_OP, hd), dtype=torch.float16, device="cuda"); vc = torch.zeros_like(kc)
    torch.cuda.synchronize()
    capi.q4_attn(tx, tw, 1e-6, q, k, v, *mats, ts, tc, q_len, past, heads, kv, hd, kc, vc, MAX_SEQ_OP)
    torch.cuda.synchronize()
    ours = [a.cpu().numpy() for a in (q, k, v, kc, vc, tx)]
    key = q4_attn_key(heads, kv, q_len, past, act)
    ref = [golden_gqa[f"{key}_{n}"] for n in ("q", "k", "v", "kc", "vc")] if (heads, kv, q_len, past, act) in REF_CASES else None
    # oracle composition: norm -> projections (fp16) -> rope of q over heads, of k over kv_heads (rope.cu:48-67)
    xn, _ = oracle.rms_norm(x.reshape(q_len, hidden), w, 1e-6)
    q16, k16, v16 = (oracle.ref64_with_act_order(xn, *t[n]).astype(np.float16) for n in ("q", "k", "v"))
    q16 = oracle.rope(q16.reshape(1, q_len * heads, hd), sin, cos, 1, q_len * heads, hd, heads, past).reshape(1, q_len, hidden)
    k16 = oracle.rope(k16.reshape(1, q_len * kv, hd), sin, cos, 1, q_len * kv, hd, kv, past).reshape(1, q_len, kv * hd)
    for i, (name, want) in enumerate((("q", q16), ("k", k16), ("v", v16.reshape(1, q_len, kv * hd)))):
        if ref is not None:
            close_to_reference(ours[i], ref[i], f"{name} vs reference q4_attn")
        close_to_reference(ours[i], want, f"{name} vs oracle")
    np.testing.assert_array_equal(ours[5], x)                   # x itself is not modified
    # cache: rows past .. past + q_len of the kv_heads caches hold k / v exactly, every other row untouched
    for who, (qq, kk, vv, kcc, vcc) in [("ours", ours[:5])] + ([("reference", ref)] if ref is not None else []):
        for tt in range(q_len):
            np.testing.assert_array_equal(kcc[0, :, past + tt], kk.reshape(q_len, kv, hd)[tt], err_msg=who)
            np.testing.assert_array_equal(vcc[0, :, past + tt], vv.reshape(q_len, kv, hd)[tt], err_msg=who)
        mask = np.ones(MAX_SEQ_OP, bool); mask[past:past + q_len] = False
        assert not kcc[0][:, mask].any() and not vcc[0][:, mask].any(), who


# ------------------------------------------------------------------------------------------------- (b) persistent decode step
@pytest.mark.parametrize("act", [False, True])
@pytest.mark.parametrize("gs", [128, 32])
@pytest.mark.parametrize("kv", [1, 2, 4])
@pytest.mark.parametrize("past", [0, 1, 16, 37, 200])
def test_fused_step_gqa_vs_oracle_and_per_op_path(oracle, stacks, kv, gs, act, past):
    import torch
    st = stacks(kv_heads=kv, gs=gs, act=act)
    st.make_plan()
    info = st.dplan.info()
    assert info["grid"] >= 100 and info["ring_stages"] >= 8, info
    rng = np.random.default_rng(past + gs + kv)
    x = (rng.standard_normal(st.shape.hidden) * 0.5).astype(np.float16)
    check_fused_step(oracle, st, torch.from_numpy(x).cuda().view(1, 1, -1), [past], f"kv {kv} g{gs} act {act}")
    assert all(kc.shape[1] == kv for kc in st.key_cache)


def test_fused_step_gqa_sequence_and_graph(oracle, stacks):
    """Five consecutive tokens on a GQA plan (8 heads over 2 KV heads), then CUDA-graph replay of the last one."""
    import torch
    st = stacks(layers=3, kv_heads=2, max_seq=128, seed=5)
    st.make_plan()
    g = torch.Generator(device="cuda"); g.manual_seed(9)
    xs = [(torch.randn((1, 1, 1024), device="cuda", generator=g) * 0.5).half() for _ in range(5)]
    check_sequence_and_graph(st, xs, [40])


def test_fused_step_gqa_short_context_after_long_one(oracle, stacks):
    """ONE GQA plan: a long context first (every partial slot written), then short ones where CTAs inside a KV head's CTA range own
    no attention unit: exl_decode_step resets the table exactly where the CPU proof says (tests/test_gqa_schedule.py)."""
    import torch
    st = stacks(kv_heads=2, max_seq=512, seed=7)
    st.make_plan()
    g = torch.Generator(device="cuda"); g.manual_seed(21)
    # 2 KV heads -> 32 CTAs take part; contexts 17 .. 240 leave some of them idle
    contexts = [[400], [37], [17], [200], [241], [3], [96], [400]]
    xs = [(torch.randn((1, 1, 1024), device="cuda", generator=g) * 0.5).half() for _ in contexts]
    check_reset_after_long_context(st, xs, contexts)


@pytest.mark.parametrize("ctx,max_seq,act", [(1920, 2048, False), (4000, 4096, False), (1920, 2048, True)])
def test_fused_step_70b_shape(oracle, stacks, ctx, max_seq, act):
    """Llama-2 70B shape (hidden 8192, inter 28672, 64 heads over 8 KV heads), 2 layers: against the per-op path."""
    import torch
    from exllama_b200.shapes import GQA_SHAPES
    s = GQA_SHAPES["70b"]
    st = stacks(hidden=s.hidden, inter=s.inter, heads=s.heads, kv_heads=s.kv_heads, max_seq=max_seq, vocab=s.vocab, seed=17, act=act)
    st.make_plan()
    assert st.dplan.info()["ring_stages"] >= 8
    x = (torch.randn((1, 1, s.hidden), device="cuda") * 0.5).half()
    check_fused_step(None, st, x, [ctx], "70B shape")


def test_plan_rejects_unsupported_gqa(oracle, stacks):
    """GQA under tensor parallelism, and a KV-head count that does not divide the heads: EXL_ERR_ARG with a message."""
    from exllama_b200 import capi
    st = stacks(layers=1, kv_heads=2, max_seq=64)
    hs = [[L.q.q4, L.k.q4, L.v.q4, L.o.q4, L.gate.q4, L.up.q4, L.down.q4] for L in st.layers]
    args = (hs, [L.ln1 for L in st.layers], [L.ln2 for L in st.layers], st.key_cache, st.value_cache, st.sin, st.cos, 8, 128, st.max_seq, 1e-6)
    with pytest.raises(capi.ExlError, match=r"error 1: .*tensor parallelism.*per-op"):
        capi.DecodePlan(*args, tp_rank=0, tp_world=2, num_kv_heads=2)
    with pytest.raises(capi.ExlError, match=r"error 1: .*num_kv_heads \(3\) must divide num_heads \(8\)"):
        capi.DecodePlan(*args, num_kv_heads=3)
