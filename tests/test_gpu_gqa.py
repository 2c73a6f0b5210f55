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

from helpers import GOLDEN, assert_close_ref64, to_cuda

pytestmark = pytest.mark.gpu

SMS = 132


@pytest.fixture(scope="module")
def golden_gqa():
    return np.load(os.path.join(GOLDEN, "ref_gpu_gqa.npz"))


def _sincos(max_seq, hd):
    inv = 1.0 / (10000 ** (np.arange(0, hd, 2, dtype=np.float64) / hd))
    ang = np.outer(np.arange(max_seq), inv)
    emb = np.concatenate([ang, ang], -1)
    return np.sin(emb).astype(np.float16), np.cos(emb).astype(np.float16)


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


def _close_to_reference(mine, ref, what):
    mine = np.asarray(mine, np.float64); ref = np.asarray(ref, np.float64)
    rms = np.sqrt(np.mean(ref ** 2))
    bad = np.abs(mine - ref) > 2e-2 * np.abs(ref) + 2e-2 * rms
    assert not bad.any(), f"{what}: {bad.sum()} / {bad.size} outside 2e-2; max {np.abs(mine - ref).max():.4g}, rms {rms:.4g}"


@pytest.mark.parametrize("heads,kv,q_len,past,act", Q4_ATTN_CASES)
def test_q4_attn_gqa_vs_reference_and_oracle(oracle, golden_gqa, heads, kv, q_len, past, act):
    import torch
    from exllama_b200 import capi
    hd = 128
    hidden = heads * hd
    t, x, w = q4_attn_inputs(oracle, heads, kv, q_len, act)
    sin, cos = _sincos(MAX_SEQ_OP, hd)
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
            _close_to_reference(ours[i], ref[i], f"{name} vs reference q4_attn")
        _close_to_reference(ours[i], want, f"{name} vs oracle")
    np.testing.assert_array_equal(ours[5], x)                   # x itself is not modified
    # cache: rows past .. past + q_len of the kv_heads caches hold k / v exactly, every other row untouched
    for who, (qq, kk, vv, kcc, vcc) in [("ours", ours[:5])] + ([("reference", ref)] if ref is not None else []):
        for tt in range(q_len):
            np.testing.assert_array_equal(kcc[0, :, past + tt], kk.reshape(q_len, kv, hd)[tt], err_msg=who)
            np.testing.assert_array_equal(vcc[0, :, past + tt], vv.reshape(q_len, kv, hd)[tt], err_msg=who)
        mask = np.ones(MAX_SEQ_OP, bool); mask[past:past + q_len] = False
        assert not kcc[0][:, mask].any() and not vcc[0][:, mask].any(), who


# ------------------------------------------------------------------------------------------------- (b) persistent decode step
def _mk_stack(hidden, inter, layers, heads, kv_heads, gs, max_seq, vocab=2048, seed=3, act=False):
    import torch
    from exllama_b200.stack import DecodeStack, LlamaShape
    shape = LlamaShape("synthetic-gqa", hidden, inter, layers, heads, vocab=vocab, kv_heads=kv_heads)
    st = DecodeStack(shape, groupsize=gs, act_order=act, device="cuda:0", max_seq=max_seq, seed=seed)
    g = torch.Generator(device="cuda"); g.manual_seed(seed + 100)
    for kc, vc in zip(st.key_cache, st.value_cache):
        kc.copy_((torch.randn(kc.shape, device="cuda", generator=g) * 0.5).half())
        vc.copy_((torch.randn(vc.shape, device="cuda", generator=g) * 0.5).half())
    return st


def _oracle_step_gqa(oracle, st, x, past):
    """float64/fp16 restatement of one decode token with grouped-query attention: returns (final hidden fp16, logits float64,
    new k/v rows [kv_heads, 128] per layer)."""
    s = st.shape
    hd, heads, kvh = s.head_dim, s.heads, s.kv_heads
    sin = st.sin.view(-1, hd).cpu().numpy(); cos = st.cos.view(-1, hd).cpu().numpy()
    x = x.reshape(1, s.hidden).copy()
    rows = []

    def mm(xin, lin, acc=None):
        xm = None if lin.g_idx is None else oracle.make_x_map(lin.g_idx.numpy(), lin.qzeros.shape[0])
        return oracle.q4_matmul_f64(xin, lin.qweight.cpu().numpy(), lin.qzeros.cpu().numpy(), lin.scales.cpu().numpy(), xm, acc)
    for i, L in enumerate(st.layers):
        xn, _ = oracle.rms_norm(x, L.ln1.cpu().numpy(), s.eps)
        q = mm(xn, L.q).astype(np.float16); k = mm(xn, L.k).astype(np.float16); v = mm(xn, L.v).astype(np.float16)
        q = oracle.rope(q.reshape(1, heads, hd), sin, cos, 1, heads, hd, heads, past).reshape(-1)
        k = oracle.rope(k.reshape(1, kvh, hd), sin, cos, 1, kvh, hd, kvh, past).reshape(kvh, hd)
        kc = st.key_cache[i][0].cpu().numpy().copy(); vc = st.value_cache[i][0].cpu().numpy().copy()
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


def _restore(st, snap):
    for (kc, vc), (k0, v0) in zip(zip(st.key_cache, st.value_cache), snap):
        kc.copy_(k0); vc.copy_(v0)


@pytest.mark.parametrize("act", [False, True])
@pytest.mark.parametrize("gs", [128, 32])
@pytest.mark.parametrize("kv", [1, 2, 4])
@pytest.mark.parametrize("past", [0, 1, 16, 37, 200])
def test_fused_step_gqa_vs_oracle_and_per_op_path(oracle, kv, gs, act, past):
    import torch
    st = _mk_stack(1024, 2816, 2, 8, kv, gs, 256, act=act)
    st.make_plan()
    info = st.dplan.info()
    assert info["grid"] >= 100 and info["ring_stages"] >= 8, info
    rng = np.random.default_rng(past + gs + kv)
    x = (rng.standard_normal(st.shape.hidden) * 0.5).astype(np.float16)
    want_x, want_logits, rows = _oracle_step_gqa(oracle, st, x, past)
    snap = [(kc.clone(), vc.clone()) for kc, vc in zip(st.key_cache, st.value_cache)]
    hid = torch.from_numpy(x).cuda().view(1, 1, -1)
    ref_logits = st.decode_step(hid.clone(), past).cpu().numpy()
    per_op_rows = [(kc[0, :, past].cpu().numpy().copy(), vc[0, :, past].cpu().numpy().copy()) for kc, vc in zip(st.key_cache, st.value_cache)]
    _restore(st, snap)
    logits = st.decode_step_fused(hid, past).cpu().numpy()
    torch.cuda.synchronize()
    got_x = st._plan_xout.cpu().numpy()
    assert_close_ref64(got_x, want_x.reshape(-1).astype(np.float64), rel=1e-2, rms=1e-2, what="final hidden vs oracle")
    assert_close_ref64(logits.reshape(-1), want_logits.reshape(-1), rel=1.5e-2, rms=1.5e-2, what="logits vs oracle")
    assert_close_ref64(logits.reshape(-1), ref_logits.reshape(-1).astype(np.float64), rel=1.5e-2, rms=1.5e-2, what="logits vs per-op path")
    for i, (kc, vc) in enumerate(zip(st.key_cache, st.value_cache)):
        assert kc.shape[1] == kv
        k_new = kc[0, :, past].cpu().numpy(); v_new = vc[0, :, past].cpu().numpy()
        assert_close_ref64(k_new, rows[i][0].astype(np.float64), rel=1e-2, rms=1e-2, what=f"layer {i} new k row vs oracle")
        assert_close_ref64(v_new, rows[i][1].astype(np.float64), rel=1e-2, rms=1e-2, what=f"layer {i} new v row vs oracle")
        assert_close_ref64(k_new, per_op_rows[i][0].astype(np.float64), rel=1e-2, rms=1e-2, what=f"layer {i} new k row vs per-op")
        assert_close_ref64(v_new, per_op_rows[i][1].astype(np.float64), rel=1e-2, rms=1e-2, what=f"layer {i} new v row vs per-op")
        mask = np.ones(st.max_seq, bool); mask[past] = False          # nothing but row `past` was written
        assert torch.equal(kc[0][:, mask], snap[i][0][0][:, mask]) and torch.equal(vc[0][:, mask], snap[i][1][0][:, mask])
    st.dplan.close(); st.close()


def test_fused_step_gqa_sequence_and_graph(oracle):
    """Five consecutive tokens on a GQA plan (8 heads over 2 KV heads), then CUDA-graph replay of the last one."""
    import torch
    st = _mk_stack(1024, 2816, 3, 8, 2, 128, 128, seed=5)
    st.make_plan()
    g = torch.Generator(device="cuda"); g.manual_seed(9)
    xs = [(torch.randn((1, 1, 1024), device="cuda", generator=g) * 0.5).half() for _ in range(5)]
    snap = [(kc.clone(), vc.clone()) for kc, vc in zip(st.key_cache, st.value_cache)]
    ref = [st.decode_step(x.clone(), 40 + i).clone() for i, x in enumerate(xs)]
    _restore(st, snap)
    got = [st.decode_step_fused(x, 40 + i).clone() for i, x in enumerate(xs)]
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(got, ref)):
        assert_close_ref64(a.cpu().numpy().reshape(-1), b.cpu().numpy().reshape(-1).astype(np.float64), rel=2e-2, rms=2e-2, what=f"token {i}")
    x = xs[-1]
    side = torch.cuda.Stream(); side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        st.decode_step_fused(x, 44)
    torch.cuda.current_stream().wait_stream(side); torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        st.decode_step_fused(x, 44)
    for _ in range(3):
        gr.replay()
    torch.cuda.synchronize()
    assert_close_ref64(st._plan_logits.cpu().numpy().reshape(-1), got[-1].cpu().numpy().reshape(-1).astype(np.float64), rel=2e-3, rms=2e-3, what="graph replay")
    st.dplan.close(); st.close()


def _needs_reset(kv_heads, past, grid):
    """decode_step_sched.h att_needs_reset under GQA: fewer attention units than the CTAs that take part (16 per KV head)."""
    nph = max(1, (past + 15) // 16)
    return nph >= 2 and kv_heads * nph < min(grid, 16 * kv_heads)


def test_fused_step_gqa_short_context_after_long_one(oracle):
    """ONE GQA plan: a long context first (every partial slot written), then short ones where CTAs inside a KV head's CTA range own
    no attention unit: exl_decode_step resets the table exactly where the CPU proof says (tests/test_gqa_schedule.py)."""
    import torch
    from exllama_b200 import capi
    st = _mk_stack(1024, 2816, 2, 8, 2, 128, 512, seed=7)
    st.make_plan()
    grid = st.dplan.info()["grid"]
    g = torch.Generator(device="cuda"); g.manual_seed(21)
    snap = [(kc.clone(), vc.clone()) for kc, vc in zip(st.key_cache, st.value_cache)]
    # 2 KV heads -> 32 CTAs take part; contexts 17 .. 240 leave some of them idle
    for past in [400, 37, 17, 200, 241, 3, 96, 400]:
        x = (torch.randn((1, 1, 1024), device="cuda", generator=g) * 0.5).half()
        ref = st.decode_step(x.clone(), past).clone()
        _restore(st, snap)
        n0 = capi.launch_count()
        got = st.decode_step_fused(x, past).clone()
        torch.cuda.synchronize()
        assert capi.launch_count() - n0 == 1 + int(_needs_reset(2, past, grid)), (past, capi.launch_count() - n0)
        _restore(st, snap)
        assert_close_ref64(got.cpu().numpy().reshape(-1), ref.cpu().numpy().reshape(-1).astype(np.float64), rel=1.5e-2, rms=1.5e-2, what=f"logits at ctx {past}")
    st.dplan.close(); st.close()


@pytest.mark.parametrize("ctx,max_seq,act", [(1920, 2048, False), (4000, 4096, False), (1920, 2048, True)])
def test_fused_step_70b_shape(oracle, ctx, max_seq, act):
    """Llama-2 70B shape (hidden 8192, inter 28672, 64 heads over 8 KV heads, vocab 32000), 2 layers: against the per-op path."""
    import torch
    from exllama_b200.shapes import GQA_SHAPES
    s = GQA_SHAPES["70b"]
    st = _mk_stack(s.hidden, s.inter, 2, s.heads, s.kv_heads, 128, max_seq, vocab=s.vocab, seed=17, act=act)
    st.make_plan()
    assert st.dplan.info()["ring_stages"] >= 8
    x = (torch.randn((1, 1, s.hidden), device="cuda") * 0.5).half()
    snap = [(kc.clone(), vc.clone()) for kc, vc in zip(st.key_cache, st.value_cache)]
    ref = st.decode_step(x.clone(), ctx).clone()
    _restore(st, snap)
    got = st.decode_step_fused(x, ctx)
    torch.cuda.synchronize()
    assert torch.isfinite(got).all()
    assert_close_ref64(got.cpu().numpy().reshape(-1), ref.cpu().numpy().reshape(-1).astype(np.float64), rel=1.5e-2, rms=1.5e-2, what="70B-shape logits")
    st.dplan.close(); st.close()


def test_plan_rejects_unsupported_gqa(oracle):
    """GQA under tensor parallelism, and a KV-head count that does not divide the heads: EXL_ERR_ARG with a message."""
    from exllama_b200 import capi
    st = _mk_stack(1024, 2816, 1, 8, 2, 128, 64)
    hs = [[L.q.q4, L.k.q4, L.v.q4, L.o.q4, L.gate.q4, L.up.q4, L.down.q4] for L in st.layers]
    args = (hs, [L.ln1 for L in st.layers], [L.ln2 for L in st.layers], st.key_cache, st.value_cache, st.sin, st.cos, 8, 128, st.max_seq, 1e-6)
    with pytest.raises(capi.ExlError, match=r"error 1: .*tensor parallelism.*per-op"):
        capi.DecodePlan(*args, tp_rank=0, tp_world=2, num_kv_heads=2)
    with pytest.raises(capi.ExlError, match=r"error 1: .*num_kv_heads \(3\) must divide num_heads \(8\)"):
        capi.DecodePlan(*args, num_kv_heads=3)
    st.close()
