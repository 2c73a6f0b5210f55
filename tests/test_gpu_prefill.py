"""Prefill: the wgmma fused-dequant GEMM (csrc/q4_gemm_tc.cu) at the projection shapes and prompt lengths prefill runs, and
DecodeStack.prefill against a float64 oracle composition.

- The GEMM at every 7B / 13B / 33B / 65B / 70B projection shape and M in {1920, 2048, 1921} (3968 for 65B), plain and accumulate,
  on a sample of rows and whole 8-column groups: restricting x . W to some rows of x and some columns of W is exact, so the float64
  oracle on the sample is the answer for those entries.
- No write outside [M, N] of the output, at partial M tiles and N % 128 != 0.
- Act-order scratch: a borrowed temp_state that is large enough and one that is not give bitwise equal results, and nothing past
  what the call may use is written.
- DecodeStack.prefill against the oracle composed with prefill's own rounding points, over the skinny, repeated-skinny and wgmma
  routes, multi-head and grouped-query attention, g128 / g32, act-order, LoRA and a batch of two; the cache rows it writes are the
  ones decode reads; and at full 7B / 13B / 70B size against T single-token decode steps.

Every test starts from a library without q4 handles or borrowed buffers and frees them all when it ends, pass or fail: exl_cleanup
frees every q4 handle on the device and resets temp_state, which a stack an earlier test failed to close would leave pointing at
freed memory that the act-order gather writes through.
"""
import numpy as np
import pytest

from helpers import REL_TOL, RMS_TOL, adapter_of, assert_close_ref64, oracle_decode_step, oracle_mm, to_cuda
from stack_harness import lib_state, restore, snapshot, stacks  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("lib_state")]

MAX_SEQ = 320                                   # the caches of the small stacks
LOGIT_TOL = dict(rel=1.5e-2, rms=1.5e-2)       # the decode tests' logit tolerance
CACHE_TOL = dict(rel=1e-2, rms=1e-2)


def _np(t):
    return t.cpu().numpy()


def _x(bsz, T, hidden, seed, scale=0.5):
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    return (torch.randn((bsz, T, hidden), device="cuda", generator=g) * scale).half()


# ---- (a) the wgmma GEMM at every prefill projection shape --------------------------------------------------------------------------
PREFILL_SHAPES = [  # (model, K, N, groupsize, act_order)
    ("7b", 4096, 4096, 128, False), ("7b", 4096, 11008, 128, False), ("7b", 11008, 4096, 128, False),
    ("13b", 5120, 5120, 128, True), ("13b", 5120, 13824, 128, True), ("13b", 13824, 5120, 128, True),
    ("33b", 6656, 6656, 32, True), ("33b", 6656, 17920, 32, True), ("33b", 17920, 6656, 32, True),
    ("65b", 8192, 22016, 128, False), ("65b", 22016, 8192, 128, False),
    ("70b", 8192, 1024, 128, False), ("70b", 8192, 28672, 128, False), ("70b", 28672, 8192, 128, False),
]


def _sample_rows(M, seed, n=24):
    """The first and last rows, both sides of every 128-row edge inside the first two 256-row tiles, the edges of the last 256- and
    128-row tiles and the middle of the last one, then random rows up to n."""
    rows = {0, 1, M - 2, M - 1}
    rows |= {r for edge in (128, 256, 384, 512) for r in (edge - 1, edge) if r < M}
    last256, last128 = (M - 1) // 256 * 256, (M - 1) // 128 * 128
    rows |= {r for r in (last256 - 1, last256, last256 + 1, last128 - 1, last128, (last256 + M) // 2) if 0 <= r < M}
    rng = np.random.default_rng(seed)
    while len(rows) < n:
        rows.add(int(rng.integers(0, M)))
    return np.array(sorted(rows))


def _sample_cols(qw, qz, sc, seed, n8=12):
    """Whole 8-column groups (one packed qzeros word each), always including the last one: (columns, qweight, qzeros, scales)."""
    N = qw.shape[1]
    c8 = np.sort(np.append(np.random.default_rng(seed).choice(N // 8 - 1, n8 - 1, replace=False), N // 8 - 1))
    cols = (c8[:, None] * 8 + np.arange(8)[None]).reshape(-1)
    return cols, np.ascontiguousarray(qw[:, cols]), np.ascontiguousarray(qz[:, c8]), np.ascontiguousarray(sc[:, cols])


@pytest.mark.parametrize("model,K,N,gs,act", PREFILL_SHAPES)
def test_tc_gemm_prefill_shapes(oracle, lib_state, model, K, N, gs, act):
    import torch
    capi = lib_state
    qw, qz, sc, g_idx = oracle.synth_q4(K, N, gs, act_order=act, seed=K + N)
    q4 = capi.Q4(*to_cuda(qw.copy(), qz, sc), None if g_idx is None else torch.from_numpy(g_idx))
    x_map, qseq = None, qw
    if act:                      # the kernel reads make_q4's sequential qweight and gathers x by x_map
        x_map = oracle.make_x_map(g_idx, K // gs)
        qseq = oracle.make_sequential(qw, x_map)
        np.testing.assert_array_equal(q4.x_map(), x_map)
    cols, sub_qw, sub_qz, sub_sc = _sample_cols(qseq, qz, sc, seed=N)
    tcols = torch.from_numpy(cols).cuda()
    gen = torch.Generator(device="cuda"); gen.manual_seed(K * 7 + N)
    for M in (1920, 2048, 1921) + ((3968,) if model == "65b" else ()):
        what = f"{model} K{K} N{N} g{gs} act{act} M{M}"
        x = torch.randn((M, K), device="cuda", generator=gen).half()
        out = capi.q4_matmul(x, q4, force_path=2)
        torch.cuda.synchronize()
        assert capi.last_q4_path() == "tc_gemm"
        auto = capi.q4_matmul(x, q4)
        torch.cuda.synchronize()
        assert capi.last_q4_path() == "tc_gemm", what
        assert torch.equal(auto, out), what
        # no atomics: each output element is the sum of one CTA over the k-blocks in order, so a second launch is bitwise equal
        assert torch.equal(capi.q4_matmul(x, q4, force_path=2), out), what
        rows = _sample_rows(M, seed=M + N)
        trows = torch.from_numpy(rows).cuda()
        xr = _np(x[trows])
        ref = oracle.q4_matmul_f64(xr, sub_qw, sub_qz, sub_sc, x_map, recons=True)
        assert_close_ref64(_np(out[trows][:, tcols]), ref, REL_TOL, RMS_TOL, what=what)
        res = torch.randn((M, N), device="cuda", generator=gen).half()
        out2 = res.clone()
        capi.q4_matmul(x, q4, out=out2, no_zero=True, force_path=2)
        ref2 = oracle.q4_matmul_f64(xr, sub_qw, sub_qz, sub_sc, x_map, acc_in=np.ascontiguousarray(_np(res[trows][:, tcols])), recons=True)
        assert_close_ref64(_np(out2[trows][:, tcols]), ref2, REL_TOL, RMS_TOL, what=what + " accumulate")


# ---- (b) no writes outside [M, N] ----------------------------------------------------------------------------------------------------
NAN_BITS = 0x7D2B               # a NaN payload no fp16 arithmetic produces


@pytest.mark.parametrize("N", [96, 1000, 8448])
@pytest.mark.parametrize("M", [49, 129, 300, 1921])
def test_tc_gemm_writes_only_its_output(oracle, lib_state, M, N):
    """The output is an M x N view inside a buffer of NaN bits, with a whole 256-row tile of room after it.  Every element outside
    the view keeps its bits, and every element inside it (a column past N would land in the next row) matches the oracle.  N = 1000
    (N % 128 != 0) is forced onto the wgmma GEMM: the auto route sends N % 32 != 0 to reconstruct + cuBLAS."""
    import torch
    capi = lib_state
    K, gs = 256, 128
    qw, qz, sc, _ = oracle.synth_q4(K, N, gs, seed=M + N)
    q4 = capi.Q4(*[torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (qw.copy(), qz, sc)])
    x = oracle.synth_x(M, K, seed=M)
    res = oracle.synth_x(M, N, seed=M + 1)
    want = x.astype(np.float64) @ oracle.reconstruct_f16(qw, qz, sc).astype(np.float64)
    force = 2 if N % 32 else 0
    pre, post = 4096, 256 * N + 4096
    for no_zero in (False, True):
        buf = torch.full((pre + M * N + post,), NAN_BITS, dtype=torch.int16, device="cuda")
        out = buf[pre:pre + M * N].view(torch.float16).view(M, N)
        if no_zero:
            out.copy_(torch.from_numpy(res).cuda())
        capi.q4_matmul(torch.from_numpy(x).cuda(), q4, out=out, no_zero=no_zero, force_path=force)
        torch.cuda.synchronize()
        assert capi.last_q4_path() == "tc_gemm"
        what = f"M{M} N{N} no_zero {no_zero}"
        assert bool((buf[:pre] == NAN_BITS).all()), f"{what}: written before the output"
        after = buf[pre + M * N:]
        assert bool((after == NAN_BITS).all()), f"{what}: {int((after != NAN_BITS).sum())} elements written after the output"
        assert_close_ref64(_np(out), want + res.astype(np.float64) if no_zero else want, REL_TOL, RMS_TOL, what=what)


# ---- (c) act-order scratch: borrowed or library-owned ---------------------------------------------------------------------------------
def test_act_order_scratch(oracle, lib_state):
    """The act-order gather of x goes to the borrowed temp_state when it holds M * K halves, else to library-owned scratch.  Both give
    the same bits; the borrowed buffer holds the gathered x and nothing past it is written, and a borrowed buffer one element too
    small is not written at all."""
    import torch
    capi = lib_state
    M, K, N, gs = 1920, 4096, 4096, 128
    qw, qz, sc, g_idx = oracle.synth_q4(K, N, gs, act_order=True, seed=5)
    q4 = capi.Q4(*[torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (qw.copy(), qz, sc)], torch.from_numpy(g_idx))
    x_np = oracle.synth_x(M, K, seed=6)
    x = torch.from_numpy(x_np).cuda()
    x_map = oracle.make_x_map(g_idx, K // gs)
    sentinel = 0x5A5A
    tm = torch.zeros((4, 64), dtype=torch.float16, device="cuda")
    tz = torch.zeros((1, 65536), dtype=torch.float32, device="cuda")
    dq = torch.zeros((1, 8), dtype=torch.float16, device="cuda")
    outs = []
    for numel, used in ((M * K + 65536, M * K), (M * K - 1, 0)):
        ts = torch.full((numel,), sentinel, dtype=torch.int16, device="cuda")
        capi.prepare_buffers(0, ts.view(torch.float16), tm, tz, dq)
        outs.append(capi.q4_matmul(x, q4, force_path=2))
        torch.cuda.synchronize()
        assert capi.last_q4_path() == "tc_gemm"
        assert bool((ts[used:] == sentinel).all()), f"temp_state of {numel}: written past {used}"
        if used:
            gathered = x[:, torch.from_numpy(x_map.astype(np.int64)).cuda()]
            assert torch.equal(ts[:used].view(torch.float16).view(M, K), gathered)
    capi.check(capi.lib().exl_cleanup())        # the borrowed buffers die with this test
    assert torch.equal(outs[0], outs[1])
    rows = _sample_rows(M, seed=1)
    cols, sub_qw, sub_qz, sub_sc = _sample_cols(oracle.make_sequential(qw, x_map), qz, sc, seed=2)
    ref = oracle.q4_matmul_f64(np.ascontiguousarray(x_np[rows]), sub_qw, sub_qz, sub_sc, x_map, recons=True)
    assert_close_ref64(_np(outs[0])[rows][:, cols], ref, REL_TOL, RMS_TOL, what="act-order scratch")


# ---- (d) DecodeStack.prefill against the float64 oracle composition -------------------------------------------------------------------
def _causal_attention(q, k, v):
    """q [T, heads, hd], k / v [T, kv_heads, hd] fp16 -> float64 [T, heads, hd]: softmax(q k^T / sqrt(hd), causal) v, query head h on
    KV head h // (heads / kv_heads) (repeat_kv)."""
    T, H, hd = q.shape
    rep = H // k.shape[1]
    qf = q.astype(np.float64).transpose(1, 0, 2)
    kf = np.repeat(k.astype(np.float64).transpose(1, 0, 2), rep, axis=0)
    vf = np.repeat(v.astype(np.float64).transpose(1, 0, 2), rep, axis=0)
    s = qf @ kf.transpose(0, 2, 1) / np.sqrt(hd)
    s[:, np.triu(np.ones((T, T), dtype=bool), 1)] = -np.inf
    p = np.exp(s - s.max(-1, keepdims=True))
    p /= p.sum(-1, keepdims=True)
    return (p @ vf).transpose(1, 0, 2)


def _add16(a, b):
    return (a.astype(np.float64) + b.astype(np.float64)).astype(np.float16)


def _oracle_prefill(oracle, st, x, M):
    """float64/fp16 restatement of DecodeStack.prefill of one sequence x [T, hidden] fp16 at past_len 0, with prefill's rounding
    points; M (rows of every q4 call, bsz * T) picks the GEMM route: fp16-rounded weights above 48 rows (wgmma), exact products at
    or below (skinny).  Returns (logits [T, vocab] float64, per layer (k, v) cache rows [kv_heads, T, hd] fp16)."""
    s = st.shape
    hd, H, KV = s.head_dim, s.heads, s.kv_heads
    T = x.shape[0]
    sin = _np(st.sin).reshape(-1, hd); cos = _np(st.cos).reshape(-1, hd)
    mm = lambda xin, i, n: oracle_mm(oracle, xin, getattr(st.layers[i], n), adapter_of(st, i, n), recons=M > 48).astype(np.float16)
    rows = []
    for i, L in enumerate(st.layers):
        xn, _ = oracle.rms_norm(x, _np(L.ln1), s.eps)
        q, k, v = (mm(xn, i, n) for n in ("q", "k", "v"))
        q = oracle.rope(q.reshape(1, T * H, hd), sin, cos, 1, T * H, hd, H, 0).reshape(T, H, hd)
        k = oracle.rope(k.reshape(1, T * KV, hd), sin, cos, 1, T * KV, hd, KV, 0).reshape(T, KV, hd)
        v = v.reshape(T, KV, hd)
        rows.append((k.transpose(1, 0, 2), v.transpose(1, 0, 2)))
        attn = _causal_attention(q, k, v).astype(np.float16).reshape(T, H * hd)
        x = _add16(x, mm(attn, i, "o"))
        xn, _ = oracle.rms_norm(x, _np(L.ln2), s.eps)
        g, u = mm(xn, i, "gate"), mm(xn, i, "up")
        g64 = g.astype(np.float64)
        act = (g64 / (1.0 + np.exp(-g64))).astype(np.float16)               # torch's fp16 silu: one rounding
        act = (act.astype(np.float64) * u.astype(np.float64)).astype(np.float16)
        x = _add16(x, mm(act, i, "down"))
    hn, _ = oracle.rms_norm(x, _np(st.norm), s.eps)
    return hn.astype(np.float64) @ _np(st.lm_head).astype(np.float64).T, rows


def _check_prefill(oracle, st, x, what):
    """prefill(x, last_only=False) against the oracle for every sequence of x [bsz, T, hidden]: logits at every position, cache rows
    [0, T) of every layer, every other cache row bitwise unchanged, and the GEMM route.  Returns the logits [bsz, T, vocab]."""
    import torch
    from exllama_b200 import capi
    bsz, T, _ = x.shape
    snap = snapshot(st)
    logits = st.prefill(x.clone(), last_only=False)
    torch.cuda.synchronize()
    assert capi.last_q4_path() == ("skinny_mma" if bsz * T <= 48 else "tc_gemm"), (what, capi.last_q4_path())
    logits = _np(logits).reshape(bsz, T, -1)
    for b in range(st.batch):
        for i, (kc, vc) in enumerate(zip(st.key_cache, st.value_cache)):
            for name, c, c0 in (("k", kc, snap[i][0]), ("v", vc, snap[i][1])):
                lo = T if b < bsz else 0
                assert torch.equal(c[b, :, lo:], c0[b, :, lo:]), f"{what}: layer {i} {name} cache of sequence {b}: rows >= {lo} written"
    for b in range(bsz):
        want, rows = _oracle_prefill(oracle, st, _np(x[b]), bsz * T)
        assert_close_ref64(logits[b], want, **LOGIT_TOL, what=f"{what} seq {b} logits")
        for i, (kc, vc) in enumerate(zip(st.key_cache, st.value_cache)):
            assert_close_ref64(_np(kc[b, :, :T]), rows[i][0].astype(np.float64), **CACHE_TOL, what=f"{what} seq {b} layer {i} k rows")
            assert_close_ref64(_np(vc[b, :, :T]), rows[i][1].astype(np.float64), **CACHE_TOL, what=f"{what} seq {b} layer {i} v rows")
    return logits


# T spans one skinny pass (<= 8), repeated skinny passes (9..48) and the wgmma GEMM (49..), with partial 128- and 256-row tiles
PREFILL_CASES = [  # (T, kv_heads, groupsize, act_order)
    (1, 8, 128, False), (1, 2, 32, True), (8, 2, 128, False), (8, 8, 32, True),
    (9, 8, 128, True), (9, 2, 32, False), (48, 2, 128, True), (48, 8, 32, False),
    (49, 8, 128, False), (49, 2, 32, True), (65, 2, 128, False), (65, 8, 32, True),
    (130, 8, 128, True), (130, 2, 32, False), (257, 2, 128, True), (257, 8, 32, False),
]


@pytest.mark.parametrize("T,kv,gs,act", PREFILL_CASES)
def test_prefill_vs_oracle(oracle, stacks, T, kv, gs, act):
    st = stacks(kv_heads=kv, max_seq=MAX_SEQ, gs=gs, act=act, seed=T + kv + gs)
    _check_prefill(oracle, st, _x(1, T, 1024, seed=T), f"T {T} kv {kv} g{gs} act {act}")


# ---- (e) LoRA in prefill -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [5, 130])
def test_prefill_lora_vs_oracle(oracle, stacks, T):
    """A rank-16 adapter on all seven projections: each adds fp16(fp16(x . A) . B) before the q4 accumulate (q4_matmul_lora)."""
    st = stacks(kv_heads=2, max_seq=MAX_SEQ, seed=40 + T)
    st.add_lora(16, "all", seed=T)
    x = _x(1, T, 1024, seed=T + 1)
    snap = snapshot(st)
    got = _check_prefill(oracle, st, x, f"LoRA T {T}")
    restore(st, snap)
    saved, st.lora = st.lora, None
    plain = _np(st.prefill(x.clone(), last_only=False)).reshape(got.shape)
    st.lora = saved
    tol = LOGIT_TOL["rms"] * np.sqrt(np.mean(got.astype(np.float64) ** 2))
    d = np.abs(got.astype(np.float64) - plain).max()
    assert d >= 20 * tol, f"the adapter moves the prefill logits by {d:.4g}, less than 20 x {tol:.4g}"


# ---- (f) prefill, then decode ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kv", [8, 2])
@pytest.mark.parametrize("T", [37, 130])
def test_prefill_then_decode(oracle, stacks, T, kv):
    """Token T after a prefill of T tokens, through the per-op decode_step and the fused step, against the whole-token oracle on the
    post-prefill caches; and the per-op logits against a prefill of all T + 1 tokens, which reads no cache row decode reads."""
    import torch
    st = stacks(kv_heads=kv, max_seq=MAX_SEQ, seed=60 + T + kv)
    x = _x(1, T + 1, 1024, seed=T + kv)
    snap0 = snapshot(st)
    whole = _np(st.prefill(x.clone())).reshape(-1)
    restore(st, snap0)
    st.prefill(x[:, :T].contiguous())
    snap = snapshot(st)
    xt = x[:, T:T + 1].contiguous()
    _, want, rows = oracle_decode_step(oracle, st, snap, _np(xt), T)
    what = f"T {T} kv {kv}"
    per_op = _np(st.decode_step(xt.clone(), T)).reshape(-1)
    assert_close_ref64(per_op, want.reshape(-1), **LOGIT_TOL, what=f"{what} per-op decode vs oracle")
    assert_close_ref64(per_op, whole.astype(np.float64), rel=2e-2, rms=2e-2, what=f"{what} per-op decode vs prefill of T + 1")
    for i, (kc, vc) in enumerate(zip(st.key_cache, st.value_cache)):
        assert_close_ref64(_np(kc[0, :, T]), rows[i][0].astype(np.float64), **CACHE_TOL, what=f"{what} layer {i} new k")
        assert_close_ref64(_np(vc[0, :, T]), rows[i][1].astype(np.float64), **CACHE_TOL, what=f"{what} layer {i} new v")
    restore(st, snap)
    st.make_plan()
    fused = st.decode_step_fused(xt, T)
    torch.cuda.synchronize()
    assert_close_ref64(_np(fused).reshape(-1), want.reshape(-1), **LOGIT_TOL, what=f"{what} fused decode vs oracle")


def test_batched_prefill_then_fused_batch_step(oracle, stacks):
    """A stack of two cache sequences: prefill of [2, T] fills both, then one fused step carries both at [T, T].  A prefill of one
    sequence fills cache sequence 0 and leaves sequence 1 alone; three sequences do not fit."""
    import torch
    T = 37
    st = stacks(kv_heads=2, max_seq=MAX_SEQ, batch=2, seed=71)
    x = _x(2, T + 1, 1024, seed=72)
    snap0 = snapshot(st)
    _check_prefill(oracle, st, x[:1, :T].contiguous(), "batch-2 stack, one sequence")
    restore(st, snap0)
    _check_prefill(oracle, st, x[:, :T].contiguous(), "batch 2")
    snap = snapshot(st)
    st.make_plan()
    xt = x[:, T:T + 1].contiguous()
    got = _np(st.decode_step_fused_batch(xt, [T, T]))
    torch.cuda.synchronize()
    for b in range(2):
        _, want, _ = oracle_decode_step(oracle, st, snap, _np(xt[b]), T, seq=b)
        assert_close_ref64(got[b], want.reshape(-1), **LOGIT_TOL, what=f"fused batch step after prefill, seq {b}")
    with pytest.raises(ValueError, match="prefill of 3 sequences into caches that hold 2"):
        st.prefill(_x(3, 4, 1024, seed=1))


# ---- (g) full size, cross-checked against T single-token decode steps -------------------------------------------------------------------
@pytest.mark.parametrize("name,act", [("7b", False), ("13b", True), ("70b", False)])
def test_full_size_prefill_vs_decode(stacks, name, act):
    """Two layers of the 7B, 13B act-order and 70B (grouped-query) shapes: prefill of 1920 tokens against 1920 per-op decode steps
    from the same caches (a float64 oracle of the prompt is too slow on the CPU; the decode path is pinned to it elsewhere)."""
    import torch
    from exllama_b200 import capi
    from exllama_b200.shapes import GQA_SHAPES, SHAPES
    s = {**SHAPES, **GQA_SHAPES}[name]
    T = 1920
    st = stacks(s, gs=128, act=act, max_seq=2048, seed=17)
    x = _x(1, T, s.hidden, seed=29)
    snap0 = snapshot(st)
    pos = sorted(set(range(0, T, 97)) | {T - 3, T - 2, T - 1})
    logits = st.prefill(x.clone(), last_only=False)[pos].cpu()
    assert capi.last_q4_path() == "tc_gemm"
    prefilled = snapshot(st)
    restore(st, snap0)
    want = []
    for p in range(T):
        lg = st.decode_step(x[:, p:p + 1].clone(), p)
        if p in pos:
            want.append(lg.view(-1).cpu())
    torch.cuda.synchronize()
    assert_close_ref64(logits.numpy(), torch.stack(want).numpy().astype(np.float64), rel=2e-2, rms=2e-2,
                       what=f"{name} prefill logits vs decode")
    for i, ((kp, vp), kc, vc) in enumerate(zip(prefilled, st.key_cache, st.value_cache)):
        assert_close_ref64(_np(kp[0, :, :T]), _np(kc[0, :, :T]).astype(np.float64), **CACHE_TOL, what=f"{name} layer {i} k rows")
        assert_close_ref64(_np(vp[0, :, :T]), _np(vc[0, :, :T]).astype(np.float64), **CACHE_TOL, what=f"{name} layer {i} v rows")
