"""Prefill over an existing KV cache: the causal attention kernel (csrc/prefill_attn.cu, exl_prefill_attn) and DecodeStack.prefill at
past_len > 0.

- The kernel against the composed float64 oracle (tests/prefill_oracle.py) over multi-head and grouped-query shapes, q_len on both
  sides of the 64-row query tile (64 / n_rep tokens) and the 64-key tile, past_len 0, 1, 37, 200 and past_len + q_len == max_seq,
  bsz 1..4 and a cache pointer offset to a middle sequence; its error against the reference's masked SDPA program's; NaN rows past
  the chunk; no write outside out; caches unchanged; two launches bitwise equal; every argument error.
- DecodeStack.prefill at past_len > 0 against the whole-prefill oracle, a follow-up turn (prefill, fused decode, prefill, fused
  decode), T = 1 against decode_step, prefill into one sequence of a batch, and chunked against single prefill at full size.

Every test starts from a library without q4 handles or borrowed buffers and frees them all when it ends (exl_cleanup).
"""
import numpy as np
import pytest

from helpers import assert_close_ref64, oracle_decode_step
from prefill_oracle import oracle_prefill, prefill_attn_f64
from stack_harness import lib_state, restore, snapshot, stacks  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("lib_state")]

HD = 128
MAX_SEQ = 384                                   # the caches of the small stacks
ATTN_TOL = dict(rel=1.5e-3, rms=1.5e-3)        # decode_attn's tolerance
LOGIT_TOL = dict(rel=1.5e-2, rms=1.5e-2)       # the decode tests' logit tolerance
CACHE_TOL = dict(rel=1e-2, rms=1e-2)
NAN_BITS = 0x7D2B                               # a NaN payload no fp16 arithmetic produces


def _np(t):
    return t.cpu().numpy()


def _inputs(bsz, q_len, heads, kv_heads, past_len, max_seq, seed, nseq=None):
    """q [bsz, q_len, heads, hd] and caches [nseq, kv_heads, max_seq, hd] (fp16, cuda); rows past past_len + q_len are NaN."""
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    nseq = bsz if nseq is None else nseq
    q = (torch.randn((bsz, q_len, heads, HD), device="cuda", generator=g) * 1.5).half()
    kc = (torch.randn((nseq, kv_heads, max_seq, HD), device="cuda", generator=g) * 1.5).half()
    vc = torch.randn((nseq, kv_heads, max_seq, HD), device="cuda", generator=g).half()
    kc[:, :, past_len + q_len:] = float("nan")
    vc[:, :, past_len + q_len:] = float("nan")
    return q, kc, vc


def _want(oracle, q, kc, vc, heads, kv_heads, past_len, max_seq):
    return np.stack([prefill_attn_f64(oracle, _np(q[b]), _np(kc[b]), _np(vc[b]), heads, kv_heads, past_len, max_seq)
                     for b in range(q.shape[0])]).reshape(q.shape[0], q.shape[1], heads * HD)


# (heads, kv_heads, bsz, past_len, q_len, max_seq): query tiles hold 64 rows = 64 / n_rep tokens, key tiles 64 keys
KERNEL_CASES = [
    (8, 8, 1, 0, 1, 64), (8, 8, 2, 1, 63, 128), (8, 8, 1, 37, 64, 128), (8, 8, 3, 37, 65, 256), (8, 8, 1, 200, 129, 384),
    (8, 8, 1, 0, 257, 257), (8, 8, 4, 200, 56, 256),
    (8, 2, 1, 0, 16, 64), (8, 2, 2, 1, 17, 64), (8, 2, 4, 37, 33, 128), (8, 2, 1, 200, 257, 512), (8, 2, 1, 63, 65, 128),
    (32, 32, 1, 0, 129, 256), (32, 32, 2, 200, 64, 264), (32, 32, 1, 1, 1, 64),
    (64, 8, 1, 0, 8, 64), (64, 8, 1, 0, 9, 64), (64, 8, 2, 37, 65, 128), (64, 8, 4, 1, 7, 128), (64, 8, 1, 200, 257, 512),
    (64, 8, 1, 191, 65, 256),
]


@pytest.mark.parametrize("heads,kv_heads,bsz,past_len,q_len,max_seq", KERNEL_CASES)
def test_kernel_vs_oracle(oracle, heads, kv_heads, bsz, past_len, q_len, max_seq):
    import torch
    from exllama_b200 import cuda_ext
    q, kc, vc = _inputs(bsz, q_len, heads, kv_heads, past_len, max_seq, seed=heads + bsz + past_len + q_len)
    out = torch.empty((bsz, q_len, heads * HD), dtype=torch.float16, device="cuda")
    cuda_ext.exllama_ext.prefill_attn(q, kc, vc, out, heads, kv_heads, HD, past_len, max_seq)
    torch.cuda.synchronize()
    assert_close_ref64(_np(out), _want(oracle, q, kc, vc, heads, kv_heads, past_len, max_seq), **ATTN_TOL,
                       what=f"{heads}/{kv_heads} bsz {bsz} past {past_len} q_len {q_len}")


def test_kernel_cache_offset_to_middle_sequence(oracle):
    """Sequences 2 and 3 of a 5-sequence cache: the kernel gets the slice's pointer and touches nothing outside it."""
    import torch
    from exllama_b200 import capi
    heads, kv_heads, past_len, q_len, max_seq = 64, 8, 37, 40, 96
    q, kc, vc = _inputs(2, q_len, heads, kv_heads, past_len, max_seq, seed=5, nseq=5)
    k0, v0 = kc.clone(), vc.clone()
    out = capi.prefill_attn(q, kc[2:4], vc[2:4], heads, kv_heads, HD, past_len, max_seq)
    torch.cuda.synchronize()
    assert torch.equal(kc.view(torch.int16), k0.view(torch.int16)) and torch.equal(vc.view(torch.int16), v0.view(torch.int16))
    assert_close_ref64(_np(out), _want(oracle, q, kc[2:4], vc[2:4], heads, kv_heads, past_len, max_seq), **ATTN_TOL, what="offset")


def _reference_program(q, kc, vc, heads, kv_heads, past_len):
    """The reference's program for a chunk at past_len > 0 on the GPU: repeat_kv, the additive fp16 mask, SDPA with that mask."""
    import torch
    from exllama_b200.stack import repeat_kv
    bsz, q_len = q.shape[:2]
    n = past_len + q_len
    keys = repeat_kv(kc[:, :, :n], heads // kv_heads)
    values = repeat_kv(vc[:, :, :n], heads // kv_heads)
    mask = torch.zeros((bsz, 1, q_len, n), dtype=torch.float16, device="cuda")
    if q_len > 1:
        mask[:, :, :q_len - 1, past_len + 1:] = torch.triu(torch.full((q_len - 1, q_len - 1), -65504.0, device="cuda")).half()
    o = torch.nn.functional.scaled_dot_product_attention(q.transpose(1, 2), keys, values, attn_mask=mask, is_causal=False)
    return o.transpose(1, 2).reshape(bsz, q_len, heads * HD)


@pytest.mark.parametrize("heads,kv_heads,past_len,q_len", [(64, 8, 200, 129), (32, 32, 37, 100), (8, 2, 300, 257)])
def test_kernel_error_vs_reference_program(oracle, heads, kv_heads, past_len, q_len):
    """RMS error against float64 at most 1.1x that of the reference's masked SDPA program on the same fp16 inputs."""
    import torch
    from exllama_b200 import capi
    max_seq = past_len + q_len + 16
    q, kc, vc = _inputs(1, q_len, heads, kv_heads, past_len, max_seq, seed=heads + q_len)
    ours = capi.prefill_attn(q, kc, vc, heads, kv_heads, HD, past_len, max_seq)
    ref = _reference_program(q, kc, vc, heads, kv_heads, past_len)
    torch.cuda.synchronize()
    want = _want(oracle, q, kc, vc, heads, kv_heads, past_len, max_seq)
    rms = lambda a: float(np.sqrt(np.mean((a.astype(np.float64) - want) ** 2)))
    e_ours, e_ref = rms(_np(ours)), rms(_np(ref))
    assert e_ours <= 1.1 * e_ref, f"kernel rms error {e_ours:.4g} > 1.1 x reference program's {e_ref:.4g}"


def test_kernel_nan_rows_guard_unchanged_caches_and_determinism():
    """Rows past past_len + q_len hold NaN: the output is finite and bitwise equal to a run on a clean cache.  The output sits between
    NaN guards that keep their bits, both caches are bitwise unchanged, and a second launch is bitwise equal."""
    import torch
    from exllama_b200 import capi
    heads, kv_heads, past_len, q_len, max_seq, bsz = 64, 8, 100, 77, 256, 2
    q, kc, vc = _inputs(bsz, q_len, heads, kv_heads, past_len, max_seq, seed=11)
    k0, v0 = kc.clone(), vc.clone()
    n = bsz * q_len * heads * HD
    pre, post = 4096, 4096
    buf = torch.full((pre + n + post,), NAN_BITS, dtype=torch.int16, device="cuda")
    out = buf[pre:pre + n].view(torch.float16).view(bsz, q_len, heads * HD)
    capi.prefill_attn(q, kc, vc, heads, kv_heads, HD, past_len, max_seq, out=out)
    again = capi.prefill_attn(q, kc, vc, heads, kv_heads, HD, past_len, max_seq)
    clean_k, clean_v = kc.clone(), vc.clone()
    clean_k[:, :, past_len + q_len:] = 0
    clean_v[:, :, past_len + q_len:] = 0
    clean = capi.prefill_attn(q, clean_k, clean_v, heads, kv_heads, HD, past_len, max_seq)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out).all())
    assert bool((buf[:pre] == NAN_BITS).all()), "written before the output"
    assert bool((buf[pre + n:] == NAN_BITS).all()), "written after the output"
    assert torch.equal(kc.view(torch.int16), k0.view(torch.int16)) and torch.equal(vc.view(torch.int16), v0.view(torch.int16))
    assert torch.equal(out.view(torch.int16), again.view(torch.int16)), "two launches differ"
    assert torch.equal(out.view(torch.int16), clean.view(torch.int16)), "NaN rows past the chunk change the output"


def test_kernel_argument_errors():
    import torch
    from exllama_b200 import capi
    q, kc, vc = _inputs(1, 4, 8, 2, 4, 16, seed=1)
    out = torch.empty((1, 4, 8 * HD), dtype=torch.float16, device="cuda")
    lib = capi.lib()
    P = lambda t: capi._ptr(t)
    call = lambda **kw: lib.exl_prefill_attn(*(kw.get(k, d) for k, d in (
        ("q", P(q)), ("kc", P(kc)), ("vc", P(vc)), ("out", P(out)), ("bsz", 1), ("q_len", 4), ("heads", 8), ("kv", 2), ("hd", HD),
        ("past", 4), ("max_seq", 16))), capi._stream())
    assert call() == 0
    for kw, text in ((dict(hd=64), "head_dim 64"), (dict(kv=3), "num_kv_heads 3"), (dict(bsz=0), "bsz 0"), (dict(q_len=0), "q_len 0"),
                     (dict(past=-5), "past_len -5"), (dict(past=13), "max_seq_len 16"), (dict(q=None), "NULL"),
                     (dict(kc=None), "NULL"), (dict(vc=None), "NULL"), (dict(out=None), "NULL")):
        assert call(**kw) == 1, kw                                        # EXL_ERR_ARG
        msg = lib.exl_last_error().decode()
        assert text in msg, (kw, msg)
    torch.cuda.synchronize()


# ---- DecodeStack.prefill at past_len > 0 --------------------------------------------------------------------------------------------
def _x(bsz, T, hidden, seed, scale=0.5):
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    return (torch.randn((bsz, T, hidden), device="cuda", generator=g) * scale).half()


def _check_prefill(oracle, st, x, past_len, what, seq=0):
    """prefill(x, past_len, seq=seq, last_only=False) against the oracle for every sequence of x [bsz, T, hidden]: logits at every
    position, the new cache rows [past_len, past_len + T) of every layer, every other row of every sequence bitwise unchanged."""
    import torch
    bsz, T, _ = x.shape
    snap = snapshot(st)
    logits = st.prefill(x.clone(), past_len, last_only=False, seq=seq)
    torch.cuda.synchronize()
    logits = _np(logits).reshape(bsz, T, -1)
    for b in range(st.batch):
        lo, hi = (past_len, past_len + T) if seq <= b < seq + bsz else (0, 0)
        for i, (kc, vc) in enumerate(zip(st.key_cache, st.value_cache)):
            for name, c, c0 in (("k", kc, snap[i][0]), ("v", vc, snap[i][1])):
                assert torch.equal(c[b, :, :lo], c0[b, :, :lo]) and torch.equal(c[b, :, hi:], c0[b, :, hi:]), \
                    f"{what}: layer {i} {name} cache of sequence {b}: a row outside [{lo}, {hi}) was written"
    caches = snapshot(st)
    for b in range(bsz):
        want, rows = oracle_prefill(oracle, st, caches, _np(x[b]), past_len, seq + b, bsz * T)
        assert_close_ref64(logits[b], want, **LOGIT_TOL, what=f"{what} seq {b} logits")
        for i, (kc, vc) in enumerate(zip(st.key_cache, st.value_cache)):
            assert_close_ref64(_np(kc[seq + b, :, past_len:past_len + T]), rows[i][0].astype(np.float64), **CACHE_TOL,
                               what=f"{what} seq {b} layer {i} k rows")
            assert_close_ref64(_np(vc[seq + b, :, past_len:past_len + T]), rows[i][1].astype(np.float64), **CACHE_TOL,
                               what=f"{what} seq {b} layer {i} v rows")
    return logits


# T <= 48 rows run the skinny GEMM route, more run the wgmma GEMM
STACK_CASES = [  # (past_len, T, kv_heads, groupsize, act_order)
    (1, 9, 8, 128, False), (37, 30, 2, 32, True), (100, 65, 8, 32, False), (200, 130, 2, 128, True), (254, 130, 8, 128, True),
]


@pytest.mark.parametrize("past_len,T,kv,gs,act", STACK_CASES)
def test_prefill_past_vs_oracle(oracle, stacks, past_len, T, kv, gs, act):
    st = stacks(kv_heads=kv, gs=gs, act=act, seed=past_len + T + kv, max_seq=MAX_SEQ)
    _check_prefill(oracle, st, _x(1, T, 1024, seed=T + past_len), past_len, f"past {past_len} T {T} kv {kv} g{gs} act {act}")


@pytest.mark.parametrize("kv", [8, 2])
def test_follow_up_turn(oracle, stacks, kv):
    """Prefill T0 tokens, three fused decode steps, prefill T1 more at the current past_len, one fused decode step; each step against
    the oracle on the caches it started from."""
    import torch
    st = stacks(kv_heads=kv, seed=80 + kv, max_seq=MAX_SEQ)
    T0, T1, steps = 50, 70, 3
    x = _x(1, T0 + steps + T1 + 1, 1024, seed=81 + kv)
    _check_prefill(oracle, st, x[:, :T0].contiguous(), 0, f"kv {kv} first turn")
    st.make_plan()
    p = T0

    def fused_step(p):
        snap = snapshot(st)
        xt = x[:, p:p + 1].contiguous()
        _, want, _ = oracle_decode_step(oracle, st, snap, _np(xt), p)
        got = st.decode_step_fused(xt, p)
        torch.cuda.synchronize()
        assert_close_ref64(_np(got).reshape(-1), want.reshape(-1), **LOGIT_TOL, what=f"kv {kv} fused decode at {p}")
    for _ in range(steps):
        fused_step(p)
        p += 1
    _check_prefill(oracle, st, x[:, p:p + T1].contiguous(), p, f"kv {kv} follow-up turn at past {p}")
    p += T1
    fused_step(p)


@pytest.mark.parametrize("kv,p", [(8, 1), (2, 77), (8, 200)])
def test_single_token_prefill_matches_decode_step(stacks, kv, p):
    """T = 1 at past_len p through prefill agrees with decode_step at p (from the same caches)."""
    st = stacks(kv_heads=kv, seed=90 + p, max_seq=MAX_SEQ)
    x = _x(1, 1, 1024, seed=p)
    snap = snapshot(st)
    got = _np(st.prefill(x.clone(), p)).reshape(-1)
    pre = snapshot(st)
    restore(st, snap)
    want = _np(st.decode_step(x.clone(), p)).reshape(-1)
    assert_close_ref64(got, want.astype(np.float64), **LOGIT_TOL, what=f"kv {kv} prefill T=1 vs decode_step at {p}")
    for (kp, vp), kc, vc in zip(pre, st.key_cache, st.value_cache):
        assert_close_ref64(_np(kp[0, :, p]), _np(kc[0, :, p]).astype(np.float64), **CACHE_TOL, what="k row")
        assert_close_ref64(_np(vp[0, :, p]), _np(vc[0, :, p]).astype(np.float64), **CACHE_TOL, what="v row")


def test_prefill_into_one_sequence_of_a_batch(oracle, stacks):
    """batch=3: sequence 1 gets a prefill at past 60 while sequences 0 and 2 sit at 40 and 90; their caches stay bitwise unchanged.
    One fused batch step at the three past_lens then matches oracle_decode_step for each sequence."""
    import torch
    st = stacks(kv_heads=2, batch=3, seed=95, max_seq=MAX_SEQ)
    lens = [40, 60, 90]
    T = 33
    x = _x(1, T, 1024, seed=96)
    _check_prefill(oracle, st, x, lens[1], "seq 1 of 3", seq=1)
    lens[1] += T
    snap = snapshot(st)
    st.make_plan()
    xt = _x(3, 1, 1024, seed=97)
    got = _np(st.decode_step_fused_batch(xt, lens))
    torch.cuda.synchronize()
    for b in range(3):
        _, want, _ = oracle_decode_step(oracle, st, snap, _np(xt[b]), lens[b], seq=b)
        assert_close_ref64(got[b], want.reshape(-1), **LOGIT_TOL, what=f"fused batch step, seq {b} at {lens[b]}")
    with pytest.raises(ValueError, match="cache sequences"):
        st.prefill(_x(2, 4, 1024, seed=1), 10, seq=2)
    with pytest.raises(ValueError, match="max_seq"):
        st.prefill(_x(1, 30, 1024, seed=1), st.max_seq - 29)


@pytest.mark.parametrize("name", ["7b", "70b"])
def test_full_size_chunked_vs_single_prefill(stacks, name):
    """Two layers of the 7B and 70B (grouped-query) shapes: 1920 tokens in chunks of 512 against one 1920-token prefill from the same
    caches, on sampled logits and every cache row."""
    import torch
    from exllama_b200.shapes import GQA_SHAPES, SHAPES
    s = {**SHAPES, **GQA_SHAPES}[name]
    T, C = 1920, 512
    st = stacks(s, gs=128, max_seq=2048, seed=17)
    x = _x(1, T, s.hidden, seed=29)
    snap0 = snapshot(st)
    pos = sorted(set(range(0, T, 97)) | {T - 3, T - 2, T - 1})
    whole = st.prefill(x.clone(), last_only=False)[pos].cpu()
    single = snapshot(st)
    restore(st, snap0)
    parts = []
    for c0 in range(0, T, C):
        lg = st.prefill(x[:, c0:c0 + C].contiguous(), c0, last_only=False)
        parts.append(lg.cpu())
    chunked = torch.cat(parts)[pos]
    torch.cuda.synchronize()
    assert_close_ref64(chunked.numpy(), whole.numpy().astype(np.float64), rel=2e-2, rms=2e-2, what=f"{name} chunked vs single logits")
    for i, ((ks, vs), kc, vc) in enumerate(zip(single, st.key_cache, st.value_cache)):
        assert_close_ref64(_np(kc[0, :, :T]), _np(ks[0, :, :T]).astype(np.float64), rel=2e-2, rms=2e-2, what=f"{name} layer {i} k rows")
        assert_close_ref64(_np(vc[0, :, :T]), _np(vs[0, :, :T]).astype(np.float64), rel=2e-2, rms=2e-2, what=f"{name} layer {i} v rows")
        assert torch.equal(kc[0, :, T:], ks[0, :, T:]) and torch.equal(vc[0, :, T:], vs[0, :, T:])
