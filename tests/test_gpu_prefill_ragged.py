"""Ragged prefill: sequences of different lengths, each at its own past_len and cache sequence, in one call.

- exl_prefill_attn_ragged against the float64 oracle (tests/prefill_oracle.py) per sequence, over multi-head and grouped-query
  shapes, q_len 1 and both sides of the query and key tile edges, past_len 0, 1, 37, 200 and past_len + q_len == max_seq, permuted
  and non-contiguous cache sequences, n_seq 1 and the cap; bitwise agreement with exl_prefill_attn on a uniform batch and on one
  sequence; NaN in every cache row no sequence may read; caches unchanged; two launches bitwise equal; every argument error.
- exl_rope_cache_ragged bit-exact against rope_ per sequence followed by the cache copy, every other cache row unchanged.
- DecodeStack.prefill_ragged against oracle_prefill per sequence with M = T (skinny and wgmma routes, MHA / GQA, g128 / g32,
  act-order, LoRA), a serving flow into a fused batch decode step, and one ragged call against one prefill per prompt at full size.

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
CAP = 64                                        # EXL_RAGGED_MAX_SEQ
ATTN_TOL = dict(rel=1.5e-3, rms=1.5e-3)
LOGIT_TOL = dict(rel=1.5e-2, rms=1.5e-2)
CACHE_TOL = dict(rel=1e-2, rms=1e-2)


def _np(t):
    return t.cpu().numpy()


def _bits_equal(a, b):
    import torch
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


def _inputs(heads, kv_heads, q_lens, past_lens, cache_seqs, n_cache, max_seq, seed):
    """Packed q [T, heads, hd] and caches [n_cache, kv_heads, max_seq, hd]; every row a sequence may not read is NaN (rows from
    past_len + q_len on in the named cache sequences, every row of the others)."""
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    T = sum(q_lens)
    q = (torch.randn((T, heads, HD), device="cuda", generator=g) * 1.5).half()
    kc = (torch.randn((n_cache, kv_heads, max_seq, HD), device="cuda", generator=g) * 1.5).half()
    vc = torch.randn((n_cache, kv_heads, max_seq, HD), device="cuda", generator=g).half()
    visible = torch.zeros((n_cache, max_seq), dtype=torch.bool, device="cuda")
    for ql, pl, cs in zip(q_lens, past_lens, cache_seqs):
        visible[cs, :pl + ql] = True
    hidden = ~visible[:, None, :, None].expand_as(kc)
    kc[hidden] = float("nan")
    vc[hidden] = float("nan")
    return q, kc, vc, hidden


def _offsets(q_lens):
    return np.concatenate([[0], np.cumsum(q_lens)]).astype(int)


def _check_vs_oracle(oracle, out, q, kc, vc, heads, kv_heads, q_lens, past_lens, cache_seqs, max_seq, what):
    off = _offsets(q_lens)
    got = _np(out).reshape(off[-1], heads * HD)
    for i, (ql, pl, cs) in enumerate(zip(q_lens, past_lens, cache_seqs)):
        want = prefill_attn_f64(oracle, _np(q[off[i]:off[i + 1]]), _np(kc[cs]), _np(vc[cs]), heads, kv_heads, pl, max_seq)
        assert_close_ref64(got[off[i]:off[i + 1]], want.reshape(ql, heads * HD), **ATTN_TOL,
                           what=f"{what}: sequence {i} (q_len {ql}, past {pl}, cache seq {cs})")


# (heads, kv_heads, q_lens, past_lens, cache_seqs, caches, max_seq): query tiles hold 64 / n_rep tokens, key tiles 64 keys
KERNEL_CASES = [
    (8, 8, [1, 63, 64, 65], [0, 1, 37, 200], [3, 0, 2, 1], 5, 265),
    (8, 8, [129, 1], [136, 0], [1, 0], 2, 265),                              # past + q_len == max_seq
    (8, 2, [15, 16, 17, 33], [200, 37, 0, 1], [4, 0, 2, 1], 6, 256),
    (8, 2, [1], [255], [2], 3, 256),
    (32, 32, [1, 129, 64], [37, 0, 200], [3, 0, 2], 5, 264),
    (64, 8, [7, 8, 9, 65], [1, 0, 37, 191], [2, 3, 0, 1], 4, 256),
    (64, 8, [257], [0], [0], 1, 257),                                        # n_seq 1, past + q_len == max_seq
]


@pytest.mark.parametrize("heads,kv_heads,q_lens,past_lens,cache_seqs,n_cache,max_seq", KERNEL_CASES)
def test_kernel_vs_oracle(oracle, heads, kv_heads, q_lens, past_lens, cache_seqs, n_cache, max_seq):
    import torch
    from exllama_b200 import cuda_ext
    q, kc, vc, _ = _inputs(heads, kv_heads, q_lens, past_lens, cache_seqs, n_cache, max_seq, seed=heads + sum(q_lens))
    out = torch.empty((sum(q_lens), heads * HD), dtype=torch.float16, device="cuda")
    cuda_ext.exllama_ext.prefill_attn_ragged(q, kc, vc, out, q_lens, past_lens, cache_seqs, heads, kv_heads, HD, max_seq)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out).all())
    _check_vs_oracle(oracle, out, q, kc, vc, heads, kv_heads, q_lens, past_lens, cache_seqs, max_seq, f"{heads}/{kv_heads}")


@pytest.mark.parametrize("heads,kv_heads", [(8, 2), (64, 8)])
def test_kernel_at_the_cap(oracle, heads, kv_heads):
    """64 sequences, q_len 1 .. 20 at past 0 .. 90, in a shuffled subset of 70 cache sequences."""
    from exllama_b200 import capi
    rng = np.random.default_rng(heads)
    q_lens = [int(v) for v in rng.integers(1, 21, CAP)]
    past_lens = [int(v) for v in rng.integers(0, 91, CAP)]
    cache_seqs = [int(v) for v in rng.permutation(70)[:CAP]]
    q, kc, vc, _ = _inputs(heads, kv_heads, q_lens, past_lens, cache_seqs, 70, 112, seed=7)
    out = capi.prefill_attn_ragged(q, kc, vc, q_lens, past_lens, cache_seqs, heads, kv_heads, HD, 112)
    _check_vs_oracle(oracle, out, q, kc, vc, heads, kv_heads, q_lens, past_lens, cache_seqs, 112, f"cap {heads}/{kv_heads}")


@pytest.mark.parametrize("heads,kv_heads,bsz,q_len,past_len", [(8, 8, 3, 65, 37), (8, 2, 4, 17, 200), (32, 32, 2, 129, 0),
                                                                 (64, 8, 4, 9, 1), (64, 8, 2, 257, 191)])
def test_uniform_batch_bitwise_equal_to_prefill_attn(heads, kv_heads, bsz, q_len, past_len):
    """A ragged description of bsz equal sequences in cache sequences 0 .. bsz-1 is bitwise exl_prefill_attn's result, and one
    sequence alone is bitwise exl_prefill_attn on that sequence's cache slice."""
    import torch
    from exllama_b200 import capi
    max_seq = past_len + q_len + 3
    q, kc, vc, _ = _inputs(heads, kv_heads, [q_len] * bsz, [past_len] * bsz, list(range(bsz)), bsz, max_seq, seed=bsz + q_len)
    uni = capi.prefill_attn(q.view(bsz, q_len, heads, HD), kc, vc, heads, kv_heads, HD, past_len, max_seq)
    rag = capi.prefill_attn_ragged(q, kc, vc, [q_len] * bsz, [past_len] * bsz, list(range(bsz)), heads, kv_heads, HD, max_seq)
    b = bsz - 1
    one_uni = capi.prefill_attn(q[b * q_len:].view(1, q_len, heads, HD), kc[b:b + 1], vc[b:b + 1], heads, kv_heads, HD, past_len,
                                max_seq)
    one_rag = capi.prefill_attn_ragged(q[b * q_len:], kc, vc, [q_len], [past_len], [b], heads, kv_heads, HD, max_seq)
    torch.cuda.synchronize()
    assert _bits_equal(rag.view(-1), uni.view(-1)), "ragged description of a uniform batch differs from exl_prefill_attn"
    assert _bits_equal(one_rag.view(-1), one_uni.view(-1)), "one-sequence ragged call differs from exl_prefill_attn"


def test_nan_rows_unchanged_caches_and_determinism():
    """NaN in every row outside each sequence's [0, past_len + q_len) and in the cache sequences the call does not name: the output
    is finite and bitwise equal to a run on a clean cache; the caches keep their bits; a second launch is bitwise equal."""
    import torch
    from exllama_b200 import capi
    heads, kv_heads, max_seq = 64, 8, 320
    q_lens, past_lens, cache_seqs = [77, 1, 130, 64], [100, 0, 190, 37], [5, 1, 3, 0]
    q, kc, vc, hidden = _inputs(heads, kv_heads, q_lens, past_lens, cache_seqs, 7, max_seq, seed=11)
    k0, v0 = kc.clone(), vc.clone()
    args = (q_lens, past_lens, cache_seqs, heads, kv_heads, HD, max_seq)
    out = capi.prefill_attn_ragged(q, kc, vc, *args)
    again = capi.prefill_attn_ragged(q, kc, vc, *args)
    ck, cv = kc.clone(), vc.clone()
    ck[hidden] = 0
    cv[hidden] = 0
    clean = capi.prefill_attn_ragged(q, ck, cv, *args)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out).all())
    assert _bits_equal(kc, k0) and _bits_equal(vc, v0), "the kernel wrote a cache"
    assert _bits_equal(out, again), "two launches differ"
    assert _bits_equal(out, clean), "NaN rows no sequence may read change the output"


@pytest.mark.parametrize("heads,kv_heads", [(8, 8), (8, 2), (64, 8)])
def test_rope_cache_ragged_bit_exact(heads, kv_heads):
    """rope_cache_ragged against rope_ of each sequence at its past_len followed by the cache copy: q, k and the written cache rows
    bitwise equal, every other cache row bitwise unchanged."""
    import torch
    from exllama_b200 import cuda_ext
    ext = cuda_ext.exllama_ext
    max_seq, n_cache = 300, 6
    q_lens, past_lens, cache_seqs = [1, 64, 130, 33], [0, 200, 170, 37], [4, 0, 2, 5]
    T = sum(q_lens)
    g = torch.Generator(device="cuda"); g.manual_seed(heads + kv_heads)
    q = (torch.randn((T, heads, HD), device="cuda", generator=g) * 2).half()
    k = (torch.randn((T, kv_heads, HD), device="cuda", generator=g) * 2).half()
    v = torch.randn((T, kv_heads, HD), device="cuda", generator=g).half()
    pos = torch.arange(max_seq, device="cuda", dtype=torch.float32)[:, None] / (10000.0 ** (torch.arange(0, HD, 2, device="cuda") / HD))
    emb = torch.cat((pos, pos), dim=-1)
    sin, cos = emb.sin()[None, None].half().contiguous(), emb.cos()[None, None].half().contiguous()
    kc = torch.randn((n_cache, kv_heads, max_seq, HD), device="cuda", generator=g).half()
    vc = torch.randn_like(kc)
    want_q, want_k, want_kc, want_vc = q.clone(), k.clone(), kc.clone(), vc.clone()
    off = _offsets(q_lens)
    for i, (ql, pl, cs) in enumerate(zip(q_lens, past_lens, cache_seqs)):
        qi = want_q[off[i]:off[i + 1]].view(1, ql, heads * HD)
        ki = want_k[off[i]:off[i + 1]].view(1, ql, kv_heads * HD)
        ext.rope_(qi, sin, cos, pl, heads, HD)
        ext.rope_(ki, sin, cos, pl, kv_heads, HD)
        want_kc[cs, :, pl:pl + ql].copy_(ki.view(ql, kv_heads, HD).transpose(0, 1))
        want_vc[cs, :, pl:pl + ql].copy_(v[off[i]:off[i + 1]].transpose(0, 1))
    ext.rope_cache_ragged(q, k, v, kc, vc, sin, cos, q_lens, past_lens, cache_seqs, heads, kv_heads, HD, max_seq)
    torch.cuda.synchronize()
    assert _bits_equal(q, want_q), "q differs from rope_"
    assert _bits_equal(k, want_k), "k differs from rope_"
    assert _bits_equal(kc, want_kc) and _bits_equal(vc, want_vc), "cache differs from rope_ + copy (or a row outside was written)"


def test_argument_errors():
    import ctypes as C
    import torch
    from exllama_b200 import capi
    heads, kv, max_seq, n_cache = 8, 2, 16, 3
    q = torch.zeros((8, heads, HD), dtype=torch.float16, device="cuda")
    k = torch.zeros((8, kv, HD), dtype=torch.float16, device="cuda")
    kc = torch.zeros((n_cache, kv, max_seq, HD), dtype=torch.float16, device="cuda")
    vc, out, sc = torch.zeros_like(kc), torch.empty((8, heads * HD), dtype=torch.float16, device="cuda"), torch.zeros((max_seq, HD), dtype=torch.float16, device="cuda")
    lib, P = capi.lib(), capi._ptr
    good = dict(q_lens=[4, 4], past_lens=[0, 12], cache_seqs=[2, 0])

    def attn(r, **kw):
        a = dict(q=P(q), kc=P(kc), vc=P(vc), out=P(out), r=r, n=n_cache, heads=heads, kv=kv, hd=HD, max_seq=max_seq)
        a.update(kw)
        return lib.exl_prefill_attn_ragged(*a.values(), capi._stream())

    def rope(r, **kw):
        a = dict(q=P(q), k=P(k), v=P(k), kc=P(kc), vc=P(vc), sin=P(sc), cos=P(sc), r=r, n=n_cache, heads=heads, kv=kv, hd=HD,
                 max_seq=max_seq)
        a.update(kw)
        return lib.exl_rope_cache_ragged(*a.values(), capi._stream())

    def ragged(**kw):
        d = dict(good)
        d.update(kw)
        return capi.ragged(d["q_lens"], d["past_lens"], d["cache_seqs"])

    too_many = ragged(q_lens=[1] * (CAP + 1), past_lens=[0] * (CAP + 1), cache_seqs=list(range(CAP + 1)))
    no_seq = ragged(); no_seq.n_seq = 0
    no_arr = ragged(); no_arr.past_len = C.POINTER(C.c_int)()
    cases = [
        (dict(r=C.byref(no_seq)), "n_seq 0"), (dict(r=C.byref(too_many)), f"n_seq {CAP + 1}"),
        (dict(r=C.byref(ragged(q_lens=[4, 0]))), "q_len[1] 0"), (dict(r=C.byref(ragged(past_lens=[-1, 12]))), "past_len[0] -1"),
        (dict(r=C.byref(ragged(past_lens=[0, 13]))), "max_seq_len 16"), (dict(r=C.byref(ragged(cache_seqs=[2, 3]))), "cache_seq[1] 3"),
        (dict(r=C.byref(ragged(cache_seqs=[-1, 0]))), "cache_seq[0] -1"), (dict(r=C.byref(ragged(cache_seqs=[2, 2]))), "repeats"),
        (dict(r=C.byref(ragged()), hd=64), "head_dim 64"), (dict(r=C.byref(ragged()), kv=3), "num_kv_heads 3"),
        (dict(r=None), "NULL"), (dict(r=C.byref(no_arr)), "NULL"), (dict(r=C.byref(ragged()), q=None), "NULL"),
        (dict(r=C.byref(ragged()), kc=None), "NULL"), (dict(r=C.byref(ragged()), vc=None), "NULL"),
    ]
    assert attn(C.byref(ragged())) == 0 and rope(C.byref(ragged())) == 0
    for fn, name, extra in ((attn, "prefill_attn_ragged", [(dict(r=C.byref(ragged()), out=None), "NULL")]),
                            (rope, "rope_cache_ragged", [(dict(r=C.byref(ragged()), sin=None), "NULL"),
                                                         (dict(r=C.byref(ragged()), k=None), "NULL")])):
        for kw, text in cases + extra:
            assert fn(**kw) == 1, (name, kw)                             # EXL_ERR_ARG
            msg = lib.exl_last_error().decode()
            assert name in msg and text in msg, (name, kw, msg)
    torch.cuda.synchronize()


# ---- DecodeStack.prefill_ragged ------------------------------------------------------------------------------------------------------
def _x(T, hidden, seed, scale=0.5):
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    return (torch.randn((T, hidden), device="cuda", generator=g) * scale).half()


# T <= 48 rows run the skinny GEMM route, more the wgmma GEMM: (kv_heads, groupsize, act_order, lora rank, q_lens, past_lens, seqs)
STACK_CASES = [
    (8, 128, False, 0, [5, 1, 30], [0, 37, 100], [2, 0, 1]),
    (2, 32, True, 0, [77, 1, 40], [200, 0, 37], [1, 2, 0]),
    (8, 32, False, 0, [65, 64], [1, 254], [0, 2]),
    (2, 128, True, 0, [130], [200], [1]),
    (8, 128, False, 8, [3, 9, 20], [0, 50, 7], [1, 2, 0]),
    (2, 128, False, 16, [100, 33], [37, 0], [2, 1]),
]


@pytest.mark.parametrize("kv,gs,act,rank,q_lens,past_lens,seqs", STACK_CASES)
def test_prefill_ragged_vs_oracle(oracle, stacks, kv, gs, act, rank, q_lens, past_lens, seqs):
    """Logits at every position and the new cache rows of every sequence against oracle_prefill with M = T; every other row of
    every cache sequence bitwise unchanged."""
    import torch
    st = stacks(kv_heads=kv, gs=gs, act=act, max_seq=MAX_SEQ, batch=3, seed=sum(q_lens) + kv)
    if rank:
        st.add_lora(rank, targets="all", seed=rank)
    T = sum(q_lens)
    x = _x(T, 1024, seed=T)
    snap = snapshot(st)
    logits = _np(st.prefill_ragged(x.clone(), q_lens, past_lens, seqs, last_only=False))
    torch.cuda.synchronize()
    what = f"kv {kv} g{gs} act {act} lora {rank} q_lens {q_lens} past {past_lens}"
    span = {cs: (pl, pl + ql) for ql, pl, cs in zip(q_lens, past_lens, seqs)}
    for b in range(st.batch):
        lo, hi = span.get(b, (0, 0))
        for i, (kc, vc) in enumerate(zip(st.key_cache, st.value_cache)):
            for name, c, c0 in (("k", kc, snap[i][0]), ("v", vc, snap[i][1])):
                assert torch.equal(c[b, :, :lo], c0[b, :, :lo]) and torch.equal(c[b, :, hi:], c0[b, :, hi:]), \
                    f"{what}: layer {i} {name} cache of sequence {b}: a row outside [{lo}, {hi}) was written"
    caches = snapshot(st)
    off = _offsets(q_lens)
    for j, (ql, pl, cs) in enumerate(zip(q_lens, past_lens, seqs)):
        want, rows = oracle_prefill(oracle, st, caches, _np(x[off[j]:off[j + 1]]), pl, cs, T)
        assert_close_ref64(logits[off[j]:off[j + 1]], want, **LOGIT_TOL, what=f"{what}: sequence {j} logits")
        for i, (kc, vc) in enumerate(zip(st.key_cache, st.value_cache)):
            assert_close_ref64(_np(kc[cs, :, pl:pl + ql]), rows[i][0].astype(np.float64), **CACHE_TOL, what=f"{what}: seq {j} layer {i} k")
            assert_close_ref64(_np(vc[cs, :, pl:pl + ql]), rows[i][1].astype(np.float64), **CACHE_TOL, what=f"{what}: seq {j} layer {i} v")


def test_prefill_ragged_last_only_and_errors(stacks):
    """last_only returns each sequence's last row of the full logits (same caches, up to the lm_head GEMM's rounding at another M);
    argument errors are ValueErrors."""
    import torch
    st = stacks(kv_heads=2, batch=3, seed=41, max_seq=MAX_SEQ)
    q_lens, past_lens = [9, 60, 1], [3, 0, 100]
    x = _x(sum(q_lens), 1024, seed=42)
    snap = snapshot(st)
    full = st.prefill_ragged(x.clone(), q_lens, past_lens, last_only=False)
    restore(st, snap)
    last = st.prefill_ragged(x.clone(), q_lens, past_lens)
    torch.cuda.synchronize()
    ends = torch.tensor(_offsets(q_lens)[1:] - 1, device="cuda")
    assert last.shape == (3, st.shape.vocab)
    assert_close_ref64(_np(last), _np(full[ends]).astype(np.float64), rel=1e-3, rms=1e-3, what="last_only rows")
    for kw, text in ((dict(q_lens=[9, 60, 0]), "at least 1"), (dict(past_lens=[3, 0, st.max_seq]), "max_seq"),
                     (dict(seqs=[0, 1, 3]), "cache sequence 3"), (dict(seqs=[0, 1, 1]), "twice"),
                     (dict(past_lens=[3, 0]), "past_lens"), (dict(q_lens=[9, 60, 2]), "hidden")):
        a = dict(q_lens=q_lens, past_lens=past_lens, seqs=None)
        a.update(kw)
        with pytest.raises(ValueError, match=text):
            st.prefill_ragged(x, a["q_lens"], a["past_lens"], a["seqs"])


def test_serving_flow_into_fused_batch_step(oracle, stacks):
    """batch=4: one prefill_ragged of prompts of 1, 77, 200 and 513 tokens at past 0, 0, 37 and 300, then one fused batch decode step
    at the resulting past_lens, against the whole-token oracle for each sequence."""
    import torch
    st = stacks(kv_heads=2, batch=4, max_seq=1024, seed=61)
    q_lens, past_lens = [1, 77, 200, 513], [0, 0, 37, 300]
    st.prefill_ragged(_x(sum(q_lens), 1024, seed=62), q_lens, past_lens)
    lens = [p + q for p, q in zip(past_lens, q_lens)]
    snap = snapshot(st)
    st.make_plan()
    xt = _x(4, 1024, seed=63).view(4, 1, 1024)
    got = _np(st.decode_step_fused_batch(xt, lens))
    torch.cuda.synchronize()
    for b in range(4):
        _, want, _ = oracle_decode_step(oracle, st, snap, _np(xt[b]), lens[b], seq=b)
        assert_close_ref64(got[b], want.reshape(-1), **LOGIT_TOL, what=f"fused batch step, seq {b} at {lens[b]}")


@pytest.mark.parametrize("name", ["7b", "70b"])
def test_full_size_ragged_vs_prefill_per_prompt(stacks, name):
    """Two layers of the 7B and 70B (grouped-query) shapes: one ragged call of five prompts, 1920 tokens in all, against one
    prefill(seq=) per prompt from the same caches, on sampled logits and every cache row."""
    import torch
    from exllama_b200.shapes import GQA_SHAPES, SHAPES
    s = {**SHAPES, **GQA_SHAPES}[name]
    q_lens, past_lens, seqs = [700, 513, 400, 250, 57], [0, 300, 0, 1000, 37], [3, 0, 4, 1, 2]
    T = sum(q_lens)
    st = stacks(s, gs=128, max_seq=2048, batch=5, seed=17)
    x = _x(T, s.hidden, seed=29)
    off = _offsets(q_lens)
    snap0 = snapshot(st)
    pos = sorted(set(range(0, T, 97)) | {T - 1} | set(int(o) - 1 for o in off[1:]))
    loop = torch.cat([st.prefill(x[off[j]:off[j + 1]].view(1, -1, s.hidden).contiguous(), past_lens[j], last_only=False, seq=seqs[j])
                      for j in range(len(q_lens))])[pos].cpu()
    looped = snapshot(st)
    restore(st, snap0)
    ragged = st.prefill_ragged(x.clone(), q_lens, past_lens, seqs, last_only=False)[pos].cpu()
    torch.cuda.synchronize()
    assert_close_ref64(ragged.numpy(), loop.numpy().astype(np.float64), rel=2e-2, rms=2e-2, what=f"{name} ragged vs per-prompt logits")
    for i, ((kl, vl), kc, vc) in enumerate(zip(looped, st.key_cache, st.value_cache)):
        for j, (ql, pl, cs) in enumerate(zip(q_lens, past_lens, seqs)):
            for nm, c, cl in (("k", kc, kl), ("v", vc, vl)):
                assert_close_ref64(_np(c[cs, :, pl:pl + ql]), _np(cl[cs, :, pl:pl + ql]).astype(np.float64), rel=2e-2, rms=2e-2,
                                   what=f"{name} layer {i} prompt {j} {nm} rows")
            assert torch.equal(kc[cs, :, :pl], kl[cs, :, :pl]) and torch.equal(kc[cs, :, pl + ql:], kl[cs, :, pl + ql:])
            assert torch.equal(vc[cs, :, :pl], vl[cs, :, :pl]) and torch.equal(vc[cs, :, pl + ql:], vl[cs, :, pl + ql:])
