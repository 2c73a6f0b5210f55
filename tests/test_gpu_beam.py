"""Beam search on the GPU (exl_beam_select, exl_kv_copy_rows, exllama_b200.beam): the selection against the float64 oracle
(oracle/beam_oracle.py) on exl_sample's own dist rows at vocab 32000 / 128256 / 262144, planted ties, short candidate lists,
the first mode's draws (exactly, and their law by chi-square), undefined rows, determinism, graph replay and argument errors; the
row copy bit for bit with nothing else written; and BeamSearch end to end on the synthetic stacks of tests/stack_harness.py --
plain sampling, greedy chains, a traced run replayed through the oracle, the cache invariant after every expansion, the hand-back
to decode_step_fused, both step routes, grouped-query attention and LoRA."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import beam_oracle as B
from stack_harness import lib_state, stacks  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

MARGIN = 1e-9            # selections the oracle decides by less are not compared
PROMPT = [5, 17, 300, 1029, 44, 2000, 7, 7, 123, 999]


def _settings(temperature=1.0, top_k=0, top_p=0.0, min_p=0.0, typical=0.0, penalty_max=1.0, sustain=-1, decay=0):
    from exllama_b200 import sampling
    s = sampling.Settings()
    s.temperature, s.top_k, s.top_p, s.min_p, s.typical = temperature, top_k, top_p, min_p, typical
    s.token_repetition_penalty_max, s.token_repetition_penalty_sustain, s.token_repetition_penalty_decay = penalty_max, sustain, decay
    return s


def _kw(s):
    return dict(temperature=s.temperature, top_k=s.top_k, top_p=s.top_p, min_p=s.min_p, typical=s.typical,
                penalty_max=s.token_repetition_penalty_max, sustain=s.token_repetition_penalty_sustain,
                decay=s.token_repetition_penalty_decay)


SETTINGS = [dict(temperature=0.95, top_k=40, top_p=0.65), dict(temperature=0.95, top_p=0.9), dict(temperature=1.0, top_k=0, typical=0.3),
            dict(temperature=1.5, top_k=500)]


def _dists(rows, vocab, seed, settings):
    """exl_sample's dist rows of seeded N(0, 3) logits [rows, vocab]."""
    import torch
    from exllama_b200 import sampling
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    lg = torch.randn((rows, vocab), device="cuda", generator=g) * 3.0
    d = torch.empty_like(lg)
    sampling.sample(lg, _settings(**settings), u=torch.zeros(rows, device="cuda"), dist=d)
    return d


def _check_expand(res, dists, scores, beams, what):
    k, par, tok, prob, sc = res.read()
    kept, m = B.expand(dists, scores, beams)
    assert k == len(kept), (what, k, len(kept))
    if m < MARGIN:
        return False
    assert [(int(r), int(t)) for r, t in zip(par, tok)] == [(r, t) for r, t, _, _ in kept], what
    np.testing.assert_array_equal(prob, np.array([p for _, _, p, _ in kept], np.float32), err_msg=what)
    np.testing.assert_allclose(sc, [s for _, _, _, s in kept], rtol=1e-14, atol=1e-12, err_msg=what)
    return True


# ---- exl_beam_select ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("beams", [1, 4, 16])
@pytest.mark.parametrize("vocab", [32000, 128256, 262144])
@pytest.mark.parametrize("rows", [1, 4, 64])
def test_select_against_oracle(rows, vocab, beams):
    """Seeded dist rows of exl_sample under one of four settings, window scores spread over a few nats: the kept (row, token) pairs,
    their probabilities and scores equal the oracle's wherever it decides with a margin of at least 1e-9."""
    from exllama_b200 import beam
    compared = 0
    for rep in range(2):
        st = SETTINGS[(rows + vocab + beams + rep) % len(SETTINGS)]
        d = _dists(rows, vocab, 1000 * rows + beams + rep, st)
        rng = np.random.default_rng(rows * 7 + beams + rep)
        scores = list(-rng.random(rows) * 3.0)
        res = beam.select(d, scores, beams)
        compared += _check_expand(res, d.cpu().numpy(), scores, beams, f"rows {rows} vocab {vocab} beams {beams} {st}")
    assert compared >= 1


def test_select_planted_ties():
    """Exact ties (equal probabilities under equal window scores) across rows go to the lower row and within a row to the lower
    token; the kept ones come out by row, then score, then token."""
    import torch
    from exllama_b200 import beam
    d = torch.zeros((3, 32000), device="cuda")
    d[0, [9, 5, 31999, 200]] = 0.25
    d[1, [7, 8, 9, 10]] = 0.25
    d[2, [1, 0]] = 0.25
    d[2, 2] = 0.125
    order = [(0, 5), (0, 9), (0, 200), (0, 31999), (1, 7), (1, 8), (1, 9), (1, 10), (2, 0), (2, 1), (2, 2)]
    for beams in (1, 3, 6, 8, 10, 11, 64):
        k, par, tok, _, sc = beam.select(d, [0.0, 0.0, 0.0], beams).read()
        assert k == min(beams, 11) and list(zip(par.tolist(), tok.tolist())) == order[:k], beams
    # a higher row score puts row 2's ties first among the kept, which are still laid out by row
    k, par, tok, _, _ = beam.select(d, [0.0, 0.0, 1.0], 3).read()
    assert list(zip(par.tolist(), tok.tolist())) == [(2, 0), (2, 1), (2, 2)]
    k, par, tok, _, _ = beam.select(d, [0.0, 0.0, 0.5], 4).read()
    assert list(zip(par.tolist(), tok.tolist())) == [(0, 5), (0, 9), (2, 0), (2, 1)]


def test_select_short_lists():
    """Fewer candidates than beams: every candidate, then -1 / NaN entries; a row with one kept token gives one candidate."""
    import torch
    from exllama_b200 import beam
    d = torch.zeros((2, 32000), device="cuda")
    d[0, 17] = 1.0
    d[1, [3, 30000]] = torch.tensor([0.75, 0.25], device="cuda")
    res = beam.select(d, [-1.0, 0.0], 16)
    k, par, tok, prob, sc = res.read()
    assert k == 3 and list(zip(par.tolist(), tok.tolist())) == [(0, 17), (1, 3), (1, 30000)]
    np.testing.assert_allclose(sc, [-1.0, math.log(0.75), math.log(0.25)], rtol=1e-15)
    assert res.parent[3:].eq(-1).all() and res.token[3:].eq(-1).all() and res.prob[3:].isnan().all()
    k, par, tok, _, _ = beam.select(d[:1], [0.0], 4).read()
    assert k == 1 and tok.tolist() == [17]


def test_select_first_mode():
    """The first mode equals beam_oracle.draw_without_replacement bit for bit (same fixed point, same double rounding), sorted by id,
    with score_host[0] + log p as the score."""
    import torch
    from exllama_b200 import beam
    for i, (vocab, st) in enumerate(((32000, SETTINGS[0]), (32000, SETTINGS[1]), (128256, SETTINGS[3]), (262144, SETTINGS[2]))):
        d = _dists(1, vocab, 50 + i, st)
        dn = d[0].cpu().numpy()
        for beams in (1, 4, 16):
            g = torch.Generator(device="cuda"); g.manual_seed(100 * i + beams)
            u = torch.rand(beams, device="cuda", generator=g)
            k, par, tok, prob, sc = beam.select(d, [-2.0], beams, first=True, u=u).read()
            want, _ = B.draw_without_replacement(dn, u.cpu().numpy())
            assert k == len(want) and tok.tolist() == sorted(want), (vocab, beams)
            assert (par == 0).all() and np.array_equal(prob, dn[tok])
            np.testing.assert_allclose(sc, -2.0 + np.log(prob.astype(np.float64)), rtol=1e-14)


def test_first_mode_law():
    """Two draws without replacement from p over six ids: the unordered pair {a, b} has probability p_a p_b / (1 - p_a) +
    p_b p_a / (1 - p_b) (chi-square, 4000 launches)."""
    import torch
    from scipy import stats
    from exllama_b200 import beam
    p = np.array([0.3, 0.0, 0.25, 0.2, 0.15, 0.1], np.float32)
    d = torch.tensor(p, device="cuda").view(1, -1)
    g = torch.Generator(device="cuda"); g.manual_seed(9)
    res = beam.SelectResult(1, 2, d.device)
    out = torch.empty((4000, 2), dtype=torch.int64, device="cuda")
    for i in range(4000):
        beam.select(d, [0.0], 2, first=True, u=torch.rand(2, device="cuda", generator=g), out=res)
        out[i] = res.token
    pairs = [tuple(r) for r in out.cpu().tolist()]
    ids = [0, 2, 3, 4, 5]
    q = p.astype(np.float64)
    keys = [(a, b) for i, a in enumerate(ids) for b in ids[i + 1:]]
    exp = np.array([q[a] * q[b] / (1 - q[a]) + q[b] * q[a] / (1 - q[b]) for a, b in keys])
    exp *= len(pairs) / exp.sum()                                 # the law sums to 1 up to the fp32 rounding of p
    obs = np.array([sum(1 for x in pairs if x == kk) for kk in keys])
    assert obs.sum() == len(pairs)
    assert stats.chisquare(obs, exp).pvalue > 1e-3, (obs, exp)


def test_select_undefined_rows():
    """exl_sample marks an undefined row with NaN in every dist entry (pinned here); such a row, a row with no positive entry and a
    row with a negative entry each give count -1 and -1 / NaN outputs, in both modes."""
    import torch
    from exllama_b200 import beam, sampling
    lg = torch.randn((2, 32000), device="cuda")
    lg[1] = -math.inf
    d = torch.full_like(lg, 7.0)
    tok, _ = sampling.sample(lg, _settings(), u=torch.zeros(2, device="cuda"), dist=d)
    assert tok[1].item() == -1 and d[1].isnan().all() and not d[0].isnan().any()
    res = beam.select(d, [0.0, 0.0], 4)
    assert res.read()[0] == -1 and res.token.eq(-1).all() and res.parent.eq(-1).all() and res.score.isnan().all()
    assert beam.select(d[1:], [0.0], 4, first=True, u=torch.rand(4, device="cuda")).read()[0] == -1
    z = torch.zeros((2, 1000), device="cuda")
    z[0, 3] = 1.0
    assert beam.select(z, [0.0, 0.0], 4).read()[0] == -1
    z[1, 4] = 1.0
    z[1, 5] = -0.5
    assert beam.select(z, [0.0, 0.0], 4).read()[0] == -1
    z[1, 5] = 0.0
    assert beam.select(z, [0.0, 0.0], 4).read()[0] == 2


def test_select_deterministic_and_graph():
    """Two launches are bitwise equal, and a CUDA-graph replay of the call equals the eager call."""
    import torch
    from exllama_b200 import beam
    d = _dists(16, 32000, 77, SETTINGS[1])
    scores = list(np.linspace(-3, 0, 16))
    a = beam.select(d, scores, 16).buf.clone()
    b = beam.select(d, scores, 16).buf.clone()
    assert torch.equal(a, b)
    res = beam.SelectResult(16, 16, d.device)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        beam.select(d, scores, 16, out=res)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        beam.select(d, scores, 16, out=res)
    res.buf.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(res.buf, a)


def test_select_errors():
    import torch
    from exllama_b200 import capi
    lib = capi.lib()
    d = torch.rand((2, 100), device="cuda")
    u = torch.rand(4, device="cuda")
    work = torch.empty(capi.beam_work_bytes(64, 64), dtype=torch.uint8, device="cuda")
    outs = [torch.empty(64, dtype=dt, device="cuda") for dt in (torch.int32, torch.int64, torch.float32, torch.float64)]
    cnt = torch.empty(1, dtype=torch.int32, device="cuda")
    P = capi._ptr

    def call(dist=P(d), rows=2, vocab=100, ld=100, scores=(0.0, 0.0), beams=4, mode=0, uu=P(u), w=P(work), wb=work.numel(),
             parent=P(outs[0]), token=P(outs[1]), prob=P(outs[2]), score=P(outs[3]), count=P(cnt)):
        sc = (C.c_double * max(len(scores), 1))(*scores) if scores is not None else None
        return lib.exl_beam_select(dist, rows, vocab, ld, sc, beams, mode, uu, w, wb, parent, token, prob, score, count, None)

    assert call() == 0
    cases = [(dict(rows=0), "rows 0 outside"), (dict(rows=65), "rows 65 outside"), (dict(beams=0), "beams 0 outside"),
             (dict(beams=65), "beams 65 outside"), (dict(vocab=0, ld=0), "vocab 0 outside"), (dict(vocab=262145, ld=262145), "vocab 262145"),
             (dict(ld=99), "dist_ld 99 < vocab 100"), (dict(mode=2), "mode 2"), (dict(mode=1), "rows 2 in first mode"),
             (dict(rows=1, scores=(0.0,), mode=1, uu=None), "u is NULL"), (dict(scores=(0.0, math.nan)), r"score_host\[1\]"),
             (dict(scores=(math.inf, 0.0)), r"score_host\[0\]"), (dict(wb=2 * 4 * 8), "work_bytes"), (dict(w=C.c_void_p(work.data_ptr() + 4)), "not 16-byte"),
             (dict(dist=None), "NULL pointer"), (dict(scores=None), "NULL pointer"), (dict(w=None), "NULL pointer"),
             (dict(parent=None), "NULL pointer"), (dict(token=None), "NULL pointer"), (dict(prob=None), "NULL pointer"),
             (dict(score=None), "NULL pointer"), (dict(count=None), "NULL pointer")]
    import re
    for kw, msg in cases:
        rc = call(**kw)
        assert rc != 0, kw
        assert re.search(msg, lib.exl_last_error().decode()), (kw, lib.exl_last_error())


# ---- exl_kv_copy_rows -----------------------------------------------------------------------------------------------------------

def _caches(layers, seqs, kvh, max_seq, seed):
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    kc = [torch.randn((seqs, kvh, max_seq, 128), device="cuda", generator=g).half() for _ in range(layers)]
    vc = [torch.randn((seqs, kvh, max_seq, 128), device="cuda", generator=g).half() for _ in range(layers)]
    return kc, vc


class _Caches:
    def __init__(self, kc, vc):
        self.key_cache, self.value_cache = kc, vc


@pytest.mark.parametrize("kvh", [8, 2])
def test_kv_copy_rows(kvh):
    """Copied rows equal their source bit for bit in every layer, K and V; no other byte of any cache changes.  Ranges touching row 0
    and max_seq, and empty ranges."""
    import torch
    from exllama_b200 import beam
    max_seq = 300
    kc, vc = _caches(3, 6, kvh, max_seq, seed=kvh)
    before = [(k.clone(), v.clone()) for k, v in zip(kc, vc)]
    pairs = [(0, 1, 0, 17), (0, 2, 250, 300), (3, 4, 5, 5), (3, 5, 0, 300)]
    beam.copy_cache_rows(_Caches(kc, vc), pairs)
    torch.cuda.synchronize()
    for l in range(3):
        for c, c0 in ((kc[l], before[l][0]), (vc[l], before[l][1])):
            want = c0.clone()
            for s, d, lo, hi in pairs:
                want[d, :, lo:hi] = c0[s, :, lo:hi]
            assert torch.equal(c, want), l


def test_kv_copy_rows_errors():
    import re
    import torch
    from exllama_b200 import beam, capi
    kc, vc = _caches(2, 4, 2, 64, seed=1)
    st = _Caches(kc, vc)
    bad = [([(0, 0, 0, 4)], "source of pair 0 and the destination of pair 0"), ([(0, 1, 0, 4), (1, 2, 0, 4)], "sequence 1 is the source"),
           ([(0, 1, 0, 4), (2, 1, 0, 4)], "destination of pairs 0 and 1"), ([(0, 1, -1, 4)], r"rows \[-1, 4\)"),
           ([(0, 1, 5, 4)], r"rows \[5, 4\)"), ([(0, 1, 0, 65)], r"rows \[0, 65\)"), ([(0, 4, 0, 4)], "the caches hold"),
           ([(-1, 1, 0, 4)], "the caches hold"), ([(0, i + 1, 0, 1) for i in range(65)], "n_pairs 65")]
    for pairs, msg in bad:
        with pytest.raises(capi.ExlError, match=msg):
            beam.copy_cache_rows(st, pairs)
    lib = capi.lib()
    ks = (C.c_void_p * 2)(*[t.data_ptr() for t in kc])
    vs = (C.c_void_p * 2)(*[t.data_ptr() for t in vc])
    pr = (capi.ExlKvCopyPair * 1)(capi.ExlKvCopyPair(0, 1, 0, 4))
    for args, msg in (((ks, vs, 0, 4, 2, 64, 128, pr, 1), "n_layers 0"), ((ks, vs, 129, 4, 2, 64, 128, pr, 1), "n_layers 129"),
                      ((ks, vs, 2, 1, 2, 64, 128, pr, 1), "num_cache_seqs 1"), ((ks, vs, 2, 4, 0, 64, 128, pr, 1), "num_kv_heads 0"),
                      ((ks, vs, 2, 4, 2, 0, 128, pr, 1), "max_seq_len 0"), ((ks, vs, 2, 4, 2, 64, 12, pr, 1), "head_dim 12"),
                      ((None, vs, 2, 4, 2, 64, 128, pr, 1), "NULL pointer"), ((ks, vs, 2, 4, 2, 64, 128, None, 1), "NULL pointer"),
                      ((ks, vs, 2, 4, 2, 64, 128, pr, 0), "n_pairs 0")):
        assert lib.exl_kv_copy_rows(*args, None) != 0, msg
        assert re.search(msg, lib.exl_last_error().decode()), (msg, lib.exl_last_error())
    odd = (C.c_void_p * 2)(kc[0].data_ptr() + 2, kc[1].data_ptr())
    assert lib.exl_kv_copy_rows(odd, vs, 2, 4, 2, 64, 128, pr, 1, None) != 0
    assert "not 16-byte aligned" in lib.exl_last_error().decode()


# ---- BeamSearch end to end ------------------------------------------------------------------------------------------------------

def _embed(st, seed=11):
    """Random N(0, 0.25) fp16 embeddings [vocab, hidden].  Tied ones (c * lm_head[token]) would make the synthetic stacks repeat
    their input token with a logit near 20 against N(0, 0.64) for the others, so every kept set would be one token and beams would
    never branch; with these the logits of a step spread like N(0, 0.64)."""
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    return (torch.randn((st.shape.vocab, st.shape.hidden), device="cuda", generator=g) * 0.5).half()


def _row_check(st, ref, slot, tokens, n, emb, what):
    """Rows [0, n) of cache sequence `slot` of st, every layer, K and V, within 1e-2 relative + 1e-2 of the row rms of what a fresh
    prefill of tokens[:n] writes into sequence 0 of ref (a stack with the same weights)."""
    import torch
    ids = torch.tensor(tokens[:n], device="cuda")
    ref.prefill(emb[ids].view(1, n, -1), 0, seq=0)
    for i in range(st.n_layers):
        for name, a, b in (("k", st.key_cache[i], ref.key_cache[i]), ("v", st.value_cache[i], ref.value_cache[i])):
            got = a[slot, :, :n].float()
            want = b[0, :, :n].float()
            rms = want.pow(2).mean(dim=(0, 2), keepdim=True).sqrt()
            err = (got - want).abs()
            bad = err > 1e-2 * want.abs() + 1e-2 * rms
            assert not bad.any(), f"{what}: layer {i} {name} slot {slot}: {int(bad.sum())} outside, max err {float(err.max()):.3g}"


def _fused_sample_loop(st, emb, s, n, seed, bos):
    """The plain generation loop: prefill, then fused step -> sampling.sample with a generator seeded `seed`."""
    import torch
    from exllama_b200 import sampling
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    ids = torch.tensor(PROMPT, device="cuda")
    hist = torch.zeros((1, st.max_seq), dtype=torch.int64, device="cuda")
    hist[0, :len(PROMPT)] = ids
    logits = st.prefill(emb[ids].view(1, len(PROMPT), -1), 0)
    st.make_plan()
    out, L = [], len(PROMPT)
    s0 = _settings(**dict(_kw(s), min_p=0.0))
    for i in range(n):
        t, _ = sampling.sample(logits, s0, history=hist, hist_lens=[L + i], generator=g, bos_token_id=bos)
        hist[0, L + i] = t
        out.append(int(t.item()))
        logits = st.decode_step_fused(emb[hist[0, L + i:L + i + 1]].view(1, 1, -1), L + i).view(1, -1)
    st.dplan.close(); st.dplan = None
    return out


def test_plain_sampling_equals_the_loop(stacks):
    """beams = beam_length = 1 is gen_single_token: bitwise the tokens of the fused step -> sampling.sample loop with the same uniforms
    (bos mask, min_p 0)."""
    import torch
    from exllama_b200.beam import BeamSearch
    s = _settings(**SETTINGS[0], penalty_max=1.15, sustain=256, decay=128, min_p=0.3)
    a, b = stacks(seed=21), stacks(seed=21)
    emb = _embed(a)
    want = _fused_sample_loop(a, emb, s, 20, seed=5, bos=7)
    g = torch.Generator(device="cuda"); g.manual_seed(5)
    bs = BeamSearch(b, emb, 1, 1, settings=s, bos_token_id=7, generator=g)
    bs.begin(PROMPT)
    assert bs.fused and bs.generate(20) == want


def _greedy_check(st, emb, emitted, what):
    """Each emitted token is the argmax of a fresh prefill's logits after the tokens before it, or within 1e-2 of the logits' rms of it."""
    import torch
    seq = list(PROMPT)
    for t in emitted:
        ids = torch.tensor(seq, device="cuda")
        lg = st.prefill(emb[ids].view(1, len(seq), -1), 0)[0].double()
        top = int(lg.argmax())
        gap = float(lg[top] - lg[t])
        assert t == top or gap <= 1e-2 * float(lg.pow(2).mean().sqrt()), (what, len(seq), t, top, gap)
        seq.append(t)


@pytest.mark.parametrize("beams,beam_length", [(1, 4), (3, 1), (4, 3), (2, 6)])
def test_greedy_chain(stacks, beams, beam_length):
    """top_k 1: every kept set is one token with p 1, so any beams and beam_length emit the greedy argmax chain."""
    from exllama_b200.beam import BeamSearch
    st = stacks(seed=31, batch=4)
    ref = stacks(seed=31)
    emb = _embed(st)
    bs = BeamSearch(st, emb, beams, beam_length, settings=_settings(top_k=1))
    bs.begin(PROMPT)
    _greedy_check(ref, emb, bs.generate(12), f"beams {beams} beam_length {beam_length}")


def _replay(trace, beams, what):
    """The traced run, decision by decision, through beam_oracle on the run's own dist rows and window scores: the first draw, every
    selection and every emitted token the oracle decides with a margin of at least 1e-9 must equal the run's; the beam list follows
    the run's own choices (so a decision inside the margin does not derail the rest).  Returns the number of decisions compared."""
    first = trace[0]
    want, m = B.draw_without_replacement(first["dist"][0], first["u"])
    compared = 0
    if m >= MARGIN:
        assert sorted(want) == first["token"], what
        compared += 1
    bl = [([t], [p]) for t, p in zip(first["token"], first["prob"])]
    for e in trace[1:]:
        if e["kind"] == "expand":
            assert [w for w, _ in bl] == e["windows"], what
            scores = [B.window_score(pr) for _, pr in bl]
            assert scores == e["scores"], what
            kept, m = B.expand(e["dist"], scores, beams)
            if m >= MARGIN:
                assert [(r, t) for r, t, _, _ in kept] == list(zip(e["parent"], e["token"])), what
                compared += 1
            bl = [(bl[r][0] + [t], bl[r][1] + [p]) for r, t, p in zip(e["parent"], e["token"], e["prob"])]
            continue
        sc = [B.window_score(pr) for _, pr in bl]
        best = max(range(len(sc)), key=lambda i: (sc[i], -i))
        gap = min((sc[best] - s for i, s in enumerate(sc) if i != best), default=math.inf)
        if gap >= MARGIN:
            assert bl[best][0][0] == e["token"], what
            compared += 1
        else:
            best = max((i for i in range(len(bl)) if bl[i][0][0] == e["token"]), key=lambda i: (sc[i], -i))
        t = e["token"]
        bl = [bl[best]] + [b for i, b in enumerate(bl) if i != best and b[0][0] == t]
        bl = [(w[1:], pr[1:]) for w, pr in bl]
    return compared


def _run_checked(st, ref, emb, beams, beam_length, s, n, seed, check_rows=True):
    """A traced BeamSearch run that clones and prunes beams; after every next() the cache invariant holds for every live slot."""
    import torch
    from exllama_b200.beam import BeamSearch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    bs = BeamSearch(st, emb, beams, beam_length, settings=s, generator=g)
    bs.trace = []
    bs.begin(PROMPT)
    emitted, pruned = [], 0
    for i in range(n):
        live = len(bs.list)
        emitted.append(bs.next())
        pruned += live > len(bs.list)
        if check_rows:
            for b in bs.list:
                _row_check(st, ref, b.slot, bs.slot_tokens(b.slot), bs.valid[b.slot], emb, f"after token {i}")
    clones = sum(len(e["parent"]) - len(set(e["parent"])) for e in bs.trace if e["kind"] == "expand")
    assert clones > 0 and pruned > 0, (clones, pruned)
    return bs, emitted


ROUTES = {
    "fused_b4": (dict(batch=4, seed=41), 4, 3),
    "ragged_act": (dict(batch=4, seed=42, act=True), 3, 3),
    "ragged_b8_6beams": (dict(batch=8, seed=43), 6, 2),
    "gqa_fused": (dict(batch=4, seed=44, kv_heads=2), 4, 4),
}


@pytest.mark.parametrize("route", list(ROUTES))
def test_traced_run(stacks, route):
    """Stochastic settings with the penalty: the run replays through beam_oracle on its own dist rows (every decision with margin,
    and the emitted tokens); after every emitted token, rows [0, valid) of every live slot equal a fresh prefill of that beam's tokens;
    after end(), decode_step_fused on sequence 0 matches a prefill of the committed sequence.  The step route is the fused batch plan
    or prefill_ragged (act-order, or more than four beams)."""
    import torch
    kw, beams, beam_length = ROUTES[route]
    st = stacks(**kw)
    ref = stacks(**dict(kw, batch=1))
    emb = _embed(st)
    s = _settings(temperature=1.0, top_k=12, top_p=0.95, penalty_max=1.15, sustain=256, decay=128)
    bs, emitted = _run_checked(st, ref, emb, beams, beam_length, s, 10, seed=7)
    assert bs.fused == route.endswith(("b4", "fused"))
    assert _replay(bs.trace, beams, route) >= 10
    # hand-back: cache sequence 0 holds rows [0, n - 1) of the committed sequence
    seq = bs.end()
    n = len(seq)
    assert seq[:len(PROMPT)] == PROMPT and seq[len(PROMPT):] == emitted
    _row_check(st, ref, 0, seq, n - 1, emb, "after end()")
    if bs.fused:
        lg = st.decode_step_fused(emb[torch.tensor(seq[-1:], device="cuda")].view(1, 1, -1), n - 1)[0].double()   # sequence 0's row
        want = ref.prefill(emb[torch.tensor(seq, device="cuda")].view(1, n, -1), 0)[0].double()
        err = float((lg - want).abs().max())
        assert err <= 2e-2 * float(want.pow(2).mean().sqrt()) + 2e-2 * float(want.abs().max()), err


def test_lora_stack(stacks):
    """A stack with a LoRA adapter on every projection: the fused batch plan carries it, and the cache invariant holds."""
    kw = dict(batch=4, seed=45)
    st = stacks(**kw)
    ref = stacks(**dict(kw, batch=1))
    st.add_lora(8, targets="all", seed=3)
    ref.add_lora(8, targets="all", seed=3)
    emb = _embed(st)
    s = _settings(temperature=1.0, top_k=12, top_p=0.95)
    bs, emitted = _run_checked(st, ref, emb, 4, 3, s, 6, seed=8)
    assert bs.fused
    assert _replay(bs.trace, 4, "lora") >= 6


def test_one_sync_per_expansion(stacks):
    """On the fused route each emitted token, once the windows are full, costs one expansion and one host synchronisation: the
    selection read."""
    import warnings
    import torch
    from exllama_b200.beam import BeamSearch
    st = stacks(batch=4, seed=46)
    emb = _embed(st)
    g = torch.Generator(device="cuda"); g.manual_seed(3)
    bs = BeamSearch(st, emb, 4, 3, settings=_settings(temperature=1.0, top_k=12, top_p=0.95, penalty_max=1.15, sustain=256, decay=128),
                    generator=g)
    bs.begin(PROMPT)
    bs.generate(2)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            bs.generate(6)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = [x for x in w if "called a synchronizing CUDA operation" in str(x.message)]
    assert bs.fused and len(syncs) == 6, [str(x.message) for x in syncs[:3]]


def test_errors(stacks):
    import torch
    from exllama_b200.beam import BeamSearch
    st = stacks(batch=4, seed=1, max_seq=32)
    emb = _embed(st)
    for beams, bl, msg in ((0, 2, "beams 0 outside"), (5, 2, "beams 5 outside"), (2, 0, "beam_length 0")):
        with pytest.raises(ValueError, match=msg):
            BeamSearch(st, emb, beams, bl)
    with pytest.raises(ValueError, match="embed must be fp16"):
        BeamSearch(st, emb[:-1], 2, 2)
    with pytest.raises(ValueError, match="embed must be fp16"):
        BeamSearch(st, emb.float(), 2, 2)
    bs = BeamSearch(st, emb, 2, 8)
    with pytest.raises(ValueError, match="leaves no room"):
        bs.begin(list(range(25)))
    with pytest.raises(ValueError, match="leaves no room"):
        bs.begin([])
    with pytest.raises(RuntimeError, match="call begin"):
        bs.next()
    bs.begin(list(range(20)))
    with pytest.raises(ValueError, match="do not fit max_seq"):
        bs.generate(10)
    headless = stacks(batch=2, seed=1, max_seq=32)
    headless.lm_head = None
    with pytest.raises(ValueError, match="no lm_head"):
        BeamSearch(headless, emb, 2, 2)
    tp = stacks(batch=2, seed=1, max_seq=32)
    tp.tp_size = 2
    try:
        with pytest.raises(NotImplementedError, match="tensor parallelism"):
            BeamSearch(tp, emb, 2, 2)
    finally:
        tp.tp_size = 1
    nan = stacks(batch=2, seed=2, max_seq=32)
    nan.lm_head[5].fill_(float("nan"))
    bs = BeamSearch(nan, emb, 2, 2, banned=None)
    with pytest.raises(RuntimeError, match="undefined"):
        bs.begin([1, 2, 3])
