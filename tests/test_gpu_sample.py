"""exl_sample (csrc/sample.cu) through exllama_b200.sampling on the GPU: against the reference's own sampler (the kept sets and final
probabilities of tests/golden/sample_ref.npz), against the float64 oracle (oracle/sample_oracle.py) on a seeded sweep, the draw,
the penalty bit for bit against exl_apply_rep_penalty, the tie rule, batches, guards, determinism and graph replay, undefined rows,
argument errors, and the logits of the fused decode step and of prefill_ragged."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import sample_oracle as S
from stack_harness import lib_state, stacks  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sample_ref.npz")
TINY = 1e-30            # the kept set on the device: ids whose final probability is at least this (denormals may differ)


def _settings(temperature=1.0, top_k=0, top_p=0.0, min_p=0.0, typical=0.0, penalty_max=1.0, sustain=-1, decay=0):
    from exllama_b200 import sampling
    s = sampling.Settings()
    s.temperature, s.top_k, s.top_p, s.min_p, s.typical = temperature, top_k, top_p, min_p, typical
    s.token_repetition_penalty_max, s.token_repetition_penalty_sustain, s.token_repetition_penalty_decay = penalty_max, sustain, decay
    return s


def _case_settings(c):
    return _settings(c["temperature"], c["top_k"], c["top_p"], c["min_p"], c["typical"], c["penalty_max"], c["sustain"], c["decay"])


def _run(logits, s, history=None, hist_lens=None, u=None, bos=None, banned=None):
    """sampling.sample on numpy / torch inputs; returns tokens, probs, dist as numpy."""
    import torch
    from exllama_b200 import sampling
    lg = torch.as_tensor(np.atleast_2d(logits), dtype=torch.float32).cuda()
    bsz, vocab = lg.shape
    h = None
    if history is not None:
        h = torch.as_tensor(np.atleast_2d(history), dtype=torch.int64).cuda()
    if u is not None:
        u = torch.as_tensor(np.atleast_1d(np.asarray(u, np.float32))).cuda()
    dist = torch.empty((bsz, vocab), dtype=torch.float32, device="cuda")
    t, p = sampling.sample(lg, s, history=h, hist_lens=hist_lens, u=u, bos_token_id=bos, banned=banned, dist=dist)
    torch.cuda.synchronize()
    return t.cpu().numpy(), p.cpu().numpy(), dist.cpu().numpy()


def _check_dist(dist_row, r, what):
    """dist against an oracle / reference kept set and probabilities: same set (>= TINY), values within 1e-5 rel + 1e-7 abs."""
    want = np.zeros(dist_row.shape[0], np.float64)
    want[r["kept"]] = r["probs"]
    np.testing.assert_array_equal(np.nonzero(dist_row >= TINY)[0], np.nonzero(want >= TINY)[0], err_msg=what)
    np.testing.assert_allclose(dist_row, want, rtol=1e-5, atol=1e-7, err_msg=what)


def _mid_u(r, rng, k=8):
    """u at the midpoints of up to k of the oracle's CDF intervals (wide ones), and the tokens they must draw."""
    cdf = r["cdf"]
    lo = np.concatenate([[0.0], cdf[:-1]])
    ok = np.nonzero(cdf - lo > 1e-5)[0]
    pick = rng.choice(ok, size=min(k, len(ok)), replace=False)
    return ((lo[pick] + cdf[pick]) / 2).astype(np.float32), r["kept"][pick], r["probs"][pick]


# ---- against the reference --------------------------------------------------------------------------------------------------------

def test_reference_cases():
    """Every case of the fixture: the kept set equals the reference's and dist matches its final probabilities."""
    for i, c in enumerate(S.golden_cases(GOLD)):
        hist = c["history"][None] if len(c["history"]) else None
        tok, prob, dist = _run(c["logits"], _case_settings(c), history=hist, u=[0.5], bos=c["bos"] if c["bos"] >= 0 else None,
                               banned=c["banned"] if len(c["banned"]) else None)
        _check_dist(dist[0], {"kept": c["kept"], "probs": c["probs"]}, f"case {i}")
        assert tok[0] in c["kept"] and prob[0] == dist[0, tok[0]], i


def test_random_sweep_against_oracle():
    """About 200 random settings on 32000-wide rows; cases the oracle decides with a margin below 1e-5 are skipped."""
    rng = np.random.default_rng(7)
    ran = 0
    for i in range(200):
        vocab = 32000
        logits = S.case_logits(1000 + i, vocab, "dominant" if i % 4 == 0 else "normal", scale=float(rng.uniform(0.5, 4)))
        top_p = float(rng.uniform(0.05, 0.99)) if rng.random() < 0.6 else 0.0
        kw = dict(temperature=float(rng.uniform(0.3, 2.0)), top_k=int(rng.choice([0, 1, 5, 40, 200, vocab])), top_p=top_p,
                  min_p=float(rng.uniform(0, 0.05)) if top_p and rng.random() < 0.4 else 0.0,
                  typical=float(rng.uniform(0.05, 0.99)) if rng.random() < 0.4 else 0.0)
        hl = int(rng.integers(0, 2000))
        history = rng.integers(0, vocab, size=hl).astype(np.int64)
        pen = dict(penalty_max=float(rng.uniform(1.0, 1.3)), sustain=int(rng.choice([-1, 0, 64, 256])), decay=int(rng.choice([0, 16, 128])))
        bos = int(rng.integers(vocab)) if rng.random() < 0.5 else -1
        r = S.sample(logits, history=history, bos=bos, **kw, **pen)
        if S.min_margin(r) < 1e-5:
            continue
        u, toks, probs = _mid_u(r, rng, k=1)
        t, p, dist = _run(logits, _settings(**kw, **pen), history=history[None] if hl else None, u=u, bos=bos if bos >= 0 else None)
        _check_dist(dist[0], r, f"sweep {i} {kw} {pen}")
        assert t[0] == toks[0], (i, t, toks)
        np.testing.assert_allclose(p[0], probs[0], rtol=1e-5, atol=1e-7)
        ran += 1
    assert ran >= 120, ran


# ---- inputs, ordering, determinism ------------------------------------------------------------------------------------------------

def test_draw_at_cdf_midpoints():
    """u at the midpoints of the oracle's CDF intervals (ascending token-id order) draws the oracle's token, with its probability."""
    rng = np.random.default_rng(3)
    history = rng.integers(0, 32000, size=1920).astype(np.int64)
    for kw in (dict(temperature=0.95, top_k=40, top_p=0.65, penalty_max=1.15, sustain=256, decay=128),
               dict(temperature=1.3, top_k=0, typical=0.5), dict(temperature=0.7, top_k=200)):
        logits = S.case_logits(11, 32000, "normal")
        r = S.sample(logits, history=history, **kw)
        u, toks, probs = _mid_u(r, rng, k=32)
        n = len(u)
        t, p, _ = _run(np.repeat(logits[None], n, 0), _settings(**kw), history=np.repeat(history[None], n, 0), u=u)
        np.testing.assert_array_equal(t, toks)
        np.testing.assert_allclose(p, probs, rtol=1e-5, atol=1e-7)
    # u past the total: the largest kept id
    logits = np.array([0.0, 1.0, 2.0, -1.0], np.float32)
    t, _, _ = _run(logits, _settings(), u=[1.0])
    assert t[0] == 3


def test_penalty_bit_exact_with_host_penalty():
    """Raw logits with the penalty on give bitwise the tokens, probs and dist of host-penalised logits (exl_apply_rep_penalty)
    with the penalty off."""
    from exllama_b200 import capi
    lib = capi.lib()
    rng = np.random.default_rng(5)
    vocab = 32000
    for sustain in (-1, 0, 256):
        for decay in (0, 128):
            for hl in (1, 17, 300, 1920):
                logits = S.case_logits(int(rng.integers(1 << 30)), vocab, "normal")
                history = rng.integers(0, 64 if hl > 40 else vocab, size=hl).astype(np.int64)   # many repeats on long histories
                pen = logits.copy()
                assert lib.exl_apply_rep_penalty(vocab, history.ctypes.data, 1.2, sustain, decay, hl, pen.ctypes.data) == 0
                u = rng.random(1).astype(np.float32)
                kw = dict(temperature=0.8, top_k=0, top_p=0.9)
                a = _run(logits, _settings(**kw, penalty_max=1.2, sustain=sustain, decay=decay), history=history[None], u=u)
                b = _run(pen, _settings(**kw), u=u)
                for x, y in zip(a, b):
                    assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), (sustain, decay, hl)


def test_ties_go_to_the_lower_id():
    vocab = 100
    logits = np.full(vocab, -5.0, np.float32)
    logits[[70, 10, 40, 20]] = 2.0
    _, _, d = _run(logits, _settings(top_k=2), u=[0.5])
    assert set(np.nonzero(d[0] > 0)[0]) == {10, 20}
    # top-p: 50 first, then the tie 5 / 60 straddles the cut: 5 stays
    logits = np.full(vocab, -8.0, np.float32)
    logits[50], logits[[60, 5]] = 3.0, 2.0
    r = S.sample(logits, 1.0)
    vals = np.sort(r["probs"])[::-1]
    top_p = float((vals[0] + vals[1] + vals[0] + vals[1] + vals[2]) / 2)
    _, _, d = _run(logits, _settings(top_p=top_p), u=[0.5])
    assert set(np.nonzero(d[0] > 0)[0]) == {50, 5}


def test_batch_rows_equal_single_rows():
    """bsz 1 .. 64, each row its own logits, history length and u: every row is bitwise the row sampled alone."""
    rng = np.random.default_rng(9)
    vocab = 32000
    s = _settings(temperature=0.9, top_k=40, top_p=0.8, penalty_max=1.15, sustain=256, decay=128)
    for bsz in (1, 3, 17, 64):
        logits = np.stack([S.case_logits(int(rng.integers(1 << 30)), vocab, "normal") for _ in range(bsz)])
        hist = rng.integers(0, vocab, size=(bsz, 700)).astype(np.int64)
        lens = [int(rng.integers(0, 701)) for _ in range(bsz)]
        u = rng.random(bsz).astype(np.float32)
        t, p, d = _run(logits, s, history=hist, hist_lens=lens, u=u)
        for b in range(bsz):
            tb, pb, db = _run(logits[b], s, history=hist[b, :max(lens[b], 1)], hist_lens=[lens[b]], u=u[b:b + 1])
            assert t[b] == tb[0] and p[b].tobytes() == pb[0].tobytes() and d[b].tobytes() == db[0].tobytes(), (bsz, b)


def test_logits_unchanged_and_guards_untouched():
    import torch
    from exllama_b200 import capi
    bsz, vocab, ld, G = 3, 32001, 32011, 64
    g = torch.Generator(device="cuda"); g.manual_seed(1)
    logits = torch.randn((bsz, ld), device="cuda", generator=g) * 3
    before = logits.clone()
    tok = torch.full((bsz + 2 * G,), -7, dtype=torch.int64, device="cuda")
    prob = torch.full((bsz + 2 * G,), float("nan"), device="cuda")
    dist = torch.full((bsz * vocab + 2 * G,), float("nan"), device="cuda")
    u = torch.rand(bsz, device="cuda", generator=g)
    hist = torch.randint(0, vocab, (bsz, 300), device="cuda", generator=g)
    lens = (C.c_int * bsz)(300, 0, 129)
    p = capi.ExlSampleParams(0.95, 40, 0.65, 0.0, 0.0, 1.15, 256, 128, 1, None, 0)
    capi.check(capi.lib().exl_sample(capi._ptr(logits), bsz, vocab, ld, capi._ptr(hist), 300, lens, C.byref(p), capi._ptr(u),
                                     C.c_void_p(tok.data_ptr() + 8 * G), C.c_void_p(prob.data_ptr() + 4 * G),
                                     C.c_void_p(dist.data_ptr() + 4 * G), capi._stream()))
    torch.cuda.synchronize()
    assert torch.equal(logits, before)
    assert (tok[:G] == -7).all() and (tok[G + bsz:] == -7).all() and (tok[G:G + bsz] >= 0).all()
    assert prob[:G].isnan().all() and prob[G + bsz:].isnan().all() and not prob[G:G + bsz].isnan().any()
    assert dist[:G].isnan().all() and dist[G + bsz * vocab:].isnan().all() and not dist[G:G + bsz * vocab].isnan().any()


def test_two_launches_bitwise_equal_and_graph_replay():
    import torch
    from exllama_b200 import sampling
    rng = np.random.default_rng(2)
    bsz, vocab = 4, 32000
    logits = torch.as_tensor(np.stack([S.case_logits(i, vocab, "normal") for i in range(bsz)])).cuda()
    hist = torch.as_tensor(rng.integers(0, vocab, size=(bsz, 1920))).cuda()
    u = torch.as_tensor(rng.random(bsz).astype(np.float32)).cuda()
    for s in (sampling.Settings(), _settings(temperature=1.2, top_k=0, top_p=0.9, typical=0.3, penalty_max=1.1, sustain=-1)):
        dist = [torch.empty((bsz, vocab), device="cuda") for _ in range(3)]
        a = sampling.sample(logits, s, history=hist, u=u, dist=dist[0])
        b = sampling.sample(logits, s, history=hist, u=u, dist=dist[1])
        torch.cuda.synchronize()
        assert all(torch.equal(x, y) for x, y in zip(a, b)) and torch.equal(dist[0], dist[1])
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            c = sampling.sample(logits, s, history=hist, u=u, dist=dist[2])
        dist[2].zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(x, y) for x, y in zip(a, c)) and torch.equal(dist[0], dist[2])


def test_undefined_rows():
    """All -inf after masking, a NaN logit, a history token >= vocab: -1 / NaN in that row only."""
    vocab = 1000
    rng = np.random.default_rng(4)
    logits = np.stack([S.case_logits(i, vocab, "normal") for i in range(5)])
    logits[1] = -np.inf
    logits[2, 17] = np.nan
    hist = rng.integers(0, vocab, size=(5, 10)).astype(np.int64)
    hist[3, 4] = vocab
    s = _settings(penalty_max=1.2)
    t, p, d = _run(logits, s, history=hist, u=rng.random(5))
    for b in range(5):
        if b in (1, 2, 3):
            assert t[b] == -1 and np.isnan(p[b]) and np.isnan(d[b]).all(), b
        else:
            assert t[b] >= 0 and not np.isnan(p[b]) and not np.isnan(d[b]).any(), b
    # every logit banned
    t, p, _ = _run(np.zeros(4, np.float32), _settings(), banned=[0, 1, 2, 3], u=[0.5])
    assert t[0] == -1 and np.isnan(p[0])


def test_argument_errors():
    import torch
    from exllama_b200 import capi
    lib = capi.lib()
    vocab = 1000
    logits = torch.zeros((64, 128256), device="cuda")
    u = torch.full((64,), 0.5, device="cuda")
    tok = torch.empty(64, dtype=torch.int64, device="cuda")
    prob = torch.empty(64, device="cuda")
    hist = torch.zeros((64, 8), dtype=torch.int64, device="cuda")

    def call(bsz=1, vocab=vocab, ld=vocab, lens=None, out=True, **kw):
        p = capi.ExlSampleParams(1.0, 0, 0.0, 0.0, 0.0, 1.0, -1, 0, -1, None, 0)
        for k, v in kw.items():
            setattr(p, k, v)
        hl = (C.c_int * 64)(*(lens or [8] * 64))
        return lib.exl_sample(capi._ptr(logits), bsz, vocab, ld, capi._ptr(hist), 8, hl, C.byref(p), capi._ptr(u),
                              capi._ptr(tok) if out else None, capi._ptr(prob), None, capi._stream())

    assert call() == 0
    for kw, text in ((dict(bsz=0), b"bsz 0"), (dict(bsz=65), b"bsz 65"), (dict(vocab=0, ld=0), b"vocab 0"),
                     (dict(vocab=262145, ld=262145), b"vocab 262145"), (dict(ld=999), b"logits_ld 999"),
                     (dict(temperature=0.0), b"temperature"), (dict(temperature=float("inf")), b"temperature"),
                     (dict(temperature=float("nan")), b"temperature"), (dict(top_k=-1), b"top_k -1"), (dict(top_k=1001), b"top_k 1001"),
                     (dict(top_p=-0.1), b"top_p"), (dict(min_p=-0.1), b"min_p"), (dict(typical=-0.1), b"typical"),
                     (dict(rep_sustain=-2), b"rep_sustain -2"), (dict(rep_decay=-1), b"rep_decay -1"),
                     (dict(lens=[9] + [8] * 63), b"hist_len[0] 9"), (dict(lens=[-1] + [8] * 63), b"hist_len[0] -1"),
                     (dict(out=False), b"NULL")):
        assert call(**kw) == 1, kw                                      # EXL_ERR_ARG
        assert text in lib.exl_last_error(), (kw, lib.exl_last_error())
    assert call(bsz=64, vocab=128256, ld=128256, top_k=0) == 0
    torch.cuda.synchronize()
    assert ((tok >= 0) & (tok < 128256)).all()


# ---- integration ------------------------------------------------------------------------------------------------------------------

def _check_against_oracle(logits_t, s, rng):
    """sampling.sample on device logits [bsz, vocab] against the oracle on their host copy, u at an oracle CDF midpoint per row."""
    import torch
    from exllama_b200 import sampling
    host = logits_t.cpu().numpy()
    us, want = [], []
    for row in host:
        r = S.sample(row, s.temperature, s.top_k, s.top_p, s.min_p, s.typical)
        assert S.min_margin(r) >= 1e-5
        u, toks, _ = _mid_u(r, rng, k=1)
        us.append(u[0]); want.append(toks[0])
    t, _ = sampling.sample(logits_t, s, u=torch.tensor(us, device=logits_t.device))
    assert t.cpu().tolist() == want


def test_fused_batch_step_then_sample(stacks):
    import torch
    st = stacks(vocab=32000, batch=3, seed=21)
    st.make_plan()
    g = torch.Generator(device="cuda"); g.manual_seed(22)
    x = (torch.randn((3, 1, 1024), device="cuda", generator=g) * 0.5).half()
    logits = st.decode_step_fused_batch(x, [5, 40, 130])
    _check_against_oracle(logits, _settings(temperature=0.3), np.random.default_rng(23))


def test_prefill_ragged_then_sample(stacks):
    import torch
    st = stacks(vocab=32000, batch=3, seed=31)
    g = torch.Generator(device="cuda"); g.manual_seed(32)
    q_lens = [7, 30, 61]
    x = (torch.randn((sum(q_lens), 1024), device="cuda", generator=g) * 0.5).half()
    logits = st.prefill_ragged(x, q_lens, [0, 12, 0])
    _check_against_oracle(logits, _settings(temperature=0.3), np.random.default_rng(33))


def test_default_rand_path_chi_square():
    """16384 draws through the default u = torch.rand(generator=...) path, against the oracle's probabilities."""
    import torch
    from scipy import stats
    from exllama_b200 import sampling
    vocab = 16
    logits = np.linspace(-2, 2, vocab).astype(np.float32)
    s = _settings(temperature=1.0)
    r = S.sample(logits, 1.0)
    lg = torch.as_tensor(np.repeat(logits[None], 64, 0)).cuda()
    gen = torch.Generator(device="cuda"); gen.manual_seed(1234)
    counts = np.zeros(vocab)
    for _ in range(256):
        t, _ = sampling.sample(lg, s, generator=gen)
        counts += np.bincount(t.cpu().numpy(), minlength=vocab)
    assert counts.sum() == 16384
    assert stats.chisquare(counts, r["probs"] * 16384).pvalue > 1e-3
