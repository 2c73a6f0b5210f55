"""Speculative sampling on the GPU (exl_spec_verify, exllama_b200.speculative): against the float64 oracle (oracle/spec_oracle.py) on a
seeded sweep; q = p accepts every draft and returns exl_sample's bonus draw; the law of the first and second emitted tokens by
chi-square; greedy on both sides is the argmax chain; undefined rows, rows past the first rejection never read, argument errors,
determinism and graph replay; and SpeculativeGenerator end to end on the synthetic stacks of tests/stack_harness.py."""
import ctypes as C
import warnings

import numpy as np
import pytest

from helpers import assert_close_ref64
from oracle import sample_oracle as S
from oracle import spec_oracle as V
from stack_harness import lib_state, restore, snapshot, stacks  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

TOL = 1e-5              # cases the oracle decides with a smaller margin (acceptance, draw, filters) are not compared


def _settings(temperature=1.0, top_k=0, top_p=0.0, min_p=0.0, typical=0.0, penalty_max=1.0, sustain=-1, decay=0):
    from exllama_b200 import sampling
    s = sampling.Settings()
    s.temperature, s.top_k, s.top_p, s.min_p, s.typical = temperature, top_k, top_p, min_p, typical
    s.token_repetition_penalty_max, s.token_repetition_penalty_sustain, s.token_repetition_penalty_decay = penalty_max, sustain, decay
    return s


SETTINGS = {
    "defaults_hist1920": (dict(temperature=0.95, top_k=40, top_p=0.65, penalty_max=1.15, sustain=256, decay=128), 1920),
    "topk0_topp0.9": (dict(temperature=0.95, top_p=0.9), 0),
    "typical0.2": (dict(temperature=0.95, top_k=0, typical=0.2), 0),
    "greedy": (dict(temperature=0.95, top_k=1), 0),
}


def _kw(s):
    return dict(temperature=s.temperature, top_k=s.top_k, top_p=s.top_p, min_p=s.min_p, typical=s.typical,
                penalty_max=s.token_repetition_penalty_max, sustain=s.token_repetition_penalty_sustain,
                decay=s.token_repetition_penalty_decay)


def _cuda(x, dtype=None):
    import torch
    return torch.as_tensor(np.asarray(x), dtype=dtype).cuda()


def _drafts(draft_logits, s, u):
    """Draft tokens and their distributions: sampling.sample(..., dist=) of the draft's logits [k, vocab]."""
    import torch
    from exllama_b200 import sampling
    lg = _cuda(draft_logits, torch.float32)
    q = torch.empty_like(lg)
    d, _ = sampling.sample(lg, s, u=_cuda(u, torch.float32), dist=q)
    return d, q


def _verify(target, d, q, s, history=None, u=None, **kw):
    """speculative.verify on numpy / torch inputs; returns (n_accepted, tokens, probs) as host values."""
    import torch
    from exllama_b200 import speculative
    h = None if history is None else _cuda(history, torch.int64)
    n, t, p = speculative.verify(_cuda(target, torch.float32), d, q, s, history=h, u=_cuda(u, torch.float32), **kw)
    torch.cuda.synchronize()
    return int(n.item()), t.cpu().tolist(), p.cpu().numpy()


# ---- the verification call ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", [1, 2, 3, 7])
@pytest.mark.parametrize("name", list(SETTINGS))
def test_against_oracle(name, k):
    """normal / dominant / flat logits, up to three seeded cases each: n_accepted, tokens and probabilities equal the oracle's wherever it
    decides with a margin of at least TOL.  Drafts come from a second logits set near the target's, so that the cases accept,
    reject and draw corrections."""
    kw, hl = SETTINGS[name]
    s = _settings(**kw)
    vocab = 32000
    ran, seen = 0, set()
    for kind in S.KINDS:
        ran_kind = 0
        for seed in range(20):
            if ran_kind == 3:
                break
            rng = np.random.default_rng(1000 * k + 100 * seed + S.KINDS.index(kind))
            target = np.stack([S.case_logits(int(rng.integers(1 << 30)), vocab, kind) for _ in range(k + 1)])
            noise = 0.01 if kind == "flat" else (0.05 if seed % 2 == 0 else 0.7)
            draft = (target[:k] + rng.standard_normal((k, vocab)) * noise).astype(np.float32)
            history = rng.integers(0, vocab, size=hl) if hl else None
            d, q = _drafts(draft, s, rng.random(k))
            u = rng.random(k + 1).astype(np.float32)
            if seed % 2 == 0:
                u[:k] *= 0.05                                          # mostly accepting
            r = V.verify(target, d.cpu().numpy(), q.cpu().numpy().astype(np.float64), u.astype(np.float64), history=history, **_kw(s))
            if V.min_margin(r) < TOL:
                continue
            n, toks, probs = _verify(target, d, q, s, history=history, u=u)
            what = f"{name} k {k} {kind} seed {seed}"
            assert n == r["n_accepted"], (what, n, r["n_accepted"])
            assert toks == r["tokens"], (what, toks, r["tokens"])
            np.testing.assert_allclose(probs, np.asarray(r["probs"], np.float64), rtol=1e-5, atol=1e-7, err_msg=what)
            ran += 1
            ran_kind += 1
            seen.add((n == k, r["residual"]))
    # top_p 0.9 over 32000 normal logits cuts among tokens of ~1e-6: only dominant and flat rows clear TOL there
    assert ran >= 3, ran
    if k <= 3 and name in ("defaults_hist1920", "typical0.2"):    # top_p's dominant and flat cases clear TOL when every draft is accepted
        assert len(seen) >= 2, seen                                   # both all-accepted and rejected cases were compared


@pytest.mark.parametrize("k", [1, 3, 7])
def test_q_equals_p_accepts_everything(k):
    """Each draft drawn by exl_sample from the target's own row (history followed by the drafts before it) and its dist row passed as
    q: every draft is accepted, each probability is bitwise that row's dist value, and the bonus is exl_sample's draw of row k
    with u_k."""
    import torch
    from exllama_b200 import sampling
    rng = np.random.default_rng(k)
    vocab, H = 32000, 1920
    s = sampling.Settings()
    target = _cuda(np.stack([S.case_logits(50 + j, vocab, "normal") for j in range(k + 1)]), torch.float32)
    hist = torch.zeros(H + k, dtype=torch.int64, device="cuda")
    hist[:H] = _cuda(rng.integers(0, vocab, size=H))
    P = torch.empty((k + 1, vocab), device="cuda")
    w = _cuda(rng.random(k + 1).astype(np.float32))
    u = _cuda(rng.random(k + 1).astype(np.float32))
    for j in range(k + 1):
        t, _ = sampling.sample(target[j:j + 1], s, history=hist.view(1, -1), hist_lens=[H + j], u=(u if j == k else w)[j:j + 1],
                               dist=P[j:j + 1])
        if j < k:
            hist[H + j:H + j + 1] = t
    bonus = t
    from exllama_b200 import speculative
    n, toks, probs = speculative.verify(target, hist[H:H + k], P[:k], s, history=hist, hist_len=H, u=u)
    torch.cuda.synchronize()
    d = hist[H:H + k]
    assert int(n.item()) == k
    assert toks.tolist() == d.tolist() + [int(bonus.item())]
    want = torch.cat([P[torch.arange(k, device="cuda"), d], P[k, bonus]])
    assert torch.equal(probs, want)


def test_law_by_chi_square():
    """Vocab 64, 20000 verifications with fixed seeds, k 2, drafts drawn from a sharper distribution than the target's: the first emitted
    token follows p_0 and the second, when d_1 was accepted, p_1 (p-value >= 1e-3 each).  Accepting a draft with probability
    p(d) instead of min(1, p(d) / q(d)) -- the same uniforms, the correction drawn from p -- fails the first test, so the test has
    power.  (Accepting a draft iff it equals the target's own independent draw, and emitting that draw otherwise, always emits the
    target's draw: it has the right law and only a lower acceptance rate.)"""
    import torch
    from scipy import stats
    from exllama_b200 import sampling, speculative
    vocab, k, N = 64, 2, 20000
    s = _settings(temperature=1.0, top_p=0.95)
    target = np.stack([S.case_logits(7 + j, vocab, "normal", scale=1.5) for j in range(k + 1)])
    draft = target[:k] * 2.0                                       # sharper than the target: q concentrates where p is largest
    p = [V.dense(S.sample(target[j], **_kw(s)), vocab) for j in range(k + 1)]
    tg, dl = _cuda(target, torch.float32), _cuda(draft, torch.float32)
    gen = torch.Generator(device="cuda"); gen.manual_seed(11)
    q = torch.empty((k, vocab), device="cuda")
    first = torch.empty(N, dtype=torch.int64, device="cuda")
    second = torch.empty(N, dtype=torch.int64, device="cuda")
    acc = torch.empty(N, dtype=torch.int32, device="cuda")
    us = torch.empty((N, k + 1), device="cuda")
    d1 = torch.empty(N, dtype=torch.int64, device="cuda")
    for i in range(N):
        d, _ = sampling.sample(dl, s, generator=gen, dist=q)
        u = torch.rand(k + 1, device="cuda", generator=gen)
        n, toks, _ = speculative.verify(tg, d, q, s, u=u)
        first[i:i + 1], second[i:i + 1], acc[i:i + 1], us[i], d1[i:i + 1] = toks[0:1], toks[1:2], n, u, d[0:1]
    first, second, acc = first.cpu().numpy(), second.cpu().numpy(), acc.cpu().numpy()
    assert (acc >= 0).all() and (acc > 0).sum() > 2000 and (acc == 0).sum() > 2000, np.bincount(acc)

    def pvalue(samples, probs):
        """Chi-square over the ids with mass; ids expected fewer than 5 times are pooled into one bin."""
        c = np.bincount(samples, minlength=vocab).astype(np.float64)
        e = probs * len(samples)
        assert c[probs == 0].sum() == 0
        big, small = e >= 5, (probs > 0) & (e < 5)
        obs, exp = list(c[big]), list(e[big])
        if small.any():
            obs.append(c[small].sum()); exp.append(e[small].sum())
        return stats.chisquare(obs, exp).pvalue

    assert pvalue(first, p[0]) >= 1e-3
    assert pvalue(second[acc >= 1], p[1]) >= 1e-3
    # the naive acceptance u < p(d) on the same uniforms and drafts
    qh = V.dense(S.sample(draft[0], **_kw(s)), vocab)
    assert np.allclose(q[0].cpu().numpy(), qh, atol=1e-6)
    us, d1 = us.cpu().numpy().astype(np.float64), d1.cpu().numpy()
    naive = np.array([d if uu[0] < p[0][d] else V.draw(p[0], uu[k])[0] for d, uu in zip(d1, us)])
    assert pvalue(naive, p[0]) < 1e-3


def test_greedy_is_the_argmax_chain():
    """top_k 1 on both sides, k 3: the emitted tokens are the target's argmax after each accepted prefix."""
    import torch
    rng = np.random.default_rng(8)
    vocab, k = 32000, 3
    s = _settings(top_k=1)
    for trial in range(12):
        target = np.stack([S.case_logits(300 + 4 * trial + j, vocab, "normal") for j in range(k + 1)])
        am = target.argmax(1).tolist()
        draft = target[:k].copy()
        a = trial % (k + 1)
        if a < k:
            draft[a, am[a]] -= 100.0                                 # the first a drafts agree, d_{a+1} does not
        d, q = _drafts(draft, s, rng.random(k))
        n, toks, probs = _verify(target, d, q, s, u=rng.random(k + 1))
        assert n == a and toks == am[:a + 1] + [-1] * (k - a), (trial, n, toks, am)
        assert (probs[:a + 1] == 1.0).all()


def test_undefined_rows_and_unread_rows():
    import torch
    rng = np.random.default_rng(9)
    vocab, k = 1000, 3
    s = _settings(temperature=0.9, top_k=50)
    target = np.stack([S.case_logits(90 + j, vocab, "normal") for j in range(k + 1)])
    d, q = _drafts(target[:k], s, rng.random(k))
    u = np.array([0.0, 0.0, 0.0, 0.5], np.float32)                  # u 0 accepts every draft the target gives mass to
    n, toks, _ = _verify(target, d, q, s, u=u)
    assert n == k, toks

    def undefined(tg=target, dd=d, qq=q):
        n, toks, probs = _verify(tg, dd, qq, s, u=u)
        return n == -1 and toks == [-1] * (k + 1) and np.isnan(probs).all()

    nan_row = target.copy(); nan_row[2, 17] = np.nan
    assert undefined(tg=nan_row)                                     # p_2 undefined, reached after d_1, d_2
    nan_last = target.copy(); nan_last[k, 3] = np.nan
    assert undefined(tg=nan_last)                                    # p_k, the bonus row
    for bad in (-1, vocab):
        dd = d.clone(); dd[1] = bad
        assert undefined(dd=dd)
    qq = q.clone(); qq[1, d[1]] = 0.0
    assert undefined(qq=qq)
    qq = q.clone(); qq[0, d[0]] = float("inf")
    assert undefined(qq=qq)
    # reject d_2 (q far above p at d_2, u just under 1): rows 2 .. k are never read, NaN there changes nothing
    qq = q.clone(); qq[1] = 0.0; qq[1, d[1]] = 1.0
    u2 = np.array([0.0, 0.9999, 0.0, 0.37], np.float32)
    ref = _verify(target, d, qq, s, u=u2)
    assert ref[0] == 1, ref
    rest = target.copy(); rest[2:] = np.nan
    got = _verify(rest, d, qq, s, u=u2)
    assert got[0] == ref[0] and got[1] == ref[1] and got[2].tobytes() == ref[2].tobytes()
    # a draft id the walk never reaches is not checked
    dd = d.clone(); dd[2] = vocab
    assert _verify(target, dd, qq, s, u=u2)[1] == ref[1]


def _bytes(t):
    return t.cpu().numpy().tobytes()


def test_two_calls_bitwise_and_graph_replay():
    import torch
    from exllama_b200 import sampling, speculative
    rng = np.random.default_rng(2)
    vocab, k = 32000, 3
    s = sampling.Settings()
    target = _cuda(np.stack([S.case_logits(20 + j, vocab, "normal") for j in range(k + 1)]), torch.float32)
    d, q = _drafts((target[:k].cpu().numpy() + rng.standard_normal((k, vocab)) * 0.5).astype(np.float32), s, rng.random(k))
    hist = _cuda(rng.integers(0, vocab, size=1920))
    for u in (_cuda(rng.random(k + 1).astype(np.float32)), _cuda(np.array([0, 0, 0, 0.3], np.float32))):
        a = speculative.verify(target, d, q, s, history=hist, u=u, bos_token_id=1)
        b = speculative.verify(target, d, q, s, history=hist, u=u, bos_token_id=1)
        torch.cuda.synchronize()
        assert all(_bytes(x) == _bytes(y) for x, y in zip(a, b))       # probs past the emitted tokens are NaN
        side = torch.cuda.Stream(); side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            speculative.verify(target, d, q, s, history=hist, u=u, bos_token_id=1)
        torch.cuda.current_stream().wait_stream(side); torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            c = speculative.verify(target, d, q, s, history=hist, u=u, bos_token_id=1)
        for t in c:
            t.fill_(-3)
        g.replay()
        torch.cuda.synchronize()
        assert all(_bytes(x) == _bytes(y) for x, y in zip(a, c))


def test_argument_errors():
    import torch
    from exllama_b200 import capi
    lib = capi.lib()
    vocab = 1000
    logits = torch.zeros((64, vocab), device="cuda")
    drafts = torch.zeros(64, dtype=torch.int64, device="cuda")
    dist = torch.full((64, vocab), 1.0 / vocab, device="cuda")
    u = torch.full((64,), 0.5, device="cuda")
    work = torch.empty((64, vocab), device="cuda")
    n_acc = torch.empty(1, dtype=torch.int32, device="cuda")
    tok = torch.empty(64, dtype=torch.int64, device="cuda")
    prob = torch.empty(64, device="cuda")
    hist = torch.zeros(8, dtype=torch.int64, device="cuda")
    P = capi._ptr

    def call(k=2, vocab=vocab, ld=vocab, dist_ld=vocab, hl=8, null=None, **kw):
        p = capi.ExlSampleParams(1.0, 0, 0.0, 0.0, 0.0, 1.1, -1, 0, -1, None, 0)
        for key, v in kw.items():
            setattr(p, key, v)
        args = dict(logits=P(logits), drafts=P(drafts), dist=P(dist), hist=P(hist), u=P(u), work=P(work), n_acc=P(n_acc), tok=P(tok),
                    prob=P(prob))
        if null:
            args[null] = None
        return lib.exl_spec_verify(args["logits"], k, vocab, ld, args["drafts"], args["dist"], dist_ld, args["hist"], hl, C.byref(p),
                                   args["u"], args["work"], args["n_acc"], args["tok"], args["prob"], capi._stream())

    assert call() == 0 and call(k=63) == 0 and call(null="hist") == 0
    cases = [(dict(k=0), b"k 0"), (dict(k=64), b"k 64"), (dict(dist_ld=999), b"dist_ld 999"), (dict(ld=999), b"logits_ld 999"),
             (dict(vocab=0, ld=0, dist_ld=0), b"vocab 0"), (dict(hl=-1), b"hist_len[0] -1"), (dict(temperature=0.0), b"temperature"),
             (dict(top_k=-1), b"top_k -1"), (dict(top_p=-0.1), b"top_p"), (dict(min_p=-0.1), b"min_p"), (dict(typical=-0.1), b"typical"),
             (dict(rep_sustain=-2), b"rep_sustain -2"), (dict(rep_decay=-1), b"rep_decay -1"), (dict(n_banned=2), b"n_banned 2")]
    cases += [(dict(null=name), b"NULL") for name in ("logits", "drafts", "dist", "u", "work", "n_acc", "tok", "prob")]
    for kw, text in cases:
        assert call(**kw) == 1, kw                                      # EXL_ERR_ARG
        assert text in lib.exl_last_error(), (kw, lib.exl_last_error())
    assert lib.exl_spec_verify(P(logits), 2, vocab, vocab, P(drafts), P(dist), vocab, None, 0, None, P(u), P(work), P(n_acc), P(tok),
                               P(prob), capi._stream()) == 1 and b"params is NULL" in lib.exl_last_error()
    torch.cuda.synchronize()


# ---- SpeculativeGenerator on synthetic stacks -------------------------------------------------------------------------------------

C_EMB = 25.0            # tied embeddings x = c * lm_head[token], as test_gpu_decode_multi's greedy loop: rows of rms ~ 0.5
PROMPT = [5, 17, 300, 1029, 44, 2000, 7, 7, 123, 999]


def _embed(st):
    return (st.lm_head.float() * C_EMB).half().contiguous()


def _greedy_reference(st, emb, n):
    """Single-step greedy decoding after a prefill of PROMPT on the one-token fused plan: the tokens and, per token, the top-2 logit
    gap over the logits' rms (the prompt's first token from the prefill, gap included).  The caches are restored afterwards."""
    import torch
    snap = snapshot(st)
    ids = torch.tensor(PROMPT, device="cuda")
    lg = st.prefill(emb[ids].view(1, len(PROMPT), -1), 0)[0].double()
    toks, gaps = [], []
    st.make_plan()
    for i in range(n):
        top = torch.topk(lg, 2).values
        gaps.append(float(top[0] - top[1]) / float(lg.pow(2).mean().sqrt()))
        toks.append(int(lg.argmax()))
        if i + 1 < n:
            lg = st.decode_step_fused(emb[toks[-1]].view(1, 1, -1), len(PROMPT) + i)[0].double()
    st.dplan.close(); st.dplan = None
    restore(st, snap)
    return toks, gaps


@pytest.mark.parametrize("negate", [False, True], ids=["same_draft", "negated_head"])
def test_greedy_generation(stacks, negate):
    """top_k 1, k 3.  A draft identical to the target (same seed) accepts all k drafts every round, so every round after the first
    starts with the two-token catch-up launch; a draft whose lm_head is negated has its first draft rejected every round.  Either
    way the tokens are single-step greedy decoding, up to the first position where its top-2 gap is within tolerance."""
    from exllama_b200.speculative import SpeculativeGenerator
    target = stacks(kv_heads=2, seed=61)
    draft = stacks(kv_heads=2, seed=61)
    if negate:
        draft.lm_head.neg_()
    emb = _embed(target)
    n = 60
    ref, gaps = _greedy_reference(target, emb, n)
    s = _settings(top_k=1)
    gen = SpeculativeGenerator(target, draft, emb, emb, k=3, settings=s)
    out = [gen.begin(PROMPT)]
    toks, accepted = gen.generate(n - 1)
    out += toks
    first_close = next((i for i, g in enumerate(gaps) if g < 5e-3), n)
    m = min(first_close, n)
    assert m >= 16, first_close
    assert out[:m] == ref[:m], (out[:m], ref[:m])
    emitted = 1
    for a in accepted:
        if emitted + a + 1 > m:
            break
        assert a == (0 if negate else 3), accepted
        emitted += a + 1
    assert emitted >= 12, (emitted, accepted)


def test_stochastic_generation_leaves_clean_caches(stacks):
    """Generator defaults (repetition penalty included) for the target, k 3, a one-layer draft: after 15 rounds every K/V row of both caches below the final
    past_len equals a fresh prefill of prompt + emitted tokens into cache sequence 1, within the multi-token step's tolerances, so no
    rejected row survives there.  Each round synchronises with the host once."""
    import torch
    from exllama_b200 import sampling
    from exllama_b200.speculative import SpeculativeGenerator
    target = stacks(kv_heads=2, batch=2, seed=71)
    draft = stacks(kv_heads=2, layers=1, batch=2, seed=71)        # the target's first layer (same seed) ...
    draft.norm, draft.lm_head = target.norm, target.lm_head          # ... and its head: an early exit of the target
    emb = _embed(target)
    g = torch.Generator(device="cuda"); g.manual_seed(72)
    # the synthetic early exit predicts the target's top token every time; drafting uniformly from its top two rejects about half
    gen = SpeculativeGenerator(target, draft, emb, emb, k=3, settings=sampling.Settings(), draft_settings=_settings(temperature=50.0, top_k=2),
                               generator=g)
    gen.begin(PROMPT)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            accepted = [gen.round() for _ in range(15)]
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = [x for x in w if "called a synchronizing CUDA operation" in str(x.message)]
    assert len(syncs) == len(accepted), [str(x.message) for x in syncs[:3]]
    toks = gen.hist[:gen.n].tolist()
    assert len(toks) == len(PROMPT) + 1 + sum(a + 1 for a in accepted) and min(toks) >= 0
    assert 0 < sum(accepted) < 3 * len(accepted), accepted          # some drafts accepted, some rejected
    for st, past in ((target, gen.n - 1), (draft, gen.n - 2 if gen.catch_up else gen.n - 1)):
        snap = snapshot(st)
        ids = torch.tensor(toks[:past], device="cuda")
        st.prefill(emb[ids].view(1, past, -1), 0, seq=1)
        for i, (kc, vc) in enumerate(zip(st.key_cache, st.value_cache)):
            for name, c in (("k", kc), ("v", vc)):
                got, want = c[0, :, :past].float().cpu().numpy(), c[1, :, :past].float().cpu().numpy()
                for r in range(past):
                    assert_close_ref64(got[:, r], want[:, r].astype(np.float64), rel=1e-2, rms=1e-2,
                                       what=f"{'draft' if st is draft else 'target'} layer {i} {name} row {r} of {past}")
        restore(st, snap)


def test_plan_errors(stacks):
    from exllama_b200.shapes import GQA_SHAPES
    from exllama_b200.speculative import SpeculativeGenerator
    st = stacks(kv_heads=2, seed=1)
    emb = _embed(st)
    with pytest.raises(ValueError, match=r"cannot take k \+ 1 = 5 tokens"):
        SpeculativeGenerator(st, st, emb, emb, k=4)
    big = stacks(GQA_SHAPES["70b"], layers=1, max_seq=64, seed=4)
    big_emb = _embed(big)
    with pytest.raises(ValueError, match=r"cannot take k \+ 1 = 2 tokens.*the largest is 1"):
        SpeculativeGenerator(big, big, big_emb, big_emb, k=1)
