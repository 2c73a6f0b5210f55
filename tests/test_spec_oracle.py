"""CPU proof of the speculative-sampling oracle's law (oracle/spec_oracle.py): enumerating the acceptance uniform on both sides of
each draft's ratio p / q and u_k at the midpoint of every cell of the final draw, the first emitted token is distributed exactly
as the target's p_0, and the second, given that d_1 was accepted, exactly as p_1 -- whatever the draft's q.  Small vocabularies,
k 1 .. 3, several filter settings and a repetition-penalty history that the drafts extend."""
import numpy as np
import pytest

from oracle import sample_oracle as S
from oracle import spec_oracle as V

SETTINGS = {
    "plain": dict(temperature=1.0),
    "defaults": dict(temperature=0.95, top_k=10, top_p=0.65, penalty_max=1.15, sustain=4, decay=6),
    "top_p": dict(temperature=0.8, top_p=0.9, min_p=0.02),
    "typical": dict(temperature=1.3, typical=0.5, penalty_max=1.2, sustain=-1),
}


def _case(seed, vocab, k, kw, draft_kw):
    """Target logits [k + 1][vocab], draft logits, a history and the draft distributions q_j (of the draft's own rows)."""
    rng = np.random.default_rng(seed)
    target = np.stack([S.case_logits(seed * 10 + j, vocab, "normal", scale=1.5) for j in range(k + 1)])
    draft = target + rng.standard_normal(target.shape).astype(np.float32) * 1.5      # a related but different model
    history = rng.integers(0, vocab, size=12)
    q = [V.dense(S.sample(draft[j], **draft_kw), vocab) for j in range(k)]
    return target, q, history


def _law(target, drafts, q, kw, history, pos):
    """The exact law of the emitted token at position pos (0 or 1; at 1 with d_1 accepted) as {token: probability}, enumerating
    the acceptance uniform of position pos on both sides of p / q for every draft id in q's support, and u_k at the midpoint of
    every cell of the final draw, each branch weighted by its probability."""
    k = len(drafts)
    law = {}

    def run(ds, us, w):
        r = V.verify(target, ds, q, us, history=history, **kw)
        assert r["n_accepted"] >= pos, r
        if r["n_accepted"] > pos:                                   # d_{pos+1} accepted: it is the token at pos
            law[ds[pos]] = law.get(ds[pos], 0.0) + w
            return
        for _, lo, hi in r["cells"]:                                # the correction / bonus: every cell of the draw
            r2 = V.verify(target, ds, q, us[:k] + [(lo + hi) / 2], history=history, **kw)
            t = r2["tokens"][pos]
            law[t] = law.get(t, 0.0) + w * (hi - lo)

    if pos == k:                                                    # k == 1, pos 1: the bonus token after d_1
        run(list(drafts), [0.0] * k + [0.5], 1.0)
        return law
    p = V.dense(S.sample(target[pos], history=list(history) + list(drafts[:pos]), **kw), target.shape[1])
    for d in np.nonzero(q[pos] > 0)[0]:
        ds = list(drafts)
        ds[pos] = int(d)
        ratio = p[d] / q[pos][d]
        us = [0.0] * (k + 1)                                        # earlier drafts: u 0 accepts any draft p gives mass to
        if ratio >= 1.0:
            run(ds, us, q[pos][d])
            continue
        us[pos] = ratio * (1 - 1e-9)
        run(ds, list(us), q[pos][d] * ratio)
        us[pos] = ratio * (1 + 1e-9)
        run(ds, list(us), q[pos][d] * (1 - ratio))
    return law


@pytest.mark.parametrize("name", list(SETTINGS))
@pytest.mark.parametrize("vocab,k", [(8, 1), (16, 2), (32, 3)])
def test_first_token_law_is_p0(name, vocab, k):
    kw = SETTINGS[name]
    target, q, history = _case(vocab + k, vocab, k, kw, dict(temperature=1.0, top_k=vocab // 2))
    drafts = [int(np.argmax(qj)) for qj in q]
    law = _law(target, drafts, q, kw, history, 0)
    p0 = V.dense(S.sample(target[0], history=list(history), **kw), vocab)
    got = np.zeros(vocab)
    for t, w in law.items():
        got[t] += w
    np.testing.assert_allclose(got, p0, rtol=0, atol=1e-12)


@pytest.mark.parametrize("name", list(SETTINGS))
@pytest.mark.parametrize("vocab,k", [(8, 1), (16, 2), (32, 3)])
def test_second_token_law_given_acceptance_is_p1(name, vocab, k):
    kw = SETTINGS[name]
    target, q, history = _case(100 + vocab + k, vocab, k, kw, dict(temperature=0.7))
    p0 = V.dense(S.sample(target[0], history=list(history), **kw), vocab)
    d1 = int(np.argmax(p0 * (q[0] > 0)))                            # a first draft the target can accept
    drafts = [d1] + [int(np.argmax(qj)) for qj in q[1:]]
    law = _law(target, drafts, q, kw, history, 1)
    p1 = V.dense(S.sample(target[1], history=list(history) + [d1], **kw), vocab)
    got = np.zeros(vocab)
    for t, w in law.items():
        got[t] += w
    np.testing.assert_allclose(got, p1, rtol=0, atol=1e-12)


def test_greedy_reproduces_the_argmax_chain():
    """top_k 1 on both sides: the emitted tokens are the target's argmax after each accepted prefix."""
    rng = np.random.default_rng(4)
    for trial in range(40):
        vocab, k = int(rng.choice([8, 16, 32])), int(rng.integers(1, 4))
        target = np.stack([S.case_logits(1000 + trial * 7 + j, vocab, "normal") for j in range(k + 1)])
        am = [int(np.argmax(t)) for t in target]
        drafts = [am[j] if rng.random() < 0.6 else (am[j] + 1) % vocab for j in range(k)]
        q = [np.eye(vocab)[d] for d in drafts]
        r = V.verify(target, drafts, q, list(rng.random(k + 1)), temperature=1.0, top_k=1)
        a = next((j for j in range(k) if drafts[j] != am[j]), k)
        assert r["n_accepted"] == a
        assert r["tokens"][:a + 1] == am[:a + 1] and r["tokens"][a + 1:] == [-1] * (k - a)
        assert all(p == 1.0 for p in r["probs"][:a + 1])


def test_undefined_rows_and_margins():
    vocab = 8
    target = np.stack([S.case_logits(j, vocab, "normal") for j in range(3)])
    q = [np.full(vocab, 1.0 / vocab)] * 2
    ok = V.verify(target, [1, 2], q, [0.0, 0.0, 0.5], temperature=1.0)
    assert ok["n_accepted"] == 2 and len(ok["accept"]) == 2 and V.min_margin(ok) > 0
    for drafts, tgt, qq in (([vocab, 2], target, q), ([1, 2], target, [np.zeros(vocab)] + q[1:]),
                            ([1, 2], np.where(np.arange(3)[:, None] == 1, np.nan, target).astype(np.float32), q)):
        r = V.verify(tgt, drafts, qq, [0.0, 0.0, 0.5], temperature=1.0)
        assert r["n_accepted"] == -1 and r["tokens"] == [-1, -1, -1], drafts
    # a NaN row past the first rejection is never read
    bad = target.copy(); bad[2] = np.nan
    rej = V.verify(target, [1, 2], [np.eye(vocab)[1], q[1]], [0.999, 0.0, 0.3], temperature=1.0)
    assert rej["n_accepted"] == 0 and rej["residual"]
    assert V.verify(bad, [1, 2], [np.eye(vocab)[1], q[1]], [0.999, 0.0, 0.3], temperature=1.0)["tokens"] == rej["tokens"]
