"""CPU checks of oracle/toplp_oracle.py, the yardstick of exl_top_logprobs: its log-probabilities against scipy's float64
log_softmax, its order (ties to the lower id, -0 and +0 one value, the logit itself rather than exp(x - m)), undefined rows (NaN,
+inf, all -inf), rows with fewer finite entries than N, and tokens outside the vocabulary; and that its bound admits an fp32
rounding of the float64 result."""
import numpy as np
import pytest
from scipy.special import log_softmax

from oracle import toplp_oracle as T


@pytest.mark.parametrize("vocab,n", [(7, 5), (7, 20), (1000, 1), (32000, 20), (128256, 5)])
def test_against_scipy(vocab, n):
    rng = np.random.default_rng(vocab + n)
    x = (rng.standard_normal(vocab) * 4).astype(np.float32)
    x[rng.integers(0, vocab, max(1, vocab // 50))] = -np.inf
    ref = log_softmax(np.where(np.isfinite(x), x.astype(np.float64), -np.inf))
    tok = int(rng.integers(0, vocab))
    r = T.top_logprobs(x, n, tok)
    assert r["lp"] == pytest.approx(ref[tok], rel=1e-12, abs=1e-12) or (np.isinf(ref[tok]) and r["lp"] == ref[tok])
    fin = np.flatnonzero(np.isfinite(x))
    want = fin[np.lexsort((fin, -x[fin]))][:n]
    assert r["ids"][:len(want)].tolist() == want.tolist()
    np.testing.assert_allclose(r["top"][:len(want)], ref[want], rtol=1e-12, atol=1e-12)
    # the fp32 rounding of the float64 value is inside the bound
    assert T.within(r["top"].astype(np.float32), r["top"], r["bound"])
    assert T.within(np.float32(r["lp"]), r["lp"], r["lp_bound"])


def test_ties_and_signed_zero():
    x = np.array([1.0, 3.0, -0.0, 3.0, 0.0, -2.0, 0.0, 3.0], np.float32)
    r = T.top_logprobs(x, 8)
    assert r["ids"].tolist() == [1, 3, 7, 0, 2, 4, 6, 5]
    assert r["top"][0] == r["top"][1] == r["top"][2] and r["top"][4] == r["top"][5] == r["top"][6]


def test_order_is_on_the_logit_not_its_exp():
    """Logits 200 apart: exp(x - m) underflows to 0 for all but the first in float64, yet the order stays strict."""
    x = np.array([0.0, -1000.0, -1200.0, -1100.0, -1000.5], np.float32)
    r = T.top_logprobs(x, 5)
    assert r["ids"].tolist() == [0, 1, 4, 3, 2]
    assert np.all(np.diff(r["top"]) < 0)


def test_fewer_finite_than_n():
    x = np.full(10, -np.inf, np.float32)
    x[[3, 8]] = [0.5, 2.0]
    r = T.top_logprobs(x, 5, 3)
    assert r["ids"].tolist() == [8, 3, -1, -1, -1]
    assert np.all(np.isneginf(r["top"][2:])) and np.isfinite(r["top"][:2]).all()
    assert r["lp"] == pytest.approx(0.5 - np.log(np.exp(0.5) + np.exp(2.0)))
    assert T.top_logprobs(x, 1, 0)["lp"] == -np.inf                       # a -inf logit's token


@pytest.mark.parametrize("bad", ["nan", "posinf", "allneginf"])
def test_undefined_rows(bad):
    x = np.zeros(16, np.float32)
    if bad == "nan":
        x[4] = np.nan
    elif bad == "posinf":
        x[9] = np.inf
    else:
        x[:] = -np.inf
    r = T.top_logprobs(x, 3, 2)
    assert np.isnan(r["lp"]) and r["ids"].tolist() == [-1, -1, -1] and np.isnan(r["top"]).all()


@pytest.mark.parametrize("tok", [-1, 16, 1 << 40, None])
def test_token_outside_the_vocabulary(tok):
    r = T.top_logprobs(np.zeros(16, np.float32), 2, tok)
    assert np.isnan(r["lp"]) and r["ids"].tolist() == [0, 1]


def test_within_rejects_an_ulp_too_far():
    x = np.linspace(-3, 3, 50).astype(np.float32)
    r = T.top_logprobs(x, 4)
    got = r["top"].astype(np.float32)
    assert T.within(got, r["top"], r["bound"])
    off = got.copy()
    off[1] = np.nextafter(np.nextafter(off[1], np.float32(-np.inf)), np.float32(-np.inf))
    assert not T.within(off, r["top"], r["bound"])
    assert not T.within(np.array([-1.0, np.nan]), np.array([-1.0, -np.inf]), np.zeros(2))
