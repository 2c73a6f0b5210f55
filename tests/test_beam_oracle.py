"""CPU checks of oracle/beam_oracle.py, the yardstick of exllama_b200.beam: it reproduces every case of tests/golden/beam_ref.npz (the
reference's own ExLlamaGenerator.beam_search on a stub model, oracle/gen_golden_beam.py) -- every emitted token and the beam windows
after every expansion -- and its selection and draw rules hold on planted cases."""
import math
import os

import numpy as np
import pytest

from oracle import beam_oracle as B

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "beam_ref.npz")
CASES = B.golden_cases(GOLDEN)


def test_golden_coverage():
    """The fixture spans beams 1-5, beam_length 1-6 and settings with top-k, top-p (with min-p), typical and the penalty."""
    assert {c["beams"] for c in CASES} == {1, 2, 3, 4, 5}
    assert {c["beam_length"] for c in CASES} == {1, 2, 3, 4, 5, 6}
    st = [c["settings"] for c in CASES]
    assert any(s["top_k"] > 0 for s in st) and any(s["top_p"] > 0 for s in st) and any(s["typical"] > 0 for s in st)
    assert any(s["min_p"] > 0 for s in st) and any(s["penalty_max"] != 1.0 for s in st)


@pytest.mark.parametrize("i", range(len(CASES)))
def test_reproduces_reference(i):
    c = CASES[i]
    r = B.run_case(c)
    assert r["emitted"] == c["emitted"]
    assert r["expansions"] == c["expansions"]
    assert B.min_margin(r) >= 1e-6


def test_expand_orders():
    """Candidates by score descending, then row, then token; the kept ones laid out by row, then score descending, then token.
    Planted exact ties: equal scores across rows go to the lower row, within a row to the lower token."""
    d = np.zeros((3, 8), np.float32)
    d[0, [1, 5]] = 0.5
    d[1, [2, 3]] = [0.25, 0.75]
    d[2, 7] = 1.0
    kept, m = B.expand(d, [0.0, math.log(2 / 3), -50.0], 3)
    # scores: row 0: log .5 (x2); row 1: log(2/3 * .75) = log .5, log(1/6); row 2: -50
    assert [(r, t) for r, t, _, _ in kept] == [(0, 1), (0, 5), (1, 3)]
    assert m == pytest.approx(math.log(0.5) - math.log(1 / 6))
    kept, _ = B.expand(d, [0.0, math.log(2 / 3), -50.0], 2)
    assert [(r, t) for r, t, _, _ in kept] == [(0, 1), (0, 5)]
    kept, m = B.expand(d, [0.0, 0.0, 0.0], 64)                   # fewer candidates than beams: every one, margin inf
    assert len(kept) == 5 and m == math.inf
    assert [(r, t) for r, t, _, _ in kept] == [(0, 1), (0, 5), (1, 3), (1, 2), (2, 7)]


def test_draw_without_replacement():
    """The first mode's draws: u = 0 takes the smallest id, each later draw is over the remaining mass, and the law of the first
    draw is p."""
    d = np.array([0.0, 0.5, 0.25, 0.0, 0.25], np.float32)
    assert B.draw_without_replacement(d, [0.0, 0.0, 0.0])[0] == [1, 2, 4]
    assert B.draw_without_replacement(d, [0.99, 0.99])[0] == [4, 2]
    assert B.draw_without_replacement(d, [0.6, 0.0, 0.0, 0.0])[0] == [2, 1, 4]    # four uniforms, three positive ids
    rng = np.random.default_rng(0)
    first = [B.draw_without_replacement(d, [u])[0][0] for u in rng.random(4000)]
    freq = np.bincount(first, minlength=5) / 4000
    assert np.abs(freq - d).max() < 0.03
