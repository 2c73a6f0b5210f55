"""CPU checks of the float64 sampling oracle (oracle/sample_oracle.py) against the reference's own ExLlamaGenerator.sample, whose
kept sets and final probabilities oracle/gen_golden_sample.py stored in tests/golden/sample_ref.npz."""
import os

import numpy as np
import pytest

from oracle import sample_oracle as S

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sample_ref.npz")


@pytest.fixture(scope="module")
def cases():
    return S.golden_cases(GOLD)


def test_oracle_reproduces_reference_cases(cases):
    assert len(cases) >= 100
    for i, c in enumerate(cases):
        r = S.run_case(c)
        assert r is not None, i
        np.testing.assert_array_equal(r["kept"], c["kept"], err_msg=f"case {i}")
        np.testing.assert_allclose(r["probs"], c["probs"], rtol=0, atol=1e-9, err_msg=f"case {i}")


def test_every_case_is_decided_with_margin(cases):
    for i, c in enumerate(cases):
        assert S.min_margin(S.run_case(c)) >= 1e-4, (i, S.run_case(c)["margins"])


def test_fixture_covers_the_settings(cases):
    """vocab 32000 / 32001 / 7 / 1, three temperatures, top_k 0 / 1 / 40 / vocab, each filter on, the generator's defaults,
    histories of 0 / 17 / 1920 tokens under each sustain / decay, bos, banned ids, dominant and flat logits."""
    seen = lambda f: {c[f] for c in cases}
    assert seen("vocab") == {32000, 32001, 7, 1}
    assert seen("temperature") == {0.3, 0.95, 1.7}
    assert {0, 1, 40}.issubset(seen("top_k")) and any(c["top_k"] == c["vocab"] for c in cases)
    assert any(c["top_p"] > 0 for c in cases) and any(c["min_p"] > 0 for c in cases) and any(c["typical"] > 0 for c in cases)
    assert any(c["top_p"] > 0 and c["typical"] > 0 for c in cases)
    assert any(c["top_k"] == 40 and abs(c["top_p"] - 0.65) < 1e-12 and c["penalty_max"] == 1.15 and (c["sustain"], c["decay"]) == (256, 128)
               for c in cases)
    assert {len(c["history"]) for c in cases} == {0, 17, 1920}
    assert {c["sustain"] for c in cases if len(c["history"])} == {-1, 0, 256}
    assert {c["decay"] for c in cases if len(c["history"])} == {0, 128}
    assert any(c["bos"] >= 0 for c in cases) and any(len(c["banned"]) for c in cases)
    assert seen("kind") == {"normal", "dominant", "flat"}


def test_oracle_draw_and_undefined_rows():
    r = S.sample(np.array([0.0, 1.0, 2.0], np.float32), 1.0, u=0.0)
    assert r["token"] == 0
    assert S.sample(np.array([0.0, 1.0, 2.0], np.float32), 1.0, u=0.9999999)["token"] == 2
    assert S.sample(np.array([0.0, 1.0], np.float32), 1.0, banned=[0, 1]) is None
    assert S.sample(np.array([0.0, np.nan], np.float32), 1.0) is None
    assert S.sample(np.array([0.0, 1.0], np.float32), 1.0, history=[5], penalty_max=1.2) is None
