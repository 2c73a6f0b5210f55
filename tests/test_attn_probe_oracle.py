"""The attention probe's construction (tests/helpers.py, "Attention probe") checked with the float64 oracle alone, so that a
failure of tests/test_gpu_decode_attn_probe.py points at a kernel, not at the harness."""
import numpy as np
import pytest

from helpers import (PROBE_GAP, cpu_probe_stack as _cpu_stack, dense_positions, identity_q4, plant_group, plant_probe,
                     probe_expectation, scaled_q_as_k, single_positions, snap_of, synth_q4_ckpt)
from stack_harness import sincos


@pytest.mark.parametrize("act", [False, True])
def test_identity_q4_contracts_to_x(oracle, act):
    """The identity o_proj gives x exactly, in the original row order and through make_q4's act-order reordering."""
    n = 1024
    x = (np.random.default_rng(1).standard_normal((1, n)) * 3).astype(np.float16)
    qw, qz, sc, g = identity_q4(n, act, seed=2)
    assert (g is not None) == act
    np.testing.assert_array_equal(oracle.ref64_with_act_order(x, qw, qz, sc, g), x.astype(np.float64))
    np.testing.assert_array_equal(oracle.dequant_f64(qw, qz, sc), np.eye(n))


@pytest.mark.parametrize("heads,kv", [(8, 8), (8, 2), (16, 2)])
def test_scaled_q_as_k_is_gamma_q_through_rope(oracle, heads, kv):
    """k tensors = the q columns of each group's first query head, scales x gamma: k_new = gamma q bit for bit after fp16
    rounding and rope (gamma a power of two)."""
    hd, hidden, gamma, past = 128, 1024, 64.0, 777
    qw, qz, sc, _ = synth_q4_ckpt(hidden, heads * hd, 128, seed=heads + kv)
    kw, kz, ks = scaled_q_as_k(qw, qz, sc, heads, kv, gamma)
    xn = np.random.default_rng(3).standard_normal((1, hidden)).astype(np.float16)
    sin, cos = sincos(1024, hd)
    q = oracle.q4_matmul_f64(xn, qw, qz, sc).astype(np.float16)
    k = oracle.q4_matmul_f64(xn, kw, kz, ks).astype(np.float16)
    q = oracle.rope(q.reshape(1, heads, hd), sin, cos, 1, heads, hd, heads, past).reshape(heads, hd)
    k = oracle.rope(k.reshape(1, kv, hd), sin, cos, 1, kv, hd, kv, past).reshape(kv, hd)
    want = (q[::heads // kv].astype(np.float64) * gamma).astype(np.float16)
    np.testing.assert_array_equal(k.view(np.uint16), want.view(np.uint16))


@pytest.mark.parametrize("n_rep", [1, 4])
@pytest.mark.parametrize("past", [1, 16, 300, 2046])
@pytest.mark.parametrize("layout", ["dense", "single"])
def test_planted_cache_answer_is_plateau_mean(oracle, n_rep, past, layout):
    """On a planted cache, decode_attn_f64 gives each planted head the mean of V over its plateau, to within the margin term;
    the poison row (overwritten by the new token) and the NaN rows past it are never read."""
    hd, max_seq, kv = 128, 2048, 2
    heads = kv * n_rep
    rng = np.random.default_rng(past + n_rep)
    q = (0.4 * rng.standard_normal((heads, hd))).astype(np.float16)
    kc = (0.5 * rng.standard_normal((kv, max_seq, hd))).astype(np.float16)
    vc = (0.5 * rng.standard_normal((kv, max_seq, hd))).astype(np.float16)
    k_new = (0.4 * rng.standard_normal((kv, hd))).astype(np.float16)
    v_new = (0.5 * rng.standard_normal((kv, hd))).astype(np.float16)
    sp = single_positions(past)
    plants = [dense_positions(past, h % n_rep, n_rep) if layout == "dense" else [sp[h % n_rep]] if h % n_rep < len(sp) else None
              for h in range(heads)]
    for g in range(kv):
        qg = q[g * n_rep:(g + 1) * n_rep]
        s_new = qg.astype(np.float64) @ k_new[g].astype(np.float64) / np.sqrt(hd)
        plant_group(qg, kc[g], vc[g], plants[g * n_rep:(g + 1) * n_rep], past, s_new, rng)
    assert np.isnan(kc[:, past + 1:]).all() and np.abs(vc[:, past]).max() == 100
    kc[:, past] = k_new; vc[:, past] = v_new
    got = oracle.decode_attn_f64(q.reshape(-1), kc, vc, heads, kv, hd, past + 1, max_seq).reshape(heads, hd)
    for h in range(heads):
        g = h // n_rep
        s = kc[g, :past + 1].astype(np.float64) @ q[h].astype(np.float64) / np.sqrt(hd)
        if plants[h] is None or len(plants[h]) == 0:
            continue
        P = np.asarray(plants[h], np.int64)
        inP = np.zeros(past + 1, bool); inP[P] = True
        gap = s[inP].min() - s[~inP].max()
        assert np.ptp(s[inP]) == 0 and gap >= PROBE_GAP, (h, gap)
        mean = vc[g, P].astype(np.float64).mean(0)
        margin = 2 * (past + 1) * np.exp(-gap) * np.abs(vc[g, :past + 1].astype(np.float64)).max()
        assert np.abs(got[h] - mean).max() <= margin, (h, np.abs(got[h] - mean).max(), margin)


# ---- the whole probe on a CPU stand-in of a DecodeStack (helpers.cpu_probe_stack) ------------------------------------------
@pytest.mark.parametrize("heads,kv", [(2, 2), (4, 1)])
def test_probe_bound_is_tight_and_sees_a_dropped_chunk(oracle, heads, kv):
    """probe_expectation on planted caches: the bound of a planted head is far below what one 16-position chunk read as
    background moves the answer by."""
    from helpers import oracle_decode_step
    past, max_seq = 300, 512
    st = _cpu_stack(oracle, heads, kv, 2, max_seq, seed=heads + kv)
    rng = np.random.default_rng(5)
    caches = [[(0.5 * rng.standard_normal((1, kv, max_seq, 128))).astype(np.float16) for _ in range(2)] for _ in range(2)]
    x = (1e-2 * rng.standard_normal(st.shape.hidden)).astype(np.float16)
    n_rep = heads // kv
    plants = plant_probe(oracle, st, caches, x, past, lambda l, h: dense_positions(past, h % n_rep, n_rep), seed=6)
    want, bound = probe_expectation(oracle, st, snap_of(caches), x, past, plants, "step")
    assert np.isfinite(bound).all() and bound.max() < 1e-2, bound.max()
    # the same token with chunk 1 of layer 1 read as background: the planted keys there lose their score
    dropped = [[c.copy() for c in kv_] for kv_ in caches]
    dropped[1][0][0, :, 16:32] = (0.5 * rng.standard_normal((kv, 16, 128))).astype(np.float16)
    moved, _, _ = oracle_decode_step(oracle, st, snap_of(dropped), x, past)
    ratio = np.abs(moved.reshape(-1).astype(np.float64) - want) / bound
    assert ratio.max() > 10, ratio.max()


def test_probe_newest_row_dominant_on_cpu(oracle):
    """k = gamma q: the new token's score clears every cached one by >= PROBE_GAP (probe_expectation asserts it), and the bound
    of those heads is as tight as a plateau's."""
    past, max_seq = 200, 256
    st = _cpu_stack(oracle, 4, 2, 1, max_seq, gamma=256.0, seed=9)
    rng = np.random.default_rng(7)
    caches = [[(0.5 * rng.standard_normal((1, 2, max_seq, 128))).astype(np.float16) for _ in range(2)]]
    x = (1e-2 * rng.standard_normal(st.shape.hidden)).astype(np.float16)
    plants = plant_probe(oracle, st, caches, x, past, lambda l, h: "new" if h % 2 == 0 else None, seed=8)
    want, bound = probe_expectation(oracle, st, snap_of(caches), x, past, plants, "step")
    b = bound.reshape(4, 128)[::2]
    assert np.isfinite(b).all() and b.max() < 5e-2, b.max()
