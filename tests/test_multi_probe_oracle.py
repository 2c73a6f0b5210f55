"""The attention probe (tests/helpers.py, "Attention probe") generalised to the multi-token step, checked with the float64 oracle
alone: a launch of n tokens at past_len, token t at position past + t reading rows [0, past + t], query vector j = t n_rep + r of a
KV group (virtual query head t * heads + h).  So that a failure of tests/test_gpu_decode_multi_probe.py points at a kernel, not at
the harness, this file shows that
  - one token is unchanged: planting and (want, bound) are bit for bit what the one-token helpers computed (tests/golden/
    attn_probe_n1.npz, written by oracle/gen_golden_attn_probe.py before the helpers took n tokens);
  - the construction holds for n tokens: every planted vector of every token answers its plateau mean, plateaus are disjoint, and
    the poison rows (the launch's own, overwritten) and the NaN rows after them are never read;
  - the probe sees the multi-token step's own bugs: each one emulated in the float64 composition misses probe_expectation's
    bound by >= 10x on at least one layout and context the GPU file runs (the matrix is printed)."""
import hashlib
import os

import numpy as np
import pytest

from helpers import (GOLDEN, PROBE_GAP, cpu_probe_stack, dense_positions, lone_positions, multi_positions, multi_probe_specs,
                     newest_inputs, oracle_decode_step, plant_group, plant_probe, probe_caches, probe_expectation, snap_of)


# ---------------------------------------------------------------------------------------------------------- n = 1 is unchanged
def _n1_cases(oracle):
    """The whole-probe cases of test_attn_probe_oracle.py: (name, stack, caches, x, past, spec, seed)."""
    for heads, kv in [(2, 2), (4, 1)]:
        past, max_seq = 300, 512
        st = cpu_probe_stack(oracle, heads, kv, 2, max_seq, seed=heads + kv)
        rng = np.random.default_rng(5)
        caches = [[(0.5 * rng.standard_normal((1, kv, max_seq, 128))).astype(np.float16) for _ in range(2)] for _ in range(2)]
        x = (1e-2 * rng.standard_normal(st.shape.hidden)).astype(np.float16)
        n_rep = heads // kv
        yield (f"dense_h{heads}_kv{kv}", st, caches, x, past, lambda l, h, n_rep=n_rep: dense_positions(300, h % n_rep, n_rep), 6)
    st = cpu_probe_stack(oracle, 4, 2, 1, 256, gamma=256.0, seed=9)
    rng = np.random.default_rng(7)
    caches = [[(0.5 * rng.standard_normal((1, 2, 256, 128))).astype(np.float16) for _ in range(2)]]
    x = (1e-2 * rng.standard_normal(st.shape.hidden)).astype(np.float16)
    yield "newest_h4_kv2", st, caches, x, 200, lambda l, h: "new" if h % 2 == 0 else None, 8


def n1_record(oracle):
    """name -> array: want, bound, sha256 of the planted caches and the plants (layer, head, position) of every _n1_cases case."""
    out = {}
    for name, st, caches, x, past, spec, seed in _n1_cases(oracle):
        plants = plant_probe(oracle, st, caches, x, past, spec, seed=seed)
        want, bound = probe_expectation(oracle, st, snap_of(caches), x, past, plants, "step")
        h = hashlib.sha256()
        for kv in caches:
            for c in kv:
                h.update(np.ascontiguousarray(c).tobytes())
        out[name + "_want"] = want
        out[name + "_bound"] = bound
        out[name + "_caches"] = np.frombuffer(h.digest(), np.uint8)
        out[name + "_plants"] = np.array([[l, hh, p] for l, d in enumerate(plants) for hh in sorted(d) for p in d[hh]], np.int64)
    return out


def test_one_token_is_unchanged(oracle):
    gold = np.load(os.path.join(GOLDEN, "attn_probe_n1.npz"))
    got = n1_record(oracle)
    assert sorted(got) == sorted(gold.files)
    for k in gold.files:
        assert got[k].dtype == gold[k].dtype and got[k].shape == gold[k].shape, k
        assert np.array_equal(got[k].view(np.uint8), gold[k].view(np.uint8)), f"{k} differs from the one-token helpers"


# ------------------------------------------------------------------------------------------------------- the construction holds
@pytest.mark.parametrize("n_rep,n", [(1, 4), (4, 3), (4, 4), (8, 4)])
@pytest.mark.parametrize("past", [1, 16, 37, 300])
@pytest.mark.parametrize("layout", ["dense", "lone"])
def test_planted_tokens_answer_their_plateau_means(oracle, n_rep, n, past, layout):
    """n tokens of n_rep query heads per KV head (m = n n_rep vectors per group, up to 32): each planted vector of each token gets
    the mean of V over its plateau, to within the margin, reading rows [0, past + t]; the plateaus of a group are disjoint; the
    poison rows past .. past + n - 1 and the NaN rows from past + n are never read."""
    hd, max_seq, kv = 128, 512, 2
    heads, m = kv * n_rep, n * n_rep
    rng = np.random.default_rng(past + 10 * n_rep + n)
    q = (0.4 * rng.standard_normal((n, heads, hd))).astype(np.float16)
    kc = (0.5 * rng.standard_normal((kv, max_seq, hd))).astype(np.float16)
    vc = (0.5 * rng.standard_normal((kv, max_seq, hd))).astype(np.float16)
    k_new = (0.4 * rng.standard_normal((n, kv, hd))).astype(np.float16)
    v_new = (0.5 * rng.standard_normal((n, kv, hd))).astype(np.float16)
    plants = [multi_positions(past, j, m) for j in range(m)] if layout == "dense" else lone_positions(past, m)
    for g in range(kv):
        qg = q[:, g * n_rep:(g + 1) * n_rep].reshape(m, hd)
        s_new = qg.astype(np.float64) @ k_new[:, g].astype(np.float64).T / np.sqrt(hd)
        plant_group(qg, kc[g], vc[g], plants, past, s_new, rng)
    sets = [set(np.asarray(P).tolist()) for P in plants if P is not None]
    assert sum(map(len, sets)) == len(set().union(*sets)), "plateaus overlap"
    assert all(max(s) < past for s in sets if s)
    assert np.isnan(kc[:, past + n:]).all() and (np.abs(vc[:, past:past + n]).max(-1) == 100).all()
    kc[:, past:past + n] = k_new.transpose(1, 0, 2); vc[:, past:past + n] = v_new.transpose(1, 0, 2)
    for t in range(n):
        got = oracle.decode_attn_f64(q[t].reshape(-1), kc, vc, heads, kv, hd, past + t + 1, max_seq).reshape(heads, hd)
        assert np.isfinite(got).all()
        for h in range(heads):
            g, r = divmod(h, n_rep)
            P = plants[t * n_rep + r]
            if P is None or len(P) == 0:
                continue
            P = np.asarray(P, np.int64)
            s = kc[g, :past + t + 1].astype(np.float64) @ q[t, h].astype(np.float64) / np.sqrt(hd)
            inP = np.zeros(past + t + 1, bool); inP[P] = True
            gap = s[inP].min() - s[~inP].max()
            assert np.ptp(s[inP]) == 0 and gap >= PROBE_GAP, (t, h, gap)
            mean = vc[g, P].astype(np.float64).mean(0)
            margin = 2 * (past + t + 1) * np.exp(-gap) * np.abs(vc[g, :past + t + 1].astype(np.float64)).max()
            assert np.abs(got[h] - mean).max() <= margin, (t, h, np.abs(got[h] - mean).max(), margin)


@pytest.mark.parametrize("past", [1, 15, 16, 17, 37, 255, 1000])
def test_layouts_cover_chunk_edges_and_the_last_row(past):
    """Across the layouts the GPU file plants, the plateaus hold the first and the last row of a 16-position chunk and past - 1,
    for every group size m = n n_rep it runs."""
    for m in (1, 2, 3, 4, 8, 12, 16, 32):
        dense = [set(multi_positions(past, j, m).tolist()) for j in range(m)]
        assert sum(map(len, dense)) == len(set().union(*dense)), m
        lone = set(p for P in lone_positions(past, m) if P is not None for p in P)
        every = set().union(*dense) | lone
        assert past - 1 in every, (m, past)
        assert 0 in every and (past <= 15 or 15 in every), (m, past)


# ------------------------------------------------------------------------------------------------------------- mutation matrix
def _attn_rows(st, q, kc, vc, rows_of):
    """float64 softmax attention of q [n, heads, hd] over the rows rows_of(t) of kc / vc [kv_heads, max_seq, hd] (zero when a
    token reads no row): [n, heads, hd]."""
    s = st.shape
    n_rep, hd = s.heads // s.kv_heads, s.head_dim
    out = np.zeros(q.shape)
    for t in range(q.shape[0]):
        idx = np.asarray(rows_of(t), np.int64)
        if len(idx) == 0:
            continue
        for h in range(s.heads):
            K = kc[h // n_rep, idx].astype(np.float64); V = vc[h // n_rep, idx].astype(np.float64)
            sc = K @ q[t, h].astype(np.float64) / np.sqrt(hd)
            w = np.exp(sc - sc.max())
            out[t, h] = w @ V / w.sum()
    return out


class _RopeQAtPast:
    """The oracle with every query head roped at past_len instead of past_len + t (the new k keeps its position: under
    grouped-query attention the k rope call has kv_heads rows per token, not heads)."""

    def __init__(self, oracle, heads):
        self._o, self._heads = oracle, heads

    def __getattr__(self, name):
        return getattr(self._o, name)

    def rope(self, x, sin, cos, bsz, rows, hd, num_heads, past):
        return self._o.rope(x, sin, cos, bsz, rows, hd, rows if num_heads == self._heads else num_heads, past)


MUTATIONS = ["future leak", "no own row", "next token's answer", "q roped at past", "history short by one",
             "launch rows twice", "other sequence"]


def _mutant(oracle, st, snap, x, past, which):
    """The final hidden state of the launch with the multi-token step's bug `which` emulated in the composition."""
    s = st.shape
    n = np.asarray(x).reshape(-1, s.hidden).shape[0]
    if which == "q roped at past":
        return oracle_decode_step(_RopeQAtPast(oracle, s.heads), st, snap, x, past)[0]
    rows = {"future leak": lambda t: np.arange(past + n),
            "no own row": lambda t: np.arange(past + t),
            "history short by one": lambda t: np.r_[np.arange(max(past - 1, 0)), past + np.arange(t + 1)],
            "launch rows twice": lambda t: np.r_[np.arange(past + n), past + np.arange(t + 1)]}

    def attend(l, q, kc, vc):
        if which == "next token's answer":
            return np.roll(_attn_rows(st, q, kc, vc, lambda t: np.arange(past + t + 1)), -1, axis=0)
        if which == "other sequence":
            ko = snap[l][0][1].numpy().copy(); vo = snap[l][1][1].numpy().copy()
            ko[:, past:past + n] = kc[:, past:past + n]; vo[:, past:past + n] = vc[:, past:past + n]
            return _attn_rows(st, q, ko, vo, lambda t: np.arange(past + t + 1))
        return _attn_rows(st, q, kc, vc, rows[which])
    return oracle_decode_step(oracle, st, snap, x, past, attend=attend)[0]


# (stack, layers, layouts, contexts): a subset of what tests/test_gpu_decode_multi_probe.py runs, at 4 tokens
MATRIX = [("kv 2", 2, ["dense", "lone+0"], [0, 1, 16, 37, 255]),
          ("kv 2 background", 1, ["dense", "lone+0"], [0, 1, 16, 37]),
          ("kv 2 newest", 1, ["newest"], [0, 1, 37])]


def test_mutation_matrix(oracle, capsys):
    """Every emulated bug misses the bound by >= 10x somewhere.  Planted plateaus clear every new row by >= 30, so a future leak
    or a double-counted launch row leaves planted heads alone: background heads at short contexts (one layer) and past 0 catch
    those.  Sequence 1 of the cache holds N(0, 0.25) rows, as the other sequences of a batched cache may."""
    n, heads, kv, max_seq = 4, 8, 2, 512
    ratios = {m: {} for m in MUTATIONS}
    for name, layers, layouts, pasts in MATRIX:
        st = cpu_probe_stack(oracle, heads, kv, layers, max_seq, gamma=256.0 if "newest" in name else None, seed=layers + 40,
                             batch=2)
        caches0 = probe_caches(st, 60 + layers)
        for i, past in enumerate(pasts):
            x = (newest_inputs(oracle, st, n, past, 70 + i) if "newest" in name else
                 (1e-2 * np.random.default_rng(70 + i).standard_normal((n, st.shape.hidden))).astype(np.float16))
            for lname, spec in multi_probe_specs(st, n, past, background="background" in name):
                if lname not in layouts:
                    continue
                caches = [[c.copy() for c in kv_] for kv_ in caches0]
                plants = plant_probe(oracle, st, caches, x, past, spec, seed=80 + i)
                snap = snap_of(caches)
                want, bound = probe_expectation(oracle, st, snap, x, past, plants, "step")
                for m in MUTATIONS:
                    got = _mutant(oracle, st, snap, x, past, m).astype(np.float64)
                    ratios[m][(name, lname, past)] = float(np.nanmax(np.abs(got - want) / bound)) if np.isfinite(got).all() else np.inf
    with capsys.disabled():
        print("\nmulti-token probe: largest |mutant - want| / bound per mutation, layout and context (4 tokens, kv 2)")
        cols = [(name, ln, p) for name, _, lns, ps in MATRIX for ln in lns for p in ps]
        for m in MUTATIONS:
            print(f"  {m:22s} " + " ".join(f"{ratios[m][c]:8.3g}" for c in cols))
        print("  columns: " + ", ".join(f"{a}/{b}/ctx {c}" for a, b, c in cols))
    for m in MUTATIONS:
        best = max(ratios[m].values())
        assert best >= 10, f"{m}: no layout misses its bound by 10x (best {best:.3g})"
