"""Float64 restatement of the generator's token sampling (generator.py:91-170, with the repetition penalty and the bos logit of
gen_single_token), the yardstick of exllama_b200/csrc/sample.cu (include/exl_b200.h exl_sample).

TEST INFRASTRUCTURE ONLY, like oracle.py.  The penalty is applied in fp32 by oracle.apply_rep_penalty (bit-exact with the
reference's rep_penalty.cpp); everything after it is float64.  Orders put ties at the lower token id.  Besides the kept set,
its final probabilities and the token for a given u, sample() reports the margin of every decision it took: how far each
threshold (top_p, typical, min_p) lies from the nearest cumulative value or probability it was compared with, and the gap
between the last kept and the first dropped key of each order (top-k, top-p, typical) -- a case with a small margin may be
decided the other way by an fp32 implementation.
"""
from __future__ import annotations

import numpy as np

from . import oracle as O


KINDS = ("normal", "dominant", "flat")


def case_logits(seed: int, vocab: int, kind: str, scale: float = 3.0) -> np.ndarray:
    """fp32 logits [vocab] of one seeded case: 'normal' (N(0, scale)), 'dominant' (one token 8 above) or 'flat' (N(0, 0.01))."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(vocab) * (0.01 if kind == "flat" else scale)
    if kind == "dominant":
        x[rng.integers(vocab)] += 8.0
    return x.astype(np.float32)


def _prefix_loop(vals, threshold, min_p=None):
    """The top-p / typical loop of generator.py:122-129 / 148-154 over vals (already ordered), in float64 .item() sums.
    Returns (kept count, margin over every comparison made)."""
    margin = np.inf
    n = 0
    cum = float(vals[0])
    while True:
        n += 1
        if n == len(vals):
            break
        if min_p is not None:
            margin = min(margin, abs(float(vals[n]) - min_p))
            if float(vals[n]) < min_p:
                break
        cum += float(vals[n])
        margin = min(margin, abs(cum - threshold))
        if cum > threshold:
            break
    return n, margin


def sample(logits, temperature, top_k=0, top_p=0.0, min_p=0.0, typical=0.0, history=None, penalty_max=1.0, sustain=-1,
           decay=0, bos=-1, banned=(), u=None):
    """One row.  Returns None for an undefined row (every logit -inf after masking, a NaN logit, a history id outside the
    vocabulary), else a dict with
      kept     int64 ids of the kept set, ascending
      probs    float64 final probabilities of those ids (what the reference's multinomial sees)
      token    the draw for u (the smallest kept id whose inclusive cumulative probability exceeds u; the largest if none)
      cdf      float64 inclusive cumulative probabilities over kept, for choosing u
      margins  {name: distance} of every threshold and order cut the case crossed"""
    x = np.array(logits, dtype=np.float32).copy()
    vocab = x.shape[0]
    if history is not None and len(history) and penalty_max != 1.0:
        h = np.asarray(history, dtype=np.int64)
        if h.min() < 0 or h.max() >= vocab:
            return None
        x = O.apply_rep_penalty(h[None], penalty_max, sustain, decay, x[None])[0]
    if bos >= 0:
        x[bos] = -10000.0
    x = x.astype(np.float64)
    banned = np.asarray(banned, dtype=np.int64)
    if banned.size and (banned.min() < 0 or banned.max() >= vocab):
        return None
    x[banned] = -np.inf
    if np.isnan(x).any() or np.all(x == -np.inf):
        return None
    y = x / temperature + 1e-8
    e = np.exp(y - y.max())
    p = e / e.sum()
    ids = np.arange(vocab)
    margins = {}
    order = np.lexsort((ids, -p))                       # probability descending, ties to the lower id
    if top_k > 0:
        if top_k < vocab:
            a, b = p[order[top_k - 1]], p[order[top_k]]
            margins["top_k_gap"] = (a - b) / a if a > 0 else 0.0
        order = order[:top_k]
        vals = p[order] / max(p[order].sum(), 1e-12)
    else:
        vals = p[order]
    if top_p > 0.0:
        n, m = _prefix_loop(vals, top_p, min_p)
        margins["top_p"] = m
        if n < len(vals):
            margins["top_p_gap"] = (vals[n - 1] - vals[n]) / vals[n - 1] if vals[n - 1] > 0 else 0.0
        order, vals = order[:n], vals[:n]
        vals = vals / max(vals.sum(), 1e-12)
    if typical > 0.0:
        lp = np.log(vals + 1e-10)
        dev = np.abs((vals * lp).sum() - lp)
        o2 = np.lexsort((order, dev))                   # entropy deviation ascending, ties to the lower id
        order, vals, dev = order[o2], vals[o2], dev[o2]
        n, m = _prefix_loop(vals, typical)
        margins["typical"] = m
        if n < len(vals):
            margins["typical_gap"] = dev[n] - dev[n - 1]
        order, vals = order[:n], vals[:n]
        vals = vals / max(vals.sum(), 1e-12)
    srt = np.argsort(order, kind="stable")
    kept, probs = order[srt].astype(np.int64), vals[srt]
    cdf = np.cumsum(probs)
    out = {"kept": kept, "probs": probs, "cdf": cdf, "margins": margins, "token": None}
    if u is not None:
        i = int(np.searchsorted(cdf, u, side="right"))
        out["token"] = int(kept[min(i, len(kept) - 1)])
    return out


def min_margin(res) -> float:
    return min(res["margins"].values(), default=np.inf)


def golden_cases(path):
    """The cases of tests/golden/sample_ref.npz (oracle/gen_golden_sample.py): per case a settings dict, its fp32 logits, history,
    banned ids, and the reference's kept ids and final probabilities."""
    g = np.load(path)
    fields = [str(f) for f in g["fields"]]
    out = []
    for i, row in enumerate(g["cases"]):
        c = dict(zip(fields, row.tolist()))
        for f in ("seed", "vocab", "top_k", "sustain", "decay", "bos"):
            c[f] = int(c[f])
        c["kind"] = KINDS[int(c["kind"])]
        c["logits"] = case_logits(c["seed"], c["vocab"], c["kind"])
        c["history"] = g["hist"][g["hist_off"][i]:g["hist_off"][i + 1]].astype(np.int64)
        c["banned"] = g["banned"][g["banned_off"][i]:g["banned_off"][i + 1]].astype(np.int64)
        c["kept"] = g["kept"][g["kept_off"][i]:g["kept_off"][i + 1]].astype(np.int64)
        c["probs"] = g["probs"][g["kept_off"][i]:g["kept_off"][i + 1]]
        out.append(c)
    return out


def run_case(c, u=None):
    """sample() on a golden_cases() entry."""
    return sample(c["logits"], c["temperature"], c["top_k"], c["top_p"], c["min_p"], c["typical"], history=c["history"],
                  penalty_max=c["penalty_max"], sustain=c["sustain"], decay=c["decay"], bos=c["bos"], banned=c["banned"], u=u)
