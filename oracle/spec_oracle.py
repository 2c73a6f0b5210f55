"""Float64 restatement of speculative sampling's verification step (Leviathan et al. 2023, Chen et al. 2023), the yardstick of
exl_spec_verify (exllama_b200/csrc/sample.cu, include/exl_b200.h).

TEST INFRASTRUCTURE ONLY, like sample_oracle.py, on which it is built: row j's target distribution p_j is sample_oracle.sample
of the target's logits row j with the history followed by the drafts d_1 .. d_j.  d_j is accepted iff u_{j-1} q_j(d_j) < p_{j-1}(d_j);
at the first rejection the correction is drawn with u_k from max(0, p_{j-1} - q_j) (from p_{j-1} if that has no mass), by inverse
CDF in ascending token-id order; if every draft is accepted the bonus token is the draw of p_k with u_k.  Besides the result,
verify() reports the margin of every decision it took -- |u q - p| of each acceptance test and how far u lies from the edges of
the CDF cell it fell in -- and the cells of the final draw, so that a test can enumerate them."""
from __future__ import annotations

import numpy as np

from . import sample_oracle as S


def dense(res, vocab):
    """A sample_oracle.sample result as a float64 [vocab] distribution (0 outside the kept set)."""
    p = np.zeros(vocab, np.float64)
    p[res["kept"]] = res["probs"]
    return p


def draw(mass, u):
    """Inverse CDF over non-negative float64 masses in ascending id order: the smallest id whose inclusive cumulative mass exceeds
    u * total, the largest id with mass if none does.  Returns (id, cells, margin): cells [(id, lo, hi)] of the ids with mass, as
    fractions of the total, and the distance of u from the edges of the chosen cell."""
    total = mass.sum()
    ids = np.nonzero(mass > 0)[0]
    cdf = np.cumsum(mass[ids]) / total
    lo = np.concatenate([[0.0], cdf[:-1]])
    i = min(int(np.searchsorted(cdf, u, side="right")), len(ids) - 1)
    cells = [(int(t), float(a), float(b)) for t, a, b in zip(ids, lo, cdf)]
    return int(ids[i]), cells, float(min(abs(u - lo[i]), abs(cdf[i] - u)))


def verify(target_logits, drafts, q, u, temperature, top_k=0, top_p=0.0, min_p=0.0, typical=0.0, history=None, penalty_max=1.0,
           sustain=-1, decay=0, bos=-1, banned=()):
    """One verification: target_logits [k + 1][vocab] (fp32 values), drafts [k] ids, q [k][vocab] the draft distributions,
    u [k + 1].  Returns a dict with
      n_accepted  a (-1 if a row the walk reached is undefined)
      tokens      [k + 1] ints: d_1 .. d_a, the correction or bonus token, then -1 (all -1 when undefined)
      probs       [k + 1] float64: p of each emitted token, NaN after them
      accept      [(|u_{j-1} q_j(d_j) - p_{j-1}(d_j)|, accepted)] of every acceptance test made
      draw        the distance of u_k from the edges of the cell it fell in (the correction's residual or p_k's CDF)
      cells       the final draw's cells [(id, lo, hi)]
      residual    whether the final token came from a residual (True) or is the bonus (False)
      rows        the sample_oracle results of the rows the walk read
      filter_margin  the smallest sample_oracle margin over those rows"""
    k = len(drafts)
    vocab = len(target_logits[0])
    hist = [] if history is None else [int(t) for t in history]
    drafts = [int(d) for d in drafts]
    kw = dict(top_k=top_k, top_p=top_p, min_p=min_p, typical=typical, penalty_max=penalty_max, sustain=sustain, decay=decay,
              bos=bos, banned=banned)
    out = {"n_accepted": -1, "tokens": [-1] * (k + 1), "probs": [np.nan] * (k + 1), "accept": [], "draw": np.inf, "cells": [],
           "residual": False, "rows": [], "filter_margin": np.inf}

    def row(j):
        h = hist + drafts[:j] if history is not None else None
        r = S.sample(target_logits[j], temperature, history=h, **kw)
        out["rows"].append(r)
        if r is not None:
            out["filter_margin"] = min(out["filter_margin"], S.min_margin(r))
        return None if r is None else dense(r, vocab)

    p = row(0)
    a, acc_p = 0, []
    while True:
        if p is None:
            return out
        if a == k:                                              # every draft accepted: the bonus draw of p_k
            tok, cells, m = draw(p, float(u[k]))
            break
        d = drafts[a]
        if not 0 <= d < vocab:
            return out
        qd = float(q[a][d])
        if not (np.isfinite(qd) and qd > 0):
            return out
        prod = float(u[a]) * qd
        ok = prod < p[d]
        out["accept"].append((abs(prod - p[d]), ok))
        if not ok:
            r = np.maximum(p - np.asarray(q[a], np.float64), 0.0)
            tok, cells, m = draw(r if r.sum() > 0 else p, float(u[k]))
            out["residual"] = True
            break
        acc_p.append(p[d])
        a += 1
        p = row(a)
    out["n_accepted"] = a
    out["tokens"][:a + 1], out["probs"][:a + 1] = drafts[:a] + [tok], acc_p + [p[tok]]
    out["draw"], out["cells"] = m, cells
    return out


def min_margin(res) -> float:
    """The smallest margin of every decision verify() took (acceptance tests, the draw, the filters of the rows it read)."""
    return min([m for m, _ in res["accept"]] + [res["draw"], res["filter_margin"]])
