"""Float64 restatement of exl_top_logprobs (include/exl_b200.h, csrc/toplp.cu): the model's log-probability of a chosen token and the
top-N alternatives of one fp32 logits row.

TEST INFRASTRUCTURE ONLY, like oracle.py.  The ids are exact (the same total order as the kernel: the logit's value with -0 read as
+0, a tie to the lower id); the log-probabilities are float64 with a per-element bound on the kernel's fp32 result:
  vocab * 2^-52 * (|lse| + 1)   the float64 sum in another order, its log and the subtraction (the + 1 covers an lse near 0),
  + 2^-24 * (|lp| + that)       the one fp32 rounding of the result.
"""
from __future__ import annotations

import numpy as np

U32 = 2.0 ** -24


def lse(x):
    """lse of one fp32 row in float64 over its finite entries, or None if the row is undefined (a NaN or +inf, or no finite entry)."""
    x = np.asarray(x, dtype=np.float32).astype(np.float64)
    if np.isnan(x).any() or (x == np.inf).any() or not np.isfinite(x).any():
        return None
    f = x[np.isfinite(x)]
    m = f.max()
    return m + np.log(np.exp(f - m).sum())


def order(x):
    """Ids of the finite entries of x, largest logit first, a tie to the lower id (-0 and +0 are one value)."""
    x = np.asarray(x, dtype=np.float32).astype(np.float64) + 0.0          # -0.0 + 0.0 == +0.0
    ids = np.flatnonzero(np.isfinite(x))
    return ids[np.lexsort((ids, -x[ids]))]


def top_logprobs(x, n, token=None):
    """One row.  Returns a dict:
      lp      float64 log-probability of token (NaN: no token, outside [0, vocab), or an undefined row)
      ids     int64 [n]: the top ids, -1 past the finite entries or on an undefined row
      top     float64 [n]: their log-probabilities; -inf past the finite entries, NaN on an undefined row
      bound   float64 [n] per-element bound on |kernel - top| (0 where top is not finite: there the kernel's value is exact)
      lp_bound  the bound for lp"""
    x = np.asarray(x, dtype=np.float32)
    V = x.shape[0]
    L = lse(x)
    ids = np.full(n, -1, np.int64)
    if L is None:
        nan = np.full(n, np.nan)
        return {"lp": np.nan, "ids": ids, "top": nan, "bound": np.zeros(n), "lp_bound": 0.0}
    e64 = V * 2.0 ** -52 * (abs(L) + 1.0)

    def lp_of(i):
        v = float(x[i]) - L
        return v, (e64 + U32 * (abs(v) + e64) if np.isfinite(v) else 0.0)

    o = order(x)[:n]
    ids[:len(o)] = o
    top = np.full(n, -np.inf)
    bound = np.zeros(n)
    for k, i in enumerate(o):
        top[k], bound[k] = lp_of(i)
    lp, lp_b = np.nan, 0.0
    if token is not None and 0 <= int(token) < V:
        lp, lp_b = lp_of(int(token))
    return {"lp": lp, "ids": ids, "top": top, "bound": bound, "lp_bound": lp_b}


def within(got, want, bound):
    """fp32 kernel values got against the oracle's want: equal where want is not finite (NaN where NaN), within bound elsewhere."""
    got = np.asarray(got, dtype=np.float64).reshape(-1)
    want = np.asarray(want, dtype=np.float64).reshape(-1)
    bound = np.asarray(bound, dtype=np.float64).reshape(-1)
    fin = np.isfinite(want)
    with np.errstate(invalid="ignore"):
        ok = np.where(fin, np.abs(got - want) <= bound, (got == want) | (np.isnan(got) & np.isnan(want)))
    return bool(ok.all())
