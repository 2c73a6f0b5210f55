"""Float64 restatement of classifier-free guidance (the reference's example_cfg.py:69-75), the yardstick of exllama_b200/csrc/cfg.cu
(include/exl_b200.h exl_cfg_mix).

TEST INFRASTRUCTURE ONLY, like oracle.py.  The penalty is applied in fp32 by oracle.apply_rep_penalty (bit-exact with the
reference's rep_penalty.cpp); the log-softmax and the mix are float64.  mix() also returns a per-element bound on the distance
between the kernel's fp32 mixed row and the float64 one, from the kernel's rounding points: lse rounded to fp32, l = x' - lse in
fp32, the weights (float)(1 - alpha) and (float)alpha, the two fp32 products and the fp32 sum.  The sampler after the mix is
sample_oracle.sample with no history and no bos mask (sample_current).

golden_cases() reads tests/golden/cfg_ref.npz (oracle/gen_golden_cfg.py).  The reference computes its mixed row in fp32 with
torch: l = (x' - max) - logsum, logsum = fp32 log of an fp32 sum, then fp32 products and sum; golden_row() restates that program
in numpy fp32 from the logsum values the fixture stores (the only quantity whose fp32 rounding depends on torch's summation
order), which reproduces the reference's row bit for bit.
"""
from __future__ import annotations

import numpy as np

from . import oracle as O
from . import sample_oracle as S

U32 = 2.0 ** -24                 # fp32 unit roundoff
U64 = 2.0 ** -53


def penalised(logits, history, penalty_max, sustain, decay):
    """fp32 logits after the repetition penalty over history (None: undefined -- a history id outside the vocabulary)."""
    x = np.array(logits, dtype=np.float32).copy()
    if history is not None and len(history) and penalty_max != 1.0:
        h = np.asarray(history, dtype=np.int64)
        if h.min() < 0 or h.max() >= x.shape[0]:
            return None
        x = O.apply_rep_penalty(h[None], penalty_max, sustain, decay, x[None])[0]
    return x


def _log_softmax64(x):
    """(l float64, lse float64) of one fp32 row, or None if the row is undefined (a NaN, or every entry -inf)."""
    if np.isnan(x).any() or np.all(x == -np.inf):
        return None
    x = x.astype(np.float64)
    m = x.max()
    lse = m + np.log(np.exp(x - m).sum())
    return x - lse, lse


def mix(la, lb, alpha, hist_a=None, hist_b=None, penalty_max=1.0, sustain=-1, decay=0):
    """One pair.  Returns None when either row is undefined (the kernel writes both rows NaN), else a dict with
      mixed    float64 (1 - alpha) * l_a + alpha * l_b of the penalised rows' float64 log-softmax
      bound    float64 per-element bound on |kernel - mixed| (0 where an l is infinite: there the kernel's value is `special`)
      special  the exact value where l_a or l_b is infinite (IEEE arithmetic on the fp32 weights), NaN elsewhere
      lse_a, lse_b  the float64 lse of each row"""
    xa = penalised(la, hist_a, penalty_max, sustain, decay)
    xb = penalised(lb, hist_b, penalty_max, sustain, decay)
    if xa is None or xb is None:
        return None
    ra, rb = _log_softmax64(xa), _log_softmax64(xb)
    if ra is None or rb is None:
        return None
    (l_a, lse_a), (l_b, lse_b) = ra, rb
    wa, wb = 1.0 - float(alpha), float(alpha)
    wa32, wb32 = float(np.float32(wa)), float(np.float32(wb))
    with np.errstate(invalid="ignore", over="ignore"):
        mixed = wa * l_a + wb * l_b
        # lse rounded to fp32 (plus the float64 sum and log), then l = x' - lse rounded to fp32
        e_lse_a = U32 * abs(lse_a) + 64 * U64 * (abs(lse_a) + 1.0)
        e_lse_b = U32 * abs(lse_b) + 64 * U64 * (abs(lse_b) + 1.0)
        e_la = e_lse_a + U32 * (np.abs(l_a) + e_lse_a)
        e_lb = e_lse_b + U32 * (np.abs(l_b) + e_lse_b)
        # weights rounded to fp32 (1 - alpha first in double), then each product rounded
        e_wa = U32 * abs(wa) + U64 * (abs(wa) + abs(alpha))
        e_wb = U32 * abs(wb)
        pa = abs(wa32) * (np.abs(l_a) + e_la)
        pb = abs(wb32) * (np.abs(l_b) + e_lb)
        e_pa = abs(wa32) * e_la + e_wa * np.abs(l_a) + U32 * pa
        e_pb = abs(wb32) * e_lb + e_wb * np.abs(l_b) + U32 * pb
        # the sum rounded to fp32 (its magnitude is at most pa + pb, products' errors included)
        bound = (e_pa + e_pb + U32 * (pa + pb + e_pa + e_pb)) * (1 + 1e-9) + 1e-300
        inf = ~np.isfinite(l_a) | ~np.isfinite(l_b)
        special = np.where(inf, wa32 * l_a + wb32 * l_b, np.nan)
    bound[inf] = 0.0
    return {"mixed": mixed, "bound": bound, "special": special, "lse_a": lse_a, "lse_b": lse_b}


def within(got, res):
    """Whether an fp32 mixed row got satisfies mix()'s result res: every finite element within the bound, and every element where
    an l is infinite equal to res["special"] (NaN where that is NaN)."""
    got = np.asarray(got, dtype=np.float64)
    sp = res["bound"] == 0.0
    with np.errstate(invalid="ignore"):
        ok = np.abs(got - res["mixed"]) <= res["bound"]
    ok_sp = (got == res["special"]) | (np.isnan(got) & np.isnan(res["special"]))
    return bool(np.all(np.where(sp, ok_sp, ok)))


def emulate32(la, lb, alpha, hist_a=None, hist_b=None, penalty_max=1.0, sustain=-1, decay=0):
    """numpy fp32 restatement of the kernel's rounding points (the lse sum in float64, in numpy's order): the mixed row, or None
    for an undefined pair."""
    xa = penalised(la, hist_a, penalty_max, sustain, decay)
    xb = penalised(lb, hist_b, penalty_max, sustain, decay)
    if xa is None or xb is None:
        return None
    out = []
    for x in (xa, xb):
        r = _log_softmax64(x)
        if r is None:
            return None
        out.append(x - np.float32(r[1]))                 # fp32 - fp32: correctly rounded
    wa, wb = np.float32(1.0 - float(alpha)), np.float32(float(alpha))
    with np.errstate(invalid="ignore", over="ignore"):
        return (wa * out[0]) + (wb * out[1])            # each an fp32 operation


def golden_row(la, lb, alpha, logsum_a, logsum_b, hist_a, hist_b, penalty_max, sustain, decay):
    """The reference's fp32 mixed row (torch: log_softmax = (x' - max) - logsum, then (1 - alpha) * l_a + alpha * l_b), restated in
    numpy fp32 with the fixture's logsum of each row."""
    ls = []
    for x, lg in ((penalised(la, hist_a, penalty_max, sustain, decay), logsum_a), (penalised(lb, hist_b, penalty_max, sustain, decay), logsum_b)):
        ls.append((x - x.max()) - np.float32(lg))
    return (np.float32(1.0 - float(alpha)) * ls[0]) + (np.float32(float(alpha)) * ls[1])


FIELDS = ["seed_a", "seed_b", "vocab", "kind", "alpha", "temperature", "top_k", "top_p", "min_p", "typical", "penalty_max", "sustain",
          "decay", "logsum_a", "logsum_b"]


def golden_cases(path):
    """The cases of tests/golden/cfg_ref.npz: per case its settings, both rows' fp32 logits (redrawn from their seeds), histories,
    the reference's logsums, and its kept ids and final probabilities."""
    g = np.load(path)
    fields = [str(f) for f in g["fields"]]
    out = []
    for i, row in enumerate(g["cases"]):
        c = dict(zip(fields, row.tolist()))
        for f in ("seed_a", "seed_b", "vocab", "top_k", "sustain", "decay"):
            c[f] = int(c[f])
        c["kind"] = S.KINDS[int(c["kind"])]
        c["logits_a"] = S.case_logits(c["seed_a"], c["vocab"], c["kind"])
        c["logits_b"] = S.case_logits(c["seed_b"], c["vocab"], c["kind"])
        for s in ("a", "b"):
            c["hist_" + s] = g["hist_" + s][g["hist_off"][i]:g["hist_off"][i + 1]].astype(np.int64)
        c["kept"] = g["kept"][g["kept_off"][i]:g["kept_off"][i + 1]].astype(np.int64)
        c["probs"] = g["probs"][g["kept_off"][i]:g["kept_off"][i + 1]]
        out.append(c)
    return out


def run_case(c):
    """The golden case through golden_row() and sample_oracle.sample (no history, no bos mask)."""
    row = golden_row(c["logits_a"], c["logits_b"], c["alpha"], c["logsum_a"], c["logsum_b"], c["hist_a"], c["hist_b"], c["penalty_max"],
                     c["sustain"], c["decay"])
    return S.sample(row, c["temperature"], c["top_k"], c["top_p"], c["min_p"], c["typical"])
