"""Generates tests/golden/sample_ref.npz by running the REFERENCE's own ExLlamaGenerator.sample (generator.py:91-170) on the CPU.

    EXLLAMA_REFERENCE=<reference checkout> python -m oracle.gen_golden_sample

generator.py imports cuda_ext, model and lora; stub modules stand in for them, so nothing is built.  For each case the
repetition penalty (oracle.apply_rep_penalty, bit-exact with the reference's rep_penalty.cpp) and the bos logit are applied
first, as gen_single_token does, then sample() runs in float64 with torch.multinomial replaced by a function that returns
every index: sample() then hands back the whole kept set with its final probabilities.  Logits are redrawn from their seed
(sample_oracle.case_logits), so the fixture stores seeds, settings, histories, kept ids and probabilities.  Every top_p /
typical / min_p is placed at the midpoint between the two values around the cut it is meant to make, and a case is kept
only if every decision it takes has a margin of at least 1e-4 and the float64 oracle agrees with the reference.
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

from . import oracle as O
from . import sample_oracle as S

MARGIN = 1e-4
FIELDS = ["seed", "vocab", "kind", "temperature", "top_k", "top_p", "min_p", "typical", "penalty_max", "sustain", "decay", "bos"]


def reference_generator():
    ref = os.environ.get("EXLLAMA_REFERENCE")
    if not ref or not os.path.exists(os.path.join(ref, "generator.py")):
        sys.exit("EXLLAMA_REFERENCE must name a checkout of the reference")
    for name, attrs in (("cuda_ext", {}), ("model", {"ExLlama": object, "ExLlamaCache": object}), ("lora", {"ExLlamaLora": object})):
        m = types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m
    sys.path.insert(0, ref)
    import generator
    return generator.ExLlamaGenerator


def run_reference(Gen, logits32, c, history, banned):
    """Penalty + bos in fp32, then the reference's sample() in float64 with every index drawn.  Returns (ids, probs) by id."""
    x = logits32.copy()
    if len(history) and c["penalty_max"] != 1.0:
        x = O.apply_rep_penalty(history[None], c["penalty_max"], c["sustain"], c["decay"], x[None])[0]
    if c["bos"] >= 0:
        x[c["bos"]] = -10000.0
    g = object.__new__(Gen)
    g.disallowed_tokens = [int(t) for t in banned] if len(banned) else None
    real = torch.multinomial
    torch.multinomial = lambda probs, num: torch.arange(probs.shape[-1])
    try:
        toks, probs = g.sample(torch.from_numpy(x.astype(np.float64))[None], c["temperature"], c["top_k"], c["top_p"], c["min_p"],
                               c["typical"])
    finally:
        torch.multinomial = real
    return toks[0].numpy().astype(np.int64), probs[0].numpy().astype(np.float64)


def oracle_run(c, logits32, history, banned):
    return S.sample(logits32, c["temperature"], c["top_k"], c["top_p"], c["min_p"], c["typical"], history=history,
                    penalty_max=c["penalty_max"], sustain=c["sustain"], decay=c["decay"], bos=c["bos"], banned=banned)


def place(c, logits32, history, banned, rng, want_p, want_typ, want_min):
    """Fill top_p / typical / min_p at midpoints around a cut the rng picks; returns False if no cut has room."""
    base = dict(c, top_p=0.0, min_p=0.0, typical=0.0)
    r = oracle_run(base, logits32, history, banned)
    vals = r["probs"][np.lexsort((r["kept"], -r["probs"]))]          # the top-k list in its order (its probabilities)
    if want_p:
        cum = np.cumsum(vals)
        ok = [n for n in range(1, min(len(vals), 400)) if vals[n] >= 2.5 * MARGIN]
        if not ok:
            return False
        n = ok[rng.integers(len(ok))]                                # keep n tokens: cum[n-1] <= top_p < cum[n]
        c["top_p"] = float((cum[n - 1] + cum[n]) / 2)
        if want_min and n > 1:
            m = int(rng.integers(1, n))                              # the min_p test cuts first, after m tokens
            if vals[m - 1] - vals[m] >= 2.5 * MARGIN:
                c["min_p"] = float((vals[m - 1] + vals[m]) / 2)
    if want_typ:
        base = dict(c, typical=0.0)
        r = oracle_run(base, logits32, history, banned)
        v = r["probs"]
        lp = np.log(v + 1e-10)
        dev = np.abs((v * lp).sum() - lp)
        o = np.lexsort((r["kept"], dev))
        vv = v[o]
        cum = np.cumsum(vv)
        ok = [n for n in range(1, min(len(vv), 400)) if vv[n] >= 2.5 * MARGIN]
        if not ok:
            return False
        n = ok[rng.integers(len(ok))]
        c["typical"] = float((cum[n - 1] + cum[n]) / 2)
    return True


def main():
    Gen = reference_generator()
    rng = np.random.default_rng(2026)
    cases, hist_all, hist_off, ban_all, ban_off, kept_all, prob_all, kept_off = [], [], [0], [], [0], [], [], [0]

    def add(c, history, banned):
        logits = S.case_logits(c["seed"], c["vocab"], c["kind"])
        r = oracle_run(c, logits, history, banned)
        if r is None or S.min_margin(r) < MARGIN:
            return False
        ids, probs = run_reference(Gen, logits, c, history, banned)
        if not np.array_equal(ids, r["kept"]) or np.abs(probs - r["probs"]).max() > 1e-9:
            return False
        cases.append([c[f] for f in FIELDS])
        hist_all.append(history); hist_off.append(hist_off[-1] + len(history))
        ban_all.append(banned); ban_off.append(ban_off[-1] + len(banned))
        kept_all.append(ids); prob_all.append(probs); kept_off.append(kept_off[-1] + len(ids))
        return True

    seed = 0
    combos = [(p, t, m) for p in (False, True) for t in (False, True) for m in (False, True) if p or not m]
    for vocab in (32000, 32001, 7, 1):
        for temp in (0.3, 0.95, 1.7):
            for top_k in sorted({0, 1, 40, vocab}):
                if top_k > vocab:
                    continue
                for want_p, want_typ, want_min in combos:
                    full = top_k in (0, vocab) and not want_p and not want_typ
                    if full and vocab >= 32000:
                        continue                                    # 32000-wide kept sets: the flat case below is the one stored
                    for attempt in range(6):
                        seed += 1
                        kind = "dominant" if seed % 3 == 0 else "normal"
                        hl = (0, 17, 1920)[seed % 3]
                        sustain, decay = ((-1, 0), (0, 128), (256, 128), (256, 0))[seed % 4]
                        history = rng.integers(0, vocab, size=hl).astype(np.int64)
                        if hl:
                            history[-5:] = history[:5]               # repeated tokens
                        bos = int(rng.integers(vocab)) if seed % 2 else -1
                        banned = rng.choice(vocab, size=min(3, vocab - 1), replace=False).astype(np.int64) if (seed % 5 == 0 and vocab > 1) else np.zeros(0, np.int64)
                        c = dict(seed=seed, vocab=vocab, kind=kind, temperature=temp, top_k=top_k, top_p=0.0, min_p=0.0, typical=0.0,
                                 penalty_max=1.15 if hl else 1.0, sustain=sustain, decay=decay, bos=bos)
                        if (want_p or want_typ) and not place(c, S.case_logits(seed, vocab, kind), history, banned, rng, want_p, want_typ, want_min):
                            continue
                        if add(c, history, banned):
                            break
    # the generator's defaults (temperature 0.95, top_k 40, top_p 0.65, penalty 1.15 / 256 / 128) on a 1920-token history
    for s in range(200, 260):
        history = rng.integers(0, 32000, size=1920).astype(np.int64)
        c = dict(seed=s, vocab=32000, kind="dominant" if s % 2 else "normal", temperature=0.95, top_k=40, top_p=0.65, min_p=0.0,
                 typical=0.0, penalty_max=1.15, sustain=256, decay=128, bos=1)
        if add(c, history, np.zeros(0, np.int64)) and sum(1 for x in cases if x[0] >= 200) >= 3:
            break
    # flat logits: the whole distribution (no cut can be placed with room on a near-flat row)
    for vocab, top_k in ((32000, 32000), (7, 0), (7, 3)):
        c = dict(seed=300 + vocab + top_k, vocab=vocab, kind="flat", temperature=0.95, top_k=top_k, top_p=0.0, min_p=0.0, typical=0.0,
                 penalty_max=1.0, sustain=-1, decay=0, bos=-1)
        add(c, np.zeros(0, np.int64), np.zeros(0, np.int64))
    rows = [[S.KINDS.index(v) if isinstance(v, str) else v for v in row] for row in cases]
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "sample_ref.npz")
    np.savez_compressed(path, fields=np.array(FIELDS), cases=np.array(rows, dtype=np.float64),
                        hist=np.concatenate(hist_all).astype(np.int32), hist_off=np.array(hist_off, np.int64),
                        banned=np.concatenate(ban_all).astype(np.int32), banned_off=np.array(ban_off, np.int64),
                        kept=np.concatenate(kept_all).astype(np.int32), probs=np.concatenate(prob_all), kept_off=np.array(kept_off, np.int64))
    print(f"{len(cases)} cases -> {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
