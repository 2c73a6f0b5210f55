"""Generates tests/golden/cfg_ref.npz by running the REFERENCE's classifier-free guidance program (example_cfg.py:70-75) with its own
ExLlamaGenerator.sample (generator.py:91-170) on the CPU.

    EXLLAMA_REFERENCE=<reference checkout> python -m oracle.gen_golden_cfg

Per case, two fp32 logits rows (the prompt's and the guidance prompt's, redrawn from their seeds by sample_oracle.case_logits) go
through the example's steps: the repetition penalty of each row over its own history (oracle.apply_rep_penalty, bit-exact with
the reference's rep_penalty.cpp), torch.log_softmax in fp32, the fp32 mix (1 - alpha) * ls[0] + alpha * ls[1] with a Python-float
alpha, and sample() -- as sample_current calls it, without a second penalty or the bos mask -- under gen_golden_sample's stubs, in
float64 with torch.multinomial replaced by a function that returns every index, so sample() hands back the whole kept set with its
final probabilities.  The fixture stores the settings, seeds, histories, the kept ids and probabilities, and each row's torch
logsum (-l at the row's maximum), from which cfg_oracle.golden_row restates the mixed row bit for bit (checked here).  Every
top_p / typical / min_p is placed at a midpoint around a cut of the mixed row (gen_golden_sample.place) and a case is kept only if
every decision has a margin of at least 1e-4 and the float64 oracle agrees with the reference.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import cfg_oracle as F
from . import sample_oracle as S
from .gen_golden_sample import MARGIN, place, reference_generator

ALPHAS = (0.0, 0.5, 1.0, -0.4, 1.4, 3.0)
FILTERS = ("top_k", "top_p_min_p", "typical", "defaults")


def reference_mix(xa, xb, alpha):
    """example_cfg.py:72-73 on two penalised fp32 rows: (mixed fp32 row, logsum of each row)."""
    ls = torch.log_softmax(torch.from_numpy(np.stack([xa, xb])), dim=-1)
    mixed = (1 - alpha) * ls[0] + alpha * ls[1]
    logsum = [-float(ls[r, int(np.argmax(x))]) for r, x in enumerate((xa, xb))]
    return mixed.numpy(), logsum


def run_reference(Gen, mixed, c):
    g = object.__new__(Gen)
    g.disallowed_tokens = None
    real = torch.multinomial
    torch.multinomial = lambda probs, num: torch.arange(probs.shape[-1])
    try:
        toks, probs = g.sample(torch.from_numpy(mixed.astype(np.float64))[None], c["temperature"], c["top_k"], c["top_p"], c["min_p"],
                               c["typical"])
    finally:
        torch.multinomial = real
    return toks[0].numpy().astype(np.int64), probs[0].numpy().astype(np.float64)


def main():
    Gen = reference_generator()
    rng = np.random.default_rng(2027)
    cases, ha_all, hb_all, hist_off, kept_all, prob_all, kept_off = [], [], [], [0], [], [], [0]
    seed = 5000
    for vocab in (32000, 7):
        for ai, alpha in enumerate(ALPHAS):
            for fi, filt in enumerate(FILTERS):
                for attempt in range(8):
                    seed += 2
                    hl = (0, 17, 1920)[(ai + fi + attempt) % 3]
                    kind = "dominant" if (seed // 2) % 3 == 0 else "normal"
                    ha = rng.integers(0, vocab, size=hl).astype(np.int64)
                    hb = rng.integers(0, vocab, size=hl).astype(np.int64)
                    if hl:
                        ha[-5:] = ha[:5]; hb[-5:] = hb[:5]              # repeated tokens
                    c = dict(seed_a=seed, seed_b=seed + 1, vocab=vocab, kind=kind, alpha=alpha, temperature=0.95, top_k=0, top_p=0.0,
                             min_p=0.0, typical=0.0, penalty_max=1.15 if hl else 1.0, sustain=(256, -1, 16)[fi % 3], decay=(128, 0, 64)[fi % 3])
                    if filt == "top_k":
                        c.update(temperature=0.7, top_k=40 if vocab > 40 else 3)
                    elif filt == "defaults":
                        c.update(top_k=40 if vocab > 40 else 3, top_p=0.65, penalty_max=1.15 if hl else 1.0, sustain=256, decay=128)
                    la, lb = S.case_logits(c["seed_a"], vocab, kind), S.case_logits(c["seed_b"], vocab, kind)
                    xa = F.penalised(la, ha, c["penalty_max"], c["sustain"], c["decay"])
                    xb = F.penalised(lb, hb, c["penalty_max"], c["sustain"], c["decay"])
                    mixed, (lga, lgb) = reference_mix(xa, xb, alpha)
                    c["logsum_a"], c["logsum_b"] = lga, lgb
                    row = F.golden_row(la, lb, alpha, lga, lgb, ha, hb, c["penalty_max"], c["sustain"], c["decay"])
                    if not np.array_equal(row.view(np.uint32), mixed.view(np.uint32)):
                        continue                                        # the numpy restatement must be the reference's row, bitwise
                    plain = dict(c, penalty_max=1.0, sustain=-1, decay=0, bos=-1)
                    if filt == "top_p_min_p" and not place(plain, mixed, np.zeros(0, np.int64), np.zeros(0, np.int64), rng, True, False, True):
                        continue
                    if filt == "typical" and not place(plain, mixed, np.zeros(0, np.int64), np.zeros(0, np.int64), rng, False, True, False):
                        continue
                    c.update(top_p=plain["top_p"], min_p=plain["min_p"], typical=plain["typical"])
                    r = S.sample(mixed, c["temperature"], c["top_k"], c["top_p"], c["min_p"], c["typical"])
                    if r is None or S.min_margin(r) < MARGIN:
                        continue
                    ids, probs = run_reference(Gen, mixed, c)
                    if not np.array_equal(ids, r["kept"]) or np.abs(probs - r["probs"]).max() > 1e-9:
                        continue
                    cases.append([S.KINDS.index(v) if isinstance(v, str) else v for v in (c[f] for f in F.FIELDS)])
                    ha_all.append(ha); hb_all.append(hb); hist_off.append(hist_off[-1] + hl)
                    kept_all.append(ids); prob_all.append(probs); kept_off.append(kept_off[-1] + len(ids))
                    break
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "cfg_ref.npz")
    np.savez_compressed(path, fields=np.array(F.FIELDS), cases=np.array(cases, dtype=np.float64),
                        hist_a=np.concatenate(ha_all).astype(np.int32), hist_b=np.concatenate(hb_all).astype(np.int32),
                        hist_off=np.array(hist_off, np.int64), kept=np.concatenate(kept_all).astype(np.int32),
                        probs=np.concatenate(prob_all), kept_off=np.array(kept_off, np.int64))
    print(f"{len(cases)} cases of {2 * len(ALPHAS) * len(FILTERS)} -> {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
