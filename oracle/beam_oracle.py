"""Float64 restatement of the generator's beam search (ExLlamaGenerator.beam_search, generator.py:497-700), the yardstick of
exl_beam_select (exllama_b200/csrc/beam.cu) and exllama_b200.beam.BeamSearch.

TEST INFRASTRUCTURE ONLY, like sample_oracle.py, on which it is built: every distribution is sample_oracle.sample of the logits
after the committed sequence and the beam's window, with that same token sequence as the penalty history.  The orders the
reference leaves to unstable torch sorts are fixed as DESIGN.md §4f states them: candidates by score descending, then parent
ascending, then token ascending; the kept candidates by parent, then score descending, then token.  Besides the emitted tokens and
the beam set after every expansion, run() reports the margin of every decision it took: the filters' margins (sample_oracle), the
gap between the beams-th and the next candidate score, the gap between the best and the second-best window score, and how far each
first-expansion draw lies from the edges of its cell -- a case with a small margin may be decided the other way by an fp32
implementation.
"""
from __future__ import annotations

import math

import numpy as np

from . import sample_oracle as S

def seq_logits(seed: int, vocab: int, seq, scale: float = 2.0) -> np.ndarray:
    """fp32 logits [vocab] as a function of the whole token sequence (the stub model of the golden fixture, oracle/gen_golden_beam.py)."""
    h = seed * 1000003 + len(seq)
    for t in seq:
        h = (h * 31 + int(t) + 7) % (1 << 61)
    rng = np.random.default_rng(h)
    return (rng.standard_normal(vocab) * scale).astype(np.float32)


def _sample(logits, history, st, bos=-1, banned=(), min_p=None):
    return S.sample(logits, st["temperature"], st["top_k"], st["top_p"], st["min_p"] if min_p is None else min_p, st["typical"],
                    history=np.asarray(history, np.int64), penalty_max=st["penalty_max"], sustain=st["sustain"], decay=st["decay"],
                    bos=bos, banned=banned)


def fix60(p):
    """The sampler's fixed point of an fp32 probability: floor(p * 2^60), exact."""
    return int(float(np.float32(p)) * 2.0 ** 60)


def draw_without_replacement(dist, u):
    """exl_beam_select's first mode on one fp32 row `dist` [vocab] with uniforms u [beams]: min(beams, #positive) successive draws,
    each the smallest remaining id whose inclusive cumulative fixed-point mass, in ascending id order, exceeds
    floor(u_j * remaining total) (in double), or the largest remaining positive id if none does.  Returns (drawn ids in draw order,
    margin: the least distance of u_j * total from the edges of its cell, as a fraction of the remaining total)."""
    ids = [int(i) for i in np.nonzero(np.asarray(dist, np.float32) > 0)[0]]
    mass = {i: fix60(dist[i]) for i in ids}
    out, margin = [], math.inf
    for j in range(min(len(u), len(ids))):
        rem = [i for i in ids if i not in out]
        total = sum(mass[i] for i in rem)
        U = int(float(np.float32(u[j])) * float(total))
        pick, cum = None, 0
        for i in rem:
            lo = cum
            cum += mass[i]
            if cum > U:
                pick = i
                if total:
                    margin = min(margin, (U - lo) / total, (cum - U) / total)
                break
        out.append(rem[-1] if pick is None else pick)
    return out, margin


def expand(dists, scores, beams):
    """exl_beam_select's expand mode in float64 over fp32 rows dists [rows][vocab] and window scores [rows]: the candidates
    (parent, token, p, score = scores[r] + log p) with p > 0, the best min(beams, n) by (score descending, parent, token), laid out
    by (parent, score descending, token).  Returns (kept list of tuples, margin: the gap between the beams-th and the next score)."""
    cands = []
    for r, d in enumerate(dists):
        d = np.asarray(d)
        ids = np.nonzero(d > 0)[0]
        if len(ids) > beams + 1:                                 # within a row the score grows with p: its best beams + 1 suffice
            v = d[ids]
            ids = ids[v >= np.partition(v, len(v) - beams - 1)[len(v) - beams - 1]]
        for t in ids:
            p = float(d[t])
            cands.append((scores[r] + math.log(p), r, int(t), p))
    cands.sort(key=lambda c: (-c[0], c[1], c[2]))
    k = min(beams, len(cands))
    margin = cands[k - 1][0] - cands[k][0] if k < len(cands) else math.inf
    kept = sorted(cands[:k], key=lambda c: (c[1], -c[0], c[2]))
    return [(r, t, p, s) for s, r, t, p in kept], margin


def window_score(probs):
    """A window's score: the float64 sum of the logs of its fp32 probabilities (BeamSearch computes it the same way)."""
    return math.fsum(math.log(p) if p > 0 else -math.inf for p in probs)


def run(logits_fn, prompt, settings, beams, beam_length, n_emit, max_seq, first_draws=None, u_first=None, dist_fn=None, bos=-1,
        banned=()):
    """Beam search over a model given as logits_fn(token sequence) -> fp32 logits [vocab].

    first_draws   the first expansion's tokens, forced (the reference's multinomial draws; any order); or
    u_first       uniforms for draw_without_replacement over the first distribution (as fp32 probabilities)
    dist_fn       optional token sequence -> fp32 [vocab] distribution to use instead of sample_oracle's (a GPU run's dist rows, so
                  that a replay follows that run's probabilities); logits_fn is then not called
    For beams == beam_length == 1 every token is a draw of gen_single_token (bos mask, min_p 0): first_draws gives them all.

    Returns dict(emitted, expansions: the beam windows (lists of tokens, in list order) after each expansion, margins: every
    decision's margin (name, value))."""
    st = dict(settings or {})
    seq = [int(t) for t in prompt]
    margins, expansions, emitted = [], [], []
    vocab = None

    def dist_of(tokens, res):
        if dist_fn is not None:
            return np.asarray(dist_fn(tokens), np.float32)
        d = np.zeros(vocab, np.float64)
        d[res["kept"]] = res["probs"]
        return d

    def sample_at(tokens, **kw):
        nonlocal vocab
        if dist_fn is not None:
            return None
        lg = logits_fn(tokens)
        vocab = lg.shape[0]
        res = _sample(lg, tokens, st, banned=banned, **kw)
        if res is None:
            raise RuntimeError("undefined distribution")
        margins.extend(("filter", v) for v in res["margins"].values())
        return res

    if beams == 1 and beam_length == 1:
        for i in range(n_emit):
            res = sample_at(seq, bos=bos, min_p=0.0)
            t = int(first_draws[i])
            assert t in set(res["kept"].tolist()), (t, res["kept"])
            seq.append(t)
            emitted.append(t)
        return dict(emitted=emitted, expansions=expansions, margins=margins)

    max_beam_length = min(max_seq - beam_length, beam_length)
    res = sample_at(seq)
    d0 = dist_of(seq, res)
    if first_draws is not None:
        toks = sorted(int(t) for t in first_draws)
    else:
        toks, m = draw_without_replacement(np.asarray(d0, np.float32), u_first)
        margins.append(("draw", m))
        toks = sorted(toks)
    beams_l = [([t], [float(d0[t])]) for t in toks]
    expansions.append([list(w) for w, _ in beams_l])
    for _ in range(n_emit):
        while len(beams_l[0][0]) < max_beam_length:
            dists, scores = [], []
            for w, pr in beams_l:
                toks_b = seq + w
                dists.append(dist_of(toks_b, sample_at(toks_b)))
                scores.append(window_score(pr))
            kept, m = expand(dists, scores, beams)
            margins.append(("select", m))
            beams_l = [(beams_l[r][0] + [t], beams_l[r][1] + [p]) for r, t, p, _ in kept]
            expansions.append([list(w) for w, _ in beams_l])
        sc = [window_score(pr) for _, pr in beams_l]
        best = max(range(len(sc)), key=lambda i: (sc[i], -i))
        others = [s for i, s in enumerate(sc) if i != best]
        if others:
            margins.append(("best", sc[best] - max(others)))
        t = beams_l[best][0][0]
        seq.append(t)
        emitted.append(t)
        beams_l = [beams_l[best]] + [b for i, b in enumerate(beams_l) if i != best and b[0][0] == t]
        beams_l = [(w[1:], pr[1:]) for w, pr in beams_l]
    return dict(emitted=emitted, expansions=expansions, margins=margins)


def min_margin(res) -> float:
    return min((v for _, v in res["margins"]), default=math.inf)


def golden_cases(path):
    """The cases of tests/golden/beam_ref.npz (oracle/gen_golden_beam.py): a list of dicts with seed, vocab, settings, beams,
    beam_length, max_seq, prompt, the reference's forced draws, emitted tokens and beam windows after each expansion."""
    import json
    g = np.load(path)
    return json.loads(str(g["cases"]))


def run_case(c):
    """run() on a golden_cases() entry, with the stub model's logits."""
    return run(lambda s: seq_logits(c["seed"], c["vocab"], s), c["prompt"], c["settings"], c["beams"], c["beam_length"],
               len(c["emitted"]), c["max_seq"], first_draws=c["draws"], bos=c.get("bos", -1))
