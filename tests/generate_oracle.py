"""Restatements of batched generation (exllama_b200/generate.py, csrc/generate.cu) for the tests: the uniform U(seed, j) in numpy
uint64 arithmetic, exl_gen_advance over numpy arrays, and a request's tokens composed from oracle/sample_oracle.py.  Test
infrastructure only."""
import numpy as np

from oracle import sample_oracle as SO

MAX_STOP = 8
LIVE, STOPPED, ERROR = 0, 1, 4


def U(seed, j):
    """splitmix64 output j (0-based) of the stream seeded with seed, top 24 bits / 2^24 (include/exl_b200.h)."""
    with np.errstate(over="ignore"):
        x = np.uint64(seed) + np.uint64(j + 1) * np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        x = x ^ (x >> np.uint64(31))
    return np.float32(int(x >> np.uint64(40)) / 16777216.0)


def advance(st, tokens, probs, slots, pos, js):
    """exl_gen_advance on the dict of numpy arrays st (hist, status, stop, seeds, embed, x_next, u_next, out_tok, out_prob), in place."""
    for r, s in enumerate(slots):
        if s < 0 or st["status"][s] != LIVE:
            continue
        t, j = int(tokens[r]), int(js[r])
        if not 0 <= t < st["embed"].shape[0]:
            st["out_tok"][s, j], st["out_prob"][s, j], st["status"][s] = -1, np.nan, ERROR
            continue
        st["hist"][s, pos[r]] = t
        st["out_tok"][s, j], st["out_prob"][s, j] = t, probs[r]
        if t in st["stop"][s]:
            st["status"][s] = STOPPED
        st["x_next"][s] = st["embed"][t]
        st["u_next"][s] = U(int(st["seeds"][s]), j + 1)


def token(logits, settings, history, seed, j, bos=None, banned=()):
    """Token j of a request by sample_oracle: (token or None for an undefined row, the smallest decision margin), with u = U(seed, j)."""
    s = settings
    u = float(U(seed, j))
    res = SO.sample(logits, s.temperature, s.top_k, s.top_p, s.min_p, s.typical, history=history,
                    penalty_max=s.token_repetition_penalty_max, sustain=s.token_repetition_penalty_sustain,
                    decay=s.token_repetition_penalty_decay, bos=-1 if bos is None else bos, banned=banned or (), u=u)
    if res is None:
        return None, np.inf
    cdf_gap = float(np.min(np.abs(res["cdf"] - u))) if len(res["cdf"]) else np.inf
    return res["token"], min(SO.min_margin(res), cdf_gap)
