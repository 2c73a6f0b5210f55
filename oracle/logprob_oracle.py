"""Float64 restatement of exl_token_logprobs (exllama_b200/csrc/logprob.cu) and the error bound its fp32 arithmetic must meet.

For final-normed hidden states hn fp16 [T, H], lm_head fp16 [V, H] and targets [T]:
    logit[t, v] = sum_k hn[t, k] lm_head[v, k]                      (float64: exact up to 2^-52 of sum_k |hn| |lm_head|)
    lse[t]      = logsumexp_v logit[t, v]
    logprob[t]  = logit[t, targets[t]] - lse[t]                      (NaN for a target outside [0, V), or a non-finite hn row)
    greedy[t]   = argmax_v logit[t, v], ties to the lower id          (-1 for a non-finite hn row)

The kernel's logits are fp32 sums of exact fp16 products on the tensor cores.  Their error is bounded, per (t, v), by
    b[t, v] = n 2^-23 sum_k |hn[t, k]| |lm_head[v, k]|,   n = H / 4 + 16
(one rounding per add of a chain of at most H / 4 partial sums plus the adds inside a k-step; 2^-23 rather than 2^-24 because the
tensor core may truncate when it aligns the products).  The log-sum-exp moves by at most max_v b[t, v] under those errors, and the
fp32 sums of exp and the expf calls add a relative error of at most SUM_REL to the sum, so
    |logprob - want| <= b[t, target] + max_v b[t, v] + SUM_REL + 1e-6 |lse|
and the greedy id is the oracle's wherever the top-two margin exceeds 2 max_v b[t, v].

Works on torch tensors on any device (the GPU tests run it on the device in float64; tests/test_logprob_oracle.py pins it against
scipy.special.log_softmax on the CPU).
"""
from __future__ import annotations

SUM_REL = 80 * 2.0 ** -24          # a 64-term fp32 sum of expf values (2 ulp each), the float64 merges, one fp32 store of the sum


def _blocks(T, V, H, budget=1 << 28):
    """Row-block length such that a [rows, V] float64 block stays within `budget` elements."""
    return max(1, min(T, budget // max(V, 1)))


def logprobs64(hn, lm_head, targets, block=None):
    """dict of float64 / int64 tensors on hn's device, per row: logprob, greedy, lse, logit of the target (NaN if out of range), bound
    (the per-row bound above without the 1e-6 |lse| term), gbound (2 max_v b), margin (top-1 minus top-2 logit over distinct ids)."""
    import torch
    T, H = hn.shape
    V = lm_head.shape[0]
    dev = hn.device
    W = lm_head.to(torch.float64)
    Wa = W.abs()
    targets = targets.reshape(-1).to(dev, torch.int64)
    n = H / 4 + 16
    out = {k: torch.empty(T, dtype=torch.float64, device=dev) for k in ("logprob", "lse", "tlogit", "bound", "gbound", "margin")}
    out["greedy"] = torch.empty(T, dtype=torch.int64, device=dev)
    step = block or _blocks(T, V, H)
    for r in range(0, T, step):
        h = hn[r:r + step].to(torch.float64)
        y = targets[r:r + step]
        logits = h @ W.t()
        bnd = n * 2.0 ** -23 * (h.abs() @ Wa.t())
        lse = torch.logsumexp(logits, dim=1)
        inr = (y >= 0) & (y < V)
        yc = y.clamp(0, V - 1)
        tl = logits.gather(1, yc[:, None])[:, 0]
        tl = torch.where(inr, tl, torch.full_like(tl, float("nan")))
        top2 = logits.topk(min(2, V), dim=1).values
        g = logits.argmax(dim=1)                   # the first maximum: the lower id on a tie
        bmax = bnd.max(dim=1).values
        finite = torch.isfinite(h).all(dim=1)
        nan = torch.full_like(lse, float("nan"))
        out["lse"][r:r + step] = torch.where(finite, lse, nan)
        out["tlogit"][r:r + step] = tl
        out["logprob"][r:r + step] = torch.where(finite, tl - lse, nan)
        out["greedy"][r:r + step] = torch.where(finite, g, torch.full_like(g, -1))
        out["bound"][r:r + step] = bnd.gather(1, yc[:, None])[:, 0] + bmax + SUM_REL
        out["gbound"][r:r + step] = 2 * bmax
        out["margin"][r:r + step] = top2[:, 0] - top2[:, -1] if V > 1 else torch.full_like(lse, float("inf"))
    return out


def torch_program(hn, lm_head, targets):
    """The reference's program (model.py:1077-1080, perplexity.py:118-121): fp16 matmul, .float(), log_softmax, gather.  Returns
    logprob fp32 [T] (targets must be in range)."""
    import torch
    logits = torch.matmul(hn, lm_head.t()).float()
    lp = torch.nn.functional.log_softmax(logits, dim=-1)
    return lp.gather(-1, targets.reshape(-1, 1)).reshape(-1)
