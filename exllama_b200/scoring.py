"""Token log-probabilities and perplexity on the device (csrc/logprob.cu, include/exl_b200.h exl_token_logprobs).

    logprob, greedy = scoring.token_logprobs(hn, lm_head, targets)

takes the final-normed hidden states hn [T, hidden] fp16 (rms_norm's output) and returns, per row, the log-probability of
targets[t] under logits = hn . lm_head^T (fp32 sums of exact fp16 products, never written to memory) and the greedy id, on the same
device and stream with no host synchronisation.  perplexity() scores token-id chunks through a DecodeStack the way the reference's
perplexity.py does, with one host read at the end.
"""
from __future__ import annotations

import ctypes as C
import math

import torch

from . import capi

_work_sizes = {}


def work_size(T, V, device):
    """Bytes of the work buffer exl_token_logprobs needs for T rows and V ids on `device` (cached: a host query, no sync)."""
    key = (int(T), int(V), int(device))
    if key not in _work_sizes:
        n = C.c_int64()
        capi.check(capi.lib().exl_token_logprobs_work_size(key[0], key[1], key[2], C.byref(n)))
        _work_sizes[key] = n.value
    return _work_sizes[key]


def token_logprobs(hn, lm_head, targets, out=None, work=None):
    """(logprob fp32 [T], greedy int64 [T]) of targets int64 [T] given hn fp16 [T, H] and lm_head fp16 [V, H], all contiguous on
    one CUDA device.  logprob[t] = logit[t, targets[t]] - logsumexp(logit[t]); greedy[t] = argmax(logit[t]), ties to the lower id.
    A target outside [0, V) gives NaN; a NaN / inf in hn[t] gives NaN and -1.  An input that does not start 16-byte aligned is
    copied first.  out: optional (logprob, greedy), 16-byte aligned, to write into; work: optional uint8 scratch of at least
    work_size(T, V, device) bytes (both needed to capture the call in a CUDA graph)."""
    if hn.dim() != 2 or hn.dtype != torch.float16 or not hn.is_cuda or not hn.is_contiguous():
        raise ValueError(f"token_logprobs: hn must be contiguous CUDA fp16 [T, H], got {hn.dtype} {tuple(hn.shape)} on {hn.device}")
    T, H = hn.shape
    if lm_head.dim() != 2 or lm_head.dtype != torch.float16 or lm_head.shape[1] != H or not lm_head.is_contiguous():
        raise ValueError(f"token_logprobs: lm_head must be contiguous fp16 [V, {H}], got {lm_head.dtype} {tuple(lm_head.shape)}")
    targets = targets.reshape(-1)
    if targets.dtype != torch.int64 or targets.numel() != T or not targets.is_contiguous():
        raise ValueError(f"token_logprobs: targets must be contiguous int64 [{T}], got {targets.dtype} {tuple(targets.shape)}")
    # the kernel reads 16-byte aligned operands (TMA, vector loads): a view that starts elsewhere is copied
    hn, lm_head, targets = (t if t.data_ptr() % 16 == 0 else t.clone() for t in (hn, lm_head, targets))
    V = lm_head.shape[0]
    dev = hn.device
    if out is None:
        out = (torch.empty(T, dtype=torch.float32, device=dev), torch.empty(T, dtype=torch.int64, device=dev))
    logprob, greedy = out
    need = work_size(T, V, dev.index or 0)
    if work is None:
        work = torch.empty(need, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        capi.check(capi.lib().exl_token_logprobs(capi._ptr(hn), T, H, capi._ptr(lm_head), V, capi._ptr(targets), capi._ptr(logprob),
                                                 capi._ptr(greedy), capi._ptr(work), work.numel() * work.element_size(),
                                                 capi._stream()))
    return logprob, greedy


def perplexity(stack, embed, chunks, per_call=None):
    """exp(-sum logprob / sum targets) over `chunks`, a list of 1-D token-id tensors, by perplexity.py's rule: chunk i's input is
    chunk[:-1] and its targets chunk[1:], and every chunk starts from an empty cache.  embed fp16 [vocab, hidden] maps ids to the
    stack's input.  The chunks go through stack.prefill_ragged(..., targets=) in calls of at most per_call sequences (default
    min(stack.batch, RAGGED_MAX_SEQ)), each into cache sequences 0 .. n-1 at past_len 0; the sum stays on the device until the one
    host read at the end."""
    cap = min(stack.batch, capi.RAGGED_MAX_SEQ)
    per_call = cap if per_call is None else int(per_call)
    if not 1 <= per_call <= cap:
        raise ValueError(f"perplexity: per_call {per_call} outside [1, {cap}]")
    chunks = [torch.as_tensor(c).reshape(-1) for c in chunks]
    for c in chunks:
        if c.numel() < 2:
            raise ValueError(f"perplexity: a chunk of {c.numel()} tokens has no target")
    dev = stack.device
    total = torch.zeros((), dtype=torch.float64, device=dev)
    count = 0
    for i in range(0, len(chunks), per_call):
        group = [c.to(dev, torch.int64) for c in chunks[i:i + per_call]]
        ids = torch.cat([c[:-1] for c in group])
        targets = torch.cat([c[1:] for c in group])
        q_lens = [c.numel() - 1 for c in group]
        logprob, _ = stack.prefill_ragged(embed[ids], q_lens, [0] * len(group), targets=targets)
        total += logprob.double().sum()
        count += targets.numel()
    return math.exp(-float(total) / count)
