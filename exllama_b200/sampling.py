"""Token sampling on the device: the generator's repetition penalty, bos mask, temperature, top-k, top-p (with min-p) and typical
filters and the draw, for every row of a logits batch in one launch (csrc/sample.cu, include/exl_b200.h exl_sample).

    tokens, probs = sampling.sample(logits, sampling.Settings(), history=ids, hist_lens=lens, bos_token_id=1)

takes the logits of DecodeStack.decode_step_fused(_batch) or prefill_ragged as they come ([bsz, vocab] fp32 on the device) and
returns int64 tokens and fp32 probabilities on the same device and stream, with no host synchronisation.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import capi


class Settings:
    """The sampling fields of ExLlamaGenerator.Settings (generator.py:9-19), same names and defaults."""

    temperature = 0.95
    top_k = 40                              # 0: off
    top_p = 0.65                            # 0.0: off
    min_p = 0.0                             # only inside the top-p loop
    typical = 0.0                           # 0.0: off

    token_repetition_penalty_max = 1.15
    token_repetition_penalty_sustain = 256  # -1: the whole history
    token_repetition_penalty_decay = 128


def params(settings: Settings, dev, bos_token_id=None, banned=None):
    """(exl_sample_params of settings, the banned ids as an int32 device tensor or None -- keep it alive until the call is made)."""
    ban = None
    if banned is not None:
        ban = torch.as_tensor(banned, dtype=torch.int32).reshape(-1).to(dev)
    p = capi.ExlSampleParams()
    p.temperature = settings.temperature
    p.top_k = settings.top_k
    p.top_p = settings.top_p
    p.min_p = settings.min_p
    p.typical = settings.typical
    p.rep_penalty_max = settings.token_repetition_penalty_max
    p.rep_sustain = settings.token_repetition_penalty_sustain
    p.rep_decay = settings.token_repetition_penalty_decay
    p.bos_token_id = -1 if bos_token_id is None else int(bos_token_id)
    p.banned = ban.data_ptr() if ban is not None and ban.numel() else None
    p.n_banned = ban.numel() if ban is not None else 0
    return p, ban


def sample(logits, settings: Settings, history=None, hist_lens=None, u=None, generator=None, bos_token_id=None, banned=None,
           dist=None):
    """One token per row of logits [bsz, vocab] fp32 (CUDA, unit stride along vocab; left unchanged).

    history   int64 [bsz, hist_ld] token ids on the logits' device, newest last, or None (no penalty)
    hist_lens the tokens of each history row to use (host ints, default hist_ld each)
    u         fp32 [bsz] uniforms in [0, 1) on the device; default torch.rand(bsz, generator=generator)
    bos_token_id  its logit becomes -10000 after the penalty (generator.py:355); None: untouched
    banned    ids whose logits become -inf (ExLlamaGenerator.disallow_tokens)
    dist      optional fp32 [bsz, vocab] that receives each row's final distribution (0 outside the kept set)

    Returns (tokens int64 [bsz], probs fp32 [bsz]): the drawn token and its final probability; -1 / NaN for a row whose
    distribution is undefined (every logit -inf after masking, a NaN logit, a history id outside the vocabulary)."""
    if logits.dim() != 2 or logits.dtype != torch.float32 or not logits.is_cuda or logits.stride(1) != 1:
        raise ValueError(f"sample: logits must be CUDA fp32 [bsz, vocab] with unit stride along vocab, got {logits.dtype} "
                         f"{tuple(logits.shape)} stride {logits.stride()} on {logits.device}")
    bsz, vocab = logits.shape
    dev = logits.device
    if u is None:
        u = torch.rand(bsz, device=dev, generator=generator)
    u = u.to(device=dev, dtype=torch.float32).contiguous()
    hist_ptr, hist_ld, lens = None, 0, None
    if history is not None:
        if history.dim() != 2 or history.shape[0] != bsz or history.dtype != torch.int64 or history.device != dev:
            raise ValueError(f"sample: history must be int64 [bsz = {bsz}, hist_ld] on {dev}, got {history.dtype} "
                             f"{tuple(history.shape)} on {history.device}")
        history = history.contiguous()
        hist_ld = history.shape[1]
        hl = [hist_ld] * bsz if hist_lens is None else [int(v) for v in hist_lens]
        if len(hl) != bsz:
            raise ValueError(f"sample: {len(hl)} hist_lens for {bsz} rows")
        lens = (C.c_int * bsz)(*hl)
        hist_ptr = C.c_void_p(history.data_ptr())
    p, ban = params(settings, dev, bos_token_id, banned)
    tokens = torch.empty(bsz, dtype=torch.int64, device=dev)
    probs = torch.empty(bsz, dtype=torch.float32, device=dev)
    if dist is not None and (dist.shape != (bsz, vocab) or dist.dtype != torch.float32 or not dist.is_contiguous()):
        raise ValueError(f"sample: dist must be contiguous fp32 [{bsz}, {vocab}], got {dist.dtype} {tuple(dist.shape)}")
    ld = logits.stride(0) if bsz > 1 else vocab          # a one-row view may carry any stride along rows
    with torch.cuda.device(dev):
        capi.check(capi.lib().exl_sample(capi._ptr(logits), bsz, vocab, ld, hist_ptr, hist_ld, lens, C.byref(p),
                                         capi._ptr(u), capi._ptr(tokens), capi._ptr(probs), capi._ptr(dist), capi._stream()))
    return tokens, probs
