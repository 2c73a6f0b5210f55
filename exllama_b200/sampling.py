"""Token sampling on the device: the generator's repetition penalty, bos mask, temperature, top-k, top-p (with min-p) and typical
filters and the draw, for every row of a logits batch in one launch (csrc/sample.cu, include/exl_b200.h exl_sample, and
exl_sample_rows when each row has its own settings).

    tokens, probs = sampling.sample(logits, sampling.Settings(), history=ids, hist_lens=lens, bos_token_id=1)

takes the logits of DecodeStack.decode_step_fused(_batch) or prefill_ragged as they come ([bsz, vocab] fp32 on the device) and
returns int64 tokens and fp32 probabilities on the same device and stream, with no host synchronisation.

    lp, ids, top = sampling.top_logprobs(logits, 5, tokens)

gives the model's log-probability of each row's token and the row's 5 most likely tokens with theirs (csrc/toplp.cu, include/exl_b200.h
exl_top_logprobs): the unprocessed distribution, before any penalty, temperature or filter.
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


def row_params(settings, bsz, dev, bos_token_id=None, banned=None):
    """(a ctypes array of bsz exl_sample_params, the banned tensors to keep alive) for exl_sample_rows: settings is a list of bsz
    Settings; bos_token_id None, one id for every row, or a list of bsz (None or an id); banned None or a list of bsz (None or ids)."""
    settings = list(settings)
    if len(settings) != bsz:
        raise ValueError(f"sample: {len(settings)} settings for {bsz} rows")
    bos = bos_token_id if isinstance(bos_token_id, (list, tuple)) else [bos_token_id] * bsz
    ban = [None] * bsz if banned is None else list(banned)
    if len(bos) != bsz or len(ban) != bsz:
        raise ValueError(f"sample: {len(bos)} bos ids and {len(ban)} banned lists for {bsz} rows")
    arr = (capi.ExlSampleParams * bsz)()
    keep = []
    for b in range(bsz):
        arr[b], t = params(settings[b], dev, bos[b], ban[b])
        keep.append(t)
    return arr, keep


def check_rows(who, t, name="logits"):
    """(rows, vocab) of t, which the row-wise kernels take only as CUDA fp32 [rows, vocab] with unit stride along vocab."""
    if t.dim() != 2 or t.dtype != torch.float32 or not t.is_cuda or t.stride(1) != 1:
        raise ValueError(f"{who}: {name} must be CUDA fp32 [rows, vocab] with unit stride along vocab, got {t.dtype} "
                         f"{tuple(t.shape)} stride {t.stride()} on {t.device}")
    return t.shape


def row_ld(t):
    """The row stride of t [rows, vocab] as the row-wise kernels take it: a one-row view may carry any stride along rows."""
    return t.stride(0) if t.shape[0] > 1 else t.shape[1]


def history_args(who, history, hist_lens, rows, dev):
    """A penalty history as the row-wise kernels take it: (history int64 [rows, hist_ld] contiguous -- keep it until the call is
    made --, hist_ld, a c_int array of each row's length), or (None, 0, None) for history None.  hist_lens: host ints, default
    hist_ld each."""
    if history is None:
        return None, 0, None
    if history.dim() != 2 or history.shape[0] != rows or history.dtype != torch.int64 or history.device != dev:
        raise ValueError(f"{who}: history must be int64 [rows = {rows}, hist_ld] on {dev}, got {history.dtype} "
                         f"{tuple(history.shape)} on {history.device}")
    history = history.contiguous()
    hist_ld = history.shape[1]
    hl = [hist_ld] * rows if hist_lens is None else [int(v) for v in hist_lens]
    if len(hl) != rows:
        raise ValueError(f"{who}: {len(hl)} hist_lens for {rows} rows")
    return history, hist_ld, (C.c_int * rows)(*hl)


def launch(logits, hist, p, u, tokens, probs, dist=None):
    """exl_sample on the current device and stream, or exl_sample_rows when p is an array of ExlSampleParams (one per row, or
    more) rather than one: logits as check_rows takes them, hist = history_args(...), u fp32 [rows] on the device; writes tokens,
    probs and dist."""
    rows, vocab = logits.shape
    history, hist_ld, lens = hist
    one = isinstance(p, capi.ExlSampleParams)
    fn = capi.lib().exl_sample if one else capi.lib().exl_sample_rows
    capi.check(fn(capi._ptr(logits), rows, vocab, row_ld(logits), capi._ptr(history), hist_ld, lens, C.byref(p) if one else p,
                  capi._ptr(u), capi._ptr(tokens), capi._ptr(probs), capi._ptr(dist), capi._stream()))


def sample(logits, settings, history=None, hist_lens=None, u=None, generator=None, bos_token_id=None, banned=None, dist=None):
    """One token per row of logits [bsz, vocab] fp32 (CUDA, unit stride along vocab; left unchanged).

    settings  a Settings for every row (exl_sample), or a list of bsz Settings, row b using settings[b] (exl_sample_rows); with a
              list, bos_token_id may also be a list of bsz ids (None: untouched) and banned a list of bsz id lists (None: none)

    history   int64 [bsz, hist_ld] token ids on the logits' device, newest last, or None (no penalty)
    hist_lens the tokens of each history row to use (host ints, default hist_ld each)
    u         fp32 [bsz] uniforms in [0, 1) on the device; default torch.rand(bsz, generator=generator)
    bos_token_id  its logit becomes -10000 after the penalty (generator.py:355); None: untouched
    banned    ids whose logits become -inf (ExLlamaGenerator.disallow_tokens)
    dist      optional fp32 [bsz, vocab] that receives each row's final distribution (0 outside the kept set)

    Returns (tokens int64 [bsz], probs fp32 [bsz]): the drawn token and its final probability; -1 / NaN for a row whose
    distribution is undefined (every logit -inf after masking, a NaN logit, a history id outside the vocabulary)."""
    bsz, vocab = check_rows("sample", logits)
    dev = logits.device
    if u is None:
        u = torch.rand(bsz, device=dev, generator=generator)
    u = u.to(device=dev, dtype=torch.float32).contiguous()
    hist = history_args("sample", history, hist_lens, bsz, dev)
    if isinstance(settings, (list, tuple)):
        p, ban = row_params(settings, bsz, dev, bos_token_id, banned)
    else:
        p, ban = params(settings, dev, bos_token_id, banned)
    tokens = torch.empty(bsz, dtype=torch.int64, device=dev)
    probs = torch.empty(bsz, dtype=torch.float32, device=dev)
    if dist is not None and (dist.shape != (bsz, vocab) or dist.dtype != torch.float32 or not dist.is_contiguous()):
        raise ValueError(f"sample: dist must be contiguous fp32 [{bsz}, {vocab}], got {dist.dtype} {tuple(dist.shape)}")
    with torch.cuda.device(dev):
        launch(logits, hist, p, u, tokens, probs, dist)
    return tokens, probs


def top_logprobs(logits, n, tokens=None):
    """The model's log-probabilities at each row of logits [rows, vocab] (as check_rows takes them; left unchanged): exl_top_logprobs.

    n       0 .. capi.TOPLP_MAX alternatives per row
    tokens  int64 [rows] on the device (e.g. sample's tokens), or None

    Returns (lp fp32 [rows], ids int64 [rows, n], top fp32 [rows, n]) on the device, without synchronising: lp the log-probability of
    tokens[r] (NaN for no token, a token outside the vocabulary or an undefined row); ids / top the n largest finite logits' ids and
    log-probabilities in descending order, a tie to the lower id (-1 / -inf past the row's finite entries; -1 / NaN on an undefined
    row: a NaN or +inf logit, or no finite one)."""
    rows, vocab = check_rows("top_logprobs", logits)
    dev = logits.device
    n = int(n)
    if tokens is not None and (tokens.shape != (rows,) or tokens.dtype != torch.int64 or tokens.device != dev or not tokens.is_contiguous()):
        raise ValueError(f"top_logprobs: tokens must be contiguous int64 [{rows}] on {dev}, got {tokens.dtype} {tuple(tokens.shape)} "
                         f"on {tokens.device}")
    lp = torch.empty(rows, dtype=torch.float32, device=dev)
    ids = torch.empty((rows, n), dtype=torch.int64, device=dev)
    top = torch.empty((rows, n), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        launch_top_logprobs(logits, tokens, n, lp, ids, top, max(n, 1))
    return lp, ids, top


def launch_top_logprobs(logits, tokens, n, lp, ids, top, top_ld, slots=None, js=None, status=None, out_ld=0):
    """exl_top_logprobs on the current device and stream (logits as check_rows takes them); with slots (host ints, -1: none), js
    (host ints) and status (int32 device), row r writes lp / ids / top row [slots[r]][js[r]] while that slot is live."""
    rows, vocab = logits.shape
    arr = lambda v: None if v is None else (C.c_int * rows)(*[int(x) for x in v])
    n_slots = 0 if status is None else status.shape[0]
    capi.check(capi.lib().exl_top_logprobs(capi._ptr(logits), rows, vocab, row_ld(logits), capi._ptr(tokens), n, arr(slots), arr(js),
                                           capi._ptr(status), n_slots, out_ld, capi._ptr(lp), capi._ptr(ids), capi._ptr(top), top_ld,
                                           capi._stream()))
