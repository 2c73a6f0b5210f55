"""What the generation drivers (generate.BatchGenerator, beam.BeamSearch, speculative.SpeculativeGenerator) share: the check of a
stack and its embedding, the opening of the stack's fused plan, and one token stepped for a set of cache slots on the fused plan
or on prefill_ragged (DESIGN.md §4f-§4h).
"""
from __future__ import annotations

import torch

from . import capi


def check_stack(who, stack, embed, contiguous=False):
    """Refuse a stack the drivers cannot step (tensor parallelism, no lm_head) and an embed that is not fp16 [vocab, hidden] of
    it.  contiguous: embed must also be contiguous (exl_gen_advance gathers its rows through the raw pointer; torch indexing does
    not need it)."""
    if stack.tp_size > 1:
        raise NotImplementedError(f"{who} under tensor parallelism is not implemented")
    if stack.lm_head is None:
        raise ValueError(f"{who}: the stack has no lm_head")
    V, H = stack.shape.vocab, stack.shape.hidden
    if embed.dtype != torch.float16 or tuple(embed.shape) != (V, H) or (contiguous and not embed.is_contiguous()):
        raise ValueError(f"{who}: embed must be {'contiguous ' if contiguous else ''}fp16 [{V}, {H}], got {embed.dtype} "
                         f"{tuple(embed.shape)}")


def open_plan(stack, **kw):
    """Close the plan stack holds and make stack.make_plan(**kw) its plan.  Returns None, or the ExlError of a stack that has no
    such plan (act-order with a batch, more sequences than the plan takes, more tokens than a multi-token plan takes); the stack
    then holds no plan."""
    if stack.dplan is not None:
        stack.dplan.close()
        stack.dplan = None
    try:
        stack.make_plan(**kw)
    except capi.ExlError as e:
        return e
    return None


def step_slots(stack, fused, x_of, live, pasts, idx):
    """One token for each cache slot in live (distinct host ints), the token of slot s at position pasts[s].

    x_of    x_of(i) -> the input rows fp16 [len, hidden] of the slots i (a slice or an int64 device tensor of slots)
    pasts   the past_len of every slot 0 .. max(live), exactly that many; the caller chooses it for a slot not in live, which the
            fused route steps too (its row past_len is written)
    idx     live on the device (the ragged route's gather), or None on the fused route

    The fused route (a plan of stack.make_plan(), fused True) is one decode_step_fused_batch over slots 0 .. max(live), or
    decode_step_fused on a one-sequence stack; otherwise one prefill_ragged with one token per live slot.  Returns (logits
    [rows, vocab] fp32, the slot of each row): slots 0 .. max(live) in order on the fused route, live in its order on the other."""
    if fused:
        n = max(live) + 1
        x = x_of(slice(0, n)).view(n, 1, -1)
        logits = stack.decode_step_fused(x, pasts[0]).view(1, -1) if stack.batch == 1 else stack.decode_step_fused_batch(x, pasts)
        return logits, list(range(n))
    n = len(live)
    return stack.prefill_ragged(x_of(idx), [1] * n, [pasts[s] for s in live], seqs=list(live), last_only=False), list(live)
