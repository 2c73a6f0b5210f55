"""Speculative sampling on the device: a small draft model proposes k tokens, the target verifies them in one multi-token step, and
the emitted tokens follow exactly the target's sampling distribution (Leviathan et al. 2023, Chen et al. 2023; csrc/sample.cu,
include/exl_b200.h exl_spec_verify).

    n_acc, tokens, probs = speculative.verify(target_logits, draft_tokens, draft_dist, sampling.Settings(), history=ids, hist_len=n)

    gen = speculative.SpeculativeGenerator(target_stack, draft_stack, target_embed, draft_embed, k=3)
    first = gen.begin(prompt_ids)
    tokens, accepted = gen.generate(128)
"""
from __future__ import annotations

import ctypes as C

import torch

from . import capi, sampling


def verify(target_logits, draft_tokens, draft_dist, settings: sampling.Settings, history=None, hist_len=None, u=None, generator=None,
           bos_token_id=None, banned=None):
    """Verify k draft tokens of one sequence (exl_spec_verify).

    target_logits  fp32 [k + 1, vocab] on the device, unit stride along vocab: row j after the prefix and d_1 .. d_j
    draft_tokens   int64 [k] on the same device
    draft_dist     fp32 [k, vocab] (any row stride, unit stride along vocab): the distribution each draft was drawn from
                   (sampling.sample(..., dist=) of the draft)
    history        int64 token ids on the device (one row, newest last), or None (no penalty); hist_len: how many of them to use
                   (a host int, default all).  Row j's penalty history is those tokens followed by d_1 .. d_j.
    u              fp32 [k + 1] uniforms in [0, 1) on the device; default torch.rand(k + 1, generator=generator)

    Returns (n_accepted int32 [1], tokens int64 [k + 1], probs fp32 [k + 1]) on the device, without synchronising: d_1 .. d_a, the
    correction or bonus token, then -1; n_accepted -1 and every token -1 when a row the walk reached is undefined."""
    for name, t, dt in (("target_logits", target_logits, torch.float32), ("draft_dist", draft_dist, torch.float32)):
        if t.dim() != 2 or t.dtype != dt or not t.is_cuda or t.stride(1) != 1:
            raise ValueError(f"verify: {name} must be CUDA fp32 2-D with unit stride along vocab, got {t.dtype} {tuple(t.shape)} "
                             f"stride {t.stride()} on {t.device}")
    rows, vocab = target_logits.shape
    k = rows - 1
    dev = target_logits.device
    if draft_tokens.shape != (k,) or draft_tokens.dtype != torch.int64 or draft_tokens.device != dev:
        raise ValueError(f"verify: draft_tokens must be int64 [{k}] on {dev}, got {draft_tokens.dtype} {tuple(draft_tokens.shape)} "
                         f"on {draft_tokens.device}")
    if draft_dist.shape != (k, vocab) or draft_dist.device != dev:
        raise ValueError(f"verify: draft_dist must be [{k}, {vocab}] on {dev}, got {tuple(draft_dist.shape)} on {draft_dist.device}")
    if u is None:
        u = torch.rand(k + 1, device=dev, generator=generator)
    u = u.to(device=dev, dtype=torch.float32).contiguous()
    hist_ptr, hl = None, 0
    if history is not None:
        history = history.reshape(-1)
        if history.dtype != torch.int64 or history.device != dev or history.stride(0) != 1:
            raise ValueError(f"verify: history must be contiguous int64 on {dev}, got {history.dtype} on {history.device}")
        hl = history.numel() if hist_len is None else int(hist_len)
        if hl > history.numel():
            raise ValueError(f"verify: hist_len {hl} > the {history.numel()} history tokens given")
        hist_ptr = C.c_void_p(history.data_ptr())
    p, ban = sampling.params(settings, dev, bos_token_id, banned)
    work = torch.empty((k + 1, vocab), dtype=torch.float32, device=dev)
    n_acc = torch.empty(1, dtype=torch.int32, device=dev)
    tokens = torch.empty(k + 1, dtype=torch.int64, device=dev)
    probs = torch.empty(k + 1, dtype=torch.float32, device=dev)
    ld = target_logits.stride(0) if rows > 1 else vocab
    dld = draft_dist.stride(0) if k > 1 else vocab
    with torch.cuda.device(dev):
        capi.check(capi.lib().exl_spec_verify(capi._ptr(target_logits), k, vocab, ld, capi._ptr(draft_tokens), capi._ptr(draft_dist), dld,
                                              hist_ptr, hl, C.byref(p), capi._ptr(u), capi._ptr(work), capi._ptr(n_acc),
                                              capi._ptr(tokens), capi._ptr(probs), capi._stream()))
    return n_acc, tokens, probs


class SpeculativeGenerator:
    """Speculative generation of one sequence with two DecodeStacks that share a vocabulary.

    target, draft          DecodeStacks with an lm_head; cache sequence 0 of each holds the sequence.  They take hidden states,
                           not token ids: target_embed / draft_embed fp16 [vocab, hidden] map a token to each stack's input.
    k                      drafts per round; the target runs on a make_plan(max_tokens=k + 1) plan, the draft on a
                           make_plan(max_tokens=2) plan (both made here; a plan a stack held is closed)
    settings               the target's sampling settings: the emitted tokens follow exactly what sampling.sample would draw
    draft_settings         the draft's (default: settings); they change how many drafts are accepted, never the output's law
    bos_token_id, banned   as sampling.sample, for both models
    generator              a CUDA torch.Generator for every uniform

    A round drafts d_1 .. d_k one token at a time (sampling.sample(..., dist=) of the draft's logits), runs the target once over
    [last token, d_1 .. d_k], and verify() keeps d_1 .. d_a plus one token of the target's.  Token ids, the history and the
    embedding gathers stay on the device; the one host synchronisation per round reads a, because the next round's past_len is a
    host argument of the step.  Rows past the accepted ones are left stale in both caches and overwritten by the next round."""

    def __init__(self, target, draft, target_embed, draft_embed, k=3, settings=None, draft_settings=None, bos_token_id=None,
                 banned=None, generator=None):
        if k < 1:
            raise ValueError(f"SpeculativeGenerator: k {k} must be at least 1")
        for name, st, emb in (("target", target, target_embed), ("draft", draft, draft_embed)):
            if st.lm_head is None:
                raise ValueError(f"SpeculativeGenerator: the {name} stack has no lm_head")
            if emb.dtype != torch.float16 or tuple(emb.shape) != (st.shape.vocab, st.shape.hidden):
                raise ValueError(f"SpeculativeGenerator: {name}_embed must be fp16 [{st.shape.vocab}, {st.shape.hidden}], got "
                                 f"{emb.dtype} {tuple(emb.shape)}")
        if target.shape.vocab != draft.shape.vocab:
            raise ValueError(f"SpeculativeGenerator: target vocab {target.shape.vocab} != draft vocab {draft.shape.vocab}")
        for st in (target, draft):
            if getattr(st, "dplan", None) is not None:
                st.dplan.close()
        try:
            target.make_plan(max_tokens=k + 1)
        except capi.ExlError as e:
            raise ValueError(f"SpeculativeGenerator: the target's multi-token plan cannot take k + 1 = {k + 1} tokens per step; "
                             f"speculation needs at least 2 (k >= 1) and k + 1 at most the plan's max_tokens ({e})") from e
        draft.make_plan(max_tokens=2)
        self.target, self.draft, self.k = target, draft, k
        self.t_emb, self.d_emb = target_embed, draft_embed
        self.settings = settings if settings is not None else sampling.Settings()
        self.draft_settings = draft_settings if draft_settings is not None else self.settings
        self.bos = bos_token_id
        self.dev = target_embed.device
        self.banned = None if banned is None else torch.as_tensor(banned, dtype=torch.int32).reshape(-1).to(self.dev)
        self.gen = generator
        self.max_seq = min(target.max_seq, draft.max_seq)
        self.hist = torch.zeros(self.max_seq + k + 1, dtype=torch.int64, device=self.dev)   # prompt, emitted tokens, drafts
        self.q = torch.empty((k, target.shape.vocab), dtype=torch.float32, device=self.dev)
        self.n = 0                          # tokens of the sequence: prompt + emitted; the last one is in neither cache yet
        self.catch_up = False               # the last round accepted every draft: the draft has not processed d_k

    def _sample(self, logits, settings, hist_len, dist=None):
        return sampling.sample(logits, settings, history=self.hist.view(1, -1), hist_lens=[hist_len], generator=self.gen,
                               bos_token_id=self.bos, banned=self.banned, dist=dist)[0]

    def begin(self, prompt_ids):
        """Prefill the prompt (a 1-D list or tensor of ids) into cache sequence 0 of both stacks and draw the first token from the
        target.  Returns it as a host int."""
        ids = torch.as_tensor(prompt_ids, dtype=torch.int64).reshape(-1).to(self.dev)
        L = ids.numel()
        if L < 1 or L + 1 + self.k > self.max_seq:
            raise ValueError(f"begin: a prompt of {L} tokens does not leave room for a round in max_seq {self.max_seq}")
        self.hist[:L] = ids
        logits = self.target.prefill(self.t_emb[ids].view(1, L, -1), 0, last_only=True)
        self.draft.prefill(self.d_emb[ids].view(1, L, -1), 0, last_only=True)
        self.hist[L:L + 1] = self._sample(logits, self.settings, L)
        self.n, self.catch_up = L + 1, False
        return int(self.hist[L])

    def round(self):
        """One round: returns the number of drafts accepted (the round emitted that many plus one)."""
        k, n = self.k, self.n
        if n + k > self.max_seq:
            raise ValueError(f"round: the sequence holds {n} tokens; a round needs rows up to {n + k} of max_seq {self.max_seq}")
        # drafts: the draft's caches hold rows [0, n - 1), or [0, n - 2) after a round that accepted every draft
        lo = n - 2 if self.catch_up else n - 1
        for j in range(k):
            x = self.d_emb[self.hist[lo:n + j]].view(n + j - lo, 1, -1)
            logits = self.draft.decode_step_fused_multi(x, lo)[-1:]
            self.hist[n + j:n + j + 1] = self._sample(logits, self.draft_settings, n + j, dist=self.q[j:j + 1])
            lo = n + j
        # the target over [last token, d_1 .. d_k] at past n - 1, then the verification
        x = self.t_emb[self.hist[n - 1:n + k]].view(k + 1, 1, -1)
        logits = self.target.decode_step_fused_multi(x, n - 1)
        n_acc, tokens, _ = verify(logits, self.hist[n:n + k], self.q, self.settings, history=self.hist, hist_len=n, generator=self.gen,
                                  bos_token_id=self.bos, banned=self.banned)
        self.hist[n:n + k + 1] = tokens
        a = int(n_acc.item())                                    # the round's one host synchronisation
        if a < 0:
            raise RuntimeError(f"round at {n} tokens: a distribution the verification reached is undefined (NaN logits, or every "
                               f"token masked)")
        self.n, self.catch_up = n + a + 1, a == k
        return a

    def generate(self, n_tokens):
        """Run rounds until at least n_tokens tokens were emitted.  Returns (the emitted token ids as a host list -- the last round
        may add up to k beyond n_tokens --, the number of drafts each round accepted)."""
        if self.n == 0:
            raise RuntimeError("generate: call begin(prompt_ids) first")
        start, accepted = self.n, []
        while self.n - start < n_tokens:
            accepted.append(self.round())
        return self.hist[start:self.n].tolist(), accepted
