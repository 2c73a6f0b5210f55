"""Beam search on the device: the generator's beams and beam_length (ExLlamaGenerator.beam_search, generator.py:384-700) over the
batched decode step, with candidate selection and cache-row copies as kernels (csrc/beam.cu, include/exl_b200.h exl_beam_select,
exl_kv_copy_rows).

    bs = beam.BeamSearch(stack, embed, beams=4, beam_length=8, settings=sampling.Settings(), generator=g)
    bs.begin(prompt_ids)
    tokens = bs.generate(128)
    committed = bs.end()          # cache sequence 0 now holds rows [0, len(committed) - 1) of the committed sequence

One expansion is one step over the live beams, one exl_sample launch (each beam's final distribution), one exl_beam_select call and
at most one exl_kv_copy_rows launch; the host reads the selection once per expansion (DESIGN.md §4f).
"""
from __future__ import annotations

import copy
import ctypes as C
import math
import time

import numpy as np
import torch

from . import capi, sampling

MAX_BEAMS = 64                                      # EXL_RAGGED_MAX_SEQ: rows and beams of one exl_beam_select call

def select(dist, scores, beams, first=False, u=None, generator=None, out=None):
    """exl_beam_select.

    dist     fp32 [rows, vocab] on the device, unit stride along vocab (sampling.sample(..., dist=) rows: 0 outside the kept set)
    scores   host floats [rows]: each row's window score (sum of the log-probabilities of its beam's window)
    beams    1 .. 64
    first    False: the best min(beams, #candidates) (row, token) pairs by scores[r] + log(p), laid out by row, then score
             descending, then token.  True (one row): min(beams, #candidates) draws without replacement with u, sorted by id.
    u        fp32 [beams] uniforms in [0, 1) on the device (first mode; default torch.rand(beams, generator=generator))
    out      optional SelectResult to write into (one allocation reused across calls)

    Returns a SelectResult on the device, without synchronising; SelectResult.read() copies it to the host in one transfer."""
    if dist.dim() != 2 or dist.dtype != torch.float32 or not dist.is_cuda or dist.stride(1) != 1:
        raise ValueError(f"select: dist must be CUDA fp32 [rows, vocab] with unit stride along vocab, got {dist.dtype} "
                         f"{tuple(dist.shape)} stride {dist.stride()} on {dist.device}")
    rows, vocab = dist.shape
    if len(scores) != rows:
        raise ValueError(f"select: {len(scores)} scores for {rows} rows")
    if not 1 <= beams <= MAX_BEAMS:
        raise ValueError(f"select: beams {beams} outside [1, {MAX_BEAMS}]")
    dev = dist.device
    if first:
        if u is None:
            u = torch.rand(beams, device=dev, generator=generator)
        u = u.to(device=dev, dtype=torch.float32).contiguous()
    res = out if out is not None and out.beams == beams and out.rows >= rows else SelectResult(rows, beams, dev)
    sc = (C.c_double * rows)(*[float(s) for s in scores])
    ld = dist.stride(0) if rows > 1 else vocab
    with torch.cuda.device(dev):
        capi.check(capi.lib().exl_beam_select(capi._ptr(dist), rows, vocab, ld, sc, beams, capi.BEAM_FIRST if first else capi.BEAM_EXPAND,
                                              capi._ptr(u) if first else None, capi._ptr(res.work), res.work.numel(),
                                              capi._ptr(res.parent), capi._ptr(res.token), capi._ptr(res.prob), capi._ptr(res.score),
                                              capi._ptr(res.count), capi._stream()))
    return res


class SelectResult:
    """exl_beam_select's outputs, carved out of one device buffer so that the host reads them in one copy: count int32 [1],
    parent int32 [beams], token int64 [beams], prob fp32 [beams], score float64 [beams]."""

    def __init__(self, rows, beams, dev):
        self.rows, self.beams = rows, beams
        self.buf = torch.empty(24 * beams + 4, dtype=torch.uint8, device=dev)     # score, token (8-byte), parent, prob, count
        self.score = self.buf[:8 * beams].view(torch.float64)
        self.token = self.buf[8 * beams:16 * beams].view(torch.int64)
        self.parent = self.buf[16 * beams:20 * beams].view(torch.int32)
        self.prob = self.buf[20 * beams:24 * beams].view(torch.float32)
        self.count = self.buf[24 * beams:24 * beams + 4].view(torch.int32)
        self.work = torch.empty(capi.beam_work_bytes(64, beams), dtype=torch.uint8, device=dev)

    def read(self):
        """(count, parent, token, prob, score) on the host: the first `count` entries of each (numpy arrays); count -1: a row was
        undefined."""
        h = self.buf.cpu().numpy()
        b = self.beams
        k = int(h[24 * b:24 * b + 4].view(np.int32)[0])
        n = max(k, 0)
        return (k, h[16 * b:20 * b].view(np.int32)[:n], h[8 * b:16 * b].view(np.int64)[:n], h[20 * b:24 * b].view(np.float32)[:n],
                h[:8 * b].view(np.float64)[:n])


def cache_pointers(stack):
    """The host arrays exl_kv_copy_rows takes for stack's caches (build once, pass to copy_cache_rows as ptrs)."""
    kc, vc = stack.key_cache, stack.value_cache
    n = len(kc)
    return ((C.c_void_p * n)(*[t.data_ptr() for t in kc]), (C.c_void_p * n)(*[t.data_ptr() for t in vc]), n, tuple(kc[0].shape),
            kc[0].device)


def copy_cache_rows(stack, pairs, ptrs=None):
    """exl_kv_copy_rows over every layer of stack's caches: pairs is a list of (src, dst, row_lo, row_hi) -- rows [row_lo, row_hi) of
    cache sequence src to the same rows of cache sequence dst.  No sequence may be both a source and a destination, and no
    destination may appear twice.  ptrs: cache_pointers(stack), if the caller keeps it."""
    pairs = [tuple(int(v) for v in p) for p in pairs]
    if not pairs:
        return
    ks, vs, n, (seqs, kvh, max_seq, hd), dev = ptrs if ptrs is not None else cache_pointers(stack)
    arr = (capi.ExlKvCopyPair * len(pairs))(*[capi.ExlKvCopyPair(*p) for p in pairs])
    with torch.cuda.device(dev):
        capi.check(capi.lib().exl_kv_copy_rows(ks, vs, n, seqs, kvh, max_seq, hd, arr, len(pairs), capi._stream()))


class _Beam:
    __slots__ = ("slot", "window", "probs")

    def __init__(self, slot, window, probs):
        self.slot, self.window, self.probs = slot, window, probs

    def score(self):
        """Sum of the log-probabilities of the window (float64 over the fp32 probabilities)."""
        return math.fsum(math.log(p) if p > 0 else -math.inf for p in self.probs)


class BeamSearch:
    """Beam search over one DecodeStack (ExLlamaGenerator.beam_search, generator.py:497-700; DESIGN.md §4f).

    stack          a DecodeStack with an lm_head and batch >= beams: beam b lives in one of cache sequences 0 .. beams - 1
    embed          fp16 [vocab, hidden]: maps a token to the stack's input
    beams          1 .. min(stack.batch, 64)
    beam_length    >= 1; windows grow to min(max_seq - beam_length, beam_length) tokens before the first token is emitted
    settings       sampling.Settings (default: its defaults); bos_token_id, banned as sampling.sample
    generator      a CUDA torch.Generator for the uniforms

    beams == 1 and beam_length == 1 is plain sampling: each token is sampling.sample of the step's logits with the bos mask and
    min_p 0, as gen_single_token does.  Otherwise each expansion steps every live beam, samples each beam's final distribution
    (penalty history: the committed sequence followed by the beam's window), keeps the best `beams` candidates across the beams'
    kept sets (exl_beam_select) and copies cache rows to the slots of cloned beams (exl_kv_copy_rows).  The step is
    decode_step_fused_batch over slots 0 .. highest live slot when stack.make_plan() succeeds, else prefill_ragged over the live
    slots.  trace: set to a list before begin() to record every selection's inputs and outputs (tests).  timings: set to a list
    to record, per expansion, six CUDA events (start, after the step, the sampler, the selection, before and after the copies and
    history updates), the host clock time of the selection read and the number of live beams (tools/beam_bench.py)."""

    def __init__(self, stack, embed, beams, beam_length, settings=None, bos_token_id=None, banned=None, generator=None):
        if stack.tp_size > 1:
            raise NotImplementedError("beam search under tensor parallelism is not implemented")
        if stack.lm_head is None:
            raise ValueError("BeamSearch: the stack has no lm_head")
        if not 1 <= int(beams) <= min(stack.batch, MAX_BEAMS):
            raise ValueError(f"BeamSearch: beams {beams} outside [1, min(stack.batch {stack.batch}, {MAX_BEAMS})]")
        if int(beam_length) < 1:
            raise ValueError(f"BeamSearch: beam_length {beam_length} must be at least 1")
        if embed.dtype != torch.float16 or tuple(embed.shape) != (stack.shape.vocab, stack.shape.hidden):
            raise ValueError(f"BeamSearch: embed must be fp16 [{stack.shape.vocab}, {stack.shape.hidden}], got {embed.dtype} "
                             f"{tuple(embed.shape)}")
        self.st, self.emb = stack, embed
        self.beams, self.beam_length = int(beams), int(beam_length)
        self.settings = settings if settings is not None else sampling.Settings()
        self.bos, self.gen = bos_token_id, generator
        self.dev = embed.device
        self.banned = None if banned is None else torch.as_tensor(banned, dtype=torch.int32).reshape(-1).to(self.dev)
        self.max_seq = stack.max_seq
        self.max_beam_length = min(self.max_seq - self.beam_length, self.beam_length)
        self.simple = self.beams == 1 and self.beam_length == 1
        if getattr(stack, "dplan", None) is not None:
            stack.dplan.close()
            stack.dplan = None
        try:
            stack.make_plan()
            self.fused = True
        except capi.ExlError:
            stack.dplan = None
            self.fused = False
        vocab = stack.shape.vocab
        self.hist = torch.zeros((self.beams, self.max_seq), dtype=torch.int64, device=self.dev)   # each slot's tokens
        self.dist = torch.empty((self.beams, vocab), dtype=torch.float32, device=self.dev)
        self.u0 = torch.zeros(self.beams, dtype=torch.float32, device=self.dev)
        self.sel = SelectResult(self.beams, self.beams, self.dev)
        self.ptrs = cache_pointers(stack)
        # slot indices go to the device through a pinned buffer: row 0 the live slots in list order, row 1 the new beams' slots.  A row
        # is rewritten only after the next selection read, by which time the stream has consumed its last copy.
        self.pin = torch.zeros((2, self.beams), dtype=torch.int64).pin_memory()
        self.idx = torch.zeros((2, self.beams), dtype=torch.int64, device=self.dev)
        self.trace = None
        self.timings = None
        self.seq = []

    # ---- host mirror -------------------------------------------------------------------------------------------------------------
    def _reset(self):
        self.seq = []                                   # the committed sequence: prompt and emitted tokens
        self.tok = np.zeros((self.beams, self.max_seq), np.int64)   # row s, first ntok[s] entries: the tokens slot s's rows are for
        self.ntok = [0] * self.beams
        self.valid = [0] * self.beams                   # leading rows of each slot that hold those tokens' K / V
        self.list = []                                  # live beams, in the reference's list order
        self.pending = None                             # simple mode: logits of the last committed token, not yet sampled

    def _sample(self, logits, rows_hist, hist_len, bos, min_p0, u=None, dist=None):
        s = self.settings
        if min_p0 and s.min_p != 0.0:                   # gen_single_token passes min_p 0 without constraints (generator.py:366)
            s = copy.copy(s)
            s.min_p = 0.0
        return sampling.sample(logits, s, history=rows_hist, hist_lens=[hist_len] * logits.shape[0], u=u, generator=self.gen,
                               bos_token_id=bos, banned=self.banned, dist=dist)

    def begin(self, prompt_ids):
        """Prefill the prompt (a 1-D list or tensor of ids) into cache sequence 0 and run the first expansion."""
        ids = [int(t) for t in torch.as_tensor(prompt_ids, dtype=torch.int64).reshape(-1).tolist()]
        L = len(ids)
        if L < 1 or L + self.beam_length > self.max_seq:
            raise ValueError(f"begin: a prompt of {L} tokens leaves no room for beam_length {self.beam_length} in max_seq {self.max_seq}")
        self._reset()
        ids_dev = torch.tensor(ids, dtype=torch.int64, device=self.dev)
        self.hist[0, :L] = ids_dev
        logits = self.st.prefill(self.emb[ids_dev].view(1, L, -1), 0, last_only=True, seq=0)
        self.seq = list(ids)
        self.tok[0, :L], self.ntok[0], self.valid[0] = ids, L, L
        if self.simple:
            self.pending = logits
            return
        # the first expansion: min(beams, |kept set|) draws without replacement from the final distribution, sorted by id
        self._sample(logits, self.hist[0:1], L, None, False, u=self.u0[:1], dist=self.dist[:1])
        u = torch.rand(self.beams, device=self.dev, generator=self.gen)
        sel = select(self.dist[:1], [0.0], self.beams, first=True, u=u, out=self.sel)
        k, _, tok, prob, _ = sel.read()
        if self.trace is not None:
            self.trace.append(dict(kind="first", dist=self.dist[:1].cpu().numpy(), scores=[0.0], u=u.cpu().numpy(), count=k,
                                   token=tok.tolist(), prob=prob.tolist()))
        if k < 0:
            raise RuntimeError("begin: the distribution after the prompt is undefined (NaN logits, or every token masked)")
        pairs = []
        for j in range(k):
            t = int(tok[j])
            self.list.append(_Beam(j, [t], [float(prob[j])]))
            if j > 0:
                pairs.append((0, j, 0, L))
                self.tok[j, :L], self.valid[j] = ids, L
            self.tok[j, L], self.ntok[j] = t, L + 1
        copy_cache_rows(self.st, pairs, self.ptrs)
        if k > 1:
            self.hist[1:k, :L] = self.hist[0, :L]
        self.hist[:k, L] = sel.token[:k]

    def slot_tokens(self, s):
        """The tokens cache sequence s's rows were computed for (its first valid[s] rows hold their K / V), as a host list."""
        return self.tok[s, :self.ntok[s]].tolist()

    def _common(self, d, src, lim):
        """Length of the common prefix of slot d's and slot src's tokens, at most lim (and at most src's token count)."""
        lim = min(lim, self.ntok[src], self.ntok[d])
        diff = np.flatnonzero(self.tok[d, :lim] != self.tok[src, :lim])
        return int(diff[0]) if diff.size else lim

    def _to_dev(self, row, values):
        """values (host ints) as an int64 device tensor, copied without a host synchronisation."""
        n = len(values)
        self.pin[row, :n] = torch.tensor(values, dtype=torch.int64)
        self.idx[row, :n].copy_(self.pin[row, :n], non_blocking=True)
        return self.idx[row, :n]

    def _step(self, pos, slots, idx=None):
        """Logits [len(slots), vocab] of every live slot's token at position pos (rows in the order of slots; idx: slots on the
        device)."""
        st = self.st
        if self.fused:
            hi = max(slots)
            pasts = [pos if s in slots else min(self.valid[s], self.max_seq - 1) for s in range(hi + 1)]
            x = self.emb[self.hist[:hi + 1, pos]].view(hi + 1, 1, -1)
            if st.batch == 1:
                lg = st.decode_step_fused(x, pos).view(1, -1)
            else:
                lg = st.decode_step_fused_batch(x, pasts)
            if slots != list(range(hi + 1)):
                lg = lg.index_select(0, idx)
            return lg
        x = self.emb[self.hist[idx, pos]]
        n = len(slots)
        return st.prefill_ragged(x, [1] * n, [pos] * n, seqs=slots, last_only=False)     # one token each: every row is a last one

    def _expand(self):
        n, m = len(self.seq), len(self.list[0].window)
        pos = n + m - 1                                 # the position of each beam's last token
        slots = [b.slot for b in self.list]
        nb = len(slots)
        ev = None
        if self.timings is not None:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
            ev[0].record()
        idx = self._to_dev(0, slots)
        logits = self._step(pos, slots, idx)
        for s in slots:
            self.valid[s] = pos + 1
        if ev:
            ev[1].record()
        self._sample(logits, self.hist.index_select(0, idx), pos + 1, None, False, u=self.u0[:nb], dist=self.dist[:nb])
        if ev:
            ev[2].record()
        scores = [b.score() for b in self.list]
        sel = select(self.dist[:nb], scores, self.beams, out=self.sel)
        if ev:
            ev[3].record()
        t0 = time.perf_counter()
        k, parent, tok, prob, score = sel.read()        # the expansion's one host synchronisation
        t_read = time.perf_counter() - t0
        if self.trace is not None:
            self.trace.append(dict(kind="expand", dist=self.dist[:nb].cpu().numpy(), scores=scores, count=k, parent=parent.tolist(),
                                   token=tok.tolist(), prob=prob.tolist(), score=score.tolist(),
                                   windows=[list(b.window) for b in self.list]))
        if k < 0:
            raise RuntimeError(f"expansion at {n} tokens: a beam's distribution is undefined (NaN logits, or every token masked)")
        # slots: a parent's first child keeps the parent's slot, a clone takes the lowest free one
        kept = {self.list[int(p)].slot for p in parent}
        free = [s for s in range(self.beams) if s not in kept]
        new, seen, pairs, hist_moves = [], set(), [], []
        for j in range(k):
            par = self.list[int(parent[j])]
            t, p = int(tok[j]), float(prob[j])
            if par.slot not in seen:
                seen.add(par.slot)
                new.append(_Beam(par.slot, par.window + [t], par.probs + [p]))
                self.tok[par.slot, pos + 1], self.ntok[par.slot] = t, pos + 2
                continue
            d, src = free.pop(0), par.slot
            lo = self._common(d, src, self.valid[d])
            hi = self.valid[src]
            if lo < hi:
                pairs.append((src, d, lo, hi))
            hist_moves.append((src, d, lo))
            self.valid[d] = hi
            self.tok[d, lo:pos + 1] = self.tok[src, lo:pos + 1]
            self.tok[d, pos + 1], self.ntok[d] = t, pos + 2
            new.append(_Beam(d, par.window + [t], par.probs + [p]))
        if ev:
            ev[4].record()
        copy_cache_rows(self.st, pairs, self.ptrs)
        for src, d, lo in hist_moves:
            self.hist[d, lo:pos + 1] = self.hist[src, lo:pos + 1]
        self.hist[self._to_dev(1, [b.slot for b in new]), pos + 1] = sel.token[:k]
        if ev:
            ev[5].record()
            self.timings.append((ev, t_read, nb))
        self.list = new

    def _emit(self):
        best, best_score = None, -math.inf
        for b in self.list:
            s = b.score()
            if best is None or s > best_score:
                best, best_score = b, s
        t = best.window[0]
        self.seq.append(t)
        self.list = [best] + [b for b in self.list if b is not best and b.window[0] == t]
        for b in self.list:
            b.window, b.probs = b.window[1:], b.probs[1:]
        if self.trace is not None:
            self.trace.append(dict(kind="emit", token=t))
        return t

    def next(self):
        """Run expansions until the windows are full, then emit one token (a host int)."""
        if not self.seq:
            raise RuntimeError("next: call begin(prompt_ids) first")
        n = len(self.seq)
        if self.simple:
            if n >= self.max_seq:
                raise ValueError(f"next: the sequence holds {n} tokens; there is no room for another in max_seq {self.max_seq}")
            if self.pending is None:
                self.pending = self._step(n - 1, [0], self._to_dev(0, [0]))
                self.valid[0] = n
            tok, _ = self._sample(self.pending, self.hist[0:1], n, self.bos, True)
            self.pending = None
            t = int(tok.item())
            if t < 0:
                raise RuntimeError(f"next at {n} tokens: the distribution is undefined (NaN logits, or every token masked)")
            self.hist[0, n] = t
            self.seq.append(t)
            self.tok[0, n], self.ntok[0] = t, n + 1
            return t
        if n + self.max_beam_length > self.max_seq:
            raise ValueError(f"next: the sequence holds {n} tokens; windows of {self.max_beam_length} do not fit max_seq {self.max_seq}")
        while len(self.list[0].window) < self.max_beam_length:
            self._expand()
        return self._emit()

    def generate(self, n_tokens):
        """n_tokens calls of next(); returns the emitted tokens as a host list."""
        return [self.next() for _ in range(int(n_tokens))]

    def end(self):
        """Leave cache sequence 0 holding rows [0, n - 1) of the committed sequence of n tokens (copied from a surviving beam's slot if
        slot 0 holds none), so that a caller can go on with decode_step_fused(embed[last], n - 1) or prefill(..., n - 1, seq=0).
        Returns the committed sequence as a host list."""
        n = len(self.seq)
        if self.list and all(b.slot != 0 for b in self.list):
            src = self.list[0].slot
            lo = self._common(0, src, min(self.valid[0], n - 1))
            if lo < n - 1:
                copy_cache_rows(self.st, [(src, 0, lo, n - 1)], self.ptrs)
            self.hist[0, :n] = self.hist[src, :n]
            self.tok[0], self.ntok[0], self.valid[0] = self.tok[src], self.ntok[src], n - 1
        out = list(self.seq)
        self.list = []
        return out
