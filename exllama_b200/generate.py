"""Batched generation on the device: many requests, each with its own settings, seed, stop ids, bos id and banned list, through the
stack's cache sequences, with a slot refilled as soon as its request finishes (continuous batching; DESIGN.md §4g).

    gen = generate.BatchGenerator(stack, embed)
    rid = gen.submit(generate.Request(prompt_ids, max_new_tokens=128, settings=s, stop_ids=[eos], seed=7))
    results = gen.run()                          # {id: Result(tokens, probs, finish, t_first)}

Cache sequence s of the stack is slot s.  Each step() steps every live request by one token, then admits waiting requests into the
lowest free slots (their prompts in one prefill_ragged, their first tokens through one exl_sample_rows and one exl_gen_advance).  A
step is one slots.step_slots (a decode_step_fused_batch over slots 0 .. highest live slot, or a ragged prefill when the stack has no
fused plan), one exl_sample_rows with each row's own settings and one exl_gen_advance, which appends the tokens, tests the stop ids
and writes the next step's input rows and uniforms on the device.  The host never waits on the step in flight: length and cache-full
finishes are decided on the host, and the device status (stop, error) of step k - 1 is read after step k has been launched.  A
request that stopped at step k - 1 is therefore stepped once more; exl_gen_advance ignores that row (the status is sticky), and its
slot is freed one step late.

Token j of a request is what sampling.sample returns for its logits row with the request's settings, bos id and banned list,
history = prompt + tokens 0 .. j - 1, and u = uniform(seed, j) (include/exl_b200.h U), so a request's tokens do not depend on
which other requests share its steps.

A guided request (Request(cfg_prompt=, cfg_alpha=), classifier-free guidance, DESIGN.md §4h) owns two slots: its prompt's and a
shadow slot for cfg_prompt, stepped with the same tokens.  Between the step and the sampler, exl_cfg_mix penalises each of its two
rows over its own slot's history and writes (1 - cfg_alpha) * l_prompt + cfg_alpha * l_cfg (log-softmaxed rows) to both; its
token j is then sampling.sample of that mixed row with the request's settings, bos id and banned list, no history (the penalty
was applied in the mix) and u = uniform(seed, j).  Both slots carry the same sampler settings and seed, so both rows draw the same
token and exl_gen_advance appends it to both.

A request with logprobs=N (1 .. capi.TOPLP_MAX) also gets, per token, the model's log-probability of that token and its N most likely
tokens with theirs (DESIGN.md §4i): exl_top_logprobs runs between the sampler and exl_gen_advance over the same logits rows the
sampler read (a guided request's mixed rows), whenever a row of the launch asks, and writes each asking row's results into its
slot's output rows under exl_gen_advance's status gate.  The tokens, probs and finishes are those of the same request without it.
"""
from __future__ import annotations

import collections
import copy
import ctypes as C
import math
import time

import torch

from . import capi, cfg, sampling
from .slots import check_stack, open_plan, step_slots

MAX_STOP = capi.GEN_MAX_STOP
_M64 = (1 << 64) - 1


def uniform(seed, j):
    """U(seed, j) of include/exl_b200.h: splitmix64 output j (0-based) of the stream seeded with seed, top 24 bits / 2^24 (a float
    that fp32 holds exactly)."""
    x = (int(seed) + (int(j) + 1) * 0x9E3779B97F4A7C15) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    x ^= x >> 31
    return (x >> 40) / float(1 << 24)


class Request:
    """One completion to generate.  prompt_ids: a non-empty 1-D list or tensor of ids; max_new_tokens >= 1; settings: a
    sampling.Settings (default its defaults), used as given; stop_ids: up to MAX_STOP ids that end the request (the stop token is
    kept); seed: the request's uniforms are uniform(seed, j); bos_token_id, banned: as sampling.sample.  cfg_prompt: None, or a
    non-empty list or tensor of ids, the guidance prompt of classifier-free guidance with weight cfg_alpha (a finite float; 0 gives
    the prompt's log-probabilities, 1 the guidance prompt's); the request then takes two slots (module docstring).  logprobs: 0 (off)
    or N in 1 .. capi.TOPLP_MAX, the number of alternatives reported per token in Result.top_logprobs."""

    def __init__(self, prompt_ids, max_new_tokens, settings=None, stop_ids=(), seed=0, bos_token_id=None, banned=None, cfg_prompt=None,
                 cfg_alpha=0.0, logprobs=0):
        self.prompt = [int(t) for t in torch.as_tensor(prompt_ids, dtype=torch.int64).reshape(-1).tolist()]
        self.max_new_tokens = int(max_new_tokens)
        self.settings = settings if settings is not None else sampling.Settings()
        self.stop_ids = [int(t) for t in stop_ids]
        self.seed = int(seed) & _M64
        self.bos_token_id = bos_token_id
        self.banned = None if banned is None else [int(t) for t in banned]
        self.cfg_prompt = None if cfg_prompt is None else [int(t) for t in torch.as_tensor(cfg_prompt, dtype=torch.int64).reshape(-1).tolist()]
        self.cfg_alpha = float(cfg_alpha)
        self.logprobs = int(logprobs)
        if not 0 <= self.logprobs <= capi.TOPLP_MAX:
            raise ValueError(f"Request: logprobs {self.logprobs} outside [0, {capi.TOPLP_MAX}]")
        if self.cfg_prompt is not None and not self.cfg_prompt:
            raise ValueError("Request: the cfg_prompt is empty")
        if not math.isfinite(self.cfg_alpha):
            raise ValueError(f"Request: cfg_alpha {self.cfg_alpha} is not finite")
        if not self.prompt:
            raise ValueError("Request: the prompt is empty")
        if self.max_new_tokens < 1:
            raise ValueError(f"Request: max_new_tokens {self.max_new_tokens} must be at least 1")
        if len(self.stop_ids) > MAX_STOP:
            raise ValueError(f"Request: {len(self.stop_ids)} stop ids, at most {MAX_STOP}")


class Result:
    """tokens, probs: host lists of the generated tokens and their final probabilities; finish: "stop" (the last token is a stop
    id), "length" (max_new_tokens), "max_seq" (the cache sequence is full) or "error" (an undefined distribution: NaN logits, or
    every token masked; tokens then holds the ones before it); t_first: seconds from submit() to the host's first sight of the
    first token (one step after it was drawn, as every status read).  For a request with logprobs=N (None otherwise): logprobs, the
    model's log-probability of each token (its raw logits row, or a guided request's mixed row, before any penalty, temperature or
    filter); top_logprobs, per token a list of the N (id, log-probability) pairs with the largest logits, in descending order (fewer
    when the row has fewer finite logits)."""

    def __init__(self):
        self.tokens, self.probs, self.finish, self.t_first = [], [], None, None
        self.logprobs, self.top_logprobs = None, None
        self._fetch, self._n = None, None

    def _settle(self):
        if self._fetch is not None:
            ev, tok, prob, *lps = self._fetch
            ev.synchronize()
            t, p = tok.tolist(), prob.tolist()
            n = t.index(-1) if -1 in t else len(t)
            self.tokens, self.probs = t[:n], p[:n]
            if lps:
                lp, ids, top = (x.tolist() for x in lps)
                self.logprobs = lp[:n]
                self.top_logprobs = [[(i, v) for i, v in zip(ids[k], top[k]) if i >= 0] for k in range(n)]
            self._fetch = None


class _Live:
    """A request in a slot.  A guided request has two: the primary (its prompt; it decides finishes and holds the tokens fetched)
    and a shadow (cfg_prompt), linked through pair; a plain request's pair is None."""
    __slots__ = ("rid", "req", "slot", "L", "n", "t0", "host_finish", "prompt", "pair", "shadow")

    def __init__(self, rid, req, slot, t0, shadow=False):
        self.prompt = req.cfg_prompt if shadow else req.prompt
        self.rid, self.req, self.slot, self.L, self.n, self.t0 = rid, req, slot, len(self.prompt), 0, t0
        self.host_finish = None
        self.pair, self.shadow = None, shadow


class Scheduler:
    """The host side of batched generation: admission, slots, positions and finishes.  dev carries out the device work (_Device for
    a DecodeStack; tests substitute a fake): admit(lives), step(lives), copy_status() -> i (an index), read_status(i) -> the status of every slot when copy i was made (host int array), fetch(live, n)
    -> (event, tokens, probs), or (event, tokens, probs, lp, ids, top) for a request with logprobs, release(slot)."""

    def __init__(self, dev, n_slots, max_seq):
        self.dev, self.n_slots, self.max_seq = dev, int(n_slots), int(max_seq)
        self.waiting = collections.deque()
        self.slots = [None] * self.n_slots
        self.results = {}
        self.order = []                     # (iteration, "admit" | "step" | "release" | "finish", ...) events, for tests
        self._next_id = 0
        self._lag = None                    # (copy index, [(live, tokens issued)]) of the previous status copy, not read yet
        self._k = 0

    def submit(self, req):
        if len(req.prompt) + 1 > self.max_seq:
            raise ValueError(f"submit: a prompt of {len(req.prompt)} tokens leaves no room for a token in max_seq {self.max_seq}")
        if req.cfg_prompt is not None:
            if self.n_slots < 2:
                raise ValueError(f"submit: a guided request takes two slots, the stack has {self.n_slots}")
            if len(req.cfg_prompt) + 1 > self.max_seq:
                raise ValueError(f"submit: a cfg_prompt of {len(req.cfg_prompt)} tokens leaves no room for a token in max_seq {self.max_seq}")
        rid = self._next_id
        self._next_id += 1
        self.waiting.append((rid, req, time.perf_counter()))
        self.results[rid] = Result()
        return rid

    def _limit(self, lv):
        """The host's finish of lv after its tokens so far, or None."""
        if lv.n >= lv.req.max_new_tokens:
            return "length"
        if max(lv.L, lv.pair.L if lv.pair is not None else 0) + lv.n >= self.max_seq:      # a guided request: its longer prompt
            return "max_seq"
        return None

    def _fetch(self, lv, n):
        res = self.results[lv.rid]
        if res._n != n:                     # an earlier fetch of a different count is replaced before the slot can be reused
            res._fetch, res._n = self.dev.fetch(lv, n), n

    def _finish(self, lv, reason, n):
        self.results[lv.rid].finish = reason
        self._fetch(lv, n)
        if self.slots[lv.slot] is lv:
            self._release(lv)
        self.order.append((self._k, "finish", lv.rid, lv.slot, reason))

    def _release(self, lv):
        for x in (lv, lv.pair) if lv.pair is not None else (lv,):
            self.slots[x.slot] = None
            self.dev.release(x.slot)
            self.order.append((self._k, "release", x.rid, x.slot))

    def step(self):
        """One iteration: one step of the live requests, admissions (prompt and first token), the status read of the previous iteration.  Returns
        False when nothing was left to do."""
        live = [lv for lv in self.slots if lv is not None]
        if not self.waiting and not live and self._lag is None:
            return False
        adm, tokens = [], 0
        # waiting requests in order into the lowest free slots (a guided request into the two lowest, and nothing overtakes one
        # that waits for them), at most max_seq prompt tokens in one admission (the prefill's scratch is sized for max_seq rows);
        # the first one always goes
        while self.waiting:
            req = self.waiting[0][1]
            free = [s for s, x in enumerate(self.slots) if x is None]
            cost = len(req.prompt) + (len(req.cfg_prompt) if req.cfg_prompt is not None else 0)
            if len(free) < (1 if req.cfg_prompt is None else 2) or (adm and tokens + cost > self.max_seq):
                break
            rid, req, t0 = self.waiting.popleft()
            tokens += cost
            lv = _Live(rid, req, free[0], t0)
            self.slots[free[0]] = lv
            adm.append(lv)
            if req.cfg_prompt is not None:
                sh = _Live(rid, req, free[1], t0, shadow=True)
                lv.pair, sh.pair = sh, lv
                self.slots[free[1]] = sh
                adm.append(sh)
        run = live
        # the step first: a fused step covers free slots at past_len 0 and writes their row 0, which the admission's prefill then
        # overwrites
        if run:
            self.dev.step(run)
            for lv in run:
                lv.n += 1
            self.order.append((self._k, "step", [(lv.slot, lv.L + lv.n - 2) for lv in run]))
        if adm:
            self.dev.admit(adm)
            for lv in adm:
                lv.n = 1
            self.order.append((self._k, "admit", [(lv.rid, lv.slot) for lv in adm]))
        snap = []
        for lv in adm + run:
            if lv.shadow:
                continue                    # a guided request finishes through its primary
            snap.append((lv, lv.n))
            lv.host_finish = self._limit(lv)
        copy = self.dev.copy_status() if snap else None
        # a request the host has finished is stepped no more: free its slot(s) now (a stop or error in its last token is settled
        # from the status read that covers it)
        for lv, _ in snap:
            if lv.host_finish is not None:
                self._fetch(lv, lv.n)
                self._release(lv)
        if self._lag is not None:
            status = self.dev.read_status(self._lag[0])
            now = time.perf_counter()
            for lv, n in self._lag[1]:
                res = self.results[lv.rid]
                if res.t_first is None:
                    res.t_first = now - lv.t0
                if res.finish is not None:
                    continue
                st = int(status[lv.slot])
                if st == capi.GEN_STOPPED:
                    self._finish(lv, "stop", n)
                elif st == capi.GEN_ERROR:
                    self._finish(lv, "error", n)
                elif lv.host_finish is not None and n == lv.n:
                    self._finish(lv, lv.host_finish, n)
        self._lag = (copy, snap) if snap else None
        self._k += 1
        return True

    def run(self):
        """step() until every submitted request has finished; returns {id: Result}."""
        while self.step():
            pass
        for res in self.results.values():
            res._settle()
        return self.results


def fused_rows(lives):
    """The rows of a fused step over the requests lives: slots 0 .. highest live slot, each live slot's request (its last token at
    position L + n - 1, the past_len it is stepped at), None and past_len 0 for a free slot (its row reads no history and the next
    prefill into that slot overwrites the row it writes).  Returns (rows, past_lens)."""
    by_slot = {lv.slot: lv for lv in lives}
    rows = [by_slot.get(s) for s in range(max(by_slot) + 1)]
    return rows, [lv.L + lv.n - 1 if lv is not None else 0 for lv in rows]


class _Device:
    """The device side of BatchGenerator over a DecodeStack: per-slot history, status, stop ids, seeds, next inputs, uniforms and
    output rows, and the launches of an admission and of a step."""

    def __init__(self, stack, embed, owner):
        st = self.st = stack
        self.emb, self.owner = embed, owner
        self.dev = embed.device
        n, ms, H, V = stack.batch, stack.max_seq, stack.shape.hidden, stack.shape.vocab
        self.n_slots, self.max_seq, self.H, self.V = n, ms, H, V
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=self.dev)
        self.hist = z((n, ms), torch.int64)
        self.status = torch.full((n,), capi.GEN_STOPPED, dtype=torch.int32, device=self.dev)
        self.stop = torch.full((n, MAX_STOP), -1, dtype=torch.int64, device=self.dev)
        self.seeds = z((n,), torch.int64)                    # uint64 bit patterns
        self.x_next = z((n, H), torch.float16)
        self.u_next = z((n,), torch.float32)
        self.out_tok = z((n, ms), torch.int64)
        self.out_prob = z((n, ms), torch.float32)
        self.out_lp = self.out_ids = self.out_top = None     # [n, ms] and [n, ms, TOPLP_MAX], made when a request first asks
        self.tokens = z((n,), torch.int64)
        self.probs = z((n,), torch.float32)
        self.pin = torch.zeros((2, n), dtype=torch.int32).pin_memory()
        self.pin_ev = [None, None]
        self.copies = 0
        self.rowp = (capi.ExlSampleParams * n)()             # each slot's sampler settings (slot order: the fused route's rows)
        self.keep = [None] * n                               # the banned tensors rowp points into
        for s in range(n):
            self.release(s)
        self.fused = open_plan(stack) is None

    def _up(self, values, dtype):
        """values (host) on the device without a host synchronisation: a pinned copy, which torch keeps until the copy is done."""
        return torch.tensor(values, dtype=dtype).pin_memory().to(self.dev, non_blocking=True)

    def release(self, s):
        self.rowp[s], _ = sampling.params(sampling.Settings(), self.dev)
        self.keep[s] = None

    def _advance(self, rows, slots, pos, js):
        n = len(slots)
        arr = lambda v: (C.c_int * n)(*[int(x) for x in v])
        capi.check(capi.lib().exl_gen_advance(capi._ptr(self.tokens), capi._ptr(self.probs), n, arr(slots), arr(pos), arr(js),
                                              capi._ptr(self.hist), self.max_seq, capi._ptr(self.status), capi._ptr(self.stop),
                                              capi._ptr(self.seeds), self.n_slots, capi._ptr(self.emb), self.V, self.H,
                                              capi._ptr(self.x_next), capi._ptr(self.u_next), capi._ptr(self.out_tok),
                                              capi._ptr(self.out_prob), self.max_seq, capi._stream()))

    def _sample(self, logits, params, history, hist_lens, u):
        """exl_sample_rows with the cached per-slot params (history: one row per logits row)."""
        hist = sampling.history_args("sample", history, hist_lens, logits.shape[0], self.dev)
        sampling.launch(logits, hist, params, u, self.tokens, self.probs)

    def _mix(self, logits, rows, history, hist_lens):
        """exl_cfg_mix over the guided requests among rows (logits row i belongs to rows[i], a _Live or None), each row penalised
        over history[i][0 .. hist_lens[i]); returns the sampler's history lengths, 0 for a guided row (it is penalised here)."""
        at = {id(lv): i for i, lv in enumerate(rows) if lv is not None}
        pairs = [(i, at[id(lv.pair)]) for i, lv in enumerate(rows) if lv is not None and lv.pair is not None and not lv.shadow]
        if not pairs:
            return hist_lens
        cfg.mix(logits, pairs, [rows[a].req.cfg_alpha for a, _ in pairs], [rows[a].req.settings for a, _ in pairs], history, hist_lens)
        return [0 if lv is not None and lv.pair is not None else h for lv, h in zip(rows, hist_lens)]

    def _top_logprobs(self, logits, rows, js):
        """exl_top_logprobs over logits (row i belongs to rows[i], a _Live or None, as its token j = js[i]) when a row asks, with the
        largest N of those rows, into the asking rows' slots under the status gate (the shadow of a guided request never asks)."""
        ask = [lv is not None and not lv.shadow and lv.req.logprobs > 0 for lv in rows]
        if not any(ask):
            return
        if self.out_lp is None:
            shape = (self.n_slots, self.max_seq)
            self.out_lp = torch.full(shape, float("nan"), dtype=torch.float32, device=self.dev)
            self.out_ids = torch.full(shape + (capi.TOPLP_MAX,), -1, dtype=torch.int64, device=self.dev)
            self.out_top = torch.full(shape + (capi.TOPLP_MAX,), float("nan"), dtype=torch.float32, device=self.dev)
        n = max(lv.req.logprobs for lv, a in zip(rows, ask) if a)
        sampling.launch_top_logprobs(logits, self.tokens, n, self.out_lp, self.out_ids, self.out_top, capi.TOPLP_MAX,
                                     [lv.slot if a else -1 for lv, a in zip(rows, ask)], js, self.status, self.max_seq)

    def _trace(self, kind, logits, lives, u):
        tr = self.owner.trace
        if tr is not None:
            tr.append(dict(kind=kind, logits=logits.cpu().numpy().copy(), rids=[lv.rid for lv in lives],
                           slots=[lv.slot for lv in lives], j=[lv.n for lv in lives], u=u.cpu().numpy().copy(),
                           shadow=[lv.shadow for lv in lives]))

    def admit(self, lives):
        n = len(lives)
        slots = [lv.slot for lv in lives]
        ids = self._up([t for lv in lives for t in lv.prompt], torch.int64)
        idx = self._up(slots, torch.int64)
        meta = self._up([lv.req.stop_ids + [-1] * (MAX_STOP - len(lv.req.stop_ids)) + [lv.req.seed - (1 << 64) if lv.req.seed >> 63 else
                                                                                     lv.req.seed] for lv in lives], torch.int64)
        self.stop[idx] = meta[:, :MAX_STOP]
        self.seeds[idx] = meta[:, MAX_STOP]
        self.status[idx] = capi.GEN_LIVE
        off = 0
        for lv in lives:
            self.hist[lv.slot, :lv.L] = ids[off:off + lv.L]
            off += lv.L
            ban = self._up(lv.req.banned, torch.int32) if lv.req.banned else None
            p, ban = sampling.params(lv.req.settings, self.dev, lv.req.bos_token_id, ban)
            self.rowp[lv.slot], self.keep[lv.slot] = p, ban
        params = (capi.ExlSampleParams * n)(*[self.rowp[s] for s in slots])
        u = self._up([uniform(lv.req.seed, 0) for lv in lives], torch.float32)
        # at most max_seq prompt tokens per prefill (its scratch rows): only a guided request's two prompts can exceed that alone
        chunks, off = [[]], 0
        for i, lv in enumerate(lives):
            if chunks[-1] and sum(lives[k].L for k in chunks[-1]) + lv.L > self.max_seq:
                chunks.append([])
            chunks[-1].append(i)
        parts = []
        for ch in chunks:
            T = sum(lives[i].L for i in ch)
            parts.append(self.st.prefill_ragged(self.emb[ids[off:off + T]], [lives[i].L for i in ch], [0] * len(ch),
                                                seqs=[slots[i] for i in ch], last_only=True))
            off += T
        logits = parts[0] if len(parts) == 1 else torch.cat(parts)
        self._trace("admit", logits, lives, u)
        history = self.hist.index_select(0, idx)
        lens = self._mix(logits, lives, history, [lv.L for lv in lives])
        self._sample(logits, params, history, lens, u)
        self._top_logprobs(logits, lives, [0] * n)
        self._advance(n, slots, [lv.L for lv in lives], [0] * n)

    def step(self, lives):
        ev = None
        if self.owner.timings is not None:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            ev[0].record()
        by_slot, pasts = fused_rows(lives)
        live = [s for s, lv in enumerate(by_slot) if lv is not None]
        idx = None if self.fused else self._up(live, torch.int64)
        logits, slots = step_slots(self.st, self.fused, lambda i: self.x_next[i], live, pasts, idx)
        rows = [by_slot[s] for s in slots]
        if self.fused:                  # the slot-ordered arrays in place: row s is slot s
            params, history, u = self.rowp, self.hist[:len(rows)], self.u_next
        else:
            params = (capi.ExlSampleParams * len(rows))(*[self.rowp[s] for s in slots])
            history, u = self.hist.index_select(0, idx), self.u_next.index_select(0, idx)
        if ev:
            ev[1].record()
        if self.owner.trace is not None:
            live_rows = [lv for lv in rows if lv is not None]
            tr_u = u[:len(rows)]
            self._trace("step", logits[[i for i, lv in enumerate(rows) if lv is not None]], live_rows,
                        tr_u[[i for i, lv in enumerate(rows) if lv is not None]])
        lens = self._mix(logits, rows, history, [lv.L + lv.n if lv is not None else 0 for lv in rows])
        self._sample(logits, params, history, lens, u)
        self._top_logprobs(logits, rows, [lv.n if lv is not None else 0 for lv in rows])
        if ev:
            ev[2].record()
        self._advance(len(rows), [lv.slot if lv is not None else -1 for lv in rows], [lv.L + lv.n if lv is not None else 0 for lv in rows],
                      [lv.n if lv is not None else 0 for lv in rows])
        if ev:
            ev[3].record()
            self.owner.timings.append((ev, len(lives)))

    def copy_status(self):
        """Copy the status into pinned buffer i % 2 behind an event; copy i is read (read_status(i)) before copy i + 2 is made."""
        i = self.copies
        self.pin[i % 2].copy_(self.status, non_blocking=True)
        self.pin_ev[i % 2] = torch.cuda.Event()
        self.pin_ev[i % 2].record()
        self.copies += 1
        return i

    def read_status(self, i):
        self.pin_ev[i % 2].synchronize()
        return self.pin[i % 2].numpy().copy()

    def fetch(self, lv, n):
        tok = torch.empty(n, dtype=torch.int64).pin_memory()
        prob = torch.empty(n, dtype=torch.float32).pin_memory()
        tok.copy_(self.out_tok[lv.slot, :n], non_blocking=True)
        prob.copy_(self.out_prob[lv.slot, :n], non_blocking=True)
        out = [tok, prob]
        N = lv.req.logprobs
        if N:
            for src in (self.out_lp[lv.slot, :n], self.out_ids[lv.slot, :n, :N], self.out_top[lv.slot, :n, :N]):
                out.append(torch.empty(src.shape, dtype=src.dtype).pin_memory())
                out[-1].copy_(src, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        return (ev, *out)


class BatchGenerator(Scheduler):
    """Batched generation over one DecodeStack (module docstring; DESIGN.md §4g).

    stack   a DecodeStack with an lm_head; its batch cache sequences are the slots, its max_seq bounds prompt + completion
    embed   fp16 [vocab, hidden]: maps a token to the stack's input

    submit(Request) -> id; step() runs one iteration; run() steps until every request has finished and returns {id: Result}.
    The step is slots.step_slots: the fused batch step when slots.open_plan makes the stack's plan (fused is then True), else a
    ragged prefill with one token per live slot (act-order, or more slots than the fused plan takes).  trace: set to a list to record
    every admission's and step's logits rows with their request ids, slots, token indices and uniforms (tests).  timings: set to a
    list to record, per step, four CUDA events (start, after the step, the sampler and exl_top_logprobs when a row asks, the advance) and the number of requests stepped
    (tools/generate_bench.py)."""

    def __init__(self, stack, embed):
        check_stack("BatchGenerator", stack, embed, contiguous=True)
        if stack.batch > capi.RAGGED_MAX_SEQ:
            raise ValueError(f"BatchGenerator: the stack holds {stack.batch} cache sequences, at most {capi.RAGGED_MAX_SEQ}")
        self.trace = None
        self.timings = None
        super().__init__(_Device(stack, embed, self), stack.batch, stack.max_seq)
        self.fused = self.dev.fused

    def submit(self, req):
        v = self.dev.V
        bad = [t for t in req.prompt + req.stop_ids if not 0 <= t < v]
        if bad:
            raise ValueError(f"submit: token id {bad[0]} outside the vocabulary [0, {v})")
        return super().submit(req)


def generate_simple(stack, embed, prompts, max_new_tokens=128, settings=None, eos_token_id=None, bos_token_id=None, banned=None,
                    seed=0):
    """ExLlamaGenerator.generate_simple over a list of prompts (lists of ids): each prompt is one request with min_p 0 and the bos
    mask, as gen_single_token samples (generator.py:355,366), seed seed + i for prompt i, max_new_tokens clipped to max_seq - the
    prompt's length, and eos_token_id as its stop id.  One difference from the reference: a row ends at its own EOS, where the
    reference steps every row until all of them have one.  Returns each prompt followed by its tokens (host lists of ids)."""
    s = copy.copy(settings if settings is not None else sampling.Settings())
    s.min_p = 0.0
    return run_prompts(stack, embed, [Request(p, 1, s, stop_ids=() if eos_token_id is None else (eos_token_id,), seed=seed + i,
                                              bos_token_id=bos_token_id, banned=banned) for i, p in enumerate(prompts)], max_new_tokens)


def run_prompts(stack, embed, reqs, max_new_tokens):
    """reqs through one BatchGenerator, each with max_new_tokens clipped to what its longer prompt leaves in max_seq; returns each
    request's prompt followed by its tokens (host lists of ids)."""
    gen = BatchGenerator(stack, embed)
    ids = []
    for req in reqs:
        req.max_new_tokens = max(1, min(int(max_new_tokens), stack.max_seq - max(len(req.prompt), len(req.cfg_prompt or ()))))
        ids.append((req.prompt, gen.submit(req)))
    res = gen.run()
    return [prompt + res[rid].tokens for prompt, rid in ids]
