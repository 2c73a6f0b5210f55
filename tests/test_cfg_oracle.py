"""CPU checks of classifier-free guidance: oracle/cfg_oracle.py against the reference's own program (tests/golden/cfg_ref.npz), its
per-element bound against a numpy-fp32 restatement of exl_cfg_mix's rounding points on a seeded sweep, and guided requests in the
host scheduler of exllama_b200/generate.py through a fake device: admission order with a guided request waiting for two slots,
both slots released together, max_seq decided on the longer prompt, and tokens equal to each request run alone."""
import math
import os

import numpy as np
import pytest

import generate_oracle as G
from exllama_b200 import generate
from oracle import cfg_oracle as F

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cfg_ref.npz")


def test_golden_cases():
    cases = F.golden_cases(GOLD)
    assert len(cases) >= 40
    assert {c["alpha"] for c in cases} == {0.0, 0.5, 1.0, -0.4, 1.4, 3.0}
    assert {len(c["hist_a"]) for c in cases} == {0, 17, 1920} and {c["vocab"] for c in cases} == {7, 32000}
    for i, c in enumerate(cases):
        r = F.run_case(c)
        assert np.array_equal(r["kept"], c["kept"]), i
        assert np.abs(r["probs"] - c["probs"]).max() <= 1e-9, i


def test_bound_holds_for_fp32_emulation():
    rng = np.random.default_rng(11)
    worst = 0.0
    for t in range(120):
        V = [7, 1000, 32000, 32001][t % 4]
        scale = [0.01, 3.0, 40.0, 2000.0, 3e4][t % 5]              # near-flat to large logits
        la = (rng.standard_normal(V) * scale).astype(np.float32)
        lb = (rng.standard_normal(V) * scale + rng.uniform(-50, 50)).astype(np.float32)
        alpha = float(rng.uniform(-3.0, 4.0)) if t % 7 else [-3.0, 0.0, 1.0, 4.0][t % 4]
        hl = [0, 17, 1920, 3000][t % 4]
        ha, hb = rng.integers(0, V, hl), rng.integers(0, V, hl)
        pen = [(1.0, -1, 0), (1.15, 256, 128), (1.3, -1, 0), (1.1, 16, 3000)][t % 4]
        r = F.mix(la, lb, alpha, ha, hb, *pen)
        got = F.emulate32(la, lb, alpha, ha, hb, *pen)
        assert F.within(got, r), (t, V, scale, alpha, pen)
        fin = r["bound"] > 0
        worst = max(worst, float((np.abs(got[fin] - r["mixed"][fin]) / r["bound"][fin]).max()))
    assert worst > 0.05                                          # the bound is not vacuous


def test_infinite_and_undefined_rows():
    la = np.array([1.0, -np.inf, 2.0, 0.5], np.float32)
    lb = np.array([0.0, 3.0, -np.inf, 1.0], np.float32)
    r = F.mix(la, lb, 0.0, None, None)                          # 0 * -inf is NaN, as torch gives it
    got = F.emulate32(la, lb, 0.0)
    assert F.within(got, r) and np.isnan(got[2]) and got[1] == -np.inf
    assert F.mix(np.full(4, -np.inf, np.float32), lb, 0.5) is None
    assert F.mix(np.array([np.nan, 0, 0, 0], np.float32), lb, 0.5) is None
    assert F.mix(la, lb, 0.5, None, np.array([4]), 1.15, -1, 0) is None     # a history id outside the vocabulary


# ---- guided requests in the scheduler ------------------------------------------------------------------------------------------

def _state(n, ms, V=40, H=8):
    return dict(hist=np.zeros((n, ms), np.int64), status=np.full(n, G.STOPPED, np.int32), stop=np.full((n, G.MAX_STOP), -1, np.int64),
                seeds=np.zeros(n, np.uint64), embed=np.arange(V * H, dtype=np.float16).reshape(V, H), x_next=np.zeros((n, H), np.float16),
                u_next=np.zeros(n, np.float32), out_tok=np.zeros((n, ms), np.int64), out_prob=np.zeros((n, ms), np.float32))


class _Ev:
    def synchronize(self):
        pass


class CfgFakeDev:
    """numpy stand-in for _Device with guided requests: a plain row draws from its history and seed; a guided pair draws one token
    from both of its slots' histories, its alpha and its seed, which goes to both rows (exl_gen_advance is generate_oracle.advance)."""

    def __init__(self, n, ms, V=40):
        self.V, self.st = V, _state(n, ms, V)
        self.copies, self.steps, self.released = [], [], []

    def draw(self, req, ha, hb=None):
        if req.banned is not None and len(set(req.banned)) >= self.V:
            return -1
        t = int(ha.sum()) * 7 + len(ha) * 3 + req.seed
        if hb is not None:
            t = t * 5 + int(hb.sum()) * 11 + len(hb) + int(req.cfg_alpha * 10)
        return int(t % self.V)

    def _tokens(self, rows, lens):
        """rows: a _Live or None per row, lens: each row's history length; both rows of a guided request must be among them."""
        hist = {lv.slot: self.st["hist"][lv.slot, :n] for lv, n in zip(rows, lens) if lv is not None}
        out = []
        for lv in rows:
            if lv is None:
                out.append(0)
            elif lv.pair is None:
                out.append(self.draw(lv.req, hist[lv.slot]))
            else:
                prim, shadow = (lv.pair, lv) if lv.shadow else (lv, lv.pair)
                out.append(self.draw(lv.req, hist[prim.slot], hist[shadow.slot]))
        return out

    def admit(self, lives):
        for lv in lives:
            s = lv.slot
            self.st["status"][s] = G.LIVE
            self.st["stop"][s] = lv.req.stop_ids + [-1] * (G.MAX_STOP - len(lv.req.stop_ids))
            self.st["seeds"][s] = lv.req.seed
            self.st["hist"][s, :lv.L] = lv.prompt
        toks = self._tokens(lives, [lv.L for lv in lives])
        G.advance(self.st, toks, [0.5] * len(lives), [lv.slot for lv in lives], [lv.L for lv in lives], [0] * len(lives))

    def step(self, lives):
        rows, pasts = generate.fused_rows(lives)
        self.steps.append((sorted(lv.slot for lv in lives), pasts))
        toks = self._tokens(rows, [lv.L + lv.n if lv else 0 for lv in rows])
        G.advance(self.st, toks, [0.5] * len(rows), [lv.slot if lv else -1 for lv in rows], [lv.L + lv.n if lv else 0 for lv in rows],
                  [lv.n if lv else 0 for lv in rows])

    def copy_status(self):
        self.copies.append(self.st["status"].copy())
        return len(self.copies) - 1

    def read_status(self, i):
        return self.copies[i]

    def fetch(self, lv, n):
        assert not lv.shadow
        return _Ev(), self.st["out_tok"][lv.slot, :n].copy(), self.st["out_prob"][lv.slot, :n].copy()

    def release(self, s):
        self.released.append(s)


def _alone(dev, req, ms):
    ha, hb, out = list(req.prompt), list(req.cfg_prompt) if req.cfg_prompt is not None else None, []
    while True:
        t = dev.draw(req, np.array(ha), None if hb is None else np.array(hb))
        if t < 0:
            return out, "error"
        out.append(t)
        ha.append(t)
        if hb is not None:
            hb.append(t)
        if t in req.stop_ids:
            return out, "stop"
        if len(out) >= req.max_new_tokens:
            return out, "length"
        if max(len(ha), len(hb or ())) >= ms:
            return out, "max_seq"


def test_scheduler_with_guided_requests():
    ms = 32
    dev = CfgFakeDev(3, ms)
    sch = generate.Scheduler(dev, 3, ms)
    R = generate.Request
    reqs = [R([1, 2, 3], 6, seed=1), R([4, 5], 9, seed=2),
            R([6, 7], 12, seed=3, cfg_prompt=[8] * 5, cfg_alpha=1.5),           # waits for two slots
            R([9], 2, seed=4),                                                  # may not overtake it
            R([3] * 4, 40, seed=5, cfg_prompt=[2] * 20, cfg_alpha=-0.4),        # max_seq on the longer (guidance) prompt
            R([1, 1], 5, seed=6, cfg_prompt=[2], cfg_alpha=0.5, banned=list(range(40))),   # every token banned
            R([5, 4, 3], 7, seed=7, cfg_prompt=[1, 2], cfg_alpha=3.0), R([2], 3, seed=8)]
    alone7, _ = _alone(dev, reqs[6], ms)
    reqs[6].stop_ids = [alone7[2]]
    ids = [sch.submit(r) for r in reqs]
    res = sch.run()
    for rid, req in zip(ids, reqs):
        want, why = _alone(dev, req, ms)
        assert (res[rid].tokens, res[rid].finish) == (want, why), (rid, res[rid].tokens, res[rid].finish, want, why)
    assert res[ids[4]].finish == "max_seq" and len(res[ids[4]].tokens) == ms - 20
    assert res[ids[5]].finish == "error" and res[ids[6]].finish == "stop"
    # admission in submission order; a guided request takes the two lowest free slots, and the plain request behind it waits
    admitted = [(k, rid, s) for k, kind, *rest in sch.order if kind == "admit" for rid, s in rest[0]]
    first = []
    for _, rid, _ in admitted:
        if rid not in first:
            first.append(rid)
    assert first == ids
    when = {rid: k for k, rid, _ in reversed(admitted)}
    assert when[ids[2]] > when[ids[1]] and when[ids[3]] >= when[ids[2]]
    for rid in ids:
        slots = [s for _, r, s in admitted if r == rid]
        assert len(slots) == (2 if reqs[ids.index(rid)].cfg_prompt is not None else 1)
    # both slots of a guided request are released in the same iteration; a slot is never taken twice
    rel = {}
    for ev in sch.order:
        if ev[1] == "release":
            rel.setdefault(ev[2], []).append((ev[0], ev[3]))
    for rid, req in zip(ids, reqs):
        if req.cfg_prompt is not None:
            assert len(rel[rid]) == 2 and rel[rid][0][0] == rel[rid][1][0], rel[rid]
    taken = set()
    for ev in sch.order:
        if ev[1] == "admit":
            for _, s in ev[2]:
                assert s not in taken
                taken.add(s)
        elif ev[1] == "release":
            taken.discard(ev[3])
    assert not taken


def test_guided_request_rejects():
    R = generate.Request
    with pytest.raises(ValueError, match="cfg_prompt is empty"):
        R([1], 4, cfg_prompt=[])
    for a in (math.nan, math.inf, -math.inf):
        with pytest.raises(ValueError, match="cfg_alpha .* not finite"):
            R([1], 4, cfg_prompt=[2], cfg_alpha=a)
    with pytest.raises(ValueError, match="two slots"):
        generate.Scheduler(CfgFakeDev(1, 8), 1, 8).submit(R([1], 4, cfg_prompt=[2]))
    sch = generate.Scheduler(CfgFakeDev(2, 8), 2, 8)
    with pytest.raises(ValueError, match="cfg_prompt of 8 tokens leaves no room"):
        sch.submit(R([1], 4, cfg_prompt=list(range(8))))
    sch.submit(R([1], 4, cfg_prompt=list(range(7))))
