"""CPU checks of batched generation: the uniform U(seed, j) against fixed splitmix64 vectors and the package's restatement, the
numpy restatement of exl_gen_advance, and the host scheduler of exllama_b200/generate.py driven through a fake device (a numpy
stand-in for the stack, the sampler and exl_gen_advance): admission order, lowest free slot, the fused rows' past_lens with free
slots at 0, host-decided length and max_seq finishes, stop and error finishes read one step late, and tokens that do not depend on
which requests share a step."""
import numpy as np
import pytest

import generate_oracle as G
from exllama_b200 import generate


def test_uniform_fixed_vectors():
    # splitmix64 seeded with 0: 0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F, 0xF88BB8A8724C81EC, 0x1B39896A51A8749B
    tops = [0xE220A8, 0x6E789E, 0x06C45D, 0xF88BB8, 0x1B3989]
    for j, t in enumerate(tops):
        assert G.U(0, j) == np.float32(t / 2 ** 24)
    for seed in (0, 1, 7, 12345, 2 ** 63, 2 ** 64 - 1):
        for j in (0, 1, 2, 255, 4095, 10 ** 6):
            u = generate.uniform(seed, j)
            assert u == G.U(seed, j) and 0.0 <= u < 1.0 and np.float32(u) == u, (seed, j)


def _state(n, ms, V=40, H=8):
    return dict(hist=np.zeros((n, ms), np.int64), status=np.full(n, G.STOPPED, np.int32), stop=np.full((n, G.MAX_STOP), -1, np.int64),
                seeds=np.zeros(n, np.uint64), embed=np.arange(V * H, dtype=np.float16).reshape(V, H), x_next=np.zeros((n, H), np.float16),
                u_next=np.zeros(n, np.float32), out_tok=np.zeros((n, ms), np.int64), out_prob=np.zeros((n, ms), np.float32))


def test_advance_restatement():
    st = _state(4, 16)
    st["status"][:] = [G.LIVE, G.LIVE, G.LIVE, G.STOPPED]
    st["stop"][1, :2] = [9, 5]
    st["seeds"][:] = [3, 4, 5, 6]
    G.advance(st, [7, 5, -1, 2], [0.5, 0.25, np.nan, 1.0], [2, 1, 0, 3], [4, 6, 3, 2], [0, 3, 1, 0])
    assert st["status"].tolist() == [G.ERROR, G.STOPPED, G.LIVE, G.STOPPED]
    assert st["hist"][2, 4] == 7 and st["out_tok"][2, 0] == 7 and st["u_next"][2] == G.U(5, 1)
    assert st["hist"][1, 6] == 5 and st["out_tok"][1, 3] == 5 and (st["x_next"][1] == st["embed"][5]).all()
    assert st["out_tok"][0, 1] == -1 and np.isnan(st["out_prob"][0, 1]) and not st["hist"][0].any()
    before = {k: v.copy() for k, v in st.items()}
    G.advance(st, [1, 1], [0.5, 0.5], [1, 3], [7, 3], [4, 1])           # finished slots: nothing written
    assert all((before[k] == st[k]).all() or k == "out_prob" for k in st)


class _Ev:
    def synchronize(self):
        pass


class FakeDev:
    """numpy stand-in for _Device: the 'sampler' draws a token from the row's history and the request's seed (or -1 when the
    request bans the whole vocabulary), and exl_gen_advance is generate_oracle.advance."""

    def __init__(self, n, ms, V=40):
        self.V, self.st = V, _state(n, ms, V)
        self.copies, self.steps, self.released = [], [], []

    def draw(self, req, hist):
        if req.banned is not None and len(set(req.banned)) >= self.V:
            return -1
        return int((int(hist.sum()) * 7 + len(hist) * 3 + req.seed) % self.V)

    def admit(self, lives):
        for lv in lives:
            s = lv.slot
            self.st["status"][s] = G.LIVE
            self.st["stop"][s] = lv.req.stop_ids + [-1] * (G.MAX_STOP - len(lv.req.stop_ids))
            self.st["seeds"][s] = lv.req.seed
            self.st["hist"][s, :lv.L] = lv.req.prompt
        toks = [self.draw(lv.req, self.st["hist"][lv.slot, :lv.L]) for lv in lives]
        G.advance(self.st, toks, [0.5] * len(lives), [lv.slot for lv in lives], [lv.L for lv in lives], [0] * len(lives))

    def step(self, lives):
        rows, pasts = generate.fused_rows(lives)
        self.steps.append((sorted(lv.slot for lv in lives), pasts))
        toks = [self.draw(lv.req, self.st["hist"][lv.slot, :lv.L + lv.n]) if lv else 0 for lv in rows]
        G.advance(self.st, toks, [0.5] * len(rows), [lv.slot if lv else -1 for lv in rows], [lv.L + lv.n if lv else 0 for lv in rows],
                  [lv.n if lv else 0 for lv in rows])

    def copy_status(self):
        self.copies.append(self.st["status"].copy())
        return len(self.copies) - 1

    def read_status(self, i):
        return self.copies[i]

    def fetch(self, lv, n):
        return _Ev(), self.st["out_tok"][lv.slot, :n].copy(), self.st["out_prob"][lv.slot, :n].copy()

    def release(self, s):
        self.released.append(s)


def _alone(dev, req, ms):
    """The request's tokens and finish when it runs by itself: the same draws, the same rules."""
    hist, out = list(req.prompt), []
    while True:
        t = dev.draw(req, np.array(hist))
        if t < 0:
            return out, "error"
        out.append(t)
        hist.append(t)
        if t in req.stop_ids:
            return out, "stop"
        if len(out) >= req.max_new_tokens:
            return out, "length"
        if len(hist) >= ms:
            return out, "max_seq"


def _requests():
    R = generate.Request
    return [R([1, 2, 3], 5, seed=1), R(list(range(10)), 3, seed=2), R([4], 1, seed=3), R([5, 6], 30, seed=4),
            R([7] * 20, 40, seed=5),                                            # reaches max_seq 32
            R([8, 9], 6, seed=6, banned=list(range(40))),                       # every token banned: fails alone
            R([2, 2], 8, seed=7), R([3, 1, 4, 1, 5], 4, seed=8)]


def test_scheduler_against_requests_alone():
    ms = 32
    dev = FakeDev(3, ms)
    sch = generate.Scheduler(dev, 3, ms)
    reqs = _requests()
    # a stop id that request 6 hits: its third token when alone
    alone6, _ = _alone(dev, reqs[6], ms)
    reqs[6].stop_ids = [alone6[2]]
    ids = [sch.submit(r) for r in reqs[:5]]
    sch.step()
    sch.step()
    ids += [sch.submit(r) for r in reqs[5:]]                                    # later arrivals
    res = sch.run()
    for rid, req in zip(ids, reqs):
        want, why = _alone(dev, req, ms)
        assert (res[rid].tokens, res[rid].finish) == (want, why), (rid, res[rid].tokens, res[rid].finish, want, why)
        assert res[rid].t_first is not None
    assert res[ids[4]].finish == "max_seq" and res[ids[5]].finish == "error" and res[ids[6]].finish == "stop"
    # admission in submission order into the lowest free slot
    admitted = [a for ev in sch.order if ev[1] == "admit" for a in ev[2]]
    assert [rid for rid, _ in admitted] == ids
    assert admitted[:3] == [(ids[0], 0), (ids[1], 1), (ids[2], 2)]
    free = {0, 1, 2}
    for ev in sch.order:
        if ev[1] == "admit":
            for rid, s in ev[2]:
                assert s == min(free), (ev, free)
                free.discard(s)
        elif ev[1] == "release":
            assert ev[3] not in free
            free.add(ev[3])
    assert free == {0, 1, 2}


def test_fused_rows_free_slots_at_zero():
    R = generate.Request
    a, b = generate._Live(0, R([1] * 5, 4), 0, 0.0), generate._Live(1, R([1] * 9, 4), 3, 0.0)
    a.n, b.n = 2, 1
    rows, pasts = generate.fused_rows([b, a])
    assert rows == [a, None, None, b] and pasts == [6, 0, 0, 9]


def test_stop_frees_the_slot_one_step_late():
    """A request whose token k is a stop id is stepped once more (the device ignores it) and its slot is freed at the iteration
    after the one that drew the stop; a length finish frees the slot at once."""
    ms = 64
    dev = FakeDev(2, ms)
    sch = generate.Scheduler(dev, 2, ms)
    r0 = generate.Request([1, 2], 20, seed=11)
    alone, _ = _alone(dev, r0, ms)
    r0.stop_ids = [alone[3]]
    k_stop = alone.index(alone[3])                                              # the first occurrence ends it
    r1 = generate.Request([3], 3, seed=12)
    i0, i1 = sch.submit(r0), sch.submit(r1)
    res = sch.run()
    assert res[i0].tokens == alone[:k_stop + 1] and res[i0].finish == "stop"
    # r0's token k_stop is drawn at iteration k_stop (token 0 at admission, iteration 0); it is stepped at iteration k_stop + 1 too
    stepped = [k for k, (slots, _) in enumerate(dev.steps, start=1) if 0 in slots]
    assert stepped[-1] == k_stop + 1
    fin = [ev for ev in sch.order if ev[1] == "finish" and ev[2] == i0]
    assert fin[0][0] == k_stop + 1
    rel = [ev for ev in sch.order if ev[1] == "release" and ev[2] == i1]
    assert rel[0][0] == 2 and res[i1].finish == "length" and len(res[i1].tokens) == 3


def test_submit_rejects_what_cannot_fit():
    sch = generate.Scheduler(FakeDev(2, 8), 2, 8)
    with pytest.raises(ValueError, match="leaves no room"):
        sch.submit(generate.Request(list(range(8)), 4))
    sch.submit(generate.Request(list(range(7)), 4))
    with pytest.raises(ValueError, match="empty"):
        generate.Request([], 4)
    with pytest.raises(ValueError, match="max_new_tokens 0"):
        generate.Request([1], 0)
    with pytest.raises(ValueError, match="stop ids"):
        generate.Request([1], 1, stop_ids=range(9))
