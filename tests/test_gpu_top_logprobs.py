"""Log-probabilities of generated tokens on the GPU (csrc/toplp.cu exl_top_logprobs, sampling.top_logprobs, Request(logprobs=),
SpeculativeGenerator(logprobs=)): the kernel against oracle/toplp_oracle.py (exact ids, per-element bound) on a seeded sweep with
planted ties, signed zeros and -inf masks; undefined rows beside defined ones; two calls bitwise equal and a graph replay; routed
writes under the status gate; argument errors naming the row.  End to end on the synthetic stacks of tests/stack_harness.py:
BatchGenerator with mixed requests (with and without logprobs, one guided) on the fused and ragged routes, every reported value
against the oracle over the traced rows (a guided request's through oracle/cfg_oracle.py's mix first), and tokens, probs and
finishes equal to a run without logprobs; one SpeculativeGenerator run against the oracle over its target rows."""
import ctypes as C
import re

import numpy as np
import pytest

from oracle import cfg_oracle, toplp_oracle as T
from stack_harness import lib_state, stacks  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu


def _logits(rows, vocab, seed):
    """Seeded fp32 rows with planted ties (a row's value copied to later ids), signed zeros, -inf masks and, in row 1 of a batch of
    more than 2, fewer finite entries than 20."""
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((rows, vocab)) * 3).astype(np.float32)
    for r in range(rows):
        k = max(1, vocab // 100)
        src = rng.integers(0, vocab, k)
        x[r, rng.integers(0, vocab, k)] = x[r, src]
        x[r, rng.integers(0, vocab, 2)] = [0.0, -0.0]
        x[r, rng.integers(0, vocab, max(1, vocab // 20))] = -np.inf
    if rows > 2:
        keep = rng.choice(vocab, min(vocab, 6), replace=False)
        x[1] = -np.inf
        x[1, keep] = [5.0, 5.0, -0.0, 0.0, -3.0, 1.0][:len(keep)]
    return x


def _check(x, toks, n, lp, ids, top, what):
    lp, ids, top = lp.cpu().numpy(), ids.cpu().numpy(), top.cpu().numpy()
    for r in range(x.shape[0]):
        w = T.top_logprobs(x[r], n, None if toks is None else int(toks[r]))
        assert ids[r].tolist() == w["ids"].tolist(), (what, r)
        assert T.within(top[r], w["top"], w["bound"]), (what, r, top[r][:5], w["top"][:5])
        assert T.within(lp[r], w["lp"], w["lp_bound"]), (what, r, lp[r], w["lp"])


@pytest.mark.parametrize("rows", [1, 4, 17, 64])
@pytest.mark.parametrize("vocab", [7, 32000, 128256])
def test_against_oracle(rows, vocab):
    import torch
    from exllama_b200 import sampling
    x = _logits(rows, vocab, rows * 7 + vocab)
    rng = np.random.default_rng(rows)
    toks = rng.integers(-2, vocab + 2, rows)
    toks[0] = int(np.argmax(x[0]))
    lg, tk = torch.from_numpy(x).cuda(), torch.from_numpy(toks).cuda()
    for n in (0, 1, 5, 20):
        lp, ids, top = sampling.top_logprobs(lg, n, tk)
        assert ids.shape == (rows, n) and top.shape == (rows, n)
        _check(x, toks, n, lp, ids, top, (rows, vocab, n))
    lp, _, _ = sampling.top_logprobs(lg, 3)
    assert torch.isnan(lp).all()                                                  # no tokens


def test_undefined_rows_leave_the_others_alone():
    import torch
    from exllama_b200 import sampling
    x = _logits(6, 32000, 5)
    x[1, 7] = np.nan
    x[3, 31999] = np.inf
    x[4] = -np.inf
    toks = np.array([0, 1, 2, 3, 4, 5])
    lp, ids, top = sampling.top_logprobs(torch.from_numpy(x).cuda(), 5, torch.from_numpy(toks).cuda())
    _check(x, toks, 5, lp, ids, top, "undefined")
    for r in (1, 3, 4):
        assert np.isnan(float(lp[r])) and (ids[r] == -1).all() and torch.isnan(top[r]).all()


def test_two_calls_bitwise_and_graph_replay():
    import torch
    from exllama_b200 import sampling
    lg = torch.from_numpy(_logits(17, 128256, 9)).cuda()
    tk = torch.arange(17, device="cuda", dtype=torch.int64) * 1000
    a = sampling.top_logprobs(lg, 20, tk)
    b = sampling.top_logprobs(lg, 20, tk)
    assert all(torch.equal(u.view(torch.int32) if u.dtype == torch.float32 else u, v.view(torch.int32) if v.dtype == torch.float32 else v)
               for u, v in zip(a, b))
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            got = sampling.top_logprobs(lg, 20, tk)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(got[1], a[1]) and torch.equal(got[0].view(torch.int32), a[0].view(torch.int32))
    assert torch.equal(got[2].view(torch.int32), a[2].view(torch.int32))


def test_routed_writes():
    """Rows land at [slot][j]; a row whose slot is not live, and a row with slot -1, write nothing."""
    import torch
    from exllama_b200 import capi, sampling
    rows, vocab, n_slots, out_ld, N = 5, 32000, 6, 9, 4
    x = _logits(rows, vocab, 11)
    lg = torch.from_numpy(x).cuda()
    toks = np.array([3, 9, 27, 81, 243])
    tk = torch.from_numpy(toks).cuda()
    status = torch.tensor([0, 0, capi.GEN_STOPPED, 0, capi.GEN_ERROR, 0], dtype=torch.int32, device="cuda")
    slots, js = [4, 0, 3, -1, 2], [1, 8, 0, 0, 5]                                  # 4 and 2 are not live
    lp = torch.full((n_slots, out_ld), 7.0, device="cuda")
    ids = torch.full((n_slots, out_ld, capi.TOPLP_MAX), 7, dtype=torch.int64, device="cuda")
    top = torch.full((n_slots, out_ld, capi.TOPLP_MAX), 7.0, device="cuda")
    sampling.launch_top_logprobs(lg, tk, N, lp, ids, top, capi.TOPLP_MAX, slots, js, status, out_ld)
    rest_lp, rest_ids, rest_top = lp.clone(), ids.clone(), top.clone()
    for r in (1, 2):
        s, j = slots[r], js[r]
        rest_lp[s, j], rest_ids[s, j, :N], rest_top[s, j, :N] = 7.0, 7, 7.0
    assert (rest_lp == 7.0).all() and (rest_ids == 7).all() and (rest_top == 7.0).all()     # nothing else written
    _check(x[[1, 2]], toks[[1, 2]], N, lp[[0, 3], [8, 0]], ids[[0, 3], [8, 0], :N], top[[0, 3], [8, 0], :N], "routed")


def test_argument_errors():
    import torch
    from exllama_b200 import capi
    lib = capi.lib()
    lg = torch.zeros((4, 100), device="cuda")
    out = torch.zeros(4 * 10 * 20, device="cuda")
    ids = torch.zeros(4 * 10 * 20, dtype=torch.int64, device="cuda")
    st = torch.zeros(4, dtype=torch.int32, device="cuda")
    arr = lambda v: (C.c_int * len(v))(*v)
    P = capi._ptr

    def call(rows=4, vocab=100, ld=100, n=5, slots=None, js=None, status=st, n_slots=4, out_ld=10, top_ld=20, logits=lg):
        return lib.exl_top_logprobs(P(logits), rows, vocab, ld, None, n, arr(slots) if slots else None, arr(js) if js else None,
                                    P(status), n_slots, out_ld, P(out), P(ids), P(out), top_ld, None)
    for kw, msg in [(dict(rows=0), r"rows 0 outside \[1, 64\]"), (dict(rows=65), r"rows 65 outside \[1, 64\]"),
                    (dict(vocab=262145, ld=262145), r"vocab 262145 outside \[1, 262144\]"), (dict(ld=99), "logits_ld 99 < vocab 100"),
                    (dict(n=21), r"n_top 21 outside \[0, 20\]"), (dict(top_ld=4), "n_top 5 with .* top_ld 4"),
                    (dict(logits=None), "NULL pointer"),
                    (dict(slots=[0, 1, 4, 2], js=[0] * 4), r"row 2: slot 4 outside \[-1, n_slots 4\)"),
                    (dict(slots=[0, 1, 1, 2], js=[0] * 4), "row 2: slot 1 named twice"),
                    (dict(slots=[0, 1, -1, 2], js=[0, 0, 0, 10]), r"row 3: j 10 outside \[0, out_ld 10\)"),
                    (dict(slots=[0, 1, 2, 3], js=[0] * 4, status=None), "slot_host without"),
                    (dict(slots=[0, 1, 2, 3], js=[0] * 4, n_slots=65), r"n_slots 65 outside \[1, 64\]")]:
        assert call(**kw) == 1, kw
        assert re.search(msg, lib.exl_last_error().decode()), (kw, lib.exl_last_error())
    assert call(slots=[0, -1, 2, 3], js=[9, 0, 0, 1]) == 0


# ---- end to end ------------------------------------------------------------------------------------------------------------------

def _settings(temperature=1.0, top_k=0, top_p=0.0, penalty=(1.0, -1, 0)):
    from exllama_b200 import sampling
    s = sampling.Settings()
    s.temperature, s.top_k, s.top_p = temperature, top_k, top_p
    s.token_repetition_penalty_max, s.token_repetition_penalty_sustain, s.token_repetition_penalty_decay = penalty
    return s


def _requests(vocab, logprobs):
    """Ten requests, every other one asking for logprobs (N 1, 5, 20 ...), request 6 guided, request 8 failing alone, request 9
    reaching max_seq; logprobs False: none asks."""
    from exllama_b200.generate import Request
    rng = np.random.default_rng(21)
    sets = [_settings(top_k=1), _settings(0.95, 40, 0.65, (1.15, 256, 128)), _settings(0.8, 0, 0.9), sampling_default()]
    Ns = [5, 0, 20, 0, 1, 0, 3, 0, 2, 7]
    out = []
    for i in range(10):
        kw = dict(settings=sets[i % 4], seed=300 + i, logprobs=Ns[i] if logprobs else 0, stop_ids=[])
        if i == 6:
            kw.update(cfg_prompt=rng.integers(0, vocab, 23), cfg_alpha=1.5)
        if i == 8:
            kw.update(banned=list(range(vocab)))
        L, m = [(5, 9), (40, 6), (300, 12), (1, 4), (17, 10), (90, 3), (12, 8), (8, 5), (60, 7), (600, 100)][i]
        out.append(Request(rng.integers(0, vocab, L), m, **kw))
    return out


def sampling_default():
    from exllama_b200 import sampling
    return sampling.Settings()


def _run(st, emb, reqs):
    from exllama_b200.generate import BatchGenerator
    gen = BatchGenerator(st, emb)
    gen.trace = []
    ids = [gen.submit(r) for r in reqs[:5]]
    for _ in range(3):
        gen.step()
    ids += [gen.submit(r) for r in reqs[5:]]
    res = gen.run()
    return gen, [res[i] for i in ids], ids


def _rows_of(gen, rid):
    """{j: (logits row, the shadow's row or None)} of request rid's traced rows."""
    out = {}
    for e in gen.trace:
        prim = {r: j for r, (x, j, sh) in enumerate(zip(e["rids"], e["j"], e["shadow"])) if x == rid and not sh}
        shad = [r for r, (x, sh) in enumerate(zip(e["rids"], e["shadow"])) if x == rid and sh]
        for r, j in prim.items():
            out[j] = (e["logits"][r], e["logits"][shad[0]] if shad else None)
    return out


@pytest.mark.parametrize("route", ["fused", "ragged_act"])
def test_batch_generator_logprobs(stacks, route):
    kw = dict(batch=4, seed=81, max_seq=640, act=route == "ragged_act")
    st = stacks(**kw)
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(82)
    emb = (torch.randn((st.shape.vocab, st.shape.hidden), device="cuda", generator=g) * 0.5).half()
    V = st.shape.vocab
    reqs = _requests(V, True)
    gen, res, ids = _run(st, emb, reqs)
    assert gen.fused == (route == "fused")
    assert res[8].finish == "error" and res[9].finish == "max_seq"
    checked = 0
    for i, (req, out, rid) in enumerate(zip(reqs, res, ids)):
        if not req.logprobs:
            assert out.logprobs is None and out.top_logprobs is None
            continue
        assert len(out.logprobs) == len(out.top_logprobs) == len(out.tokens), i
        rows = _rows_of(gen, rid)
        for j, tok in enumerate(out.tokens):
            x, xs = rows[j]
            tol = 0.0
            if req.cfg_prompt is not None:                           # the mixed row, as exl_cfg_mix wrote it
                s = req.settings
                pen = (s.token_repetition_penalty_max, s.token_repetition_penalty_sustain, s.token_repetition_penalty_decay)
                ha, hb = req.prompt + out.tokens[:j], req.cfg_prompt + out.tokens[:j]
                m = cfg_oracle.mix(x, xs, req.cfg_alpha, ha, hb, *pen)
                x = cfg_oracle.emulate32(x, xs, req.cfg_alpha, ha, hb, *pen)
                tol = 2 * float(np.max(m["bound"][np.isfinite(m["mixed"])]))
            w = T.top_logprobs(x, req.logprobs, tok)
            got_ids = [a for a, _ in out.top_logprobs[j]]
            got_top = np.array([b for _, b in out.top_logprobs[j]])
            n_fin = int((w["ids"] >= 0).sum())
            assert len(got_ids) == n_fin, (i, j)
            assert abs(out.logprobs[j] - w["lp"]) <= w["lp_bound"] + tol, (i, j, out.logprobs[j], w["lp"])
            assert np.all(np.abs(got_top - w["top"][:n_fin]) <= w["bound"][:n_fin] + tol), (i, j)
            if tol == 0.0:
                assert got_ids == w["ids"][:n_fin].tolist(), (i, j)
            else:                                                    # ids may swap only between values within the mix's bound
                assert set(got_ids[:-1]) <= set(T.order(x)[:n_fin + 2].tolist()), (i, j)
            checked += 1
    assert checked >= 20
    # the same requests without logprobs: equal tokens, probs and finishes while both runs saw the same logits rows
    gen0, res0, ids0 = _run(st, emb, _requests(V, False))
    same = 0
    for i, (a, b) in enumerate(zip(res, res0)):
        ra, rb = _rows_of(gen, ids[i]), _rows_of(gen0, ids0[i])
        diverged = False
        for j in range(max(len(a.tokens), len(b.tokens)) + 1):
            if j not in ra or j not in rb or not (np.array_equal(ra[j][0].view(np.int32), rb[j][0].view(np.int32)) and
                                                   (ra[j][1] is None or np.array_equal(ra[j][1].view(np.int32), rb[j][1].view(np.int32)))):
                diverged = j < max(len(a.tokens), len(b.tokens))
                break
            if j < len(a.tokens):
                assert a.tokens[j] == b.tokens[j] and np.float32(a.probs[j]).tobytes() == np.float32(b.probs[j]).tobytes(), (i, j)
                same += 1
        if not diverged:
            assert a.tokens == b.tokens and a.finish == b.finish, i
    # the ragged route is deterministic, so every token compares; the fused step's atomics can part the runs after a few steps
    assert same >= (20 if route == "ragged_act" else 1), same


def test_speculative_logprobs(stacks):
    import torch
    from exllama_b200 import sampling
    from exllama_b200.speculative import SpeculativeGenerator
    target = stacks(kv_heads=2, seed=91)
    draft = stacks(kv_heads=2, layers=1, seed=91)
    draft.norm, draft.lm_head = target.norm, target.lm_head
    g = torch.Generator(device="cuda"); g.manual_seed(92)
    emb = (torch.randn((target.shape.vocab, target.shape.hidden), device="cuda", generator=g) * 0.5).half()
    prompt = list(range(3, 40, 3))

    def run(logprobs):
        rec = []
        for st in (target, draft):
            f = st.decode_step_fused_multi
            st.decode_step_fused_multi = (lambda f: lambda x, p: rec.append(f(x, p).clone()) or rec[-1])(f)
        try:
            gg = torch.Generator(device="cuda"); gg.manual_seed(93)
            gen = SpeculativeGenerator(target, draft, emb, emb, k=3, settings=sampling.Settings(),
                                       draft_settings=_settings(temperature=50.0, top_k=2), generator=gg, logprobs=logprobs)
            gen.begin(prompt)
            rounds = []
            for _ in range(8):
                n = gen.n
                a = gen.round()
                rounds.append((n, a, rec[-1].cpu().numpy()))
            return gen, rounds, [r.cpu().numpy() for r in rec]
        finally:
            del target.decode_step_fused_multi, draft.decode_step_fused_multi
    gen, rounds, rec = run(5)
    toks = gen.hist[:gen.n].tolist()
    k = 0
    for n, a, x in rounds:
        for i in range(a + 1):
            w = T.top_logprobs(x[i], 5, toks[n + i])
            lp, top = gen.token_logprobs[k], gen.top_logprobs[k]
            assert abs(lp - w["lp"]) <= w["lp_bound"], (n, i)
            assert [t for t, _ in top] == w["ids"][:len(top)].tolist() and len(top) == int((w["ids"] >= 0).sum()), (n, i)
            assert np.all(np.abs(np.array([v for _, v in top]) - w["top"][:len(top)]) <= w["bound"][:len(top)]), (n, i)
            k += 1
    assert k == len(gen.token_logprobs) == gen.n - len(prompt) - 1
    gen0, rounds0, rec0 = run(0)
    assert gen0.token_logprobs == [] and gen0.top_logprobs == []
    # the emitted tokens equal the run without logprobs up to the first step whose logits differ in any bit (fp32 atomics)
    same = next((c for c in range(min(len(rec), len(rec0))) if not np.array_equal(rec[c].view(np.int32), rec0[c].view(np.int32))), None)
    toks0 = gen0.hist[:gen0.n].tolist()
    if same is None:
        assert toks == toks0
    else:
        upto, calls = len(prompt) + 1, 0
        for n, a, _ in rounds:
            calls += 4                                               # k draft steps and one target step per round
            if calls > same:
                break
            upto = n + a + 1
        assert toks[:upto] == toks0[:upto]
