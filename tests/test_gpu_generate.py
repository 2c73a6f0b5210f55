"""Batched generation on the GPU (exl_sample_rows, exl_gen_advance, exllama_b200.generate): per-row sampler settings bitwise equal
to exl_sample on each row alone, per-row argument errors, graph replay; exl_gen_advance bitwise against its numpy restatement
(tests/generate_oracle.py); and BatchGenerator end to end on the synthetic stacks of tests/stack_harness.py, on the fused route and
on the prefill_ragged route (act-order): every token equals sampling.sample of its traced logits row with the request's settings,
history and U(seed, j); the traced logits match a fresh prefill; reused slots hold the new request's rows; stop ids, max_new_tokens
1, a full cache sequence and a request that fails alone."""
import ctypes as C

import numpy as np
import pytest

import generate_oracle as G
from stack_harness import lib_state, stacks  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu


def _settings(temperature=1.0, top_k=0, top_p=0.0, min_p=0.0, typical=0.0, penalty=(1.0, -1, 0)):
    from exllama_b200 import sampling
    s = sampling.Settings()
    s.temperature, s.top_k, s.top_p, s.min_p, s.typical = temperature, top_k, top_p, min_p, typical
    s.token_repetition_penalty_max, s.token_repetition_penalty_sustain, s.token_repetition_penalty_decay = penalty
    return s


MIXED = [dict(top_k=1), dict(temperature=0.95, top_k=40), dict(temperature=0.9, top_k=0, top_p=0.8, min_p=0.02),
         dict(temperature=1.0, typical=0.3), dict(temperature=0.95, top_k=40, top_p=0.65, penalty=(1.15, 256, 128)),
         dict(temperature=1.3, top_k=200, penalty=(1.3, -1, 0)), dict(temperature=0.7, top_p=0.9, typical=0.5, penalty=(1.1, 16, 64))]


def _rows(bsz, vocab, seed):
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    logits = torch.randn((bsz, vocab), device="cuda", generator=g) * 3
    hist = torch.randint(0, vocab, (bsz, 300), device="cuda", generator=g)
    u = torch.rand(bsz, device="cuda", generator=g)
    return logits, hist, u


def test_sample_rows_equal_rows_is_exl_sample():
    import torch
    from exllama_b200 import sampling
    logits, hist, u = _rows(8, 32000, 1)
    lens = [300, 0, 17, 299, 256, 1, 128, 300]
    for kw in MIXED:
        s = _settings(**kw)
        d1 = torch.empty_like(logits); d2 = torch.empty_like(logits)
        t1, p1 = sampling.sample(logits, s, history=hist, hist_lens=lens, u=u, bos_token_id=3, banned=[5, 6], dist=d1)
        t2, p2 = sampling.sample(logits, [s] * 8, history=hist, hist_lens=lens, u=u, bos_token_id=3, banned=[[5, 6]] * 8, dist=d2)
        assert torch.equal(t1, t2) and torch.equal(p1, p2) and torch.equal(d1, d2), kw


def test_sample_rows_mixed_settings():
    """Each row, with its own settings, bos id and banned list, is bitwise exl_sample run on that row alone."""
    import torch
    from exllama_b200 import sampling
    bsz, vocab = len(MIXED) + 2, 32000
    logits, hist, u = _rows(bsz, vocab, 2)
    sets = [_settings(**kw) for kw in MIXED] + [_settings(**MIXED[1]), _settings(**MIXED[4])]
    bos = [None, 1, 2, None, 1, None, 0, 1, None]
    banned = [None, [7, 8, 9], None, list(range(100, 600)), [1], None, None, list(range(vocab)), [3]]   # row 7 bans every token
    lens = [300, 12, 0, 300, 250, 299, 64, 5, 1]
    dist = torch.empty_like(logits)
    tok, prob = sampling.sample(logits, sets, history=hist, hist_lens=lens, u=u, bos_token_id=bos, banned=banned, dist=dist)
    assert int(tok[7]) == -1
    for b in range(bsz):
        d = torch.empty((1, vocab), device="cuda")
        t, p = sampling.sample(logits[b:b + 1], sets[b], history=hist[b:b + 1], hist_lens=[lens[b]], u=u[b:b + 1], bos_token_id=bos[b],
                               banned=banned[b], dist=d)
        assert int(t) == int(tok[b]) and torch.equal(p, prob[b:b + 1], ) if b != 7 else int(t) == -1, b
        assert torch.equal(d[0], dist[b]) or (b == 7 and bool(torch.isnan(d).all())), b


def test_sample_rows_graph_replay():
    import torch
    from exllama_b200 import sampling
    logits, hist, u = _rows(len(MIXED), 32000, 3)
    sets = [_settings(**kw) for kw in MIXED]
    lens = [300] * len(MIXED)
    want = sampling.sample(logits, sets, history=hist, hist_lens=lens, u=u)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            got = sampling.sample(logits, sets, history=hist, hist_lens=lens, u=u)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def test_sample_rows_errors_name_the_row():
    import torch
    from exllama_b200 import capi, sampling
    logits, hist, u = _rows(4, 1000, 4)
    good = _settings()
    for b, kw, msg in [(3, dict(top_k=1001), r"sample: row 3: top_k 1001 outside \[0, vocab 1000\]"),
                       (1, dict(temperature=0.0), "sample: row 1: temperature 0 is not finite and positive"),
                       (2, dict(top_p=-0.5), "sample: row 2: top_p -0.5 is negative"),
                       (0, dict(min_p=-1.0), "sample: row 0: min_p -1 is negative"),
                       (2, dict(typical=-1.0), "sample: row 2: typical -1 is negative"),
                       (1, dict(penalty=(1.1, -2, 0)), "sample: row 1: rep_sustain -2 < -1"),
                       (3, dict(penalty=(1.1, 5, -1)), "sample: row 3: rep_decay -1 < 0")]:
        sets = [good] * 4
        sets[b] = _settings(**kw)
        with pytest.raises(capi.ExlError, match=msg):
            sampling.sample(logits, sets, history=hist, u=u)
    p, _ = sampling.row_params([good] * 4, 4, logits.device)
    p[2].n_banned = 3
    tok = torch.empty(4, dtype=torch.int64, device="cuda"); prob = torch.empty(4, device="cuda")
    rc = capi.lib().exl_sample_rows(capi._ptr(logits), 4, 1000, 1000, None, 0, None, p, capi._ptr(u), capi._ptr(tok), capi._ptr(prob),
                                    None, None)
    assert rc == 1 and "sample: row 2: n_banned 3 with banned" in capi.lib().exl_last_error().decode()
    assert capi.lib().exl_sample_rows(capi._ptr(logits), 4, 1000, 1000, None, 0, None, None, capi._ptr(u), capi._ptr(tok),
                                      capi._ptr(prob), None, None) == 1
    assert "p_rows is NULL" in capi.lib().exl_last_error().decode()
    with pytest.raises(ValueError, match="3 settings for 4 rows"):
        sampling.sample(logits, [good] * 3, u=u)


# ---- exl_gen_advance ------------------------------------------------------------------------------------------------------------

def _advance(dev, rows_tok, rows_prob, slots, pos, js):
    from exllama_b200 import capi
    n = len(slots)
    arr = lambda v: (C.c_int * n)(*v)
    return capi.lib().exl_gen_advance(capi._ptr(rows_tok), capi._ptr(rows_prob), n, arr(slots), arr(pos), arr(js), capi._ptr(dev["hist"]),
                                      dev["hist"].shape[1], capi._ptr(dev["status"]), capi._ptr(dev["stop"]), capi._ptr(dev["seeds"]),
                                      dev["hist"].shape[0], capi._ptr(dev["embed"]), dev["embed"].shape[0], dev["embed"].shape[1],
                                      capi._ptr(dev["x_next"]), capi._ptr(dev["u_next"]), capi._ptr(dev["out_tok"]),
                                      capi._ptr(dev["out_prob"]), dev["out_tok"].shape[1], None)


def test_gen_advance_against_numpy():
    import torch
    rng = np.random.default_rng(5)
    n, ms, V, H = 8, 64, 500, 256
    host = dict(hist=rng.integers(0, V, (n, ms)), status=np.array([0, 0, 1, 0, 4, 0, 0, 0], np.int32),
                stop=np.full((n, G.MAX_STOP), -1, np.int64), seeds=rng.integers(0, 2 ** 63, n).astype(np.uint64) * np.uint64(2),
                embed=rng.standard_normal((V, H)).astype(np.float16), x_next=np.zeros((n, H), np.float16), u_next=np.zeros(n, np.float32),
                out_tok=rng.integers(0, V, (n, ms)), out_prob=rng.random((n, ms)).astype(np.float32))
    host["stop"][3, :3] = [11, 12, 13]
    host["stop"][6, 7] = 40
    dev = {k: torch.from_numpy(v.view(np.int64) if v.dtype == np.uint64 else v).cuda() for k, v in host.items()}
    tok = np.array([13, 40, 7, -1, 99, 40, 5], np.int64)                       # slot 3 stops (13), 6 stops (40), 7 errors
    prob = rng.random(7).astype(np.float32)
    slots, pos, js = [3, 6, 2, 7, -1, 0, 5], [10, 20, 30, 40, 0, 63, 1], [0, 5, 9, 63, 0, 12, 2]   # 2 already stopped; a -1 gap
    assert _advance(dev, torch.from_numpy(tok).cuda(), torch.from_numpy(prob).cuda(), slots, pos, js) == 0
    G.advance(host, tok, prob, slots, pos, js)
    for k, v in host.items():
        got = dev[k].cpu().numpy()
        want = v.view(np.int64) if v.dtype == np.uint64 else v
        assert np.array_equal(got, want, equal_nan=np.issubdtype(got.dtype, np.floating)), k
    assert host["status"].tolist() == [0, 0, 1, 1, 4, 0, 1, 4]
    # a second advance leaves every finished slot untouched
    before = {k: v.clone() for k, v in dev.items()}
    assert _advance(dev, torch.from_numpy(tok).cuda(), torch.from_numpy(prob).cuda(), [3, 6, 7, 2], [11, 21, 41, 31], [1, 6, 0, 10]) == 0
    assert all(torch.equal(before[k], dev[k]) for k in dev if k not in ("out_prob",))
    assert torch.equal(before["out_prob"].nan_to_num(), dev["out_prob"].nan_to_num())


def test_gen_advance_errors():
    import torch
    from exllama_b200 import capi
    n, ms, V, H = 4, 16, 50, 64
    dev = dict(hist=torch.zeros((n, ms), dtype=torch.int64, device="cuda"), status=torch.zeros(n, dtype=torch.int32, device="cuda"),
               stop=torch.full((n, 8), -1, dtype=torch.int64, device="cuda"), seeds=torch.zeros(n, dtype=torch.int64, device="cuda"),
               embed=torch.zeros((V, H), dtype=torch.float16, device="cuda"), x_next=torch.zeros((n, H), dtype=torch.float16, device="cuda"),
               u_next=torch.zeros(n, device="cuda"), out_tok=torch.zeros((n, ms), dtype=torch.int64, device="cuda"),
               out_prob=torch.zeros((n, ms), device="cuda"))
    t = torch.zeros(2, dtype=torch.int64, device="cuda"); p = torch.zeros(2, device="cuda")
    for slots, pos, js, msg in [([0, 4], [0, 0], [0, 0], r"row 1: slot 4 outside \[-1, n_slots 4\)"),
                                ([1, 1], [0, 0], [0, 0], "row 1: slot 1 named twice"),
                                ([0, 1], [16, 0], [0, 0], r"row 0: pos 16 outside \[0, hist_ld 16\)"),
                                ([0, 1], [0, 0], [0, -1], r"row 1: j -1 outside \[0, out_ld 16\)")]:
        assert _advance(dev, t, p, slots, pos, js) == 1
        import re
        assert re.search(msg, capi.lib().exl_last_error().decode()), capi.lib().exl_last_error()


# ---- BatchGenerator end to end --------------------------------------------------------------------------------------------------

def _embed(st, seed=11):
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    return (torch.randn((st.shape.vocab, st.shape.hidden), device="cuda", generator=g) * 0.5).half()


LENS = [1, 17, 200, 513]


def _requests(vocab, stop=None):
    from exllama_b200.generate import Request
    rng = np.random.default_rng(9)
    sets = [_settings(**kw) for kw in MIXED]
    out = []
    for i in range(10):
        L = LENS[i % 4]
        out.append(Request(rng.integers(0, vocab, L), [12, 1, 9, 30, 6, 20, 8, 15, 10, 7][i], settings=sets[i % len(sets)], seed=1000 + i,
                           bos_token_id=[None, 1][i % 2], banned=[None, [4, 5]][i % 3 == 0]))
    out[2].max_new_tokens = 1
    out[5].banned = list(range(vocab))                                         # fails alone
    out.append(Request(rng.integers(0, vocab, 620), 100, settings=sets[1], seed=77))   # reaches max_seq 640
    if stop is not None:
        out[stop[0]].stop_ids = [stop[1]]
    return out


def _run(st, emb, reqs):
    from exllama_b200.generate import BatchGenerator
    gen = BatchGenerator(st, emb)
    gen.trace = []
    ids = [gen.submit(r) for r in reqs[:6]]
    for _ in range(3):
        gen.step()
    ids += [gen.submit(r) for r in reqs[6:9]]
    for _ in range(4):
        gen.step()
    ids += [gen.submit(r) for r in reqs[9:]]
    res = gen.run()
    return gen, [res[i] for i in ids], ids


def _check_trace(gen, reqs, res, ids):
    """Every token is sampling.sample of its traced logits row with the request's settings, history and U(seed, j), bitwise."""
    import torch
    from exllama_b200 import sampling
    rid_req = dict(zip(ids, zip(reqs, res)))
    seen = 0
    for e in gen.trace:
        for r, (rid, j) in enumerate(zip(e["rids"], e["j"])):
            req, out = rid_req[rid]
            if j > len(out.tokens) or (j == len(out.tokens) and out.finish != "error"):
                continue                                                        # the extra step after a stop
            hist = torch.tensor([req.prompt + out.tokens[:j]], device="cuda")
            u = torch.tensor([G.U(req.seed, j)], device="cuda")
            assert float(e["u"][r]) == float(u[0]), (rid, j)
            t, p = sampling.sample(torch.from_numpy(e["logits"][r:r + 1]).cuda(), req.settings, history=hist, u=u,
                                   bos_token_id=req.bos_token_id, banned=req.banned)
            if j == len(out.tokens):
                assert int(t) == -1 and out.finish == "error", (rid, j)
            else:
                assert int(t) == out.tokens[j] and float(p) == out.probs[j], (rid, j, int(t), out.tokens[j])
            seen += 1
    return seen


def _prefill_check(ref, emb, trace, rid, req, out, what):
    """The request's last traced logits row against a fresh prefill of its prompt and tokens before it."""
    import torch
    last = [(e, r) for e in trace for r, x in enumerate(e["rids"]) if x == rid]
    e, r = last[-1]
    j = e["j"][r]
    ids = torch.tensor(req.prompt + out.tokens[:j], device="cuda")
    want = ref.prefill(emb[ids].view(1, len(ids), -1), 0)[0].double().cpu().numpy()
    got = e["logits"][r].astype(np.float64)
    err = np.abs(got - want).max()
    assert err <= 2e-2 * np.sqrt((want ** 2).mean()) + 2e-2 * np.abs(want).max(), (what, rid, err)


def _row_check(st, ref, slot, tokens, n, emb, what):
    """Rows [1, n) of cache sequence slot against a fresh prefill of tokens[:n] (row 0 of a free slot is rewritten whenever a fused
    step covers it at past_len 0)."""
    import torch
    ids = torch.tensor(tokens[:n], device="cuda")
    ref.prefill(emb[ids].view(1, n, -1), 0, seq=0)
    for i in range(st.n_layers):
        for name, a, b in (("k", st.key_cache[i], ref.key_cache[i]), ("v", st.value_cache[i], ref.value_cache[i])):
            got, want = a[slot, :, 1:n].float(), b[0, :, 1:n].float()
            rms = want.pow(2).mean(dim=(0, 2), keepdim=True).sqrt()
            bad = (got - want).abs() > 1e-2 * want.abs() + 1e-2 * rms
            assert not bad.any(), f"{what}: layer {i} {name} slot {slot}: {int(bad.sum())} outside"


@pytest.mark.parametrize("route", ["fused", "ragged_act"])
def test_batch_generator(stacks, route):
    kw = dict(batch=4, seed=51, max_seq=640, act=route == "ragged_act")
    st = stacks(**kw)
    ref = stacks(**dict(kw, batch=1))
    emb = _embed(st)
    V = st.shape.vocab
    reqs = _requests(V)
    gen, res, ids = _run(st, emb, reqs)
    assert gen.fused == (route == "fused")
    # a stop id the second run hits: request 3's fourth token (its first occurrence ends it)
    stop_tok = res[3].tokens[3]
    reqs2 = _requests(V, stop=(3, stop_tok))
    gen2, res2, ids2 = _run(st, emb, reqs2)
    k = res[3].tokens.index(stop_tok)              # both runs step the same rows until request 3 stops: the same tokens so far
    assert res2[3].tokens == res[3].tokens[:k + 1] and res2[3].finish == "stop"
    assert res2[2].finish == "length" and len(res2[2].tokens) == 1
    assert res2[5].finish == "error" and res2[5].tokens == []
    assert res2[10].finish == "max_seq" and len(res2[10].tokens) == 640 - 620
    for i, r in enumerate(res2):
        if i not in (3, 5, 10):
            assert r.finish == "length" and len(r.tokens) == reqs2[i].max_new_tokens, i
    assert _check_trace(gen2, reqs2, res2, ids2) >= sum(len(r.tokens) for r in res2)
    for i in (0, 3, 7, 10):
        _prefill_check(ref, emb, gen2.trace, ids2[i], reqs2[i], res2[i], route)
    # every slot holds the last request admitted into it: rows [0, L + n - 1) equal a fresh prefill of its tokens
    last = {}
    for ev in gen2.order:
        if ev[1] == "admit":
            for rid, s in ev[2]:
                last[s] = rid
    for s, rid in last.items():
        i = ids2.index(rid)
        toks = reqs2[i].prompt + res2[i].tokens
        n = len(toks) - (res2[i].finish != "error")
        _row_check(st, ref, s, toks, n, emb, f"{route} slot {s}")


def test_greedy_batch_equals_alone(stacks):
    """top_k 1 on tied embeddings (c * lm_head): each request's tokens in a batch of 4 equal the same request run alone, up to the
    first position whose top-2 logit gap is within tolerance."""
    import torch
    from exllama_b200.generate import BatchGenerator, Request
    st = stacks(batch=4, seed=61, max_seq=256)
    one = stacks(batch=1, seed=61, max_seq=256)
    emb = (st.lm_head.float() * 40).half().contiguous()
    rng = np.random.default_rng(3)
    reqs = [Request(rng.integers(0, st.shape.vocab, L), 24, settings=_settings(top_k=1), seed=i) for i, L in enumerate([5, 40, 90, 17])]
    gen = BatchGenerator(st, emb)
    gen.trace = []
    ids = [gen.submit(r) for r in reqs]
    res = gen.run()
    for rid, req in zip(ids, reqs):
        alone = BatchGenerator(one, emb)
        alone.trace = []
        aid = alone.submit(req)
        a = alone.run()[aid]
        b = res[rid]
        rows = [(e["j"][r], e["logits"][r]) for e in alone.trace for r, x in enumerate(e["rids"]) if x == aid]
        for j, lg in rows:
            top2 = np.sort(lg.astype(np.float64))[-2:]
            if top2[1] - top2[0] <= 2e-2 * np.sqrt((lg.astype(np.float64) ** 2).mean()):
                break
            assert a.tokens[j] == b.tokens[j], (rid, j)


def test_steady_steps_never_wait_on_the_device(stacks):
    """On the fused route a step() of live requests launches the step, the sampler and the advance and reads the status copied one
    step earlier behind its event: over 8 steady steps of 4 live requests torch's sync debug mode sees no synchronising call."""
    import warnings
    import torch
    from exllama_b200.generate import BatchGenerator, Request
    st = stacks(batch=4, seed=53, max_seq=256)
    gen = BatchGenerator(st, _embed(st))
    rng = np.random.default_rng(4)
    for b in range(4):
        gen.submit(Request(rng.integers(0, st.shape.vocab, 20 + b), 40, settings=_settings(**MIXED[b]), seed=b))
    for _ in range(3):
        gen.step()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            for _ in range(8):
                gen.step()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = [x for x in w if "called a synchronizing CUDA operation" in str(x.message)]
    assert gen.fused and len(syncs) == 0, [str(x.message) for x in syncs[:3]]
    assert all(r.finish == "length" and len(r.tokens) == 40 for r in gen.run().values())
