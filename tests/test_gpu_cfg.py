"""Classifier-free guidance on the GPU (csrc/cfg.cu exl_cfg_mix, exllama_b200/cfg.py, guided requests in exllama_b200/generate.py):
the mix against the float64 oracle (oracle/cfg_oracle.py) within its per-element bound, both rows of a pair bitwise equal and every
other row bitwise unchanged, over vocabularies 1 .. 262144, every alpha, three penalty triples and 1, 2 and 32 pairs; undefined
input; determinism and graph replay; every argument error; the reference's own cases (tests/golden/cfg_ref.npz) through the mix
and exl_sample's dist; and BatchGenerator with guided and plain requests on the fused and ragged routes, checked token by token
against cfg.mix + sampling.sample of the traced row pairs, with each slot's cache rows against a fresh prefill."""
import ctypes as C
import os

import numpy as np
import pytest

import generate_oracle as G
from oracle import cfg_oracle as F
from stack_harness import lib_state, stacks  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cfg_ref.npz")
ALPHAS = [0.0, 0.5, 1.0, -0.4, 1.4, 3.0]
PENALTIES = [(1.0, -1, 0), (1.15, 256, 128), (1.3, -1, 0)]


def _settings(temperature=1.0, top_k=0, top_p=0.0, min_p=0.0, typical=0.0, penalty=(1.0, -1, 0)):
    from exllama_b200 import sampling
    s = sampling.Settings()
    s.temperature, s.top_k, s.top_p, s.min_p, s.typical = temperature, top_k, top_p, min_p, typical
    s.token_repetition_penalty_max, s.token_repetition_penalty_sustain, s.token_repetition_penalty_decay = penalty
    return s


def _inputs(rows, vocab, seed, ld=None, hist_ld=2000):
    rng = np.random.default_rng(seed)
    ld = ld or vocab
    lg = (rng.standard_normal((rows, ld)) * rng.choice([0.5, 3.0, 30.0], size=(rows, 1))).astype(np.float32)
    hist = rng.integers(0, vocab, (rows, hist_ld)).astype(np.int64)
    lens = [int(x) for x in rng.choice([0, 1, 17, 300, 1920, hist_ld], size=rows)]
    return lg, hist, lens


def _check_mix(vocab, rows, pairs, alphas, pen, seed, ld=None):
    import torch
    from exllama_b200 import cfg
    lg, hist, lens = _inputs(rows, vocab, seed, ld)
    t = torch.from_numpy(lg).cuda()
    view = t[:, :vocab]
    cfg.mix(view, pairs, alphas, _settings(penalty=pen), history=torch.from_numpy(hist).cuda(), hist_lens=lens)
    got = t.cpu().numpy()
    in_pair = {r for p in pairs for r in p}
    for r in range(rows):
        if r not in in_pair:
            assert np.array_equal(got[r].view(np.uint32), lg[r].view(np.uint32)), f"row {r} outside the pairs changed"
    assert np.array_equal(got[:, vocab:].view(np.uint32), lg[:, vocab:].view(np.uint32)), "columns past vocab changed"
    for (a, b), alpha in zip(pairs, alphas):
        assert np.array_equal(got[a, :vocab].view(np.uint32), got[b, :vocab].view(np.uint32)), (a, b)
        res = F.mix(lg[a, :vocab], lg[b, :vocab], alpha, hist[a, :lens[a]], hist[b, :lens[b]], *pen)
        assert F.within(got[a, :vocab], res), (vocab, a, b, alpha, pen, float(np.nanmax(np.abs(got[a, :vocab] - res["mixed"]) / res["bound"])))


@pytest.mark.parametrize("vocab", [1, 7, 32000, 32001, 128256, 262144])
def test_mix_against_oracle(vocab):
    for i, pen in enumerate(PENALTIES):
        # one pair per alpha, a > b, non-adjacent rows, a padded leading dimension
        _check_mix(vocab, 9, [(7, 2)], [ALPHAS[(2 * i) % 6]], pen, 10 * i + 1, ld=vocab + 5)
        _check_mix(vocab, 6, [(0, 5), (3, 1)], [ALPHAS[(2 * i + 1) % 6], ALPHAS[(2 * i + 2) % 6]], pen, 10 * i + 2)
    if vocab <= 128256:
        rng = np.random.default_rng(vocab)
        perm = rng.permutation(64)
        pairs = [(int(perm[2 * k]), int(perm[2 * k + 1])) for k in range(32)]
        _check_mix(vocab, 64, pairs, [ALPHAS[k % 6] for k in range(32)], PENALTIES[1], 77)


def test_every_alpha_and_penalty_at_32000():
    for alpha in ALPHAS:
        for j, pen in enumerate(PENALTIES):
            _check_mix(32000, 4, [(1, 3)], [alpha], pen, 100 + j)


def test_undefined_input():
    import torch
    from exllama_b200 import cfg
    vocab = 1000
    lg, hist, _ = _inputs(8, vocab, 5)
    lg[1, 10] = np.nan                                 # pair (1, 0)
    lg[3, :] = -np.inf                                 # pair (2, 3)
    hist[4, 5] = vocab                                 # pair (5, 4): a bad id inside the penalty window
    t = torch.from_numpy(lg).cuda()
    cfg.mix(t, [(1, 0), (2, 3), (5, 4), (6, 7)], [0.5] * 4, _settings(penalty=(1.15, -1, 0)), history=torch.from_numpy(hist).cuda(),
            hist_lens=[50] * 8)
    got = t.cpu().numpy()
    for r in range(6):
        assert np.isnan(got[r]).all(), r
    res = F.mix(lg[6], lg[7], 0.5, hist[6, :50], hist[7, :50], 1.15, -1, 0)
    assert F.within(got[6], res) and np.array_equal(got[6], got[7])
    # the sampler returns -1 for both rows of an undefined pair
    from exllama_b200 import sampling
    tok, _ = sampling.sample(t, _settings(), u=torch.full((8,), 0.5, device="cuda"))
    assert tok.cpu().tolist()[:6] == [-1] * 6 and min(tok.cpu().tolist()[6:]) >= 0


def test_two_calls_bitwise_and_graph_replay():
    import torch
    from exllama_b200 import cfg
    lg, hist, lens = _inputs(6, 32000, 9)
    h = torch.from_numpy(hist).cuda()
    s = _settings(penalty=(1.15, 256, 128))
    pairs, alphas = [(0, 3), (4, 1), (2, 5)], [1.4, -0.4, 3.0]
    a = torch.from_numpy(lg).cuda(); b = a.clone(); g_in = a.clone()
    cfg.mix(a, pairs, alphas, s, history=h, hist_lens=lens)
    cfg.mix(b, pairs, alphas, s, history=h, hist_lens=lens)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=st):
            cfg.mix(g_in, pairs, alphas, s, history=h, hist_lens=lens)
    g_in.copy_(torch.from_numpy(lg).cuda())
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(g_in.view(torch.int32), a.view(torch.int32))


def test_argument_errors():
    import torch
    from exllama_b200 import capi
    lib = capi.lib()
    lg = torch.zeros((4, 100), device="cuda")
    hist = torch.zeros((4, 8), dtype=torch.int64, device="cuda")

    def call(pairs, rows=4, vocab=100, ld=100, lens=(0, 0, 0, 0), history=True, logits=True, n=None):
        arr = (capi.ExlCfgPair * len(pairs))(*[capi.ExlCfgPair(*p) for p in pairs]) if pairs is not None else None
        hl = (C.c_int * 4)(*lens) if lens is not None else None
        rc = lib.exl_cfg_mix(capi._ptr(lg) if logits else None, rows, vocab, ld, capi._ptr(hist) if history else None, 8, hl, arr,
                             n if n is not None else len(pairs or [ok]), None)
        return rc, lib.exl_last_error().decode()

    ok = (0, 1, 0.5, 1.1, -1, 0)
    assert call([ok])[0] == 0
    for kw, msg in [(dict(pairs=[(0, 4, 0.5, 1.1, -1, 0)]), r"pair 0: row b 4 outside \[0, rows 4\)"),
                    (dict(pairs=[(-1, 2, 0.5, 1.1, -1, 0)]), r"pair 0: row a -1 outside"),
                    (dict(pairs=[(2, 2, 0.5, 1.1, -1, 0)]), "pair 0: a == b == 2"),
                    (dict(pairs=[ok, (3, 1, 0.5, 1.1, -1, 0)]), "pair 1: row 1 is already in pair 0"),
                    (dict(pairs=[(0, 1, float("nan"), 1.1, -1, 0)]), "pair 0: alpha nan is not finite"),
                    (dict(pairs=[(0, 1, float("inf"), 1.1, -1, 0)]), "pair 0: alpha inf is not finite"),
                    (dict(pairs=[(0, 1, 0.5, 1.1, -2, 0)]), "pair 0: rep_sustain -2 < -1"),
                    (dict(pairs=[(0, 1, 0.5, 1.1, 4, -1)]), "pair 0: rep_decay -1 < 0"),
                    (dict(pairs=[ok], lens=(0, 9, 0, 0)), r"hist_len\[1\] 9 outside \[0, hist_ld 8\]"),
                    (dict(pairs=[ok], lens=(0, 0, -1, 0)), r"hist_len\[2\] -1 outside"),
                    (dict(pairs=[ok], lens=None), "history without hist_len_host"),
                    (dict(pairs=[ok], ld=99), "ld 99 < vocab 100"),
                    (dict(pairs=[ok], rows=0), r"rows 0 outside \[1, 64\]"),
                    (dict(pairs=[ok], rows=65), r"rows 65 outside"),
                    (dict(pairs=[ok], vocab=0, ld=100), r"vocab 0 outside \[1, 262144\]"),
                    (dict(pairs=[ok], vocab=262145, ld=262145), "vocab 262145 outside"),
                    (dict(pairs=[ok], n=0), r"n_pairs 0 outside \[1, 32\]"),
                    (dict(pairs=[ok], n=33), "n_pairs 33 outside"),
                    (dict(pairs=[ok], logits=False), "NULL pointer"),
                    (dict(pairs=None), "NULL pointer")]:
        import re
        rc, err = call(**kw)
        assert rc == 1 and re.search(msg, err), (kw, err)
    assert call([ok], history=False, lens=None)[0] == 0                  # no history: no penalty, no lengths needed


def test_reference_cases():
    """Every case of the fixture through exl_cfg_mix and exl_sample's dist: the reference's kept set, its probabilities within 1e-5."""
    import torch
    from exllama_b200 import cfg, sampling
    for i, c in enumerate(F.golden_cases(GOLD)):
        V = c["vocab"]
        hl = len(c["hist_a"])
        t = torch.from_numpy(np.stack([c["logits_a"], c["logits_b"]])).cuda()
        h = torch.from_numpy(np.stack([c["hist_a"], c["hist_b"]]) if hl else np.zeros((2, 1), np.int64)).cuda()
        pen = (c["penalty_max"], c["sustain"], c["decay"])
        cfg.mix(t, [(0, 1)], [c["alpha"]], _settings(penalty=pen), history=h, hist_lens=[hl, hl])
        dist = torch.empty((1, V), device="cuda")
        sampling.sample(t[:1], _settings(c["temperature"], c["top_k"], c["top_p"], c["min_p"], c["typical"]),
                        u=torch.full((1,), 0.5, device="cuda"), dist=dist)
        d = dist[0].cpu().numpy()
        want = np.zeros(V)
        want[c["kept"]] = c["probs"]
        np.testing.assert_array_equal(np.nonzero(d >= 1e-30)[0], np.nonzero(want >= 1e-30)[0], err_msg=f"case {i}")
        np.testing.assert_allclose(d, want, rtol=1e-5, atol=1e-7, err_msg=f"case {i}")


# ---- guided requests in BatchGenerator ------------------------------------------------------------------------------------------

def _embed(st, seed=11):
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    return (torch.randn((st.shape.vocab, st.shape.hidden), device="cuda", generator=g) * 0.5).half()


def _requests(vocab, stop=None):
    from exllama_b200.generate import Request
    rng = np.random.default_rng(19)
    P = lambda n: rng.integers(0, vocab, n)
    sets = [_settings(temperature=0.95, top_k=40, top_p=0.65, penalty=(1.15, 256, 128)), _settings(temperature=0.9, top_p=0.8, min_p=0.02),
            _settings(temperature=1.0, typical=0.3, penalty=(1.3, -1, 0)), _settings(top_k=1)]
    out = [Request(P(17), 10, sets[0], seed=1, cfg_prompt=P(40), cfg_alpha=1.4),
           Request(P(200), 8, sets[1], seed=2),
           Request(P(5), 12, sets[2], seed=3, cfg_prompt=P(1), cfg_alpha=-0.4, bos_token_id=1),
           Request(P(30), 6, sets[3], seed=4, cfg_prompt=P(9), cfg_alpha=3.0, banned=list(range(vocab))),          # error
           Request(P(600), 100, sets[0], seed=5, cfg_prompt=P(610), cfg_alpha=0.5),                             # max_seq: 30 tokens
           Request(P(9), 5, sets[1], seed=6),
           Request(P(60), 14, sets[0], seed=7, cfg_prompt=P(33), cfg_alpha=0.0, banned=[4, 5]),
           Request(P(3), 9, sets[2], seed=8, cfg_prompt=P(120), cfg_alpha=1.0)]
    if stop is not None:
        out[stop[0]].stop_ids = [stop[1]]
    return out


def _run(st, emb, reqs):
    from exllama_b200.generate import BatchGenerator
    gen = BatchGenerator(st, emb)
    gen.trace = []
    ids = [gen.submit(r) for r in reqs[:4]]
    for _ in range(3):
        gen.step()
    ids += [gen.submit(r) for r in reqs[4:6]]
    for _ in range(2):
        gen.step()
    ids += [gen.submit(r) for r in reqs[6:]]
    res = gen.run()
    return gen, [res[i] for i in ids], ids


def _check_trace(gen, reqs, res, ids):
    """Every guided token is bitwise cfg.mix + sampling.sample of its traced row pair; every plain one sampling.sample of its row."""
    import torch
    from exllama_b200 import cfg, sampling
    rid_req = dict(zip(ids, zip(reqs, res)))
    seen = 0
    for e in gen.trace:
        rows = {}
        for r, (rid, sh) in enumerate(zip(e["rids"], e["shadow"])):
            rows.setdefault(rid, [None, None])[int(sh)] = r
        for rid, (r, r2) in rows.items():
            req, out = rid_req[rid]
            j = e["j"][r]
            if j > len(out.tokens) or (j == len(out.tokens) and out.finish != "error"):
                continue
            u = torch.tensor([G.U(req.seed, j)], device="cuda")
            assert float(e["u"][r]) == float(u[0])
            if req.cfg_prompt is None:
                hist = torch.tensor([req.prompt + out.tokens[:j]], device="cuda")
                t, p = sampling.sample(torch.from_numpy(e["logits"][r:r + 1]).cuda(), req.settings, history=hist, u=u,
                                       bos_token_id=req.bos_token_id, banned=req.banned)
            else:
                assert e["j"][r2] == j and float(e["u"][r2]) == float(u[0])
                ha, hb = req.prompt + out.tokens[:j], req.cfg_prompt + out.tokens[:j]
                hist = torch.zeros((2, max(len(ha), len(hb))), dtype=torch.int64)
                hist[0, :len(ha)] = torch.tensor(ha); hist[1, :len(hb)] = torch.tensor(hb)
                lg = torch.from_numpy(np.stack([e["logits"][r], e["logits"][r2]])).cuda()
                cfg.mix(lg, [(0, 1)], [req.cfg_alpha], req.settings, history=hist.cuda(), hist_lens=[len(ha), len(hb)])
                t, p = sampling.sample(lg[:1], req.settings, u=u, bos_token_id=req.bos_token_id, banned=req.banned)
            if j == len(out.tokens):
                assert int(t) == -1 and out.finish == "error", (rid, j)
            else:
                assert int(t) == out.tokens[j] and float(p) == out.probs[j], (rid, j, int(t), out.tokens[j])
            seen += 1
    return seen


def _row_check(st, ref, slot, tokens, n, emb, what):
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
def test_batch_generator_guided(stacks, route):
    kw = dict(batch=4, seed=71, max_seq=640, act=route == "ragged_act")
    st = stacks(**kw)
    ref = stacks(**dict(kw, batch=1))
    emb = _embed(st)
    V = st.shape.vocab
    gen, res, ids = _run(st, emb, _requests(V))
    assert gen.fused == (route == "fused")
    stop_tok = res[0].tokens[4]
    reqs = _requests(V, stop=(0, stop_tok))
    gen, res, ids = _run(st, emb, reqs)
    k = res[0].tokens.index(stop_tok)
    assert res[0].finish == "stop" and len(res[0].tokens) == k + 1
    assert res[3].finish == "error" and res[3].tokens == []
    assert res[4].finish == "max_seq" and len(res[4].tokens) == 640 - 610
    for i in (1, 2, 5, 6, 7):
        assert res[i].finish == "length" and len(res[i].tokens) == reqs[i].max_new_tokens, i
    assert _check_trace(gen, reqs, res, ids) >= sum(len(r.tokens) for r in res)
    # both slots of every guided request wrote the same tokens; each slot holds its own prompt followed by the tokens
    slots = {}
    for ev in gen.order:
        if ev[1] == "admit":
            for rid, s in ev[2]:
                slots.setdefault(rid, []).append(s)
    last = {}
    for rid, ss in slots.items():
        for s in ss:
            last[s] = (rid, ss)
    for s, (rid, ss) in last.items():
        i = ids.index(rid)
        req, out = reqs[i], res[i]
        n_tok = len(out.tokens)
        if len(ss) == 2 and last[ss[0]][0] == last[ss[1]][0] == rid:
            assert np.array_equal(gen.dev.out_tok[ss[0], :n_tok].cpu().numpy(), gen.dev.out_tok[ss[1], :n_tok].cpu().numpy()), rid
        prompt = req.prompt if s == ss[0] else req.cfg_prompt
        toks = prompt + out.tokens
        n = len(toks) - (out.finish != "error")
        _row_check(st, ref, s, toks, n, emb, f"{route} slot {s}")


def test_generate_cfg_alpha_zero_greedy_is_plain(stacks):
    """top_k 1 on tied embeddings: an alpha 0 guided request emits the plain request's tokens (log-softmax keeps the argmax), up to
    the first near-tie of the plain run's logits."""
    from exllama_b200 import cfg
    from exllama_b200.generate import BatchGenerator, Request
    st = stacks(batch=4, seed=81, max_seq=256)
    emb = (st.lm_head.float() * 40).half().contiguous()
    rng = np.random.default_rng(5)
    s = _settings(top_k=1)
    prompts = [(rng.integers(0, st.shape.vocab, 23).tolist(), rng.integers(0, st.shape.vocab, 41).tolist()),
               (rng.integers(0, st.shape.vocab, 7).tolist(), rng.integers(0, st.shape.vocab, 3).tolist())]
    guided = cfg.generate_cfg(st, emb, prompts, 0.0, max_new_tokens=20, settings=s)
    gen = BatchGenerator(st, emb)
    gen.trace = []
    pid = [gen.submit(Request(p, 20, s, seed=i)) for i, (p, _) in enumerate(prompts)]
    res = gen.run()
    for i, ((p, _), rid) in enumerate(zip(prompts, pid)):
        plain = res[rid].tokens
        assert guided[i][:len(p)] == p
        rows = sorted((e["j"][r], e["logits"][r]) for e in gen.trace for r, x in enumerate(e["rids"]) if x == rid)
        for j, lg in rows:
            top2 = np.sort(lg.astype(np.float64))[-2:]
            if top2[1] - top2[0] <= 2e-2 * np.sqrt((lg.astype(np.float64) ** 2).mean()):
                break
            assert guided[i][len(p) + j] == plain[j], (i, j)
