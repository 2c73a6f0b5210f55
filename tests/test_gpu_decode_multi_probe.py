"""The multi-token decode step (exl_decode_step_multi) checked on its own output: planted-key caches through attention probe stacks,
and phase-probe stacks, on multi-token plans.

test_gpu_decode_multi.py sees this path through logits, final hidden state and new k / v rows at 1e-2 of their rms, where a
nearly flat softmax over N(0, 0.25) caches makes attention a small share of the residual: a causal tail that leaks the next
token's row, a token handed its neighbour's partial, q roped at past_len instead of past_len + t, or history read from another
cache sequence all stay inside that tolerance.  Here (tests/helpers.py, "Attention probe", with n tokens: virtual query head
t * heads + h) every planted query vector of every token answers the mean of V over its own plateau, background heads are held
to the q-error bound, rows past..past+n-1 hold poison keys the launch must overwrite before reading, and rows after them are NaN.
tests/test_multi_probe_oracle.py shows on the CPU that each of those bugs misses this file's bounds by >= 10x.

The phase probes (test_gpu_decode_phase_probe.py) on multi-token plans: each token's new k / v rows (QKV), x_out - x_in (MLP),
the layer hand-off and every token's logits, bounded element by element at position past + t.  Act-order and LoRA plans are
refused for multi-token steps (test_gpu_decode_multi.py::test_rejected_arguments)."""
import numpy as np
import pytest

from helpers import (assert_within_any, assert_within_bound, attn_probe_stack, mlp_expectation, multi_probe_specs, newest_inputs,
                     phase_probe_edit, plant_probe, probe_caches, probe_expectation, qkv_expectation, snap_of)
from stack_harness import check_head, lib_state, stacks  # noqa: F401

pytestmark = pytest.mark.gpu

# the most tokens a plan of the 1024-wide, 8-head probe stacks takes (max_tokens_for on an H100): 4, but 2 under 8 query heads per
# KV head, whose 4 tokens would be 32 query vectors per KV head in shared memory
MAX_TOKENS = {8: 4, 4: 4, 2: 4, 1: 2}


def _shape(hidden, inter, heads, kv_heads=None):
    from exllama_b200.stack import LlamaShape
    return LlamaShape("multi-probe", hidden, inter, 1, heads, vocab=32000, kv_heads=kv_heads)


def _x(n, hidden, seed):
    return (1e-2 * np.random.default_rng(seed).standard_normal((n, hidden))).astype(np.float16)


def _load(st, caches):
    import torch
    for kc, vc, (k0, v0) in zip(st.key_cache, st.value_cache, caches):
        kc.copy_(torch.from_numpy(k0)); vc.copy_(torch.from_numpy(v0))
    torch.cuda.synchronize()


def _report(capsys, what, worst):
    with capsys.disabled():
        print(f"\n{what}: tightest margin (largest |got - want| / bound) {worst:.3g}")


def run_multi(st, caches, x, past, seq=0):
    """Load the caches, launch the n tokens of x [n, hidden] at past_len on cache sequence seq: final hidden states [n, hidden]."""
    import torch
    _load(st, caches)
    n = x.shape[0]
    st.decode_step_fused_multi(torch.from_numpy(x).cuda().view(n, 1, -1), past, seq=seq)
    torch.cuda.synchronize()
    return st._plan_xout[:n].cpu().numpy()


def _probe(oracle, st, past, spec, seed, caches0, x, seq=0, nan_others=False):
    """Plant a copy of caches0 for the launch of x at past (sequence seq; nan_others: every other sequence all NaN), run the
    multi-token step: (got, want, bound) [n, hidden]."""
    caches = [[c.copy() for c in kv] for kv in caches0]
    plants = plant_probe(oracle, st, caches, x, past, spec, seed, seq=seq)
    if nan_others:
        for kc, vc in caches:
            for b in range(kc.shape[0]):
                if b != seq:
                    kc[b] = np.nan; vc[b] = np.nan
    got = run_multi(st, caches, x, past, seq)
    want, bound = probe_expectation(oracle, st, snap_of(caches), x, past, plants, "step", seq=seq)
    return got.reshape(want.shape), want, bound


def _check(oracle, st, past, spec, seed, caches0, x, what, **kw):
    got, want, bound = _probe(oracle, st, past, spec, seed, caches0, x, **kw)
    return assert_within_bound(got, bound, want, what)


def _sweep(oracle, st, pasts, seed, what, layouts, max_tokens=4, background=False):
    """Every layout of `layouts` (multi_probe_specs names) at every context of `pasts`, in order, on one plan; the token count
    runs max_tokens, max_tokens - 1, .., 1 and round again.  Returns the largest err / bound."""
    caches0 = probe_caches(st, seed)
    worst = 0.0
    for i, past in enumerate(pasts):
        n = min(max_tokens - i % max_tokens, st.max_seq - past)
        x = _x(n, st.shape.hidden, seed + i)
        for name, spec in multi_probe_specs(st, n, past, background):
            if name in layouts:
                worst = max(worst, _check(oracle, st, past, spec, seed + 7 * i, caches0, x, f"{what} ctx {past} n {n} {name}"))
    return worst


# -------------------------------------------------------------------------------------------------------------- attention probes
@pytest.mark.parametrize("kv", [8, 4, 2, 1])
def test_multi_probe_contexts(oracle, capsys, kv):
    """Two layers, ONE plan swept from the longest context down (every partial slot written first), then short contexts where a
    KV head's CTA range holds CTAs without a unit (att_needs_reset_multi): n_rep 1, 2, 4, 8 (kv 1 at its 2-token limit), so up to 16 query vectors
    per KV head, each with its own plateau."""
    st = attn_probe_stack(_shape(1024, 2816, 8, kv), 2, 1024, seed=20 + kv)
    st.make_plan(with_head=False, max_tokens=MAX_TOKENS[kv])
    worst = _sweep(oracle, st, [1024 - MAX_TOKENS[kv], 0, 1, 15, 16, 17, 37, 255, 1000], 1000 + 10 * kv, f"kv {kv}",
                   ("dense", "lone+0"), max_tokens=MAX_TOKENS[kv])
    _report(capsys, f"contexts kv {kv}", worst)
    st.dplan.close(); st.close()


@pytest.mark.parametrize("kv", [8, 2])
def test_multi_probe_background_heads(oracle, capsys, kv):
    """One layer, the odd KV heads' query vectors on the plain cache: at short contexts the launch's own rows carry a large share
    of their softmax, so the causal tail (which new rows each token reads, and with which scores) is held to the q-error bound.
    A future leak or a missing own row is invisible to planted heads and shows here."""
    st = attn_probe_stack(_shape(1024, 2816, 8, kv), 1, 512, seed=30 + kv)
    st.make_plan(with_head=False, max_tokens=4)
    worst = _sweep(oracle, st, [0, 1, 16, 37, 0, 1, 16, 37], 1100 + kv, f"background kv {kv}", ("dense", "lone+0"),
                   background=True)
    _report(capsys, f"background kv {kv}", worst)
    st.dplan.close(); st.close()


@pytest.mark.parametrize("kv", [8, 2])
def test_multi_probe_newest_row_dominant(oracle, capsys, kv):
    """k = 256 q of each group's first query head: token t's first query head of a group scores its own new row far above the
    history and the earlier tokens' rows (newest_inputs picks such inputs), so its answer is its own new v row -- written by this
    launch, read back from fp32 scratch in the causal tail.  q roped at past_len instead of past_len + t breaks it."""
    st = attn_probe_stack(_shape(1024, 2816, 8, kv), 1, 1024, seed=40 + kv, gamma=256.0)
    st.make_plan(with_head=False, max_tokens=4)
    caches0 = probe_caches(st, 1200 + kv)
    worst = 0.0
    for i, past in enumerate([1020, 0, 1, 37, 255]):
        n = 4 - i % 4
        x = newest_inputs(oracle, st, n, past, 1210 + 10 * kv + i)
        spec = dict(multi_probe_specs(st, n, past))["newest"]
        worst = max(worst, _check(oracle, st, past, spec, 1220 + i, caches0, x, f"newest kv {kv} ctx {past} n {n}"))
    _report(capsys, f"newest kv {kv}", worst)
    st.dplan.close(); st.close()


def test_multi_probe_sequence_isolation(oracle, capsys):
    """Sequence 2 of a four-sequence cache, every other sequence all NaN: the history is streamed from sequence 2 only and the
    new rows go there."""
    st = attn_probe_stack(_shape(1024, 2816, 8, 2), 2, 512, seed=50, batch=4)
    st.make_plan(with_head=False, max_tokens=4)
    caches0 = probe_caches(st, 1300)
    worst = 0.0
    for i, (past, n) in enumerate([(37, 4), (255, 3), (0, 2), (16, 4)]):
        name, spec = multi_probe_specs(st, n, past)[i % 2]
        worst = max(worst, _check(oracle, st, past, spec, 1310 + i, caches0, _x(n, 1024, 1320 + i), f"seq 2 ctx {past} n {n} {name}",
                                  seq=2, nan_others=True))
    _report(capsys, "sequence isolation", worst)
    st.dplan.close(); st.close()


@pytest.mark.parametrize("model,n", [("7b", 4), ("13b", 4), ("33b", 3), ("65b", 2), ("70b", 1)])
def test_multi_probe_full_shapes(oracle, capsys, model, n):
    """One layer of each model at its full width and its largest token count (max_tokens_for: the tightest shared-memory
    layouts), at context 1920, where speculative decoding runs."""
    from exllama_b200.shapes import GQA_SHAPES, SHAPES
    s = GQA_SHAPES[model] if model == "70b" else SHAPES[model]
    st = attn_probe_stack(_shape(s.hidden, s.inter, s.heads, s.kv_heads), 1, 2048, seed=60)
    st.make_plan(with_head=False, max_tokens=n)
    caches0 = probe_caches(st, 1400)
    spec = dict(multi_probe_specs(st, n, 1920))["dense"]
    worst = _check(oracle, st, 1920, spec, 1410, caches0, _x(n, s.hidden, 1420), f"{model} n {n}")
    _report(capsys, f"{model} n {n}", worst)
    st.dplan.close(); st.close()


def test_multi_probe_liveness(oracle, monkeypatch):
    """A plan built with EXL_DS_DEBUG=2 (read at plan creation) skips the history's attention math: the probe misses by >= 100x."""
    st = attn_probe_stack(_shape(1024, 2816, 8, 2), 1, 512, seed=70)
    monkeypatch.setenv("EXL_DS_DEBUG", "2")
    st.make_plan(with_head=False, max_tokens=4)
    monkeypatch.delenv("EXL_DS_DEBUG")
    spec = dict(multi_probe_specs(st, 4, 300))["dense"]
    got, want, bound = _probe(oracle, st, 300, spec, 1500, probe_caches(st, 1500), _x(4, 1024, 1501))
    miss = np.nanmax(np.abs(got.astype(np.float64) - want) / bound)
    assert miss >= 100, miss
    st.dplan.close(); st.close()


# ------------------------------------------------------------------------------------------------------------------ phase probes
def _phase(stacks, *, o_off=(), mlp_off=(), seed=0, max_tokens=4, **kw):
    """A phase-probe stack (make_stack, phase_probe_edit) with a multi-token plan and its head."""
    st = stacks(seed=seed, **kw)
    phase_probe_edit(st, o_off, mlp_off, seed)
    st.make_plan(max_tokens=max_tokens)
    return st


def _run(st, xs, past):
    """One multi-token launch of xs [n, hidden] at past: (x_out [n, hidden], new rows rows[l][t] = (k, v) [kv_heads, hd]); every
    token's logits checked against the kernel's own x_out (check_head)."""
    import torch
    n = xs.shape[0]
    lg = st.decode_step_fused_multi(torch.from_numpy(xs).cuda().view(n, 1, -1), past)
    torch.cuda.synchronize()
    xo = st._plan_xout[:n].cpu().numpy()
    lg = lg.cpu().numpy()
    for t in range(n):
        check_head(st, lg[t], xo[t], f"ctx {past} token {t}/{n}")
    rows = [[(kc[0, :, past + t].cpu().numpy(), vc[0, :, past + t].cpu().numpy()) for t in range(n)]
            for kc, vc in zip(st.key_cache, st.value_cache)]
    return xo, rows


def _qkv_sweep(oracle, st, l, pasts, seed, what, x_of=None):
    """Each launch's tokens' new k / v rows of layer l against qkv_expectation at past + t; layer l's input is x_in (l = 0) or
    x_out (the hand-off stacks, whose layer 1 adds nothing)."""
    worst = 0.0
    for i, (past, n) in enumerate(pasts):
        xs = _x(n, st.shape.hidden, seed + i)
        xo, rows = _run(st, xs, past)
        xin = xs if l == 0 else xo
        for t in range(n):
            worst = max(worst, assert_within_any(rows[l][t], qkv_expectation(oracle, st, l, xin[t], past + t),
                                                 f"{what} ctx {past} token {t}/{n}"))
    return worst


@pytest.mark.parametrize("gs", [32, 64, 128, 256, None])
def test_multi_qkv_probe_group_sizes(oracle, stacks, capsys, gs):
    st = _phase(stacks, gs=gs, layers=1, max_seq=256, seed=71)
    worst = _qkv_sweep(oracle, st, 0, [(0, 4), (37, 3), (252, 4), (1, 2), (16, 1)], 1600, f"qkv g{gs}")
    _report(capsys, f"qkv g{gs}", worst)


@pytest.mark.parametrize("kv", [8, 4, 2, 1])
def test_multi_qkv_probe_gqa(oracle, stacks, capsys, kv):
    st = _phase(stacks, kv_heads=kv, layers=1, seed=72 + kv, max_tokens=MAX_TOKENS[kv])
    pasts = [(1, 4), (200, 3), (17, 2)] if MAX_TOKENS[kv] == 4 else [(1, 2), (200, 1), (17, 2)]
    worst = _qkv_sweep(oracle, st, 0, pasts, 1700 + kv, f"qkv kv {kv}")
    _report(capsys, f"qkv kv {kv}", worst)


@pytest.mark.parametrize("kv", [8, 2])
def test_multi_mlp_probe(oracle, stacks, capsys, kv):
    """o off, inter 512 (the silu term of the bound grows as sqrt(inter)): each token's x_out - x_in against mlp_expectation."""
    st = _phase(stacks, kv_heads=kv, inter=512, layers=1, o_off=(0,), seed=80 + kv)
    worst = 0.0
    for i, (past, n) in enumerate([(0, 4), (37, 3), (200, 2)]):
        xs = _x(n, 1024, 1800 + 10 * kv + i)
        xo, _ = _run(st, xs, past)
        for t in range(n):
            worst = max(worst, assert_within_any(xo[t], mlp_expectation(oracle, st, 0, xs[t]), f"mlp kv {kv} ctx {past} token {t}"))
    _report(capsys, f"mlp kv {kv}", worst)


@pytest.mark.parametrize("kv", [8, 2, 1])
def test_multi_handoff_probe(oracle, stacks, capsys, kv):
    """Layer 0 a full random layer over random caches, layer 1 with o and MLP off: each token's layer-1 k / v rows against the QKV
    bound on rms_norm(x_out, ln1[1]) -- the residual carry, ln1 preload and accumulator clean-up between layers, per token row."""
    st = _phase(stacks, kv_heads=kv, layers=2, o_off=(1,), mlp_off=(1,), seed=90 + kv, max_tokens=MAX_TOKENS[kv])
    pasts = [(0, 4), (16, 3), (200, 4)] if MAX_TOKENS[kv] == 4 else [(0, 2), (16, 1), (200, 2)]
    worst = _qkv_sweep(oracle, st, 1, pasts, 1900 + kv, f"hand-off kv {kv}")
    _report(capsys, f"hand-off kv {kv}", worst)
