"""Decode attention checked on its own output: planted-key caches through an attention probe stack (tests/helpers.py, "Attention
probe"), whose final hidden state is the residual plus each layer's attention output.

The whole-stack tests (test_gpu_decode_step.py, test_gpu_gqa.py, ...) see attention only through logits, where a nearly flat
softmax over N(0, 0.25) caches makes it about 1 % of the residual: a dropped chunk, a dropped new token or a lost CTA slot stays
inside their tolerance.  Here every planted head's answer is the mean of V over its plateau (random +-1 rows), so losing one chunk
moves it by about 1 / |P|, and every other head is held to a bound derived from q's error (probe_expectation).  Rows past the
context are NaN and row `past` holds a poison key (V = 100 x a signature) that the step must overwrite before attention reads it.

Covered: the persistent step (multi-head and GQA paths, the CTA-slot combine, act-order's attn_vec route, batches with unused NaN
sequences, LoRA on q / v, 7B and 70B head counts) and the per-op path q4_attn -> decode_attn -> q4_attn_2 at 1, 4, 5, 6, 7 and 8
splits with several sub-blocks per split."""
import numpy as np
import pytest

from helpers import (assert_within_bound, attn_probe_stack, dense_positions, plant_probe, probe_caches, probe_expectation,
                     single_positions, snap_of)

pytestmark = pytest.mark.gpu


def _shape(hidden, inter, heads, kv_heads=None):
    from exllama_b200.stack import LlamaShape
    return LlamaShape("attn-probe", hidden, inter, 1, heads, vocab=32000, kv_heads=kv_heads)


def _x(hidden, seed):
    return (1e-2 * np.random.default_rng(seed).standard_normal(hidden)).astype(np.float16)


def _load(st, caches):
    import torch
    for kc, vc, (k0, v0) in zip(st.key_cache, st.value_cache, caches):
        kc.copy_(torch.from_numpy(k0)); vc.copy_(torch.from_numpy(v0))
    torch.cuda.synchronize()


def _specs(st, past, background=False):
    """Plateau layouts for one context: "dense", then two sweeps of lone planted keys (each planted head its own position; with 8
    heads the first sweep already puts a key at every position of single_positions).
    Query head r of a KV group takes the dense residues {r, 15 - r}.  background: the query heads of the odd KV heads of a
    one-layer plan keep the plain N(0, 0.25) cache and are held to the q-error bound.  (Under a second layer their loose bound
    would reach every head through the next layer's rms norm, so multi-layer plans plant every head.)"""
    n_rep = st.shape.heads // st.shape.kv_heads
    assert not background or len(st.layers) == 1
    single = single_positions(past)

    def bg(h):
        return background and (h // n_rep) % 2 == 1
    out = [("dense", lambda l, h: None if bg(h) else dense_positions(past, h % n_rep, n_rep))]
    for off in (0, 3):
        if single:
            out.append((f"single+{off}", lambda l, h, off=off: None if bg(h) else [single[(h + l + off) % len(single)]]))
    return out


def _probe(oracle, st, past, spec, seed, kind, run, caches0, x):
    """Plant a copy of caches0, run (run(caches, x, past) -> final hidden state), check against the oracle within
    probe_expectation's bound: (got, want, bound)."""
    caches = [[c.copy() for c in kv] for kv in caches0]
    plants = plant_probe(oracle, st, caches, x, past, spec, seed)
    got = run(caches, x, past)
    want, bound = probe_expectation(oracle, st, snap_of(caches), x, past, plants, kind)
    return got, want, bound


def _check(oracle, st, past, spec, seed, kind, run, caches0, x, what):
    got, want, bound = _probe(oracle, st, past, spec, seed, kind, run, caches0, x)
    return assert_within_bound(got, bound, want, what)


def run_fused(st):
    import torch

    def run(caches, x, past):
        _load(st, caches)
        st.decode_step_fused(torch.from_numpy(x).cuda().view(1, 1, -1), past)
        torch.cuda.synchronize()
        return st._plan_xout.cpu().numpy().reshape(-1)
    return run


def run_per_op(st):
    import torch

    def run(caches, x, past):
        _load(st, caches)
        h = torch.from_numpy(x.copy()).cuda().view(1, 1, -1)
        st.decode_step(h, past)
        torch.cuda.synchronize()
        return h.cpu().numpy().reshape(-1)
    return run


def _sweep(oracle, st, pasts, run, kind, seed, what, background=False, n_specs=None):
    """Every layout of _specs at every context of `pasts`, in order, on one stack / plan."""
    caches0 = probe_caches(st, seed)
    for i, past in enumerate(pasts):
        x = _x(st.shape.hidden, seed + i)
        for name, spec in _specs(st, past, background)[:n_specs]:
            _check(oracle, st, past, spec, seed + 7 * i, kind, run, caches0, x, f"{what} ctx {past} {name}")


# ---------------------------------------------------------------------------------------------------------- persistent step
def test_probe_step_mha_contexts(oracle):
    """8 heads, 2 layers (layer l must read layer l's cache), one plan: the longest context first (every partial slot written),
    then short ones, where CTAs of a head's range own no unit (att_needs_reset)."""
    st = attn_probe_stack(_shape(1024, 2816, 8), 2, 2048, seed=1)
    st.make_plan(with_head=False)
    _sweep(oracle, st, [2047, 0, 1, 16, 17, 255, 1000], run_fused(st), "step", 100, "mha", n_specs=2)
    st.dplan.close(); st.close()


@pytest.mark.parametrize("kv", [8, 2])
def test_probe_step_background_heads(oracle, kv):
    """One layer, the query heads of the odd KV heads on the plain cache: at short contexts the new token carries a large share of
    their softmax, so its score (q . k_new / sqrt(128)) and its v row are checked against the q-error bound -- in the multi-head
    path and in the GQA path (att_gqa's own new-token partial)."""
    st = attn_probe_stack(_shape(1024, 2816, 8, kv), 1, 1024, seed=14 + kv)
    st.make_plan(with_head=False)
    _sweep(oracle, st, [1, 16, 600], run_fused(st), "step", 150 + kv, f"background kv {kv}", background=True, n_specs=2)
    st.dplan.close(); st.close()


@pytest.mark.parametrize("kv", [4, 2, 1])
def test_probe_step_gqa(oracle, kv):
    """n_rep 2, 4, 8: every query head of a group has its own plateau over the shared KV rows."""
    st = attn_probe_stack(_shape(1024, 2816, 8, kv), 2, 1024, seed=2 + kv)
    st.make_plan(with_head=False)
    _sweep(oracle, st, [1023, 0, 17], run_fused(st), "step", 200 + kv, f"gqa kv {kv}", n_specs=2)
    st.dplan.close(); st.close()


@pytest.mark.parametrize("kv", [8, 2])
def test_probe_step_newest_row_dominant(oracle, kv):
    """k = 256 q (the q projection's tensors, scales x 256; under GQA the group's first query head): the new token's score is far
    above every cached one, so that head's answer is the new v row, which the step writes in the same launch.  The other query
    heads of a group see gamma q_r . q_0, of either sign and any size: they are held to the q-error bound, which is loose, so the
    GQA plan has one layer (a second layer's rms norm would carry that looseness to every head)."""
    st = attn_probe_stack(_shape(1024, 2816, 8, kv), 2 if kv == 8 else 1, 2048, seed=5, gamma=256.0)
    st.make_plan(with_head=False)
    n_rep = 8 // kv
    run = run_fused(st)
    caches0 = probe_caches(st, 300)
    for i, past in enumerate([2047, 0, 1, 255]):
        spec = lambda l, h: "new" if h % n_rep == 0 else None
        _check(oracle, st, past, spec, 310 + i, "step", run, caches0, _x(1024, 320 + i), f"newest kv {kv} ctx {past}")
    st.dplan.close(); st.close()


def test_probe_step_batch(oracle):
    """Batches of mixed contexts; a launch of 3 sequences on a 4-sequence plan, the 4th sequence all NaN."""
    import torch
    st = attn_probe_stack(_shape(1024, 2816, 8), 2, 2048, seed=6, batch=4)
    st.make_plan(with_head=False)
    for j, pasts in enumerate([[0, 255, 16, 2047], [1000, 17, 256]]):
        bsz = len(pasts)
        caches = probe_caches(st, 400 + j)
        xs = [_x(1024, 410 + 10 * j + b) for b in range(bsz)]
        plants = []
        for b, past in enumerate(pasts):
            name, spec = _specs(st, past)[(b + j) % 2]
            plants.append(plant_probe(oracle, st, caches, xs[b], past, spec, 450 + 10 * j + b, seq=b))
        for kc, vc in caches:
            kc[bsz:] = np.nan; vc[bsz:] = np.nan
        _load(st, caches)
        got = st.decode_step_fused_batch(torch.from_numpy(np.stack(xs)).cuda().view(bsz, 1, -1), pasts).cpu().numpy()
        for b, past in enumerate(pasts):
            want, bound = probe_expectation(oracle, st, snap_of(caches), xs[b], past, plants[b], "step", seq=b)
            assert_within_bound(got[b], bound, want, f"batch {pasts}: sequence {b} at ctx {past}")
    st.dplan.close(); st.close()


def test_probe_step_act_order(oracle):
    """Act-order plan: the combined attention goes through L2 (attn_vec) and o_proj gathers it with its own x_map."""
    st = attn_probe_stack(_shape(1024, 2816, 8), 2, 1024, act=True, seed=7)
    st.make_plan(with_head=False)
    _sweep(oracle, st, [1000, 17, 300], run_fused(st), "step", 500, "act-order")
    st.dplan.close(); st.close()


def test_probe_step_lora(oracle):
    """Rank-16 adapters on q and v (o_proj stays the identity); every head planted."""
    st = attn_probe_stack(_shape(1024, 2816, 8), 2, 1024, seed=8, lora_rank=16)
    st.make_plan(with_head=False)
    _sweep(oracle, st, [700, 33], run_fused(st), "step", 600, "lora")
    st.dplan.close(); st.close()


@pytest.mark.parametrize("model,pasts,max_seq", [("7b", [1920, 2047], 2048), ("70b", [4095], 4096)])
def test_probe_step_full_head_counts(oracle, model, pasts, max_seq):
    """7B (32 heads) and Llama-2 70B (64 query heads over 8 KV heads) at their full widths, 1 layer."""
    from exllama_b200.shapes import GQA_SHAPES, SHAPES
    s = {"7b": SHAPES["7b"], "70b": GQA_SHAPES["70b"]}[model]
    st = attn_probe_stack(_shape(s.hidden, s.inter, s.heads, s.kv_heads), 1, max_seq, seed=9)
    st.make_plan(with_head=False)
    _sweep(oracle, st, pasts, run_fused(st), "step", 700, model, n_specs=2)
    st.dplan.close(); st.close()


def test_probe_step_liveness(oracle, monkeypatch):
    """A plan built with EXL_DS_DEBUG=2 (read at plan creation) skips the attention math: the probe misses by >= 100x its bound."""
    st = attn_probe_stack(_shape(1024, 2816, 8), 1, 512, seed=10)
    monkeypatch.setenv("EXL_DS_DEBUG", "2")
    st.make_plan(with_head=False)
    monkeypatch.delenv("EXL_DS_DEBUG")
    past = 300
    name, spec = _specs(st, past)[0]
    got, want, bound = _probe(oracle, st, past, spec, 800, "step", run_fused(st), probe_caches(st, 800), _x(1024, 801))
    miss = np.nanmax(np.abs(got.astype(np.float64) - want) / bound)
    assert miss >= 100, miss
    st.dplan.close(); st.close()


# ---------------------------------------------------------------------------------------------------------------- per-op path
# decode_attn splits a context of seq = past + 1 rows over nsplit = min(8, ceil(seq / 256)) CTAs of a cluster (at least 4 from
# seq 256 on); a split walks ceil(chunk / 256) sub-blocks of 256 rows.
PER_OP_PASTS = [100, 700, 1100, 1400, 1600, 3000]                # 1, 4, 5, 6, 7, 8 splits (2 sub-blocks each at 3000)


@pytest.mark.parametrize("kv", [8, 2])
def test_probe_per_op(oracle, kv):
    """DecodeStack.decode_step (q4_attn -> decode_attn under programmatic dependent launch -> q4_attn_2 -> q4_mlp) on the probe."""
    st = attn_probe_stack(_shape(1024, 2816, 8, kv), 2, 4096, seed=11 + kv)
    _sweep(oracle, st, PER_OP_PASTS if kv == 8 else [1100, 3000], run_per_op(st), "gemv", 900 + kv, f"per-op kv {kv}", n_specs=2)
    st.close()


def test_probe_per_op_background_heads(oracle):
    """The per-op path, one layer, odd heads on the plain cache (see test_probe_step_background_heads)."""
    st = attn_probe_stack(_shape(1024, 2816, 8), 1, 1024, seed=15)
    _sweep(oracle, st, [1, 16, 17, 300], run_per_op(st), "gemv", 160, "per-op background", background=True)
    st.close()


def test_probe_per_op_newest_row_dominant(oracle):
    """decode_attn reads the newest row after griddepcontrol.wait and every other row before it: with k = 256 q the new token is
    the answer, and the poison key in row `past` before the launch shows a stale read."""
    st = attn_probe_stack(_shape(1024, 2816, 8), 1, 4096, seed=13, gamma=256.0)
    run = run_per_op(st)
    caches0 = probe_caches(st, 950)
    for i, past in enumerate([0, 255, 1300, 3000]):
        _check(oracle, st, past, lambda l, h: "new", 960 + i, "gemv", run, caches0, _x(1024, 970 + i), f"per-op newest ctx {past}")
    st.close()
