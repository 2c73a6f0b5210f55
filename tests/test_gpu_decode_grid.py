"""The persistent decode step at the grid sizes and ring depths its schedule is proven for, not only at the card's SM count.

decode_step_kernel cuts the GEMV, ATT and HEAD phases with range_lo(U, cta, grid) (decode_step_sched.h), so the grid decides which of
its code paths run: a CTA range that crosses q|k, k|v or gate|up (the producer's matrix switch inside one range), a range longer than
one tile's K stages, an ATT phase that the grid rather than the per-head cap limits, the partial-table reset, and compact or full x
staging for batches.  An H100 has 132 (SXM) or 114 (PCIe) SMs, both divisible by 6, so at the native grid the gate|up crossing never
happens.  EXL_DS_GRID (read at plan creation) runs every plan kind here at smaller grids, and EXL_DS_DEPTH the ring at depths below
the largest that fits.  Every case is checked with the checks the other decode-step files use: the whole token against the float64
oracle and the per-op path, short contexts after a long one, consecutive tokens with CUDA-graph replay, the phase and attention probes,
and the multi-token check.  tests/test_decode_grid_regimes.py proves every case's schedule on the CPU and shows that the table reaches
every regime.  Grids above the card's SM count are skipped.
"""
from collections import namedtuple

import numpy as np
import pytest

import test_gpu_decode_attn_probe as attn_probe
import test_gpu_decode_multi as multi_step
import test_gpu_decode_phase_probe as phase_probe
import test_gpu_lora as lora_tests
from helpers import assert_close_ref64, attn_probe_stack
from stack_harness import (check_fused_step, check_head, check_reset_after_long_context, check_sequence_and_graph,  # noqa: F401
                           fused_step, lib_state, per_op, restore, snapshot, stacks)

pytestmark = pytest.mark.gpu

NATIVE_SMS = 132     # what grid None (the card's SM count) stands for in the CPU regime proof: an H100 SXM

# check: what the GPU test runs; stack: make_stack's keyword arguments; grid: EXL_DS_GRID (None: the card's SM count); launches:
# per launch the contexts of its sequences, or (k, past) of a multi-token launch; max_tokens: a multi-token plan; lora: (rank,
# projections) of an adapter on every layer.
Case = namedtuple("Case", "id check stack grid launches max_tokens lora", defaults=(None, None))

STD = dict(hidden=1024, inter=2816, heads=8)                 # the standard synthetic stack, 2 layers
NARROW = dict(hidden=1024, inter=2816, heads=4)              # 4 heads of 128 under a 1024-wide residual: DOWN ranges pass one tile
ONE = [(255,), (0,), (1,), (37,)]                             # the longest context first: every partial slot is written
BATCH = [(255, 0, 37, 1), (17, 200, 3)]                       # the second launch: 3 sequences of 4, the 4th all NaN
MULTI = [(4, 200), (4, 0), (4, 37), (2, 17)]
RESET = [(200,), (37,), (17,), (100,), (49,), (3,), (96,), (200,)]
FULL = [(1920,)]


def _cases():
    c = []
    for gs in (128, 32):
        for g in (8, 9, 13, 32, 57, 114, 131, None):
            c.append(Case(f"mha-g{gs}-grid{g or 'native'}", "whole", dict(STD, gs=gs), g, ONE))
    for g in (4, 5, 7):
        c.append(Case(f"narrow-grid{g or 'native'}", "whole", dict(NARROW), g, ONE))
    for kv in (2, 1):
        for g in (8, 9, 32, 57, 114):
            c.append(Case(f"gqa{kv}-grid{g or 'native'}", "whole", dict(STD, kv_heads=kv), g, ONE))
    for g in (8, 13, 57, 114):
        c.append(Case(f"act-grid{g or 'native'}", "whole", dict(STD, act=True), g, ONE))
    for g in (13, 32):
        c.append(Case(f"reset-grid{g or 'native'}", "reset", dict(STD), g, RESET))
    for kv, g in ((2, 8), (2, 13), (8, 33), (8, 57), (8, 114)):
        c.append(Case(f"batch-kv{kv}-grid{g or 'native'}", "whole", dict(STD, kv_heads=kv, batch=4), g, BATCH))
    for kv in (8, 2):
        for g in (8, 13, 57, 114):
            c.append(Case(f"multi-kv{kv}-grid{g or 'native'}", "multi", dict(STD, kv_heads=kv), g, MULTI, max_tokens=4))
    for g in (9, 57, 114):                                    # test_gpu_lora.py's r 16 single-sequence and r 128 batch cases
        c.append(Case(f"lora-grid{g}", "lora", dict(STD), g, [(1,)], lora=(16, "all")))
        c.append(Case(f"lora-batch-grid{g}", "lora", dict(STD, kv_heads=2, batch=4), g, [(0, 200, 16, 37)], lora=(128, "all")))
    for kv, g in ((8, 8), (8, 13), (2, 9)):
        c.append(Case(f"qkv-probe-kv{kv}-grid{g or 'native'}", "qkv_probe", dict(STD, kv_heads=kv, layers=1), g, [(0,), (37,), (255,)]))
        c.append(Case(f"mlp-probe-kv{kv}-grid{g or 'native'}", "mlp_probe", dict(STD, kv_heads=kv, inter=512, layers=1), g, [(0,), (37,)]))
        c.append(Case(f"handoff-probe-kv{kv}-grid{g or 'native'}", "handoff_probe", dict(STD, kv_heads=kv), g, [(0,), (16,), (200,)]))
        c.append(Case(f"attn-probe-kv{kv}-grid{g or 'native'}", "attn_probe", dict(STD, kv_heads=kv, vocab=0), g, [(255,), (17,)]))
    c.append(Case("13b-act-grid114", "full", dict(hidden=5120, inter=13824, heads=40, vocab=32000, act=True, max_seq=2048), 114, FULL))
    c.append(Case("7b-grid131", "full", dict(hidden=4096, inter=11008, heads=32, vocab=32000, max_seq=2048), 131, FULL))
    c.append(Case("70b-grid114", "full", dict(hidden=8192, inter=28672, heads=64, kv_heads=8, vocab=32000, max_seq=2048), 114, FULL))
    for g in (None, 13):
        c.append(Case(f"depth-grid{g or 'native'}", "depth", dict(STD), g, [(40 + t,) for t in range(5)]))
    return c


CASES = _cases()


def dims(case):
    """(hidden, attention width, intermediate width, heads, KV heads, vocab, act-order, max_batch, max_seq) of a case's plan."""
    s = {**dict(hidden=1024, inter=2816, heads=8, kv_heads=None, vocab=2048, act=False, batch=1, max_seq=256), **case.stack}
    kv = s["kv_heads"] or s["heads"]
    return (s["hidden"], s["heads"] * 128, s["inter"], s["heads"], kv, s["vocab"], s["act"], s["batch"], s["max_seq"])


def _of(check):
    return [pytest.param(c, id=c.id) for c in CASES if c.check == check]


def _grid(grid):
    """The grid a plan gets with EXL_DS_GRID = grid (None: the card's SM count); skips a grid above the SM count."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if grid is not None and grid > sms:
        pytest.skip(f"grid {grid} > {sms} SMs")
    return grid or sms


def _planned(monkeypatch, grid, make):
    """make() creates the plan with EXL_DS_GRID = grid set (plan creation reads it); the plan must report that grid."""
    want = _grid(grid)
    if grid is not None:
        monkeypatch.setenv("EXL_DS_GRID", str(grid))
    try:
        st = make()
    finally:
        monkeypatch.delenv("EXL_DS_GRID", raising=False)
    assert st.dplan.info()["grid"] == want, st.dplan.info()
    return st


def _stack(stacks, case, seed, **plan):
    """The case's stack with its plan (make_plan(**plan))."""
    st = stacks(seed=seed, **case.stack)
    st.make_plan(**plan)
    return st


def _x(bsz, hidden, seed, scale=0.5):
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    return (torch.randn((bsz, 1, hidden), device="cuda", generator=g) * scale).half()


def _check_nan_fourth(st, xs, pasts, what):
    """A launch of len(pasts) sequences on a larger plan whose other sequences' caches are all NaN: every sequence against the per-op
    path, the logits against the kernel's own hidden state, and the NaN sequences untouched."""
    import torch
    n = len(pasts)
    snap = snapshot(st)
    ref, _ = per_op(st, snap, xs, pasts)
    for kc, vc in zip(st.key_cache, st.value_cache):
        kc[n:] = float("nan"); vc[n:] = float("nan")
    got = fused_step(st, xs, pasts).cpu().numpy()
    xo = st._plan_xout.view(-1, st.shape.hidden)[:n].cpu().numpy()
    for kc, vc in zip(st.key_cache, st.value_cache):
        assert torch.isnan(kc[n:]).all() and torch.isnan(vc[n:]).all(), what
    restore(st, snap)
    assert np.isfinite(got).all(), what
    for b in range(n):
        check_head(st, got[b], xo[b], f"{what} seq {b}")
        assert_close_ref64(got[b], ref[b].cpu().numpy().reshape(-1).astype(np.float64), rel=1.5e-2, rms=1.5e-2, what=f"{what} seq {b} vs per-op")


# ------------------------------------------------------------------------------------------------------------------- whole token
@pytest.mark.parametrize("case", _of("whole"))
def test_whole_token(oracle, stacks, monkeypatch, case):
    """Each launch against the float64 oracle and the per-op path (check_fused_step); a launch of 3 on a 4-sequence plan with the
    4th sequence NaN against the per-op path."""
    seed = 3 + sum(map(ord, case.id)) % 97
    st = _planned(monkeypatch, case.grid, lambda: _stack(stacks, case, seed))
    for j, pasts in enumerate(case.launches):
        xs = _x(len(pasts), st.shape.hidden, seed + j)
        if len(pasts) < st.batch:
            _check_nan_fourth(st, xs, list(pasts), f"{case.id} ctx {pasts}")
        else:
            check_fused_step(oracle, st, xs, list(pasts), f"{case.id} ctx {pasts}")


@pytest.mark.parametrize("case", _of("lora"))
def test_lora(oracle, stacks, monkeypatch, case):
    """test_gpu_lora.py's cases (their stacks, adapters and inputs) at other grids: the LA step's (matrix, K stage) units and the
    CTA that adds a tile's B term both follow the grid.  Against the oracle and the per-op path, and the adapter must matter."""
    rank, targets = case.lora
    kv, bsz = case.stack.get("kv_heads") or 8, len(case.launches[0])
    past = case.launches[0]
    # the seeds of test_gpu_lora.test_fused_step_vs_oracle_and_per_op (one sequence) and test_batched_fused_step (a batch)
    seed, lora_seed, x_seed = (3 + kv + 128 + rank, rank + past[0], past[0] + rank) if bsz == 1 else (50 + bsz + kv, bsz, 7 * bsz)

    def make():
        st = stacks(seed=seed, **case.stack)
        lora_tests._add(st, rank, targets, seed=lora_seed)
        st.make_plan()
        return st
    st = _planned(monkeypatch, case.grid, make)
    lora_tests._check_step(oracle, st, lora_tests._xs(bsz, 1024, x_seed), list(past), case.id)


def test_batch_larger_than_the_grid_takes_is_rejected(stacks, monkeypatch):
    """4 sequences of 8 heads need 32 CTAs: at grid 31 the largest batch is 3."""
    from exllama_b200 import capi
    _grid(31)
    st = stacks(batch=4, layers=1, max_seq=64)
    monkeypatch.setenv("EXL_DS_GRID", "31")
    with pytest.raises(capi.ExlError, match=r"max_batch 4 does not fit.*31 CTAs.*the largest batch is 3$"):
        st.make_plan()


@pytest.mark.parametrize("kind", ["mha", "gqa", "multi"])
def test_grid_below_the_head_count_is_rejected(stacks, monkeypatch, kind):
    """A plan whose grid (EXL_DS_GRID) has fewer CTAs than heads is refused at creation: ATT keeps at most two head segments per CTA,
    and no schedule is proven for such a grid.  No plan is ever stepped here."""
    from exllama_b200 import capi
    st = stacks(layers=1, max_seq=64, kv_heads=None if kind == "mha" else 2)
    monkeypatch.setenv("EXL_DS_GRID", "7")
    with pytest.raises(capi.ExlError, match=r"error 1: .*more heads \(8\) than the grid's 7 CTAs"):
        st.make_plan(max_tokens=4 if kind == "multi" else None)


# ------------------------------------------------------------------------------------------------------ reset after a long context
@pytest.mark.parametrize("case", _of("reset"))
def test_short_contexts_after_a_long_one(oracle, stacks, monkeypatch, case):
    from helpers import att_needs_reset
    grid = _grid(case.grid)
    st = _planned(monkeypatch, case.grid, lambda: _stack(stacks, case, 7))
    contexts = [list(p) for p in case.launches]
    seen = check_reset_after_long_context(st, [_x(1, 1024, 21 + j) for j in range(len(contexts))], contexts)
    assert seen == {att_needs_reset(8, 8, p[0], grid) for p in contexts}


# ---------------------------------------------------------------------------------------------------------------- multi-token
@pytest.mark.parametrize("case", _of("multi"))
def test_multi_token_every_position(oracle, stacks, monkeypatch, case):
    seed = 5 + sum(map(ord, case.id)) % 97
    st = _planned(monkeypatch, case.grid, lambda: _stack(stacks, case, seed, max_tokens=case.max_tokens))
    for j, (k, past) in enumerate(case.launches):
        multi_step.check_multi_step(oracle, st, multi_step.rand_x(k, seed + j), past, 0, f"{case.id} k {k}")


# --------------------------------------------------------------------------------------------------------------------- probes
def _phase_probe(stacks, monkeypatch, case, **kw):
    return _planned(monkeypatch, case.grid, lambda: phase_probe._probe(stacks, seed=11, **case.stack, **kw))


@pytest.mark.parametrize("case", _of("qkv_probe"))
def test_qkv_probe(oracle, stacks, monkeypatch, case):
    st = _phase_probe(stacks, monkeypatch, case)
    for i, (past,) in enumerate(case.launches):
        x = phase_probe._xs(1, 1024, 100 + i)
        _, _, rows = phase_probe._run(st, x, [past])
        phase_probe._check_qkv(oracle, st, 0, x[0], past, rows[0][0], f"{case.id} ctx {past}")


@pytest.mark.parametrize("case", _of("mlp_probe"))
def test_mlp_probe(oracle, stacks, monkeypatch, case):
    st = _phase_probe(stacks, monkeypatch, case, o_off=(0,))
    for i, (past,) in enumerate(case.launches):
        phase_probe._check_mlp(oracle, st, phase_probe._xs(1, 1024, 500 + i), [past], f"{case.id} ctx {past}")


@pytest.mark.parametrize("case", _of("handoff_probe"))
def test_handoff_probe(oracle, stacks, monkeypatch, case):
    st = _phase_probe(stacks, monkeypatch, case, o_off=(1,), mlp_off=(1,))
    for i, (past,) in enumerate(case.launches):
        phase_probe._check_handoff(oracle, st, phase_probe._xs(1, 1024, 600 + i), [past], f"{case.id}")


@pytest.mark.parametrize("case", _of("attn_probe"))
def test_attention_probe(oracle, lib_state, monkeypatch, case):
    """Planted plateaus (dense, then lone keys) at every context of the case, on one two-layer probe plan."""
    s = case.stack
    made = []

    def make():
        made.append(attn_probe_stack(attn_probe._shape(s["hidden"], s["inter"], s["heads"], s["kv_heads"]), 2, 256, seed=1))
        made[-1].make_plan(with_head=False)
        return made[-1]
    try:
        st = _planned(monkeypatch, case.grid, make)
        attn_probe._sweep(oracle, st, [p for (p,) in case.launches], attn_probe.run_fused(st), "step", 100, case.id, n_specs=2)
    finally:
        for st in made:
            if st.dplan is not None:
                st.dplan.close()
            st.close()


# ------------------------------------------------------------------------------------------------------------------ full sizes
@pytest.mark.parametrize("case", _of("full"))
def test_full_size_vs_per_op(oracle, stacks, monkeypatch, case):
    """Two layers of a real model's widths at a grid of a smaller part (114: an H100 PCIe) or an odd one, ctx 1920, against the per-op
    path: 13B's QKV ranges at 114 CTAs are longer than one tile's 40 K stages."""
    st = _planned(monkeypatch, case.grid, lambda: _stack(stacks, case, 13))
    for pasts in case.launches:
        check_fused_step(None, st, _x(1, st.shape.hidden, 23), list(pasts), case.id)


# ----------------------------------------------------------------------------------------------------------------- ring depth
@pytest.mark.parametrize("case", _of("depth"))
def test_ring_depths(oracle, stacks, monkeypatch, case):
    """EXL_DS_DEPTH 2, 3 and one below the largest that fits: the plan has 4 x depth ring stages, and five consecutive tokens plus a
    CUDA-graph replay match the per-op path (at depth 2 and 3 every stage of the ring is in flight, kmid == depth)."""
    st = _planned(monkeypatch, case.grid, lambda: _stack(stacks, case, 5))
    native = st.dplan.info()["ring_stages"] // 4
    st.dplan.close(); st.dplan = None
    assert native >= 4
    starts = [case.launches[0][0]]

    def replan():
        st.make_plan()
        return st
    for depth in (2, 3, native - 1):
        monkeypatch.setenv("EXL_DS_DEPTH", str(depth))
        try:
            _planned(monkeypatch, case.grid, replan)
        finally:
            monkeypatch.delenv("EXL_DS_DEPTH", raising=False)
        assert st.dplan.info()["ring_stages"] == 4 * depth, (depth, st.dplan.info())
        check_sequence_and_graph(st, [_x(1, 1024, 90 + 7 * depth + t) for t in range(len(case.launches))], starts)
        st.dplan.close(); st.dplan = None
