"""The persistent decode step's GEMV phases and lm_head checked on their own outputs: phase-probe stacks (tests/helpers.py, "Phase
probes") whose new k / v rows, x_out - x_in or logits are one phase's output, each bounded element by element on the kernel's
own upstream output.

The whole-stack tests hold the final hidden state, the logits and the new k / v rows to 1e-2 of the rms, about ten times the
step's own GEMV error, and see o_proj and the MLP only through a residual they add a few percent to.  Here:
  QKV       layer 0's new k and v rows against step_gemv on rms_norm(x_in, ln1) (a 0.4 % gain error in the x segment scale, or a
            wrong scale row, breaks it);
  o_proj    MLP off, o random: x_out - x_in against W_o . attn, with attn the step's own new v row at context 0, or the plateau
            mean of planted caches (probe_expectation's attention bound, carried through |W_o|) at longer contexts;
  MLP       o off: x_out - x_in against down(silu(gate) * up) of rms_norm(x_in, ln2);
  hand-off  two layers, the second with o and MLP off: its new k / v rows against the QKV bound on rms_norm(x_out, ln1[1]), which
            pins the residual carry, the ln1 preload and the accumulator clean-up between layers;
  HEAD      every probe also checks the logits against the kernel's own x_out (head_expectation), about 1e-4 of their rms.
Norm weights are log-uniform over [0.05, 4] with exact zeros, different per tensor, so a wrong or stale norm row is gross."""
import numpy as np
import pytest

from helpers import (assert_within_any, assert_within_bound, dense_positions, mlp_expectation, o_expectation_ctx0, oracle_mm,
                     oracle_qkv, phase_probe_edit, plant_probe, probe_caches, probe_expectation, qkv_expectation, snap_of)
from stack_harness import check_head, fused_step, lib_state, snapshot, stacks  # noqa: F401

pytestmark = pytest.mark.gpu

# (groupsize, act-order): every x staging and segment layout of the GEMV (gs 64 is gemv_t<UPSEG = 2>)
GS_KINDS = [(32, False), (64, False), (128, False), (256, False), (None, False), (128, True), (32, True)]


def _xs(bsz, hidden, seed):
    """Layer inputs of about 1e-2 rms: the block outputs dominate x_out."""
    return (1e-2 * np.random.default_rng(seed).standard_normal((bsz, hidden))).astype(np.float16)


def _probe(stacks, *, o_off=(), mlp_off=(), lora=None, seed=0, with_head=True, **kw):
    """A phase-probe stack with its plan: make_stack(**kw), phase_probe_edit, then an adapter (rank 16 on the projections `lora`)."""
    st = stacks(seed=seed, **kw)
    phase_probe_edit(st, o_off, mlp_off, seed)
    if lora:
        st.add_lora(16, targets=lora, seed=seed)
    st.make_plan(with_head=with_head)
    return st


def _nan_unused(st, bsz):
    for kc, vc in zip(st.key_cache, st.value_cache):
        kc[bsz:] = float("nan"); vc[bsz:] = float("nan")


def _run(st, xs, pasts):
    """One fused step of xs [bsz, hidden] at contexts pasts: (x_out [bsz, hidden], logits [bsz, vocab] or None, new rows
    rows[l][b] = (k [kv_heads, hd], v [kv_heads, hd]))."""
    import torch
    bsz = len(pasts)
    logits = fused_step(st, torch.from_numpy(xs).cuda().view(bsz, 1, -1), pasts)
    torch.cuda.synchronize()
    xo = st._plan_xout.view(-1, st.shape.hidden)[:bsz].cpu().numpy()
    rows = [[(kc[b, :, p].cpu().numpy(), vc[b, :, p].cpu().numpy()) for b, p in enumerate(pasts)]
            for kc, vc in zip(st.key_cache, st.value_cache)]
    lg = logits.view(bsz, -1).cpu().numpy() if st._plan_logits is not None else None
    if lg is not None:
        for b in range(bsz):
            check_head(st, lg[b], xo[b], f"seq {b}")
    return xo, lg, rows


def _check_qkv(oracle, st, l, x, past, row, what):
    return assert_within_any(row, qkv_expectation(oracle, st, l, x, past), what)


# ------------------------------------------------------------------------------------------------------------------------------ QKV
@pytest.mark.parametrize("gs,act", GS_KINDS)
def test_qkv_probe_group_sizes(oracle, stacks, gs, act):
    st = _probe(stacks, gs=gs, act=act, layers=1, max_seq=256, seed=11)
    for i, past in enumerate([0, 37, 255]):
        x = _xs(1, 1024, 100 + i)
        _, _, rows = _run(st, x, [past])
        _check_qkv(oracle, st, 0, x[0], past, rows[0][0], f"g{gs} act {act} ctx {past}")


@pytest.mark.parametrize("kv", [8, 4, 2, 1])
def test_qkv_probe_gqa(oracle, stacks, kv):
    st = _probe(stacks, kv_heads=kv, layers=1, seed=12 + kv)
    for i, past in enumerate([1, 200]):
        x = _xs(1, 1024, 110 + i)
        _, _, rows = _run(st, x, [past])
        _check_qkv(oracle, st, 0, x[0], past, rows[0][0], f"kv {kv} ctx {past}")


@pytest.mark.parametrize("gs,lora", [(128, None), (64, None), (128, ("q", "k", "v"))])
def test_qkv_probe_batch(oracle, stacks, gs, lora):
    """Batch 4 at ragged contexts, then 3 sequences on the 4-sequence plan with the 4th all NaN; each sequence its own x_in."""
    st = _probe(stacks, gs=gs, batch=4, kv_heads=2, layers=1, lora=lora, seed=13)
    for j, pasts in enumerate([[0, 200, 16, 37], [255, 1, 37]]):
        if len(pasts) < 4:
            _nan_unused(st, len(pasts))
        xs = _xs(len(pasts), 1024, 120 + j)
        _, _, rows = _run(st, xs, pasts)
        for b, past in enumerate(pasts):
            _check_qkv(oracle, st, 0, xs[b], past, rows[0][b], f"g{gs} lora {lora} batch {pasts} seq {b}")


def test_qkv_probe_lora_single(oracle, stacks):
    st = _probe(stacks, layers=1, lora=("q", "k", "v"), seed=14)
    for i, past in enumerate([0, 37]):
        x = _xs(1, 1024, 130 + i)
        _, _, rows = _run(st, x, [past])
        _check_qkv(oracle, st, 0, x[0], past, rows[0][0], f"lora ctx {past}")


# --------------------------------------------------------------------------------------------------------------------------- o_proj
@pytest.mark.parametrize("gs,act", GS_KINDS)
def test_o_probe_ctx0_group_sizes(oracle, stacks, gs, act):
    st = _probe(stacks, gs=gs, act=act, layers=1, mlp_off=(0,), seed=21)
    x = _xs(1, 1024, 200)
    xo, _, rows = _run(st, x, [0])
    assert_within_any(xo[0], [o_expectation_ctx0(oracle, st, 0, x[0], rows[0][0][1])], f"o g{gs} act {act}")


@pytest.mark.parametrize("kv,bsz,lora", [(4, 1, None), (2, 1, None), (1, 1, None), (8, 1, ("o",)), (2, 4, ("o",)), (8, 4, None)])
def test_o_probe_ctx0_gqa_batch_lora(oracle, stacks, kv, bsz, lora):
    st = _probe(stacks, kv_heads=kv, batch=bsz, layers=1, mlp_off=(0,), lora=lora, seed=22 + kv)
    xs = _xs(bsz, 1024, 210 + kv)
    xo, _, rows = _run(st, xs, [0] * bsz)
    for b in range(bsz):
        assert_within_any(xo[b], [o_expectation_ctx0(oracle, st, 0, xs[b], rows[0][b][1])], f"o kv {kv} lora {lora} seq {b}")


def _o_planted(oracle, st, pasts, seed, what):
    """One layer, MLP off, o random: every head planted with its dense plateau, x_out checked against probe_expectation with the
    attention bound carried through |W_o| (o_prop)."""
    import torch
    s = st.shape
    n_rep = s.heads // s.kv_heads
    bsz = len(pasts)
    caches = probe_caches(st, seed)
    xs = _xs(bsz, s.hidden, seed + 1)
    plants = [plant_probe(oracle, st, caches, xs[b], p, lambda l, h, p=p: dense_positions(p, h % n_rep, n_rep), seed + 2 + b, seq=b)
              for b, p in enumerate(pasts)]
    for kc, vc in caches:
        kc[bsz:] = np.nan; vc[bsz:] = np.nan
    for kc, vc, (k0, v0) in zip(st.key_cache, st.value_cache, caches):
        kc.copy_(torch.from_numpy(k0)); vc.copy_(torch.from_numpy(v0))
    xo, _, _ = _run(st, xs, pasts)
    for b, p in enumerate(pasts):
        want, bound = probe_expectation(oracle, st, snap_of(caches), xs[b], p, plants[b], "step", seq=b, o_prop=True)
        assert_within_bound(xo[b], bound, want, f"{what} seq {b} ctx {p}")


@pytest.mark.parametrize("kv,act", [(8, False), (2, False), (8, True)])
def test_o_probe_planted_contexts(oracle, stacks, kv, act):
    st = _probe(stacks, kv_heads=kv, act=act, layers=1, mlp_off=(0,), max_seq=512, seed=31 + kv)
    for i, past in enumerate([511, 1, 16, 37, 200]):
        _o_planted(oracle, st, [past], 300 + 10 * i, f"o planted kv {kv} act {act}")


def test_o_probe_planted_batch(oracle, stacks):
    st = _probe(stacks, kv_heads=2, batch=4, layers=1, mlp_off=(0,), max_seq=256, seed=35)
    _o_planted(oracle, st, [200, 1, 37, 16], 400, "o planted batch")
    _o_planted(oracle, st, [16, 255, 0], 420, "o planted batch of 3")


# ------------------------------------------------------------------------------------------------------------------------------ MLP
def _check_mlp(oracle, st, xs, pasts, what):
    xo, _, _ = _run(st, xs, pasts)
    for b in range(len(pasts)):
        assert_within_any(xo[b], mlp_expectation(oracle, st, 0, xs[b]), f"{what} seq {b}")


@pytest.mark.parametrize("gs,act", GS_KINDS)
def test_mlp_probe_group_sizes(oracle, stacks, gs, act):
    """inter 512: the silu term of the bound grows as sqrt(inter) against down's output, so a narrow MLP keeps it tight."""
    st = _probe(stacks, gs=gs, act=act, inter=512, layers=1, o_off=(0,), seed=41)
    for i, past in enumerate([0, 37]):
        _check_mlp(oracle, st, _xs(1, 1024, 500 + i), [past], f"mlp g{gs} act {act} ctx {past}")


@pytest.mark.parametrize("kv,bsz,lora", [(2, 4, None), (8, 1, ("gate", "up", "down")), (4, 4, ("gate", "up", "down"))])
def test_mlp_probe_batch_lora(oracle, stacks, kv, bsz, lora):
    st = _probe(stacks, kv_heads=kv, batch=bsz, inter=512, layers=1, o_off=(0,), lora=lora, seed=42 + kv)
    pasts = [0, 200, 16, 37][:bsz]
    _check_mlp(oracle, st, _xs(bsz, 1024, 510 + kv), pasts, f"mlp kv {kv} lora {lora}")


# ------------------------------------------------------------------------------------------------------------------------- hand-off
def _check_handoff(oracle, st, xs, pasts, what):
    xo, _, rows = _run(st, xs, pasts)
    for b, p in enumerate(pasts):
        _check_qkv(oracle, st, 1, xo[b], p, rows[1][b], f"{what} seq {b} ctx {p} layer 1")


@pytest.mark.parametrize("gs,act", GS_KINDS)
def test_handoff_probe_group_sizes(oracle, stacks, gs, act):
    """Layer 0 a full random layer over random caches, layer 1 with o and MLP off: x_out is layer 0's output exactly."""
    st = _probe(stacks, gs=gs, act=act, layers=2, o_off=(1,), mlp_off=(1,), seed=51)
    for i, past in enumerate([0, 16, 200]):
        _check_handoff(oracle, st, _xs(1, 1024, 600 + i), [past], f"hand-off g{gs} act {act}")


@pytest.mark.parametrize("kv,bsz", [(2, 1), (1, 1), (8, 4), (2, 3)])
def test_handoff_probe_gqa_batch(oracle, stacks, kv, bsz):
    st = _probe(stacks, kv_heads=kv, batch=bsz, layers=2, o_off=(1,), mlp_off=(1,), seed=52 + kv)
    pasts = [37, 0, 255, 16][:bsz]
    _check_handoff(oracle, st, _xs(bsz, 1024, 610 + kv), pasts, f"hand-off kv {kv} batch {bsz}")


# ------------------------------------------------------------------------------------------------------------------------ 7B widths
def test_probes_7b_widths(oracle, stacks):
    """hidden 4096, inter 11008, 32 heads: QKV and hand-off on one two-layer stack, then o_proj at context 0 and the MLP."""
    kw = dict(hidden=4096, inter=11008, heads=32, vocab=32000, max_seq=256)
    st = _probe(stacks, layers=2, o_off=(1,), mlp_off=(1,), seed=61, **kw)
    x = _xs(1, 4096, 700)
    _, _, rows = _run(st, x, [200])
    _check_qkv(oracle, st, 0, x[0], 200, rows[0][0], "7B qkv")
    _check_handoff(oracle, st, _xs(1, 4096, 701), [37], "7B hand-off")
    st.dplan.close(); st.dplan = None
    st = _probe(stacks, layers=1, mlp_off=(0,), seed=62, **kw)
    x = _xs(1, 4096, 702)
    xo, _, rows = _run(st, x, [0])
    assert_within_any(xo[0], [o_expectation_ctx0(oracle, st, 0, x[0], rows[0][0][1])], "7B o")
    st.dplan.close(); st.dplan = None
    st = _probe(stacks, layers=1, o_off=(0,), seed=63, **kw)
    _check_mlp(oracle, st, _xs(1, 4096, 703), [37], "7B mlp")


# ---------------------------------------------------------------------------------------------------------- phase shares, measured
def test_phase_shares_of_standard_stack(oracle, stacks, capsys):
    """rms(o_proj output) / rms(residual) and rms(MLP output) / rms(residual) of layer 0 of the standard synthetic stack (the one
    the whole-stack tests use: inputs of 0.5 rms, N(0, 0.25) caches), through the oracle: how much of x_out each block is."""
    st = stacks(layers=1, seed=3)
    snap = snapshot(st)
    L = st.layers[0]
    out = []
    for past in (0, 37, 200):
        x = (np.random.default_rng(past + 128).standard_normal((1, 1024)) * 0.5).astype(np.float16)
        _, q, k, v = oracle_qkv(oracle, st, 0, x, past)
        kc = snap[0][0][0].cpu().numpy().copy(); vc = snap[0][1][0].cpu().numpy().copy()
        kc[:, past] = k; vc[:, past] = v
        attn = oracle.decode_attn_f64(q, kc, vc, 8, 8, 128, past + 1, st.max_seq).astype(np.float16).reshape(1, -1)
        o = oracle_mm(oracle, attn, L.o)
        x1 = (x.astype(np.float64) + o).astype(np.float16)
        xn, _ = oracle.rms_norm(x1, L.ln2.cpu().numpy(), st.shape.eps)
        act = oracle.silu_mul(oracle_mm(oracle, xn, L.gate).astype(np.float16), oracle_mm(oracle, xn, L.up).astype(np.float16))
        m = oracle_mm(oracle, act, L.down)
        rms = lambda a: float(np.sqrt(np.mean(np.asarray(a, np.float64) ** 2)))
        out.append((past, rms(o) / rms(x), rms(m) / rms(x1)))
    with capsys.disabled():
        print("\nphase shares of x_out (ctx, o / residual, MLP / residual):", [(p, round(a, 4), round(b, 4)) for p, a, b in out])
    assert all(a < 1 and b < 1 for _, a, b in out)
