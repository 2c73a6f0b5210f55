"""The decode GEMVs' 16-bit x quantisation at its edges, on the GPU: one-group (GPTQ groupsize -1) and 256 / 512 groups, outlier
("massive") activations, saturated weights and the int32 headroom of q4_gemv's segment value.

(a) q4_matmul (skinny kernel, and the auto route's repeated skinny passes at 9 <= M <= 48) against helpers.quant_error_bound, a
    float64 bound proved on the CPU by tests/test_quant_bound.py.
(b) Exact answers at the largest integer sums: constant x and saturated weights put every x_q at 32767 and every q - zp at -16
    (or +14), on one-group matrices as long and wide as Llama-2 70B's and beyond.
(c) The fused per-op blocks (q4_attn, q4_attn_2, q4_mlp) with one group and gs 256 on outlier x.
(d) The persistent decode step with one group per matrix (DecodeStack(groupsize=None)) against the oracle and the per-op path.
(e) Our error against float64 is no larger than the reference kernel's on outlier and one-group inputs (tests/golden/ref_gpu_quant.npz,
    oracle/gen_golden_ref_gpu_quant.py)."""
import os

import numpy as np
import pytest

from helpers import (GOLDEN, adapter_of, assert_close_ref64, assert_within_bound, gen_x, oracle_decode_step,
                     outlier_channels, q4_column_sample, quant_error_bound, sample_cols, synth_q4_ckpt, synth_q4_saturated, to_cuda,
                     ulp_diff_f16)
from stack_harness import fused_step, lib_state, per_op, restore, sincos, snapshot, stacks  # noqa: F401

# No q4 handle or borrowed buffer outlives a test (the 70B-width matrices here are large).
pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("lib_state")]


def _q4(capi, qw, qz, sc, g_idx):
    import torch
    tq, tz, ts = to_cuda(qw.copy(), qz, sc)
    return capi.Q4(tq, tz, ts, None if g_idx is None else torch.from_numpy(g_idx))


def _bound_on_cols(oracle, x, qw, qz, sc, g_idx, cols, kind="gemv"):
    """(B, ref64) of the output columns `cols`, in make_q4's sequential layout with the act-order x gather."""
    sub = q4_column_sample(qw, qz, sc, cols)
    x_map = None
    if g_idx is not None:
        x_map = oracle.make_x_map(g_idx, qz.shape[0])
        sub = (oracle.make_sequential(sub[0], x_map),) + sub[1:]
    return quant_error_bound(oracle, x, *sub, x_map=x_map, kind=kind)


# ------------------------------------------------------------------------------------------------------- (a) q4_matmul vs the bound
A_CASES = [  # (M, K, N, gs, act, x kind, outlier variant, weights)
    (1, 1024, 128, None, False, "outlier1000", 0, "ckpt"),
    (1, 8192, 28672, None, False, "outlier1000", 3, "ckpt"),      # Llama-2 70B gate / up, one group
    (1, 11008, 4096, None, True, "outlier64", 3, "ckpt"),
    (2, 4224, 4096, 128, False, "outlier1000", 1, "ckpt"),        # 33 stages: odd stage count, ragged k-warp split
    (2, 4224, 256, None, False, "outlier64", 0, "sat-"),
    (8, 8192, 4096, 256, True, "outlier1000", 4, "ckpt"),
    (8, 8192, 1024, 512, False, "outlier64", 2, "ckpt"),
    (1, 11008, 4096, 256, False, "silu", 0, "ckpt"),
    (2, 1024, 4096, 32, True, "zeros", 0, "ckpt"),
    (3, 8192, 2048, None, False, "zeros", 0, "ckpt"),
    (1, 4224, 128, 32, False, "subnormal", 0, "ckpt"),
    (2, 8192, 28672, 128, False, "big", 0, "ckpt"),
    (1, 8192, 4096, 512, True, "outlier1000", 0, "ckpt"),
    (1, 8192, 28672, 256, False, "outlier1000", 1, "ckpt"),
    (4, 1024, 512, 512, False, "const", 0, "sat+"),
    (9, 8192, 4096, None, False, "outlier1000", 0, "ckpt"),       # auto route: repeated skinny passes
    (48, 4224, 1024, 128, True, "outlier1000", 1, "ckpt"),
    (9, 1024, 128, 512, False, "gauss", 0, "ckpt"),
    (48, 11008, 4096, 256, False, "silu", 0, "ckpt"),
    (16, 1024, 128, None, True, "outlier1000", 2, "ckpt"),
]


def _a_inputs(M, K, N, gs, act, xkind, variant, wkind, seed):
    cols = sample_cols(N, 24, seed)
    x = gen_x(xkind, M, K, seed=seed, channels=outlier_channels(K, gs, variant), gs=gs)
    if wkind == "ckpt":
        w = synth_q4_ckpt(K, N, gs, act, seed=seed, cols=cols, scale=1e-3 if xkind == "big" else 1.0)
    else:
        w = synth_q4_saturated(K, N, gs, sign=-1 if wkind == "sat-" else 1, act=act, seed=seed)
    return x, w, cols


@pytest.mark.parametrize("M,K,N,gs,act,xkind,variant,wkind", A_CASES)
def test_q4_matmul_within_quant_bound(oracle, M, K, N, gs, act, xkind, variant, wkind):
    import torch
    from exllama_b200 import capi
    seed = M * 7 + K + N % 97 + (gs or 3) + variant
    x, (qw, qz, sc, g_idx), cols = _a_inputs(M, K, N, gs, act, xkind, variant, wkind, seed)
    q4 = _q4(capi, qw, qz, sc, g_idx)
    out = capi.q4_matmul(to_cuda(x), q4, force_path=1 if M <= 8 else 0)
    torch.cuda.synchronize()
    assert capi.last_q4_path() == "skinny_mma"
    B, ref = _bound_on_cols(oracle, x, qw, qz, sc, g_idx, cols)
    assert_within_bound(out.cpu().numpy()[:, cols], B, ref, what=f"M{M} K{K} N{N} g{gs} act{act} {xkind}/{variant} {wkind}")


# -------------------------------------------------------------------------------------------------------- (b) integer headroom
def _exact_scales(K, N, seed, mult):
    """fp16 scales s_n whose exact output mult * K * s_n is a normal fp16 number between 1 and 30000."""
    rng = np.random.default_rng(seed)
    s = (10.0 ** rng.uniform(0, np.log10(30000), N) / (abs(mult) * K)).astype(np.float16)
    want = mult * K * s.astype(np.float64)
    assert (np.abs(want) >= 2.0 ** -14).all() and (np.abs(want) < 65504).all()
    return s[None, :], want


@pytest.mark.parametrize("M", [1, 2, 8])
@pytest.mark.parametrize("K,N,sign", [(8192, 28672, -1), (8192, 28672, 1), (16384, 28672, -1), (65536, 128, -1)])
def test_q4_matmul_headroom_exact(oracle, M, K, N, sign):
    """x = +-1 (one sign per row) against saturated one-group weights: x_q = +-32767 everywhere and the output is
    -+16 K s_n (nibble 0, zero nibble 15) or +-14 K s_n (nibble 15, zero nibble 0), up to its final fp16 rounding.
    K 8192 / 16384 at N 28672: 224 tiles leave no room for a cluster, so one CTA streams all of K; K 65536 at N 128: a cluster of
    8 CTAs of 64 stages each.  Every segment is one 128-k stage, so |val| = 16 * 32767 * 128 (before segments were cut at the
    stage, the M = 1 case summed 4096 k into one value, 65,535 short of INT32_MAX)."""
    import torch
    from exllama_b200 import capi
    mult = -16 if sign < 0 else 14
    sc, want1 = _exact_scales(K, N, K + N + M, mult)
    qw, qz, sc, _ = synth_q4_saturated(K, N, None, sign=sign, scales=sc)
    signs = np.where(np.arange(M) % 2 == 0, 1.0, -1.0)
    x = np.repeat(signs[:, None], K, axis=1).astype(np.float16)
    out = capi.q4_matmul(to_cuda(x), _q4(capi, qw, qz, sc, None), force_path=1)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    want = (signs[:, None] * want1[None, :])
    assert (want == want.astype(np.float16)).all() or mult == 14
    d = ulp_diff_f16(got, want.astype(np.float16))
    assert d.max() <= 1, f"M{M} K{K} N{N} x{mult}: {int((d > 1).sum())} outputs off by more than 1 ulp (max {int(d.max())}), " \
                         f"e.g. got {got.reshape(-1)[d.argmax()]} want {want.reshape(-1)[d.argmax()]}"


def test_q4_mlp_headroom_70b_widths(oracle):
    """q4_mlp at Llama-2 70B widths with one group (hidden 8192, inter 28672, M = 1): constant x normalises to exactly 1, and
    saturated gate / up make gate = -16 * 8192 * s_gate and up = -16 * 8192 * s_up exact fp16 numbers -- the fused SILU_MUL launch
    carries the largest integer sums.  down (g128, checkpoint-like) is checked on a column sample against the oracle composition within its
    quantisation bound, plus the residual's share of the fp16 rounding and 8 fp16 ulps of each silu(gate) * up (the GPU's hexp /
    hrcp against the correctly rounded restatement, test_gpu_ops.test_silu_mul)."""
    import torch
    from exllama_b200 import capi
    H, I = 8192, 28672
    rng = np.random.default_rng(70)
    sg = (rng.uniform(0.25, 6, I) / (16 * H)).astype(np.float16)[None, :]     # gate in [-6, -0.25]: silu(gate) far from 0
    g_want = -16.0 * H * sg.astype(np.float64)[0]
    su = (np.where(rng.random(I) < 0.01, 300.0, rng.uniform(0.1, 3, I)) / (16 * H)).astype(np.float16)[None, :]
    gate = synth_q4_saturated(H, I, None, sign=-1, scales=sg)
    up = synth_q4_saturated(H, I, None, sign=-1, scales=su)
    cols = sample_cols(H, 24, 5)
    down = synth_q4_ckpt(I, H, 128, seed=71, cols=cols)
    x = np.ones((1, H), np.float16)
    w = np.ones(H, np.float16)
    xn, _ = oracle.rms_norm(x, w, 1e-6)
    assert (xn == 1).all()
    g16 = g_want.astype(np.float16)[None, :]
    u16 = (-16.0 * H * su.astype(np.float64)).astype(np.float16)
    assert (g16.astype(np.float64) == g_want).all()
    act16 = oracle.silu_mul(g16, u16)
    tx = to_cuda(x.copy())
    capi.q4_mlp(tx, to_cuda(w), 1e-6, _q4(capi, *gate), _q4(capi, *up), _q4(capi, *down))
    torch.cuda.synchronize()
    B, ref = _bound_on_cols(oracle, act16, *down, cols)
    sub_w = np.abs(oracle.dequant_f64(*q4_column_sample(*down[:3], cols)))
    B = B + 2.0 ** -11 * np.abs(x[:, cols].astype(np.float64)) + (8 * np.spacing(np.abs(act16)).astype(np.float64)) @ sub_w
    assert_within_bound(tx.cpu().numpy()[:, cols], B, ref + x[:, cols].astype(np.float64), what="q4_mlp 70B one group, down")


# ----------------------------------------------------------------------------------------------- (c) fused per-op blocks
def _block_weights(hidden, inter, gs, seed, kv=None, act=False):
    """Checkpoint-like weights of one layer.  With act-order, q / k / v share one g_idx and gate / up another, as a checkpoint's
    projections of one input may; make_q4 still gives every matrix its own x_map, so q4_attn and q4_mlp then take their general
    paths (capi.cu) -- the fused launches (rope + cache, silu * mul epilogues) run in the cases without act-order."""
    kv = kv or hidden
    names = [("q", hidden, hidden), ("k", hidden, kv), ("v", hidden, kv), ("o", hidden, hidden),
             ("gate", hidden, inter), ("up", hidden, inter), ("down", inter, hidden)]
    shared = {"k": "q", "v": "q", "up": "gate"}
    t = {}
    for i, (n, K, N) in enumerate(names):
        g = t[shared[n]][3] if n in shared else None
        t[n] = synth_q4_ckpt(K, N, gs, act, seed=seed + i, g_idx=g)
    return t


def _rope_allowance(B, ref, sin, cos, heads, hd, past):
    """The bound of q / k after rope: rope mixes element i with i +- 64 by |cos| and |sin| (the bound of each enters with those
    weights).  The fp16 roundings: the oracle rounds ref where the kernel rounds its own result (2^-11 |ref|, once), and rope's
    product and fma round differently on the two sides (2 x 2^-11 of |cos r| + 2 |sin r'| each): at most 5 x 2^-11 of
    |cos r| + |sin r'| in all."""
    n = B.shape[-1]
    b = B.reshape(-1, heads, hd)
    r16 = np.abs(ref.astype(np.float16).astype(np.float64)).reshape(-1, heads, hd)
    c, s = np.abs(cos[past].astype(np.float64)), np.abs(sin[past].astype(np.float64))
    rot = lambda a: np.concatenate([a[..., hd // 2:], a[..., :hd // 2]], axis=-1)   # noqa: E731
    mixed = c * b + s * rot(b)
    fp16 = 5 * 2.0 ** -11 * (c * r16 + s * rot(r16))
    return (mixed + fp16).reshape(-1, n) + 2.0 ** -24


@pytest.mark.parametrize("gs,kvh,act", [(None, 8, False), (256, 8, False), (None, 1, False), (256, 1, False),
                                         (None, 1, True), (256, 8, True)])
def test_q4_attn_and_mlp_blocks_outliers(oracle, gs, kvh, act):
    """q4_attn with multi-head (8 KV heads) and grouped-query attention (8 query heads over 1 KV head: Llama-2 70B's ratio of 64 over 8
    as test_gpu_gqa builds it, scaled to hidden 1024), q4_attn_2 and q4_mlp on outlier x with checkpoint-like weights.
    Without act-order q4_attn / q4_mlp run as one fused launch each; with act-order they take their general paths (_block_weights).
    v and attn_2 are plain projections: within B.  q, k (after rope) and q4_mlp get B plus the fp16 roundings between their steps,
    composed as written beside each check.  The fused RMS norm may move the fp16 row factor by one ulp against the oracle's
    (test_gpu_ops.test_rms_norm), so every projection of a normalised x also gets 2 fp16 ulps of each x element through |W|."""
    import torch
    from exllama_b200 import capi
    hidden, inter, hd, max_seq, past = 1024, 2816, 128, 64, 37
    heads = hidden // hd
    kvw = kvh * hd
    t = _block_weights(hidden, inter, gs, seed=500 + (gs or 1), kv=kvw, act=act)
    x = gen_x("outlier1000", 1, hidden, seed=5, channels=outlier_channels(hidden, gs, 1)).reshape(1, 1, hidden)
    w = (1 + 0.1 * np.random.default_rng(6).standard_normal(hidden)).astype(np.float16)
    sin, cos = sincos(max_seq, hd)

    def mk(n):
        return _q4(capi, *t[n])

    def bound(xin, n):
        qw, qz, sc, g = t[n]
        return _bound_on_cols(oracle, xin, qw, qz, sc, g, np.arange(qw.shape[1]))

    def through(dx, n):
        """sum_k dx_k |w_kn|: how far a change of dx in the input can move the output."""
        qw, qz, sc, g = t[n]
        if g is not None:
            xm = oracle.make_x_map(g, qz.shape[0])
            dx, qw = dx[:, xm.astype(np.int64)], oracle.make_sequential(qw, xm)
        return dx @ np.abs(oracle.dequant_f64(qw, qz, sc))

    def bound_norm(xn_, n):
        B_, r_ = bound(xn_, n)
        return B_ + through(2 * np.spacing(np.abs(xn_)).astype(np.float64), n), r_

    xn, _ = oracle.rms_norm(x.reshape(1, hidden), w, 1e-6)
    tq = torch.empty((1, 1, hidden), dtype=torch.float16, device="cuda")
    tk = torch.empty((1, 1, kvw), dtype=torch.float16, device="cuda"); tv = torch.empty_like(tk)
    kc = torch.zeros((1, kvh, max_seq, hd), dtype=torch.float16, device="cuda"); vc = torch.zeros_like(kc)
    capi.q4_attn(to_cuda(x), to_cuda(w), 1e-6, tq, tk, tv, mk("q"), mk("k"), mk("v"), to_cuda(sin), to_cuda(cos), 1, past,
                 heads, kvh, hd, kc, vc, max_seq)
    torch.cuda.synchronize()
    Bv, rv = bound_norm(xn, "v")
    assert_within_bound(tv.cpu().numpy().reshape(1, -1), Bv, rv, what="v")
    for name, got, nh in (("q", tq, heads), ("k", tk, kvh)):
        Bp, rp = bound_norm(xn, name)
        want = oracle.rope(rp.astype(np.float16).reshape(1, nh, hd), sin, cos, 1, nh, hd, nh, past).reshape(1, -1).astype(np.float64)
        # |got - want| <= rope of the projection's bound + the fp16 roundings of the projection output and of rope's own steps
        assert_within_bound(got.cpu().numpy().reshape(1, -1), _rope_allowance(Bp, rp, sin, cos, nh, hd, past), want,
                            what=f"{name} after rope")

    # q4_attn_2: x += attn . o  (one fp16 rounding of the sum: B's 2^-11 |ref| plus the residual's 2^-11 |x|)
    attn = gen_x("outlier64", 1, hidden, seed=8, channels=outlier_channels(hidden, gs, 4))
    x2 = gen_x("gauss", 1, hidden, seed=9)
    tx = to_cuda(x2.copy())
    capi.q4_attn_2(tx, to_cuda(attn), mk("o"))
    Bo, ro = bound(attn, "o")
    x2d = x2.astype(np.float64)
    assert_within_bound(tx.cpu().numpy(), Bo + 2.0 ** -11 * np.abs(x2d), ro + x2d, what="attn_2")

    # q4_mlp: x += down(silu(gate(n)) * up(n)).  gate and up are rounded to fp16 before the silu: each may sit up to its bound
    # plus one fp16 rounding away from the oracle's, which moves silu(g) * u by at most |silu'(g)| |u| dg + |silu(g)| du (|silu'| <=
    # 1.1); the GPU silu adds its 8 ulps; each change of an act element reaches the output through |w_down|.
    x3 = gen_x("outlier1000", 1, hidden, seed=10, channels=outlier_channels(hidden, gs, 0))
    xn3, _ = oracle.rms_norm(x3, w, 1e-6)
    Bg, rg = bound_norm(xn3, "gate"); Bu, ru = bound_norm(xn3, "up")
    g16, u16 = rg.astype(np.float16), ru.astype(np.float16)
    act16 = oracle.silu_mul(g16, u16)
    dg = Bg + 2.0 ** -11 * np.abs(rg); du = Bu + 2.0 ** -11 * np.abs(ru)
    sg = np.abs(g16.astype(np.float64)) / (1 + np.exp(-g16.astype(np.float64)))
    dact = 1.1 * np.abs(u16.astype(np.float64)) * dg + (sg + 1.1 * dg) * du + 8 * np.spacing(np.abs(act16)).astype(np.float64)
    Bd, rd = bound(act16, "down")
    x3d = x3.astype(np.float64)
    tx = to_cuda(x3.copy())
    capi.q4_mlp(tx, to_cuda(w), 1e-6, mk("gate"), mk("up"), mk("down"))
    torch.cuda.synchronize()
    assert_within_bound(tx.cpu().numpy(), Bd + through(dact, "down") + 2.0 ** -11 * np.abs(x3d), rd + x3d, what="q4_mlp")


# ------------------------------------------------------------------------------------- (d) the persistent step with one group
def _check_step(oracle, st, xs, pasts, what):
    """Fused step vs the per-op path and the float64 oracle composition for every sequence of xs [bsz, 1, hidden].  The two kernels
    quantise x with different steps (32767 and 32639 per segment), so the fused step meets the per-op path on the logits only."""
    import torch
    bsz = len(pasts)
    snap = snapshot(st)
    per_op_logits = [lg.cpu().numpy().reshape(-1) for lg in per_op(st, snap, xs, pasts)[0]]
    st.make_plan()
    logits = fused_step(st, xs, pasts).cpu().numpy()
    torch.cuda.synchronize()
    got_x = st._plan_xout.view(-1, st.shape.hidden)[:bsz].cpu().numpy()
    new_rows = [[(kc[b, :, pasts[b]].cpu().numpy(), vc[b, :, pasts[b]].cpu().numpy()) for kc, vc in zip(st.key_cache, st.value_cache)]
                for b in range(bsz)]
    for b in range(bsz):
        w = f"{what} seq {b} (ctx {pasts[b]})"
        assert np.isfinite(logits[b]).all(), w
        assert_close_ref64(logits[b], per_op_logits[b].astype(np.float64), rel=1.5e-2, rms=1.5e-2, what=f"{w} logits vs per-op")
        want_x, want_logits, rows = oracle_decode_step(oracle, st, snap, xs[b].cpu().numpy(), pasts[b], b)
        assert_close_ref64(got_x[b], want_x.reshape(-1).astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} final hidden vs oracle")
        assert_close_ref64(logits[b], want_logits.reshape(-1), rel=1.5e-2, rms=1.5e-2, what=f"{w} logits vs oracle")
        assert_close_ref64(per_op_logits[b], want_logits.reshape(-1), rel=1.5e-2, rms=1.5e-2, what=f"{w} per-op logits vs oracle")
        for i in range(len(st.layers)):
            assert_close_ref64(new_rows[b][i][0], rows[i][0].astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} layer {i} new k")
            assert_close_ref64(new_rows[b][i][1], rows[i][1].astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} layer {i} new v")
    restore(st, snap)


def _xs(bsz, hidden, seed, scale=0.5, outliers=()):
    import torch
    x = (np.random.default_rng(seed).standard_normal((bsz, 1, hidden)) * scale)
    for c in outliers:
        x[:, :, c] = 300 * scale * (1 if c % 2 else -1)
    return torch.from_numpy(x.astype(np.float16)).cuda()


def test_one_group_stack_layout(oracle, stacks):
    """DecodeStack(groupsize=None): every matrix holds one group (GPTQ groupsize -1), act-order g_idx is all zeros, and tensor
    parallelism is refused."""
    from exllama_b200.stack import DecodeStack, LlamaShape
    st = stacks(layers=1, kv_heads=2, gs=None, max_seq=64, act=True)
    for n in st.PROJ:
        lin = getattr(st.layers[0], n)
        assert lin.qzeros.shape[0] == 1 and lin.scales.shape[0] == 1, n
        assert lin.g_idx is not None and not lin.g_idx.any(), n
    with pytest.raises(NotImplementedError, match="one quantisation group"):
        DecodeStack(LlamaShape("x", 1024, 2816, 1, 8, vocab=2048), groupsize=None, tp_rank=0, tp_size=2)


@pytest.mark.parametrize("act", [False, True])
@pytest.mark.parametrize("kv", [8, 2])
@pytest.mark.parametrize("past", [0, 37, 200])
def test_fused_step_one_group(oracle, stacks, kv, act, past):
    st = stacks(kv_heads=kv, gs=None, seed=40 + kv, act=act)
    _check_step(oracle, st, _xs(1, 1024, past + kv), [past], f"one group kv{kv} act{act}")


def test_fused_step_one_group_batch(oracle, stacks):
    st = stacks(kv_heads=2, gs=None, seed=61, batch=3)
    _check_step(oracle, st, _xs(3, 1024, 62), [5, 200, 37], "one group, batch of 3")


def test_fused_step_one_group_lora(oracle, stacks):
    st = stacks(kv_heads=2, gs=None, seed=63)
    st.add_lora(16, targets="all", alpha=128, seed=2)
    _check_step(oracle, st, _xs(1, 1024, 64, scale=0.05), [37], "one group, LoRA")
    assert adapter_of(st, 0, "down") is not None


def test_fused_step_one_group_70b_shape(oracle, stacks):
    """Llama-2 70B widths (hidden 8192, inter 28672, 64 query heads over 8 KV heads), 2 layers at ctx 1920, one group."""
    from exllama_b200.shapes import GQA_SHAPES
    s = GQA_SHAPES["70b"]
    st = stacks(hidden=s.hidden, inter=s.inter, heads=s.heads, kv_heads=s.kv_heads, gs=None, max_seq=2048, vocab=s.vocab, seed=17)
    _check_step(oracle, st, _xs(1, s.hidden, 70), [1920], "70B one group")


@pytest.mark.parametrize("gs", [128, None])
def test_fused_step_outlier_embedding(oracle, stacks, gs):
    """An embedding row with two channels at 300x the rest (a "massive activation"): both paths against the oracle."""
    st = stacks(kv_heads=2, gs=gs, seed=80)
    _check_step(oracle, st, _xs(1, 1024, 81, outliers=(77, 640)), [37], f"outlier embedding g{gs}")


# ------------------------------------------------------------------------------------------ (e) against the reference kernel
E_CASES = [  # (M, K, N, gs, act, x kind, outlier variant, quiet outlier rows)
    (1, 8192, 4096, None, False, "outlier1000", 0, True),          # the outlier channel's weights are 0 in 90 % of the columns
    (1, 8192, 4096, None, False, "outlier1000", 3, False),
    (4, 4096, 4096, 256, True, "outlier1000", 4, True),
    (1, 8192, 4096, 512, False, "outlier64", 2, True),
    (2, 4096, 4096, None, True, "silu", 0, False),
    (1, 11008, 4096, 256, False, "outlier1000", 1, False),
]


def e_inputs(M, K, N, gs, act, xkind, variant, quiet):
    """Seeded inputs of an E_CASES entry: (x, (qweight, qzeros, scales, g_idx)), shared with oracle/gen_golden_ref_gpu_quant.py."""
    seed = 900 + M + K // 64 + variant
    ch = outlier_channels(K, gs, variant)
    x = gen_x(xkind, M, K, seed=seed, channels=ch, gs=gs)
    return x, synth_q4_ckpt(K, N, gs, act, seed=seed, cols=e_cols(N), quiet_rows=ch if quiet else ())


def e_cols(N):
    """The stored column sample: 64 whole 8-column groups (a restriction the oracle can contract exactly)."""
    return sample_cols(N, 64, seed=N)


def e_key(M, K, N, gs, act, xkind, variant, quiet):
    return f"quant_{M}_{K}_{N}_{gs or 0}_{int(act)}_{xkind}_{variant}_{int(quiet)}"


@pytest.fixture(scope="module")
def golden_quant():
    return np.load(os.path.join(GOLDEN, "ref_gpu_quant.npz"))


@pytest.mark.parametrize("case", E_CASES, ids=[e_key(*c) for c in E_CASES])
def test_error_no_larger_than_reference_kernel(oracle, golden_quant, case):
    """Our rms error against float64 is at most 1.05 x the reference's own on the same inputs (SURVEY.md 8c), on a fixed
    column sample, and the two agree within 2e-2."""
    from exllama_b200 import capi
    M, K, N, gs, act, xkind, variant, quiet = case
    x, (qw, qz, sc, g_idx) = e_inputs(*case)
    c = e_cols(N)
    mine = capi.q4_matmul(to_cuda(x), _q4(capi, qw, qz, sc, g_idx)).cpu().numpy().astype(np.float64)[:, c]
    theirs = golden_quant[e_key(*case)].astype(np.float64)
    sub = q4_column_sample(qw, qz, sc, c)
    ref = oracle.ref64_with_act_order(x, *sub, g_idx)
    rms = np.sqrt(np.mean(theirs ** 2))
    assert np.all(np.abs(mine - theirs) <= 2e-2 * np.abs(theirs) + 2e-2 * rms)
    e_mine = np.sqrt(np.mean((mine - ref) ** 2)); e_ref = np.sqrt(np.mean((theirs - ref) ** 2))
    assert e_mine <= 1.05 * e_ref + 1e-6, (e_mine, e_ref)
