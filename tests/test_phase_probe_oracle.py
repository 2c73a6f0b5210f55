"""CPU proof of the phase-probe bounds (tests/helpers.py, "Phase probes"): the fused decode step's arithmetic emulated in numpy
lands inside every bound over many seeds, and each arithmetic mutation the GPU probes target, emulated the same way, breaks the
bound it targets -- so a failure of tests/test_gpu_decode_phase_probe.py points at the kernel, and a pass means something.

Emulated: the RMS row factor from an fp32 sum in a random order, rounded to fp16, then x * rm * w in fp16; the GEMVs with x
quantised per segment (group cut at the 128-k stage) with Q = 32639, exact int segment sums and fp32 fmas of the segments in a
random order; adapters with fp32 t, fp16(t) and an fp32 B sum; silu_h with hexp and hrcp each landing on either fp16 neighbour
of the exact value; the HEAD's per-lane fhfma2 chains, shuffle tree and fp32 atomics in a random order."""
from types import SimpleNamespace

import numpy as np
import pytest

from helpers import (STAGE_K, head_expectation, hmul, mlp_expectation, o_expectation_ctx0, qkv_expectation, synth_q4_ckpt)
from stack_harness import sincos

f16, f32 = np.float16, np.float32


# ---- the step's arithmetic ------------------------------------------------------------------------------------------------------
def emu_norm(x, w, eps, rng, w_group0=None):
    """The kernel's normalised x: fp32 sum of squares in a random order, 1 / sqrt in fp32, rounded to fp16; then two fp16
    multiplies.  w_group0: weights for the first 8 elements (a mutation)."""
    x = np.asarray(x, f16).reshape(-1)
    ss = np.add.accumulate((x.astype(f32) ** 2)[rng.permutation(x.size)], dtype=f32)[-1]
    rm = f16(f32(1.0) / np.sqrt(f32(ss / f32(x.size) + f32(eps))))
    w = np.asarray(w, f16).copy()
    if w_group0 is not None:
        w[:8] = w_group0
    return hmul(hmul(x, rm), w), rm


def _fma_chain(terms, rng):
    """fp32 sum of float64-exact terms [n, N] in a random order, each addition rounded to fp32."""
    acc = np.zeros(terms.shape[1], f32)
    for i in rng.permutation(len(terms)):
        acc = (acc.astype(np.float64) + terms[i]).astype(f32)
    return acc


def emu_gemv(oracle, x, lin, ab, rng, q_scale=32639.0, upseg_row0=False):
    """The fused step's fp32 accumulator of one GEMV on its fp16 input x [K] (checkpoint order).  q_scale: the Q of the segment
    scale absmax * (1 / Q) (the quantiser uses 32639); upseg_row0: the second 64-k segment of a 128-k stage reads the first one's
    scale / zero row."""
    qw, qz, sc = (t.numpy() for t in (lin.qweight, lin.qzeros, lin.scales))
    K8, N = qw.shape
    K, G = K8 * 8, qz.shape[0]
    gs = K // G
    sh = np.arange(8, dtype=np.uint32) * 4
    q = ((qw.view(np.uint32)[:, None, :] >> sh[None, :, None]) & 0xF).reshape(K, N).astype(np.int64)
    z1 = ((qz.view(np.uint32)[:, :, None] >> sh[None, None, :]) & 0xF).reshape(G, N).astype(np.int64) + 1
    xg = np.asarray(x, f16).reshape(-1)
    if lin.g_idx is not None:
        xg = xg[np.asarray(oracle.make_x_map(lin.g_idx.numpy(), G), np.int64)]
    win = min(gs, STAGE_K)
    terms = []
    for lo in range(0, K, win):
        g = lo // gs
        if upseg_row0 and gs == 64 and (lo % STAGE_K) == 64:
            g -= 1
        xs = xg[lo:lo + win].astype(f32)
        mx = f32(np.abs(xs).max())
        inv = f32(32639.0) / mx if mx > 0 else f32(0)
        xq = np.rint((xs * inv).astype(f32)).astype(np.int64)
        sx = f32(mx * f32(1.0 / q_scale))
        val = xq @ (q[lo:lo + win] - z1[g])
        terms.append((sc[g].astype(f32) * sx).astype(f32).astype(np.float64) * val)
    acc = _fma_chain(np.array(terms), rng)
    if ab is not None:
        A, B = (t.numpy() for t in ab)
        t = _fma_chain(np.asarray(x, f16).astype(np.float64)[:, None] * A.astype(np.float64), rng)
        acc = _fma_chain(np.vstack([acc.astype(np.float64)[None],
                                    t.astype(f16).astype(np.float64)[:, None] * B.astype(np.float64)]), rng)
    return acc


def _either(v, rng):
    """Exact v rounded to an fp16 neighbour at random (an fp32 approximation rounded to fp16: within one ulp)."""
    with np.errstate(over="ignore"):
        r = np.asarray(v, np.float64).astype(f16)
        other = np.nextafter(r, np.where(r > v, f16(-np.inf), f16(np.inf)).astype(f16))
    return np.where(rng.random(r.shape) < 0.5, r, np.where(np.isfinite(other), other, r)).astype(f16)


def emu_silu_h(g, rng):
    """hmul(g, hrcp(hadd(1, hexp(-g)))) with hexp and hrcp each on either fp16 neighbour of the exact value."""
    g = np.asarray(g, f16)
    with np.errstate(over="ignore", divide="ignore"):
        e = _either(np.exp(-g.astype(np.float64)), rng)
        s = (1.0 + e.astype(np.float64)).astype(f16)
        r = _either(1.0 / s.astype(np.float64), rng)
    return hmul(g, r)


def emu_head(x_out, norm, W, eps, rng, unrounded_rm=False, w_group0=None):
    """The HEAD phase: h = the kernel's normalised x_out; per vocabulary row the chunks of 512 go to warps two at a time (chunk
    pairs of the row-major [vocab, H] order), a lane chains 8 fhfma2 over its 16 values of each chunk, the warp reduces with 5
    xor shuffles and adds its partial to the logit with an fp32 atomic, in a random order."""
    x_out = np.asarray(x_out, f16).reshape(-1)
    H = x_out.size
    if unrounded_rm:
        ss = np.add.accumulate((x_out.astype(f32) ** 2)[rng.permutation(H)], dtype=f32)[-1]
        rmf = f32(1.0) / np.sqrt(f32(ss / f32(H) + f32(eps)))
        h = hmul((x_out.astype(f32) * rmf).astype(f16), norm)
    else:
        h, _ = emu_norm(x_out, norm, eps, rng, w_group0)
    V = W.shape[0]
    cpr = H // 512
    P = W.astype(np.float64) * h.astype(np.float64)[None]                       # exact products
    P = P.reshape(V, cpr, 2, 32, 8).transpose(0, 1, 3, 2, 4).reshape(V, cpr, 32, 16)   # [row, chunk, lane, chain order]
    parts = {}
    for row_chunk in range(V * cpr):
        row, kc = divmod(row_chunk, cpr)
        key = (row, row_chunk // 2)
        lane = parts.get(key, np.zeros(32, f32))
        for j in range(16):
            lane = (lane.astype(np.float64) + P[row, kc, :, j]).astype(f32)
        parts[key] = lane
    logits = np.zeros(V, f32)
    by_row = {}
    for (row, _), lane in parts.items():
        for off in (16, 8, 4, 2, 1):
            lane = (lane + lane[np.arange(32) ^ off]).astype(f32)
        by_row.setdefault(row, []).append(lane[0])
    for row, ps in by_row.items():
        for i in rng.permutation(len(ps)):
            logits[row] = f32(logits[row] + ps[i])
    return logits


# ---- a CPU stand-in of a phase-probe DecodeStack ------------------------------------------------------------------------------
def _distinct(n, seed):
    from helpers import distinct_norm
    return distinct_norm(n, seed)


def cpu_stack(oracle, gs=128, act=False, heads=4, kv=2, inter=512, layers=1, lora=(), o_off=(), mlp_off=(), seed=0):
    import torch
    from exllama_b200.shapes import LlamaShape
    hd = 128
    hidden = heads * hd
    shape = LlamaShape("cpu-phase-probe", hidden, inter, layers, heads, vocab=512, kv_heads=kv)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    rng = np.random.default_rng(seed)

    def lin(K, N, j, scale=0.2):
        qw, qz, sc, g = synth_q4_ckpt(K, N, gs, act, seed=seed * 100 + j, scale=scale)
        if g is not None:
            qw = oracle.make_sequential(qw, oracle.make_x_map(g, qz.shape[0]))
        return SimpleNamespace(qweight=t(qw), qzeros=t(qz), scales=t(sc), g_idx=None if g is None else t(g))
    Ls, lo = [], []
    for i in range(layers):
        L = SimpleNamespace(q=lin(hidden, hidden, 10 * i), k=lin(hidden, kv * hd, 10 * i + 1), v=lin(hidden, kv * hd, 10 * i + 2),
                            o=lin(hidden, hidden, 10 * i + 3), gate=lin(hidden, inter, 10 * i + 4), up=lin(hidden, inter, 10 * i + 5),
                            down=lin(inter, hidden, 10 * i + 6),
                            ln1=t(_distinct(hidden, seed * 101 + 3 * i)), ln2=t(_distinct(hidden, seed * 101 + 3 * i + 1)))
        if i in o_off:
            L.o.scales.zero_()
        if i in mlp_off:
            L.ln2.zero_()
        ad = {}
        for n in lora:
            K, N = getattr(L, n).qweight.shape[0] * 8, getattr(L, n).qweight.shape[1]
            ad[n] = (t((rng.standard_normal((K, 16)) / np.sqrt(K)).astype(f16)), t((rng.standard_normal((16, N)) * 0.05).astype(f16)))
        Ls.append(L); lo.append(ad)
    sin, cos = sincos(256, hd)
    return SimpleNamespace(shape=shape, layers=Ls, sin=t(sin), cos=t(cos), max_seq=256, lora=lo if lora else None,
                           norm=t(_distinct(hidden, seed * 101 + 99)),
                           lm_head=t((rng.standard_normal((512, hidden)) * 0.02).astype(f16)))


def _ad(st, l, n):
    return (st.lora[l] or {}).get(n) if st.lora is not None else None


def emu_layer_qkv(oracle, st, l, x, past, rng, ln=None, **mut):
    """Layer l's new (k, v) rows [kv_heads, hd] as the kernel computes them on its fp16 layer input x."""
    s = st.shape
    L = st.layers[l]
    xn, _ = emu_norm(x, L.ln1.numpy() if ln is None else ln, s.eps, rng)
    k = emu_gemv(oracle, xn, L.k, _ad(st, l, "k"), rng, **mut).astype(f16)
    v = emu_gemv(oracle, xn, L.v, _ad(st, l, "v"), rng, **mut).astype(f16)
    k = oracle.rope(k.reshape(1, s.kv_heads, 128), st.sin.numpy(), st.cos.numpy(), 1, s.kv_heads, 128, s.kv_heads, past)
    return k.reshape(s.kv_heads, 128), v.reshape(s.kv_heads, 128)


def emu_mlp(oracle, st, l, x, rng, down_k8_0_up=False):
    """x_out of a layer with o off: fp16(x + down(hmul(silu_h(fp16(gate)), fp16(up))))."""
    L = st.layers[l]
    xn, _ = emu_norm(x, L.ln2.numpy(), st.shape.eps, rng)
    g = emu_gemv(oracle, xn, L.gate, _ad(st, l, "gate"), rng).astype(f16)
    u = emu_gemv(oracle, xn, L.up, _ad(st, l, "up"), rng).astype(f16)
    if down_k8_0_up:
        g = g.copy(); g[:8] = u[:8]
    act = hmul(emu_silu_h(g, rng), u)
    d = emu_gemv(oracle, act, L.down, _ad(st, l, "down"), rng)
    return (np.asarray(x, f16).astype(f32) + d).astype(f16)


def _fits(got, cands):
    if not isinstance(got, tuple):
        got, cands = (got,), [(c,) for c in cands]
    return min(max(float(np.max(np.abs(np.asarray(gv, np.float64).reshape(np.shape(w)) - w) / b)) for gv, (w, b) in zip(got, c))
               for c in cands)


def _x(n, seed):
    return (1e-2 * np.random.default_rng(seed).standard_normal(n)).astype(f16)


# ---- every bound holds on the emulated step -----------------------------------------------------------------------------------
PLANS = [dict(gs=32), dict(gs=64), dict(gs=128), dict(gs=None), dict(gs=128, act=True), dict(gs=32, act=True), dict(gs=128, kv=1),
         dict(gs=64, lora=("k", "v", "o", "gate", "up", "down"))]


@pytest.mark.parametrize("plan", range(len(PLANS)))
def test_emulated_step_within_every_bound(oracle, plan):
    """QKV rows, o_proj at context 0, the MLP and the HEAD over 4 seeds each: the emulated kernel is inside every bound, and the
    bounds are tight (QKV rms below 1e-2 of the row's rms, HEAD below 3e-4 of the logits' rms: 50x inside 1.5e-2)."""
    kw = PLANS[plan]
    for seed in range(4):
        rng = np.random.default_rng(1000 * plan + seed)
        st = cpu_stack(oracle, seed=seed, **kw)
        x = _x(st.shape.hidden, seed)
        past = [0, 37, 200, 255][seed]
        k, v = emu_layer_qkv(oracle, st, 0, x, past, rng)
        c = qkv_expectation(oracle, st, 0, x, past)
        assert _fits((k, v), c) <= 1
        assert np.sqrt(np.mean(c[0][1][1] ** 2) / np.mean(c[0][1][0] ** 2)) < 1e-2
        # o_proj at context 0 (MLP off): attn = the new v row
        st_o = cpu_stack(oracle, seed=seed, mlp_off=(0,), **kw)
        _, v0 = emu_layer_qkv(oracle, st_o, 0, x, 0, rng)
        attn = np.repeat(v0.reshape(st_o.shape.kv_heads, 1, 128), st_o.shape.heads // st_o.shape.kv_heads, axis=1).reshape(-1)
        xo = (x.astype(f32) + emu_gemv(oracle, attn, st_o.layers[0].o, _ad(st_o, 0, "o"), rng)).astype(f16)
        assert _fits(xo, [o_expectation_ctx0(oracle, st_o, 0, x, v0)]) <= 1
        # the MLP (o off)
        st_m = cpu_stack(oracle, seed=seed, o_off=(0,), **kw)
        xm = emu_mlp(oracle, st_m, 0, x, rng)
        assert _fits(xm, mlp_expectation(oracle, st_m, 0, x)) <= 1
        # the HEAD on that x_out
        lg = emu_head(xm, st_m.norm.numpy(), st_m.lm_head.numpy(), st_m.shape.eps, rng)
        hc = head_expectation(xm, st_m.norm.numpy(), st_m.lm_head.numpy(), st_m.shape.eps)
        assert _fits(lg, hc) <= 1
        assert np.sqrt(np.mean(hc[0][1] ** 2) / np.mean(hc[0][0] ** 2)) < 3e-4


@pytest.mark.parametrize("H", [1024, 1536])
def test_emulated_head_within_bound_many_orders(oracle, H):
    """The HEAD alone at a width whose chunk pairs line up with the rows (1024) and one where they straddle rows (1536)."""
    rng = np.random.default_rng(H)
    W = (rng.standard_normal((256, H)) * 0.02).astype(f16)
    norm = _distinct(H, 5)
    for seed in range(6):
        x = (rng.standard_normal(H) * rng.uniform(0.01, 3)).astype(f16)
        assert _fits(emu_head(x, norm, W, 1e-6, rng), head_expectation(x, norm, W, 1e-6)) <= 1


# ---- each mutation the GPU probes target breaks its bound ---------------------------------------------------------------------
def _breaks(values):
    """The mutation escapes the bound (ratio > 1) in at least three of four seeds."""
    return sum(v > 1 for v in values) >= 3


def test_mutation_segment_scale_32767_breaks_qkv(oracle):
    """absmax * (1 / 32767) instead of (1 / 32639): every projection 0.39 % small."""
    r = []
    for seed in range(4):
        st = cpu_stack(oracle, seed=seed)
        x = _x(st.shape.hidden, seed)
        k, v = emu_layer_qkv(oracle, st, 0, x, 37, np.random.default_rng(seed), q_scale=32767.0)
        r.append(_fits((k, v), qkv_expectation(oracle, st, 0, x, 37)))
    assert _breaks(r), r


def test_mutation_upseg2_scale_row_breaks_qkv(oracle):
    """Groups of 64: the second segment of a stage with the first one's scale / zero row."""
    r = []
    for seed in range(4):
        st = cpu_stack(oracle, gs=64, seed=seed)
        x = _x(st.shape.hidden, seed)
        k, v = emu_layer_qkv(oracle, st, 0, x, 37, np.random.default_rng(seed), upseg_row0=True)
        r.append(_fits((k, v), qkv_expectation(oracle, st, 0, x, 37)))
    assert _breaks(r), r


def test_mutation_stale_ln1_breaks_handoff(oracle):
    """Layer 1's QKV normalised with layer 0's ln1 (a preload of the wrong layer's weights)."""
    r = []
    for seed in range(4):
        st = cpu_stack(oracle, layers=2, seed=seed)
        x = _x(st.shape.hidden, seed)                   # stands for layer 0's output
        k, v = emu_layer_qkv(oracle, st, 1, x, 16, np.random.default_rng(seed), ln=st.layers[0].ln1.numpy())
        r.append(_fits((k, v), qkv_expectation(oracle, st, 1, x, 16)))
    assert _breaks(r), r


def test_mutation_down_reads_up_for_gate_breaks_mlp(oracle):
    """DOWN staging: silu(up) * up instead of silu(gate) * up in the first 8-wide column group."""
    r = []
    for seed in range(4):
        st = cpu_stack(oracle, o_off=(0,), seed=seed)
        x = _x(st.shape.hidden, seed)
        r.append(_fits(emu_mlp(oracle, st, 0, x, np.random.default_rng(seed), down_k8_0_up=True), mlp_expectation(oracle, st, 0, x)))
    assert _breaks(r), r


@pytest.mark.parametrize("mut", ["unrounded_rm", "neighbour_group"])
def test_mutation_head_breaks_head(oracle, mut):
    """HEAD with the fp32 row factor unrounded, or the first 8 elements normalised with the next 8's weights."""
    r = []
    H = 1024
    for seed in range(4):
        rng = np.random.default_rng(seed)
        W = (rng.standard_normal((256, H)) * 0.02).astype(f16)
        norm = _distinct(H, seed)
        x = (rng.standard_normal(H) * 0.3).astype(f16)
        kw = dict(unrounded_rm=True) if mut == "unrounded_rm" else dict(w_group0=norm[8:16])
        r.append(_fits(emu_head(x, norm, W, 1e-6, rng, **kw), head_expectation(x, norm, W, 1e-6)))
    assert _breaks(r), r


# ---- the switches give exact zeros ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gs,act", [(128, False), (64, True), (None, False)])
def test_zero_scales_and_zero_ln2_give_exact_zeros(oracle, gs, act):
    """o off: zero scales contract any x to exactly 0 (oracle and emulation).  MLP off: ln2 = 0 normalises to exactly 0, so gate,
    up, silu * mul and down are exactly 0."""
    st = cpu_stack(oracle, gs=gs, act=act, o_off=(0,), mlp_off=(0,), seed=3)
    L = st.layers[0]
    rng = np.random.default_rng(0)
    a = rng.standard_normal((1, st.shape.hidden)).astype(f16)
    xm = None if L.o.g_idx is None else oracle.make_x_map(L.o.g_idx.numpy(), L.o.qzeros.shape[0])
    assert not oracle.q4_matmul_f64(a, L.o.qweight.numpy(), L.o.qzeros.numpy(), L.o.scales.numpy(), xm).any()
    assert not emu_gemv(oracle, a, L.o, None, rng).any()
    xn, _ = oracle.rms_norm(a, L.ln2.numpy(), st.shape.eps)
    assert not xn.astype(np.float64).any()
    gm = None if L.gate.g_idx is None else oracle.make_x_map(L.gate.g_idx.numpy(), L.gate.qzeros.shape[0])
    g = oracle.q4_matmul_f64(xn, L.gate.qweight.numpy(), L.gate.qzeros.numpy(), L.gate.scales.numpy(), gm).astype(f16)
    act_ = oracle.silu_mul(g, g)
    dm = None if L.down.g_idx is None else oracle.make_x_map(L.down.g_idx.numpy(), L.down.qzeros.shape[0])
    assert not oracle.q4_matmul_f64(act_, L.down.qweight.numpy(), L.down.qzeros.numpy(), L.down.scales.numpy(), dm).any()
    assert (emu_mlp(oracle, st, 0, a[0], rng) == a[0]).all()
