"""Shared helpers for the parity tests (test infrastructure; may import the oracle)."""
import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Stated fp16 tolerance for q4_matmul (SURVEY.md 8c): ours accumulates exact fp16 products in fp32, so the
# only error against the float64 restatement is the final fp16 rounding (2^-11 relative) plus fp32 summation.
REL_TOL = 1.5e-3
RMS_TOL = 1.5e-3


def assert_close_ref64(got_f16, ref64, rel=REL_TOL, rms=RMS_TOL, what=""):
    got = np.asarray(got_f16, dtype=np.float64)
    ref = np.asarray(ref64, dtype=np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert np.isfinite(got).all(), f"{what}: non-finite output"
    r = np.sqrt(np.mean(ref * ref))
    err = np.abs(got - ref)
    bound = rel * np.abs(ref) + rms * r
    bad = err > bound
    assert not bad.any(), (f"{what}: {bad.sum()} / {bad.size} outside tolerance; max err {err.max():.4g} "
                           f"(rms ref {r:.4g}) at {np.unravel_index(err.argmax(), err.shape)}")
    return float(np.sqrt(np.mean(err * err)) / max(r, 1e-30))


def close_to_reference(mine, ref, what):
    """Within 2e-2 relative plus 2e-2 of the rms of the reference kernel's output (its own fp16 rounding points differ from ours)."""
    mine = np.asarray(mine, np.float64); ref = np.asarray(ref, np.float64)
    rms = np.sqrt(np.mean(ref ** 2))
    bad = np.abs(mine - ref) > 2e-2 * np.abs(ref) + 2e-2 * rms
    assert not bad.any(), f"{what}: {bad.sum()} / {bad.size} outside 2e-2; max {np.abs(mine - ref).max():.4g}, rms {rms:.4g}"


def att_needs_reset(heads, kv_heads, longest, grid, bsz=1):
    """decode_step_sched.h att_needs_reset: whether exl_decode_step resets the attention-partial table before a launch whose longest
    context is `longest`.  The attention phase has bsz x kv_heads x ceil(longest / 16) units (at least one per virtual KV head) for
    min(grid, bsz x kv_heads x cap) CTAs, cap 16 per KV head under grouped-query attention and 7 per head without; with two or more
    units per head and fewer units than CTAs, some CTA inside a head's range owns none (tests/test_batch_schedule.py proves this
    restatement against the header)."""
    nph = max(1, (longest + 15) // 16)
    cap = 16 if kv_heads < heads else 7
    return nph >= 2 and bsz * kv_heads * nph < min(grid, bsz * kv_heads * cap)


def ulp_diff_f16(a, b):
    """Distance in fp16 ulps (monotone integer mapping of the bit patterns)."""
    def key(x):
        u = np.asarray(x, dtype=np.float16).view(np.uint16).astype(np.int32)
        return np.where(u & 0x8000, -(u & 0x7fff), u & 0x7fff)
    return np.abs(key(a) - key(b))


GOLDEN = os.path.join(ROOT, "tests", "golden")


def golden_cols(n, seed, k=512):
    """The fixed sample of output columns stored for a golden array whose last axis has n entries (all of them when n <= k)."""
    if n <= k:
        return np.arange(n)
    return np.sort(np.random.default_rng(seed).choice(n, k, replace=False))


def _np(t):
    return t.cpu().numpy()


def adapter_of(st, i, name):
    """(A, B) of projection `name` of layer i of a DecodeStack, or None."""
    return (st.lora[i] or {}).get(name) if st.lora is not None else None


def oracle_mm(oracle, xin, lin, ab=None, acc=None, recons=False):
    """x . W of a stack projection in float64 (act-order: the x gather of make_q4's sequential layout), accumulated onto acc, with an
    adapter (A, B): acc + fp16(fp16(x . A) . B) as q4_matmul_lora and the per-op blocks compose it.

    recons=True contracts against the fp16-rounded reconstructed weights (what the wgmma GEMM's B operand holds, bit-identical to
    reconstruct_kernel).  Those weights come from oracle.reconstruct_f16 once and are contracted in float64 by numpy: the same exact
    sum as oracle.q4_matmul_f64(..., recons=True), which re-dequantises every weight for every row and is too slow for a prefill."""
    xm = None if lin.g_idx is None else oracle.make_x_map(lin.g_idx.numpy(), lin.qzeros.shape[0])
    if ab is not None:
        t = oracle.half_matmul_f64(xin, _np(ab[0])).astype(np.float16)
        acc = oracle.half_matmul_f64(t, _np(ab[1]), acc_in=acc).astype(np.float16)
    if not recons:
        return oracle.q4_matmul_f64(xin, _np(lin.qweight), _np(lin.qzeros), _np(lin.scales), xm, acc)
    w = oracle.reconstruct_f16(_np(lin.qweight), _np(lin.qzeros), _np(lin.scales)).astype(np.float64)
    xg = np.asarray(xin, np.float64) if xm is None else np.asarray(xin, np.float64)[:, xm]
    out = xg @ w
    return out if acc is None else out + np.asarray(acc, np.float64)


def oracle_qkv(oracle, st, i, x, past):
    """Layer i of a DecodeStack on the fp16 layer inputs x [n, hidden] of n consecutive tokens, token t at position past + t, as
    oracle_decode_step computes them: (normed x [n, hidden], roped fp16 q [n, heads * hd], roped fp16 k [n, kv_heads, hd], fp16 v
    [n, kv_heads, hd]).  One token (n = 1): q [heads * hd], k and v [kv_heads, hd]."""
    s = st.shape
    hd, heads, kvh = s.head_dim, s.heads, s.kv_heads
    sin = st.sin.view(-1, hd).cpu().numpy(); cos = st.cos.view(-1, hd).cpu().numpy()
    L = st.layers[i]
    x = np.asarray(x, np.float16).reshape(-1, s.hidden)
    n = x.shape[0]
    xn, _ = oracle.rms_norm(x, _np(L.ln1), s.eps)
    q, k, v = (oracle_mm(oracle, xn, getattr(L, m), adapter_of(st, i, m)).astype(np.float16) for m in ("q", "k", "v"))
    # the oracle's rope puts row r at position past + r // num_heads: token t's heads at past + t
    q = oracle.rope(q.reshape(1, n * heads, hd), sin, cos, 1, n * heads, hd, heads, past).reshape(n, heads * hd)
    k = oracle.rope(k.reshape(1, n * kvh, hd), sin, cos, 1, n * kvh, hd, kvh, past).reshape(n, kvh, hd)
    v = v.reshape(n, kvh, hd)
    return (xn, q[0], k[0], v[0]) if n == 1 else (xn, q, k, v)


def causal_attn(oracle, st, q, kc, vc, past):
    """Attention of n consecutive tokens of one sequence: q [n, heads, hd] fp16 (token t at position past + t), kc / vc [kv_heads,
    max_seq, hd] fp16 holding the launch's own rows at past .. past + n - 1.  Token t reads rows [0, past + t]: one decode query
    of oracle.decode_attn_f64 per token.  Returns float64 [n, heads, hd]."""
    from prefill_oracle import prefill_attn_f64
    s = st.shape
    return prefill_attn_f64(oracle, q, kc, vc, s.heads, s.kv_heads, past, st.max_seq, s.head_dim)


def oracle_decode_step(oracle, st, snap, x, past, seq=0, n_layers=None, attend=None):
    """float64/fp16 restatement of one decode launch of a DecodeStack (grouped-query attention, cache sequence `seq`, the stack's
    adapter) on the cache snapshot `snap` (per layer (key_cache, value_cache) tensors), with the fused step's rounding points:
    x [n, hidden] holds n consecutive tokens, token t at position past + t.  Per layer every token's k / v rows go into rows
    past .. past + n - 1 of a copy of the cache, then token t attends rows [0, past + t] (causal_attn).  Returns (final hidden fp16
    [n, hidden], logits float64 [n, vocab] or None for a stack without a head, new k / v rows per layer: [kv_heads, n, hd] each, or
    [kv_heads, hd] for one token).  n_layers: stop after that many layers (hidden state after them, no logits).  attend(l, q, kc,
    vc): the attention of layer l in place of causal_attn (a test emulating a kernel bug)."""
    s = st.shape
    hd, heads, kvh = s.head_dim, s.heads, s.kv_heads
    x = np.asarray(x, np.float16).reshape(-1, s.hidden).copy()
    n = x.shape[0]
    rows = []
    for i, L in enumerate(st.layers):
        _, q, k, v = oracle_qkv(oracle, st, i, x, past)
        q, k, v = q.reshape(n, heads, hd), k.reshape(n, kvh, hd), v.reshape(n, kvh, hd)
        kc = _np(snap[i][0][seq]).copy(); vc = _np(snap[i][1][seq]).copy()
        kc[:, past:past + n] = k.transpose(1, 0, 2); vc[:, past:past + n] = v.transpose(1, 0, 2)
        rows.append((k[0].copy(), v[0].copy()) if n == 1 else (kc[:, past:past + n].copy(), vc[:, past:past + n].copy()))
        a = causal_attn(oracle, st, q, kc, vc, past) if attend is None else attend(i, q, kc, vc)
        attn = a.astype(np.float16).reshape(n, -1)
        x = oracle_mm(oracle, attn, L.o, adapter_of(st, i, "o"), acc=x).astype(np.float16)
        xn, _ = oracle.rms_norm(x, _np(L.ln2), s.eps)
        act = oracle.silu_mul(oracle_mm(oracle, xn, L.gate, adapter_of(st, i, "gate")).astype(np.float16),
                              oracle_mm(oracle, xn, L.up, adapter_of(st, i, "up")).astype(np.float16))
        x = oracle_mm(oracle, act, L.down, adapter_of(st, i, "down"), acc=x).astype(np.float16)
        if i + 1 == n_layers:
            return x, None, rows
    if st.lm_head is None:
        return x, None, rows
    hn, _ = oracle.rms_norm(x, _np(st.norm), s.eps)
    return x, hn.astype(np.float64) @ _np(st.lm_head).astype(np.float64).T, rows


def q4_column_sample(qweight, qzeros, scales, cols):
    """(qweight, qzeros, scales) of the output columns `cols` (whole groups of 8, ascending): an exact restriction of the matrix, so
    the float64 oracle can check a sample of a matrix too wide to contract in full."""
    cols = np.asarray(cols)
    G = qzeros.shape[0]
    sub_qw = np.ascontiguousarray(qweight[:, cols]); sub_sc = np.ascontiguousarray(scales[:, cols])
    zfull = ((qzeros.view(np.uint32)[:, :, None] >> (np.arange(8, dtype=np.uint32) * 4)[None, None]) & 0xF).reshape(G, -1)
    zsub = zfull[:, cols].reshape(G, -1, 8)
    sub_qz = (zsub.astype(np.uint32) << (np.arange(8, dtype=np.uint32) * 4)).sum(-1).astype(np.uint32).view(np.int32)
    return sub_qw, np.ascontiguousarray(sub_qz), sub_sc


def sample_cols(N, groups8, seed=0):
    """`groups8` whole 8-column groups of an N-wide output (all columns when that covers N), ascending."""
    if groups8 * 8 >= N:
        return np.arange(N)
    c = np.sort(np.random.default_rng(seed).choice(N // 8, groups8, replace=False)) * 8
    return (c[:, None] + np.arange(8)[None]).reshape(-1)


# ---------------------------------------------------------------------------------------------------------------------------------
# x quantisation of the decode GEMVs: an error bound, and the inputs that stress it
#
# q4_gemv_kernel (q4_gemv.cu) and decode_step_kernel (decode_step.cu) carry x as a 16-bit integer per quantisation segment:
#     x_q = rn(x * Q / absmax(segment)),   x ~ x_q * absmax / Q,   Q = 32767 (q4_gemv) or 32639 (decode_step: the high byte
#     (x_q + 128) >> 8 must fit in s8),
# and contract x_q with the 4-bit weights exactly in int32.  In both kernels a segment lies inside one quantisation group and one
# aligned 128-k ring stage.  Which segments a launch uses (q4_gemv also cuts them at its staging chunk and cluster slice) is the
# launch's business; the bound below takes the largest window a segment can have, so it holds for any split.
# ---------------------------------------------------------------------------------------------------------------------------------

QUANT_Q = {"gemv": 32767, "step": 32639}
STAGE_K = 128
FP16_TINY = 2.0 ** -24            # smallest fp16 subnormal
# The fp32 term.  Every fp32 rounding on the way to an output -- Q / absmax and x * (Q / absmax), the x scale absmax * (1/Q), scale
# * x scale, (float)val and the fma of each segment, then the k-warp, cluster and atomic sums of the partials -- is a relative error
# of at most 2^-24 of a partial no larger than (1 + 2^-22) sum_k |x_k w_kn|.  A segment costs at most 4 of them plus one addition,
# an output sees at most one segment per window plus one per 128-k stage where a chunk or a cluster slice cuts a window, and fewer
# than QUANT_C more in the k-warp / cluster / atomic reductions: n_fp32 = 5 * (windows + K / 128) + QUANT_C roundings in all.
QUANT_C = 16


def quant_windows(K, groups):
    """Window index of every k (gathered order): the largest range of k one quantisation segment may cover, the group
    intersected with the aligned 128-k stage."""
    return np.arange(K) // min(K // groups, STAGE_K)


def quant_error_bound(oracle, x, qweight, qzeros, scales, x_map=None, kind="gemv"):
    """(B, ref64): a float64 bound B[m, n] >= |kernel - ref64| of one decode GEMV, and ref64 itself.

    qweight is in the sequential layout make_q4 leaves (groups contiguous in k, oracle.make_sequential) and x is gathered through
    x_map before the contraction, as the kernels do.

        B = (1 + 2^-10) * ( sum_k A(k) / (2Q) |w_kn|  +  n_fp32 2^-24 sum_k |x_mk w_kn| )  +  2^-11 |ref|  +  2^-24

    A(k) = absmax of x over the window of k (quant_windows): rounding x to the 16-bit grid costs at most half a step A / Q per
    element.  n_fp32 (QUANT_C's comment) is 5 (K / min(gs, 128) + K / 128) + 16: about K / 5 at groups of 32, K / 13 from
    groups of 128 up.  2^-11 |ref| + 2^-24 is the final fp16 rounding (relative for normal results,
    absolute below 2^-14), and 1 + 2^-10 lets that rounding act on the error itself."""
    assert kind in QUANT_Q
    xg = np.asarray(x, np.float16).astype(np.float64)
    if x_map is not None:
        xg = xg[:, np.asarray(x_map, np.int64)]
    W = oracle.dequant_f64(qweight, qzeros, scales)
    ref = xg @ W
    M, K = xg.shape
    win = quant_windows(K, qzeros.shape[0])
    starts = np.flatnonzero(np.r_[True, win[1:] != win[:-1]])
    A = np.maximum.reduceat(np.abs(xg), starts, axis=1)[:, win]
    aw = np.abs(W)
    t1 = (A / (2.0 * QUANT_Q[kind])) @ aw
    n_fp32 = 5 * (win[-1] + 1 + -(-K // STAGE_K)) + QUANT_C
    t2 = n_fp32 * 2.0 ** -24 * (np.abs(xg) @ aw)
    return (1 + 2.0 ** -10) * (t1 + t2) + 2.0 ** -11 * np.abs(ref) + FP16_TINY, ref


def assert_within_bound(got_f16, bound, ref, what=""):
    got = np.asarray(got_f16, np.float64)
    assert np.isfinite(got).all(), f"{what}: non-finite output"
    err = np.abs(got - ref)
    bad = err > bound
    i = np.unravel_index(np.argmax(err / bound), err.shape)
    assert not bad.any(), (f"{what}: {bad.sum()} / {bad.size} outside the quantisation bound; worst at {i}: err {err[i]:.4g} > "
                           f"bound {bound[i]:.4g} (ref {ref[i]:.4g})")
    return float((err / bound).max())


# ---- weights ----------------------------------------------------------------------------------------------------------------------

def pack_q4(nib, znib, scales, g_idx=None):
    """nibbles q [K, N] and stored zero nibbles z [G, N] (0..15) -> GPTQ (qweight [K/8, N], qzeros [G, N/8], scales, g_idx)."""
    K, N = nib.shape
    sh = np.arange(8, dtype=np.uint32) * 4
    qw = (nib.astype(np.uint32).reshape(K // 8, 8, N) << sh[None, :, None]).sum(1, dtype=np.uint32).view(np.int32)
    G, Nz = znib.shape
    qz = (znib.astype(np.uint32).reshape(G, Nz // 8, 8) << sh[None, None, :]).sum(-1, dtype=np.uint32).view(np.int32)
    return np.ascontiguousarray(qw), np.ascontiguousarray(qz), np.asarray(scales, np.float16), g_idx


def _groups(K, gs):
    return 1 if gs is None else K // gs


def _g_idx(K, gs, act, rng):
    if not act:
        return None
    g = np.zeros(K, np.int32) if gs is None else (np.arange(K) // gs).astype(np.int32)
    return g[rng.permutation(K)]


def synth_q4_ckpt(K, N, gs, act=False, seed=0, cols=None, scale=1.0, quiet_rows=(), quiet_frac=0.9, g_idx=None):
    """Checkpoint-like GPTQ tensors (gs None = one group): stored zero nibbles 7 or 8, nibbles a discretised normal (sd 2.5)
    around z + 1 clipped to 0..15, scales log-uniform over two decades (x `scale`) with 1 % of the columns at 30x.
    cols: only these columns get checkpoint-like nibbles (the rest uniform), so a sampled-column check of a very wide matrix stays
    cheap.  quiet_rows: k (original order) whose weights are exactly 0 (q = z + 1) in `quiet_frac` of the columns -- an outlier
    channel the layer mostly ignores.  g_idx: use this act-order permutation (matrices that share one x order, e.g. q / k / v)."""
    rng = np.random.default_rng(seed)
    G = _groups(K, gs)
    znib = rng.integers(7, 9, size=(G, N))
    sc = 10.0 ** rng.uniform(-3.5, -1.5, size=(G, N)) * scale
    sc[:, rng.random(N) < 0.01] *= 30
    cols = np.arange(N) if cols is None else np.asarray(cols)
    g_idx = _g_idx(K, gs, act, rng) if g_idx is None else g_idx
    grp = (np.zeros(K, np.int64) if gs is None else np.arange(K) // gs) if g_idx is None else g_idx.astype(np.int64)
    zc = znib[:, cols][grp] + 1
    nc = np.clip(np.rint(zc + 2.5 * rng.standard_normal((K, len(cols)))), 0, 15)
    for k in quiet_rows:
        quiet = rng.random(len(cols)) < quiet_frac
        nc[k, quiet] = zc[k, quiet]
    qw_c, qz, sc16, _ = pack_q4(nc.astype(np.uint8), znib, sc.astype(np.float16))
    if len(cols) == N:
        return qw_c, qz, sc16, g_idx
    qw = rng.integers(0, 2**32, size=(K // 8, N), dtype=np.uint32).view(np.int32)
    qw[:, cols] = qw_c
    return qw, qz, sc16, g_idx


def synth_q4_saturated(K, N, gs, sign=-1, scales=None, act=False, seed=0):
    """Every weight at the end of the 4-bit range: sign -1 = nibble 0 with zero nibble 15 (q - z - 1 = -16), sign +1 = nibble 15
    with zero nibble 0 (q - z - 1 = +14).  The packed words are built directly (all nibbles equal), so 70B widths stay cheap."""
    rng = np.random.default_rng(seed)
    G = _groups(K, gs)
    wq, wz = (0, -1) if sign < 0 else (-1, 0)                       # -1 = 0xffffffff: eight nibbles of 15
    if scales is None:
        scales = 10.0 ** rng.uniform(-3, -2, size=(G, N))
    return (np.full((K // 8, N), wq, np.int32), np.full((G, N // 8), wz, np.int32), np.asarray(scales, np.float16),
            _g_idx(K, gs, act, rng))


# ---- activations ------------------------------------------------------------------------------------------------------------------

def outlier_channels(K, gs, variant):
    """Channels for the outlier generator (gs None = one group): variant 0 = the first k of a group, stage and chunk; 1 = the last k
    of a group and the first of the next stage; 2 = three channels in one group; 3 = the last k of the first 8192-k staging chunk
    and the last k of the matrix; 4 = one channel inside a group, one in another group."""
    g = K if gs is None else gs
    c = {0: [0],
         1: [g - 1, min(K - 1, 128 if g > 128 else g)],
         2: [min(g - 1, 5), min(g - 1, 77), min(g - 1, 126)],
         3: [min(K, 8192) - 1, K - 1],
         4: [g // 3, min(K - 1, g + g // 2 + 1)]}[variant]
    return sorted(set(c))


X_KINDS = ("gauss", "outlier64", "outlier1000", "silu", "zeros", "const", "big", "subnormal")


def gen_x(kind, M, K, seed=0, channels=(0,), gs=None):
    """Seeded fp16 activations [M, K] for the quantisation edges:
    gauss: standard normal;  outlier64 / outlier1000: standard normal with `channels` at +-64 / +-1000 (signs alternate by row);
    silu: silu(g) * u with g ~ N(1, 1.5), u ~ N(0.3, 1) (sign-biased, as the input of down_proj);  zeros: row 0 all zero (M > 1) and,
    in the last row, an all-zero group (the group of k = 0 when gs is None: the first 128 k);  const: every row constant (its own
    value), so every x_q is +-Q and quantisation is exact;  big: N(0, 100) with absmax 60000 (pair it with weights scaled down so
    the output stays finite);  subnormal: random fp16 subnormals."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((M, K))
    if kind.startswith("outlier"):
        mag = float(kind[len("outlier"):])
        for m in range(M):
            for j, c in enumerate(channels):
                x[m, c] = mag * (1 if (m + j) % 2 == 0 else -1)
    elif kind == "silu":
        g = 1 + 1.5 * x
        x = g / (1 + np.exp(-g)) * (0.3 + rng.standard_normal((M, K)))
    elif kind == "zeros":
        if M > 1:
            x[0] = 0
        w = 128 if gs is None else gs
        x[M - 1, :w] = 0
    elif kind == "const":
        x = np.repeat(rng.choice([-1, 1], M)[:, None] * rng.uniform(0.1, 3, (M, 1)), K, axis=1)
    elif kind == "big":
        x = 100 * x
        x[np.arange(M), rng.integers(0, K, M)] = 60000 * rng.choice([-1, 1], M)
    elif kind == "subnormal":
        x = rng.integers(-1023, 1024, (M, K)) * 2.0 ** -24
    else:
        assert kind == "gauss", kind
    return x.astype(np.float16)


def to_cuda(*arrays):
    import torch
    out = []
    for a in arrays:
        out.append(None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda())
    return out if len(out) > 1 else out[0]


# ---------------------------------------------------------------------------------------------------------------------------------
# Attention probe: a DecodeStack whose final hidden state is, up to fp16 rounding, the residual plus the attention outputs
#
# o_proj is the identity (stored zero nibble 7, nibble 9 on the diagonal and 8 elsewhere, scale 1), ln2 is zero so the MLP adds an
# exact 0, the residual is small (1e-2 N(0, 1): the rms norm makes q / k / v independent of its scale) and there is no head.  Keys
# planted in the caches then pin each head's answer: a set P of positions holding the same key bits, scoring >= PROBE_GAP above every
# other position of the head, makes the answer the mean of V over P whatever small error the kernel's q has.
# ---------------------------------------------------------------------------------------------------------------------------------

PROBE_SCORE = 40.0                # planted keys score at least this, and 30 above the head's other keys
PROBE_GAP = 25.0                  # the setup asserts every other score of a planted head is this far below its plateau
POISON_LIFT = 20.0                # the poison row scores this far above everything else


def identity_q4(n, act=False, seed=0, gs=128):
    """GPTQ tensors (qweight, qzeros, scales, g_idx) of the n x n identity in original row order: stored zero nibble 7 (z + 1 = 8),
    nibble 9 on the diagonal and 8 elsewhere, scale 1.  act: a random g_idx (make_q4 reorders the rows; the x gather undoes it)."""
    qw = np.full((n // 8, n), 0x88888888, np.uint32)
    k = np.arange(n)
    qw[k // 8, k] += (np.uint32(1) << (4 * (k % 8)).astype(np.uint32))
    qz = np.full((n // gs, n // 8), 0x77777777, np.uint32)
    return (qw.view(np.int32), qz.view(np.int32), np.ones((n // gs, n), np.float16),
            _g_idx(n, gs, act, np.random.default_rng(seed)))


def scaled_q_as_k(qweight, qzeros, scales, heads, kv_heads, gamma, hd=128):
    """k projection tensors whose output is gamma times the q projection's first query head of each KV group (q4_column_sample
    of those columns, scales x gamma, gamma a power of two): k_new = gamma q up to the GEMV's accumulation order."""
    n_rep = heads // kv_heads
    cols = (np.arange(kv_heads)[:, None] * n_rep * hd + np.arange(hd)[None]).reshape(-1)
    kw, kz, ks = q4_column_sample(qweight, qzeros, scales, cols)
    return kw, kz, (ks.astype(np.float64) * gamma).astype(np.float16)


def attn_probe_stack(shape, layers, max_seq, act=False, batch=1, seed=0, gamma=None, lora_rank=0):
    """A DecodeStack (groupsize 128, no head) turned into an attention probe: identity o_proj (its own g_idx under act-order),
    ln2 = 0.  gamma: k projection = gamma x the q projection of each KV group's first query head (scaled_q_as_k).  lora_rank:
    adapters on q and v only, so o_proj stays the identity."""
    import torch
    from exllama_b200.stack import DecodeStack, Q4Linear
    st = DecodeStack(shape, groupsize=128, act_order=act, max_seq=max_seq, layers=layers, seed=seed, with_head=False, batch=batch)
    for i, L in enumerate(st.layers):
        qw, qz, sc, g = identity_q4(shape.heads * shape.head_dim, act, seed * 31 + i)
        L.o = Q4Linear(*to_cuda(qw, qz, sc), None if g is None else torch.from_numpy(g), st.dev_index)
        L.ln2.zero_()
        if gamma is not None:
            assert not act, "gamma needs the q projection in original row order"
            kw, kz, ks = scaled_q_as_k(_np(L.q.qweight), _np(L.q.qzeros), _np(L.q.scales), shape.heads, shape.kv_heads, gamma)
            L.k = Q4Linear(*to_cuda(kw, kz, ks), None, st.dev_index)
    if lora_rank:
        st.add_lora(lora_rank, targets=("q", "v"), seed=seed)
    torch.cuda.synchronize()
    return st


def cpu_probe_stack(oracle, heads, kv, layers, max_seq, gamma=None, seed=0, batch=1):
    """What the probe helpers read of an attn_probe_stack, on the CPU (hidden heads x 128, inter 512): q / k / v / gate / up /
    down checkpoint-like, o the identity, ln2 = 0, no head, caches of `batch` sequences.  gamma: k = gamma q as in
    attn_probe_stack."""
    import torch
    from types import SimpleNamespace
    from exllama_b200.shapes import LlamaShape
    from stack_harness import sincos
    hd = 128
    hidden, inter = heads * hd, 512
    shape = LlamaShape("cpu-probe", hidden, inter, layers, heads, vocab=32000, kv_heads=kv)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    lin = lambda qw, qz, sc: SimpleNamespace(qweight=t(qw), qzeros=t(qz), scales=t(sc), g_idx=None)
    rng = np.random.default_rng(seed)
    Ls = []
    for i in range(layers):
        mk = lambda K, N, j: lin(*synth_q4_ckpt(K, N, 128, seed=seed * 100 + 10 * i + j, scale=0.2)[:3])
        L = SimpleNamespace(q=mk(hidden, hidden, 0), k=mk(hidden, kv * hd, 1), v=mk(hidden, kv * hd, 2),
                            o=lin(*identity_q4(hidden)[:3]), gate=mk(hidden, inter, 3), up=mk(hidden, inter, 4), down=mk(inter, hidden, 5),
                            ln1=t((1 + 0.05 * rng.standard_normal(hidden)).astype(np.float16)), ln2=t(np.zeros(hidden, np.float16)))
        if gamma is not None:
            L.k = lin(*scaled_q_as_k(L.q.qweight.numpy(), L.q.qzeros.numpy(), L.q.scales.numpy(), heads, kv, gamma))
        Ls.append(L)
    sin, cos = sincos(max_seq, hd)
    kc = [torch.zeros((batch, kv, max_seq, hd), dtype=torch.float16) for _ in range(layers)]
    return SimpleNamespace(shape=shape, layers=Ls, sin=t(sin), cos=t(cos), max_seq=max_seq, lora=None, lm_head=None,
                           key_cache=kc)


def probe_caches(st, seed):
    """Background caches for a probe stack: per layer [key_cache, value_cache] numpy fp16 [batch, kv_heads, max_seq, hd] of
    N(0, 0.25)."""
    rng = np.random.default_rng(seed)
    return [[(0.5 * rng.standard_normal(tuple(kc.shape))).astype(np.float16) for _ in range(2)] for kc in st.key_cache]


def dense_positions(past, r=0, n_rep=1):
    """The dense plateau of query head r of a KV group of n_rep heads: positions p < past with p mod 16 in {r, 15 - r} -- for r = 0
    the first and the last position of every 16-position chunk (16k and 16k - 1) -- and past - 1 for the head whose residues hold
    it (head 0 when none does)."""
    p = np.arange(past)
    sel = p[(p % 16 == r) | (p % 16 == 15 - r)]
    if past > 0:
        m = (past - 1) % 16
        owner = min(m, 15 - m)
        if (owner if owner < n_rep else 0) == r:
            sel = np.union1d(sel, [past - 1])
    return sel


def single_positions(past):
    """Where a lone planted key goes: 0, 15, 16, the first / a middle / the last 16-position chunk, past - 1 (those below past)."""
    nch = (past + 15) // 16
    c = [0, 15, 16, 7, 16 * (nch // 2) + 9, 16 * (nch - 1) + 3, past - 1]
    return sorted({p for p in c if 0 <= p < past})


def multi_positions(past, j, m):
    """The dense plateau of query vector j of the m = n n_rep vectors of a KV group in an n-token launch (j = t n_rep + r), each
    disjoint from the others': m <= 8, dense_positions(past, j, m) (residues {j, 15 - j}); m <= 16, the positions p < past with
    p mod 16 = j; m > 16 (at most 32), residue j mod 16 on the 16-position chunks of parity j // 16.  past - 1 goes to the vector
    whose residue (and parity) holds it, or to vector 0 when no vector's does."""
    if m <= 8:
        return dense_positions(past, j, m)
    assert m <= 32, m
    p = np.arange(past)
    own = p % 16 + (16 * (p // 16 % 2) if m > 16 else 0)
    sel = p[own == j]
    if past > 0 and own[-1] >= m and j == 0:
        sel = np.append(sel, past - 1)
    return sel


def lone_positions(past, m, off=0):
    """One planted key for each of m query vectors, at distinct positions: single_positions(past) first, then evenly spread rows
    of the context, rotated by `off`.  Entry j (None when the context has fewer rows than vectors) is vector j's plateau."""
    single = single_positions(past)
    spread = [p for p in np.unique(np.linspace(0, past - 1, 2 * m).astype(np.int64)).tolist() if p not in single] if past else []
    order = single + spread
    return [[order[(j + off) % len(order)]] if j < len(order) else None for j in range(m)]


def multi_probe_specs(st, n, past, background=False):
    """Plant specs (plant_probe) of an n-token launch at past_len, by name: "dense" (multi_positions), "lone+0" / "lone+3" (one
    key per query vector, lone_positions rotated by the offset and the layer) and "newest" (each token's first query head of a
    group answers with its own new row: a stack whose k is gamma q).  Vector j = t n_rep + r of KV group g is virtual head
    t * heads + g * n_rep + r.  background: the odd KV groups stay unplanted (one-layer plans: a second layer would carry their
    loose bound to every head)."""
    heads = st.shape.heads
    n_rep = heads // st.shape.kv_heads
    m = n * n_rep

    def vec(h):
        t, hh = divmod(h, heads)
        g, r = divmod(hh, n_rep)
        return g, t * n_rep + r, r

    def bg(g):
        return background and g % 2 == 1
    out = [("dense", lambda l, h: None if bg(vec(h)[0]) else multi_positions(past, vec(h)[1], m))]
    for off in (0, 3):
        out.append((f"lone+{off}", lambda l, h, off=off: None if bg(vec(h)[0]) else lone_positions(past, m, off + l)[vec(h)[1]]))
    out.append(("newest", lambda l, h: "new" if vec(h)[2] == 0 else None))
    return out


def newest_inputs(oracle, st, n, past, seed, margin=PROBE_GAP + 15.0):
    """Inputs x [n, hidden] (1e-2 N(0, 1)) of a one-layer k = gamma q stack for the "newest" layout: token by token, a draw is
    kept when each KV group's first query head scores its own new row at least `margin` above the new rows of the tokens before
    it.  (A q dominated by a few high-scale columns is nearly collinear with the other tokens' q, so a larger earlier q can
    outscore the token's own row.)"""
    s = st.shape
    n_rep = s.heads // s.kv_heads
    rng = np.random.default_rng(seed)
    xs = []
    for t in range(n):
        for _ in range(200):
            x = np.stack(xs + [(1e-2 * rng.standard_normal(s.hidden)).astype(np.float16)])
            _, q, k, _ = oracle_qkv(oracle, st, 0, x, past)
            q = q.reshape(t + 1, s.heads, s.head_dim)[t, ::n_rep].astype(np.float64)
            k = k.reshape(t + 1, s.kv_heads, s.head_dim).astype(np.float64)
            sc = np.einsum("gd,jgd->gj", q, k) / np.sqrt(s.head_dim)
            if (sc[:, t:] - margin >= sc[:, :t].max(1, initial=-np.inf)[:, None]).all():
                xs.append(x[t])
                break
        else:
            raise AssertionError(f"no input for token {t} lets its own row dominate")
    return np.stack(xs)


def plant_group(q, kc, vc, plants, past, s_new, rng, poison=True):
    """Plant keys for the query vectors of one KV group (numpy, in place).

    q [m, hd] the group's roped fp16 query vectors: the n_rep heads of one token, or for a launch of n tokens m = n n_rep vectors,
    vector j = t n_rep + r token t's head r; kc / vc [max_seq, hd] the group's cache rows of one sequence; plants[j] the positions
    (< past) of vector j's plateau, or None; s_new [m] or [m, n] the vectors' scores against the launch's n new rows.  The key
    of vector r is the least-norm k with q_j . k / sqrt(hd) = T_r for j = r and 0 for the other vectors of the group, T_r =
    max(PROBE_SCORE, 30 + every other score of vector r, the new rows' included), written in fp16 at every position of
    plants[r], with a random +-1 V row per position.  poison: rows past .. past + n - 1 (which the launch overwrites with its new
    rows) get a key scoring POISON_LIFT above everything for every vector and V = 100 x a signature, and the rows from past + n
    on NaN: a kernel that reads either shows it."""
    hd = q.shape[1]
    Q = q.astype(np.float64)
    G = Q @ Q.T
    s_new = np.asarray(s_new, np.float64).reshape(len(Q), -1)
    n = s_new.shape[1]
    bg = (kc[:past].astype(np.float64) @ Q.T).max(0) / np.sqrt(hd) if past > 0 else np.full(len(Q), -np.inf)
    top = np.maximum(bg, s_new.max(1))
    tmax = top.max()
    for r, P in enumerate(plants):
        if P is None or len(P) == 0:
            continue
        assert np.max(P) < past, (P, past)
        T = max(PROBE_SCORE, top[r] + 30.0)
        tmax = max(tmax, T)
        t = np.zeros(len(Q)); t[r] = T * np.sqrt(hd)
        kc[P] = (Q.T @ np.linalg.solve(G, t)).astype(np.float16)
        assert np.isfinite(kc[P]).all(), f"plateau key of head {r} at score {T:.0f} overflows fp16"
        vc[P] = rng.choice([-1.0, 1.0], (len(P), hd)).astype(np.float16)
    if poison and past < kc.shape[0]:
        t = np.full(len(Q), (tmax + POISON_LIFT) * np.sqrt(hd))
        key = (Q.T @ np.linalg.solve(G, t)).astype(np.float16)
        assert np.isfinite(key).all(), "poison key overflows fp16"
        for p in range(past, min(past + n, kc.shape[0])):
            kc[p] = key
            vc[p] = 100 * rng.choice([-1.0, 1.0], hd).astype(np.float16)
        kc[past + n:] = np.nan; vc[past + n:] = np.nan


def snap_of(caches):
    import torch
    return [(torch.from_numpy(kc), torch.from_numpy(vc)) for kc, vc in caches]


def plant_probe(oracle, st, caches, x, past, spec, seed, seq=0, poison=True):
    """Plant every layer of cache sequence `seq` of a probe stack (caches from probe_caches, modified in place) for the launch of
    x [n, hidden] (token t at position past + t), layer by layer: layer l's q depends on the layers below, so they are planted
    first.  Query heads are virtual, as the multi-token step numbers them: h = t * heads + h' is token t's query head h' (for one
    token h = h').  spec(l, h) -> positions of head h's plateau, "new" (the token's own new row, past + t, dominates: nothing to
    plant) or None (background).  Returns plants[l] = {virtual head: positions} for probe_expectation."""
    s = st.shape
    hd, heads, kvh = s.head_dim, s.heads, s.kv_heads
    n_rep = heads // kvh
    rng = np.random.default_rng(seed)
    x = np.asarray(x, np.float16).reshape(-1, s.hidden)
    n = x.shape[0]
    out = []
    for l in range(len(st.layers)):
        xl = x
        if l > 0:
            xl = oracle_decode_step(oracle, st, snap_of(caches), x, past, seq, n_layers=l)[0]
        _, q, k, _ = oracle_qkv(oracle, st, l, xl, past)
        q = q.reshape(n, heads, hd); k = k.reshape(n, kvh, hd)
        pl = {}
        for g in range(kvh):
            qg = q[:, g * n_rep:(g + 1) * n_rep].reshape(n * n_rep, hd)
            q64 = qg.astype(np.float64)
            s_new = np.stack([q64 @ k[t, g].astype(np.float64) for t in range(n)], 1) / np.sqrt(hd)
            ps = []
            for j in range(n * n_rep):
                t, r = divmod(j, n_rep)
                hv = t * heads + g * n_rep + r
                P = spec(l, hv)
                if isinstance(P, str):
                    assert P == "new"
                    pl[hv] = np.array([past + t])
                    P = None
                elif P is not None:
                    taken = np.concatenate([np.zeros(0, np.int64)] + [p for p in ps if p is not None])
                    P = np.setdiff1d(np.asarray(P, np.int64), taken)          # a position serves one vector of the group
                    if len(P):
                        pl[hv] = P
                    else:
                        P = None
                ps.append(P)
            plant_group(qg, caches[l][0][seq, g], caches[l][1][seq, g], ps, past, s_new, rng, poison)
        out.append(pl)
    return out


def _rope_err(v, e, sin_row, cos_row):
    """Bound on |kernel - oracle| after rope (l' = hfma(l, cos, hmul(r, -sin)), both in fp16) of rows v [n, hd] whose pre-rope
    values differ by at most e [n, hd]: the propagated difference plus one fp16 rounding difference (2^-10 relative) for each
    of the two operations."""
    hd = v.shape[1]
    c = np.abs(cos_row.astype(np.float64)); sn = np.abs(sin_row.astype(np.float64))
    partner = np.r_[np.arange(hd // 2, hd), np.arange(hd // 2)]
    v64 = np.abs(v.astype(np.float64))
    lin = c * e + sn * e[:, partner]
    return 1.01 * (lin + 2.0 ** -10 * (sn * (v64[:, partner] + e[:, partner]) + v64 + lin)) + 2 * FP16_TINY


def probe_expectation(oracle, st, snap, x, past, plants, kind, seq=0, o_prop=False):
    """(want, bound): the oracle's final hidden state of a probe stack (oracle_decode_step on the cache snapshot) for the launch
    of x [n, hidden] (token t at position past + t) and a float64 bound B >= |kernel - want| per element: [n, hidden] each, or
    [hidden] for one token.

    Per layer and token t, with the layer input known to within bx (0 for layer 0):
      q, k, v  The GEMV error is quant_error_bound(kind) of each projection, plus the oracle's own fp16 rounding 2^-11 |ref|,
               plus the effect of a perturbed input: rms norm moves xn by at most |w| rm (bx + |x| rms(bx) / rms(x)) + 2 ulps,
               contracted with |W| (adapters: the same for x . A, a rounding of x . A, and the 16-bit x grid, contracted with
               |B|).  Rope at position past + t adds the propagated error and 2 fp16 ulps (_rope_err): Dq, Dk, Dv.
      scores   Token t reads the cached rows [0, past) and the launch's new rows j = 0 .. t (kn_j, token j's k).  A score
               q . k_p / sqrt(hd) moves by at most delta_h = max(sum_d Dq_d max_p |k_pd|, max_j sum_d Dq_d |kn_jd| + (|q_d| +
               Dq_d) Dk_jd) / sqrt(hd) (cached rows hold the same bits in kernel and oracle), plus 2^-20 of sum_d |q_d| max_p
               |k_pd| / sqrt(hd) for the fp32 dot product and scale.
      softmax  Scores within delta of the oracle's move every weight by a factor in [e^-2delta, e^2delta], so the output moves by
               at most (e^{2 delta} - 1) max|V| (and never more than 2 max|V|: both are averages of the same rows).  A planted
               head (plants[l][h] = P, h the virtual head t * heads + h') whose P scores at least gap above every other position
               has its answer within 2 n e^{-(gap - 2 delta)} max|V| of the mean of V over P in both kernel and oracle (n = past
               + t + 1 positions): that bound is used instead, and the setup asserts gap >= PROBE_GAP.  At past = 0 token 0's
               own row is the only one and has weight 1.  Add the largest Dv of the new rows 0 .. t times the most weight they
               can have (1, or n e^{-(gap - 2 delta)} when they are off the plateau), and (past / 16 + 64) 2^-23 max|V| for fp32
               accumulation along a chain of at most past / 16 + 64 additions and the exponential approximations (the causal
               tail adds at most 4 to the chain).
      o_proj   Two fp16 roundings of the attention output, then the identity o GEMV's x quantisation: quant_error_bound(kind)
               of the identity at an upper bound of |attention| (segments: group and 128-k stage, so a head under plain order).
               o_prop: o_proj is any matrix (no adapter): the attention bound goes through |W_o| instead of unchanged, and the
               quantisation term is the same bound for that matrix.
      x_out    bx + the attention bound + the o bound + two fp16 roundings of the residual sum; the MLP adds an exact 0.
    The fp16 roundings are taken relative (2^-11 |value|) with FP16_TINY for the subnormal range."""
    s = st.shape
    hd, heads, kvh = s.head_dim, s.heads, s.kv_heads
    n_rep = heads // kvh
    sin = st.sin.view(-1, hd).cpu().numpy(); cos = st.cos.view(-1, hd).cpu().numpy()
    x = np.asarray(x, np.float16).reshape(-1, s.hidden)
    n = x.shape[0]
    want, _, rows = oracle_decode_step(oracle, st, snap, x, past, seq)
    xs = [x] + [oracle_decode_step(oracle, st, snap, x, past, seq, n_layers=l)[0] for l in range(1, len(st.layers))] + [want]
    bx = np.zeros((n, s.hidden))
    sq = np.sqrt(hd)
    for l, L in enumerate(st.layers):
        xn, q, k, v = oracle_qkv(oracle, st, l, xs[l], past)
        q, k = q.reshape(n, heads, hd), k.reshape(n, kvh, hd)
        xn64 = xn.astype(np.float64)
        dxn = None
        if bx.any():
            w = np.abs(_np(L.ln1).astype(np.float64))
            dxn = np.empty((n, s.hidden))
            for t in range(n):
                xl = xs[l][t].astype(np.float64)
                r = np.sqrt(np.mean(xl * xl) + s.eps)
                dxn[t] = 1.01 * (w / r * (bx[t] + np.abs(xl) * (np.sqrt(np.mean(bx[t] * bx[t])) / r + 2.0 ** -9)) +
                                 2.0 ** -9 * np.abs(xn64[t]))

        def proj_err(name):
            lin = getattr(L, name)
            xm = None if lin.g_idx is None else oracle.make_x_map(lin.g_idx.numpy(), lin.qzeros.shape[0])
            qw, qz, sc = _np(lin.qweight), _np(lin.qzeros), _np(lin.scales)
            B, ref = quant_error_bound(oracle, xn, qw, qz, sc, xm, kind)
            e = B + 2.0 ** -11 * np.abs(ref) + FP16_TINY
            if dxn is not None:
                W = np.abs(oracle.dequant_f64(qw, qz, sc))
                e = e + 1.01 * np.stack([(d if xm is None else d[np.asarray(xm, np.int64)]) @ W for d in dxn])
            ab = adapter_of(st, l, name)
            if ab is not None:
                A, Bm = (np.abs(_np(t).astype(np.float64)) for t in ab)
                for t in range(n):
                    ex = 2.0 ** -9 * np.abs(xn64[t]) + np.abs(xn64[t]).max() / QUANT_Q["step"] + (0 if dxn is None else dxn[t])
                    t16 = np.abs(oracle.half_matmul_f64(xn[t:t + 1], _np(ab[0])))
                    e[t] = e[t] + 1.01 * ((ex @ A + 2.0 ** -10 * t16[0]) @ Bm) + 2.0 ** -10 * (t16[0] @ Bm)
            return e
        eq, ek, ev = proj_err("q"), proj_err("k"), proj_err("v")
        dq = [_rope_err(q[t], eq[t].reshape(heads, hd), sin[past + t], cos[past + t]) for t in range(n)]
        dk = [_rope_err(k[t], ek[t].reshape(kvh, hd), sin[past + t], cos[past + t]) for t in range(n)]
        dv = [ev[t].reshape(kvh, hd) for t in range(n)]
        kc = _np(snap[l][0][seq]).copy(); vc = _np(snap[l][1][seq]).copy()
        kc[:, past:past + n] = rows[l][0].reshape(kvh, n, hd); vc[:, past:past + n] = rows[l][1].reshape(kvh, n, hd)
        attn = causal_attn(oracle, st, q, kc, vc, past)
        battn = np.empty((n, s.hidden))
        for t in range(n):
            npos = past + t + 1
            K = kc[:, :npos].astype(np.float64); V = vc[:, :npos].astype(np.float64)
            q64 = q[t].astype(np.float64)
            bh = np.zeros(heads)
            for h in range(heads):
                g = h // n_rep
                kmax = np.abs(K[g]).max(0)
                kold = np.abs(K[g, :past]).max(0) if past > 0 else np.zeros(hd)
                dnew = [dq[t][h] @ np.abs(K[g, past + j]) + (np.abs(q64[h]) + dq[t][h]) @ dk[j][g] for j in range(t + 1)]
                delta = max([dq[t][h] @ kold] + dnew) / sq
                delta = delta * (1 + 2.0 ** -10) + 2.0 ** -20 * (np.abs(q64[h]) @ kmax) / sq
                dvn = max(dv[j][g].max() for j in range(t + 1))
                vmax = np.abs(V[g]).max() + dvn
                P = plants[l].get(t * heads + h) if plants is not None else None
                if P is not None:
                    sc_h = K[g] @ q64[h] / sq
                    inP = np.zeros(npos, bool); inP[P] = True
                    assert len(set(sc_h[inP].tolist())) == 1 or P.tolist() == [past + t], f"layer {l} token {t} head {h}: planted keys differ"
                    gap = sc_h[inP].min() - sc_h[~inP].max() if (~inP).any() else np.inf
                    assert gap >= PROBE_GAP, f"layer {l} token {t} head {h}: plateau only {gap:.2f} above the other scores"
                    w_off = min(1.0, npos * np.exp(min(50.0, 2 * delta - gap))) if np.isfinite(gap) else 0.0
                    b = 2 * w_off * vmax + dvn * (1.0 if inP[past:].any() else w_off)
                elif past == 0 and t == 0:
                    b = dvn                                       # one row: weight 1 whatever the scores
                else:
                    b = min(2.0, np.expm1(min(50.0, 2 * delta))) * vmax + dvn
                bh[h] = b + (past / 16 + 64) * 2.0 ** -23 * vmax
            battn[t] = (bh[:, None] + 2.0 ** -10 * np.abs(attn[t]) + 2 * FP16_TINY).reshape(-1)
        attn = attn.reshape(n, -1)
        lin = L.o
        xm = None if lin.g_idx is None else oracle.make_x_map(lin.g_idx.numpy(), lin.qzeros.shape[0])
        amax = ((np.abs(attn) + battn) * (1 + 2.0 ** -9)).astype(np.float16)
        Bo, _ = quant_error_bound(oracle, amax, _np(lin.qweight), _np(lin.qzeros), _np(lin.scales), xm, kind)
        if o_prop:
            assert adapter_of(st, l, "o") is None, "o_prop carries no adapter on o"
            Wo = np.abs(oracle.dequant_f64(_np(lin.qweight), _np(lin.qzeros), _np(lin.scales)))
            battn = np.stack([(b if xm is None else b[np.asarray(xm, np.int64)]) @ Wo for b in battn])
        bx = bx + battn + Bo + 2.0 ** -10 * np.abs(xs[l + 1].astype(np.float64)) + 2 * FP16_TINY
    return (want.reshape(-1), bx[0]) if n == 1 else (want, bx)


class RefLib:
    """oracle/_ref/libexllama_ref.so: the reference's own kernels compiled for sm_90a (oracle/gen_golden_ref_gpu.py and tools only;
    the tests read what it computed from tests/golden/ref_gpu.npz)."""

    def __init__(self):
        from oracle import oracle as O
        path = O.ref_cuda_lib_path()
        if path is None:
            raise FileNotFoundError("oracle/_ref/libexllama_ref.so not built")
        self.lib = C.CDLL(path)
        self.lib.ref_make_q4.restype = C.c_void_p
        self.lib.ref_make_q4.argtypes = [C.c_void_p] * 4 + [C.c_int] * 4
        self.lib.ref_q4_matmul.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        self.lib.ref_reconstruct.argtypes = [C.c_void_p, C.c_void_p]
        self.lib.ref_q4_get_x_map.argtypes = [C.c_void_p, C.c_void_p]
        self.lib.ref_prepare_buffers.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        self.lib.ref_rms_norm.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_int, C.c_int, C.c_int]
        self.lib.ref_rope.argtypes = [C.c_void_p] * 3 + [C.c_int] * 5
        self.lib.ref_column_remap.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        self.lib.ref_half_matmul_cublas.argtypes = [C.c_void_p] * 3 + [C.c_int] * 4
        self.lib.ref_q4_attn.argtypes = ([C.c_void_p, C.c_void_p, C.c_float] + [C.c_void_p] * 8 + [C.c_int] * 7 +
                                         [C.c_void_p, C.c_void_p, C.c_int, C.c_int])
        self.lib.ref_q4_attn_2.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        self.lib.ref_q4_mlp.argtypes = [C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
        self.keep = []

    def prepare_buffers(self, inter, max_rows=2048, dq_numel=0):
        import torch
        ts = torch.zeros((max_rows, inter), dtype=torch.float16, device="cuda")
        tm = torch.zeros((4, inter), dtype=torch.float16, device="cuda")
        tz = torch.zeros((1, 65536), dtype=torch.float32, device="cuda")
        dq = torch.zeros((1, max(dq_numel, 8)), dtype=torch.float16, device="cuda")
        self.keep += [ts, tm, tz, dq]
        torch.cuda.synchronize()
        self.lib.ref_prepare_buffers(0, ts.data_ptr(), ts.numel(), tm.data_ptr(), tz.data_ptr(), dq.data_ptr(), 65536)

    def make_q4(self, qweight, qzeros, scales, g_idx_np=None):
        """qweight etc. are CUDA tensors (qweight is rewritten in place for act-order)."""
        import torch
        torch.cuda.synchronize()
        g = None
        if g_idx_np is not None:
            g = np.ascontiguousarray(g_idx_np, dtype=np.int32)
            self.keep.append(g)
        h = self.lib.ref_make_q4(qweight.data_ptr(), qzeros.data_ptr(), scales.data_ptr(),
                                 g.ctypes.data if g is not None else None,
                                 qweight.shape[0] * 8, qweight.shape[1], qzeros.shape[0], 0)
        self.keep += [qweight, qzeros, scales]
        self.lib.ref_sync()
        return h

    def q4_matmul(self, x, h, N, out=None, no_zero=False, mode=0):
        import torch
        if out is None:
            out = torch.empty((x.shape[0], N), dtype=torch.float16, device="cuda")
        torch.cuda.synchronize()
        self.lib.ref_q4_matmul(x.data_ptr(), x.shape[0], h, out.data_ptr(), int(no_zero), mode)
        self.lib.ref_sync()
        return out

    def sync(self):
        self.lib.ref_sync()


# ---------------------------------------------------------------------------------------------------------------------------------
# Phase probes: stacks whose new k / v rows, x_out - x_in or logits are ONE phase's output, bounded element by element on the
# kernel's own upstream output
#
# A stack from stack_harness.make_stack is edited in place before make_plan (the q4 handles borrow the tensors): o_proj's scales
# zeroed makes its GEMV add exactly 0 (cs * sx * val = 0); ln2 zeroed stages an all-zero x, whose absmax 0 quantises it to 0, so
# silu(0) * 0 = 0 and down adds exactly 0.  Norm weights log-uniform over [0.05, 4] with exact zeros, different for every tensor,
# make a wrong tensor or a stale row a gross error.  With a residual of 1e-2 rms the block outputs dominate x_out.
# ---------------------------------------------------------------------------------------------------------------------------------

def distinct_norm(n, seed):
    """Norm weights [n] fp16: log-uniform over [0.05, 4], n / 128 of them exactly 0 (at least two), a different draw per seed."""
    rng = np.random.default_rng(seed)
    w = np.exp(rng.uniform(np.log(0.05), np.log(4.0), n))
    w[rng.choice(n, max(2, n // 128), replace=False)] = 0
    return w.astype(np.float16)


def phase_probe_edit(st, o_off=(), mlp_off=(), seed=0):
    """Edit a DecodeStack in place (before make_plan): distinct_norm weights for ln1 / ln2 of every layer and the final norm,
    o_proj's scales zeroed in the layers o_off, ln2 zeroed in the layers mlp_off."""
    import torch
    h = st.shape.hidden
    for i, L in enumerate(st.layers):
        L.ln1.copy_(torch.from_numpy(distinct_norm(h, seed * 101 + 3 * i)))
        L.ln2.copy_(torch.from_numpy(distinct_norm(h, seed * 101 + 3 * i + 1)))
        if i in o_off:
            L.o.scales.zero_()
        if i in mlp_off:
            L.ln2.zero_()
    st.norm.copy_(torch.from_numpy(distinct_norm(h, seed * 101 + 99)))
    torch.cuda.synchronize()


def hmul(a, b):
    """fp16 x fp16 rounded to fp16 (the product is exact in float64, so this is __hmul's single rounding)."""
    return (np.asarray(a, np.float16).astype(np.float64) * np.asarray(b, np.float16).astype(np.float64)).astype(np.float16)


def norm_candidates(x, w, eps):
    """rms_norm(x, w) of x [rows, dim] fp16, as (x * rm) * w in fp16 (rms_norm.cu:118-131), for rm = the fp16 row factor
    rounded from float64 and its two fp16 neighbours: the kernel sums x^2 in fp32 in its own order and takes rsqrtf, so where the
    exact factor lies near an fp16 rounding boundary its fp16 factor may be the neighbour.  Given the factor both compute the same
    two roundings, so one of the three is the kernel's normalised x bit for bit.  Returns [rm, rm + 1 ulp, rm - 1 ulp] rows."""
    x = np.asarray(x, np.float16).reshape(-1, np.shape(x)[-1])
    x64 = x.astype(np.float64)
    rm = (1.0 / np.sqrt(np.mean(x64 * x64, axis=1) + eps)).astype(np.float16)[:, None]
    w = np.asarray(w, np.float16).reshape(1, -1)
    return [hmul(hmul(x, r), w) for r in (rm, np.nextafter(rm, np.float16(np.inf)), np.nextafter(rm, np.float16(-np.inf)))]


def step_gemv(oracle, x, lin, ab=None, dx=None):
    """(ref, err) of one GEMV of the fused step (q4 `lin`, adapter ab = (A, B) or None) on its phase input x [M, K] in the
    checkpoint's order, before the fp32 accumulator is rounded anywhere: ref = x . W + fp16(x . A) . B in float64 (t = x . A
    rounded to nearest) and err >= |accumulator - ref|.  x may be float64 (an exact value the kernel only approximates); dx >= |x'
    - x| bounds the kernel's own input x' (None: x' = x bit for bit).  With |x'| <= X = |x| + dx:

        err = (1 + 2^-10) ( sum_k A(k) / (2Q) |w_kn| + n_fp32 2^-24 sum_k X_k |w_kn| + sum_k dx_k |w_kn| )
            + sum_j |B_jn| e_j + (rank + 4) 2^-24 sum_j (|t16_j| + e_j) |B_jn|

    The first line is quant_error_bound without its final fp16 rounding (A(k) the absmax of X over k's window, 4 more fp32
    roundings for the adapter's atomics into the accumulator) plus the input's own error through |W|.  The adapter: the kernel's
    fp32 t' = x' . A is within dt = (K + 8) 2^-24 (X . |A|) + dx . |A| of t, and its fp16(t') within e = dt + 2^-10 (|t| + dt) +
    2^-24 of fp16(t) (each rounded to nearest, so less than one ulp apart whichever way t' falls); the B sum is a chain of rank
    fp32 fmas and an atomic add."""
    x64 = np.asarray(x, np.float64)
    x64 = x64.reshape(-1, x64.shape[-1])
    M, K = x64.shape
    dx = np.zeros_like(x64) if dx is None else np.broadcast_to(np.asarray(dx, np.float64), x64.shape)
    qw, qz, sc = _np(lin.qweight), _np(lin.qzeros), _np(lin.scales)
    xm = None if lin.g_idx is None else np.asarray(oracle.make_x_map(lin.g_idx.numpy(), qz.shape[0]), np.int64)
    g = slice(None) if xm is None else xm
    W = oracle.dequant_f64(qw, qz, sc)
    aw = np.abs(W)
    ref = x64[:, g] @ W
    X = np.abs(x64) + dx
    Xg = X[:, g]
    win = quant_windows(K, qz.shape[0])
    starts = np.flatnonzero(np.r_[True, win[1:] != win[:-1]])
    A = np.maximum.reduceat(Xg, starts, axis=1)[:, win]
    n_fp32 = 5 * (win[-1] + 1 + -(-K // STAGE_K)) + QUANT_C + 4
    err = (1 + 2.0 ** -10) * ((A / (2.0 * QUANT_Q["step"])) @ aw + n_fp32 * 2.0 ** -24 * (Xg @ aw) + dx[:, g] @ aw)
    del W, aw
    if ab is not None:
        Am, Bm = (_np(t).astype(np.float64) for t in ab)
        t = x64 @ Am
        t16 = t.astype(np.float16).astype(np.float64)
        ref = ref + t16 @ Bm
        dt = (K + 8) * 2.0 ** -24 * (X @ np.abs(Am)) + dx @ np.abs(Am)
        e = dt + 2.0 ** -10 * (np.abs(t) + dt) + FP16_TINY
        err = err + e @ np.abs(Bm) + (Am.shape[1] + 4) * 2.0 ** -24 * ((np.abs(t16) + e) @ np.abs(Bm))
    return ref, err


def rounded_bound(ref, err, base=None):
    """Bound on |fp16(base + acc) - (base + ref)| for an fp32 accumulator acc within err of ref (base: the fp16 residual the
    accumulator is added to, or None): the error itself and one fp16 rounding of a value no larger than |base + ref| + err."""
    v = np.abs(ref if base is None else np.asarray(base, np.float64) + ref)
    return (1 + 2.0 ** -11) * err + 2.0 ** -11 * v + FP16_TINY


def qkv_expectation(oracle, st, l, x, past):
    """Layer l's new k and v rows on its fp16 layer input x [hidden] at position `past`: per norm candidate (norm_candidates of
    ln1), ((k want [kv_heads, hd], k bound), (v want, v bound)).  v = fp16(accumulator): step_gemv's error and its rounding
    (rounded_bound).  k: the kernel rounds its accumulator and ropes it in fp16 (hfma(l, cos, hmul(r, -sin))); want is the oracle's
    rope of fp16(ref), and the pre-rope rows differ by at most the v-style bound plus the oracle's own rounding of ref, which
    _rope_err carries through rope."""
    s = st.shape
    hd, kvh = s.head_dim, s.kv_heads
    L = st.layers[l]
    sin = st.sin.view(-1, hd).cpu().numpy(); cos = st.cos.view(-1, hd).cpu().numpy()
    out = []
    for xn in norm_candidates(x, _np(L.ln1), s.eps):
        kr, ke = step_gemv(oracle, xn, L.k, adapter_of(st, l, "k"))
        vr, ve = step_gemv(oracle, xn, L.v, adapter_of(st, l, "v"))
        k16 = kr.astype(np.float16)
        kw = oracle.rope(k16.reshape(1, kvh, hd), sin, cos, 1, kvh, hd, kvh, past).reshape(kvh, hd)
        ek = (rounded_bound(kr, ke) + 2.0 ** -11 * np.abs(kr) + FP16_TINY).reshape(kvh, hd)
        kb = _rope_err(kw, ek, sin[past], cos[past])
        out.append(((kw.astype(np.float64), kb), (vr.reshape(kvh, hd), rounded_bound(vr, ve).reshape(kvh, hd))))
    return out


# silu_h (decode_step.cu) = hmul(x, hrcp(hadd(1, hexp(-x)))); hexp and hrcp are an fp32 approximation rounded to fp16 (cuda_fp16.hpp),
# so each lands within one fp16 ulp (2^-10 relative) of the exact value, and hadd / hmul round to nearest (2^-11): silu_h(x) is
# within 2^-10 + 2^-11 + 2^-10 + 2^-11 (+ second order) = SILU_REL of silu(x), for every fp16 x above -11.  Below -11, exp(-x)
# overflows fp16 and silu_h gives 0 where |silu(x)| <= 11 e^-11 < SILU_FLOOR.
SILU_REL = 3.1 * 2.0 ** -10
SILU_FLOOR = 2e-4


def silu64(g):
    g = np.asarray(g, np.float64)
    return g / (1.0 + np.exp(-g))


def mlp_expectation(oracle, st, l, x):
    """The MLP of layer l on its fp16 input x [hidden] (o_proj off, so x is also the residual): per norm candidate of ln2,
    (want, bound) of x_out = fp16(x + down(act)), act = silu(gate) * up in float64 on the exact projections.

    gate / up: the kernel's fp16 values are within Bg / Bu (rounded_bound of step_gemv) of the exact g / u.  silu moves by at most
    1.1 Bg (|silu'| <= 1.1), and silu_h adds SILU_REL of its value (SILU_FLOOR where g may lie below -11): ds.  The product
    rounds once more: |act' - act| <= (|s| + ds) Bu + |u| ds + 2^-11 (|act| + that).  down: step_gemv on act with that dx, then
    the residual add's rounding."""
    s = st.shape
    L = st.layers[l]
    out = []
    for xn in norm_candidates(x, _np(L.ln2), s.eps):
        gr, ge = step_gemv(oracle, xn, L.gate, adapter_of(st, l, "gate"))
        ur, ue = step_gemv(oracle, xn, L.up, adapter_of(st, l, "up"))
        bg, bu = rounded_bound(gr, ge), rounded_bound(ur, ue)
        sr = silu64(gr)
        ds = 1.1 * bg + SILU_REL * (np.abs(sr) + 1.1 * bg) + np.where(gr - bg < -11.0, SILU_FLOOR, 0.0) + 2 * FP16_TINY
        act = sr * ur
        da = (np.abs(sr) + ds) * bu + np.abs(ur) * ds
        da = da + 2.0 ** -11 * (np.abs(act) + da) + FP16_TINY
        dr, de = step_gemv(oracle, act, L.down, adapter_of(st, l, "down"), dx=da)
        x64 = np.asarray(x, np.float16).astype(np.float64).reshape(1, -1)
        out.append(((x64 + dr).reshape(-1), rounded_bound(dr, de, x64).reshape(-1)))
    return out


def o_expectation_ctx0(oracle, st, l, x, v_new):
    """o_proj of layer l at context 0 on its fp16 residual x [hidden] (MLP off): the attention over one row gives that row weight
    exactly 1, so every query head's output is its KV group's new v row v_new [kv_heads, hd] bit for bit (the kernel's own, read
    from the cache).  (want, bound) of x_out = fp16(x + o(attn)): step_gemv on that exact input, and the residual's rounding."""
    s = st.shape
    n_rep = s.heads // s.kv_heads
    attn = np.repeat(np.asarray(v_new, np.float16).reshape(s.kv_heads, 1, s.head_dim), n_rep, axis=1).reshape(1, -1)
    r, e = step_gemv(oracle, attn, st.layers[l].o, adapter_of(st, l, "o"))
    x64 = np.asarray(x, np.float16).astype(np.float64).reshape(1, -1)
    return (x64 + r).reshape(-1), rounded_bound(r, e, x64).reshape(-1)


def head_expectation(x_out, norm, lm_head, eps):
    """Logits of the HEAD phase on the kernel's own final hidden state x_out [hidden]: per norm candidate (norm_candidates of the
    final norm), (want, bound) with want = h . lm_head^T in float64 on the fp16 normalised h.  The products of two fp16 values
    are exact in fp32, so the only error is fp32 summation (decode_step.cu, HEAD): a lane's fhfma2 chain over at most 2 chunks of
    512 (32 fmas), 5 shuffle adds, and one atomic add per warp partial of the row (at most H / 1024 + 2 of them), each rounding
    a partial sum no larger than sum_k |h_k w_k|: bound = n 2^-24 (1 + 2^-18) sum_k |h_k w_k|, n = 32 + 5 + H / 1024 + 2."""
    x_out = np.asarray(x_out, np.float16).reshape(1, -1)
    H = x_out.shape[1]
    lm_head = np.asarray(lm_head, np.float16)
    n = 32 + 5 + H // 1024 + 2
    h = np.concatenate(norm_candidates(x_out, norm, eps)).astype(np.float64).T          # [H, 3]
    want, s = np.empty((lm_head.shape[0], 3)), np.empty((lm_head.shape[0], 3))
    for r in range(0, lm_head.shape[0], 2048):                                           # float64 in row blocks: 70B widths stay small
        W = lm_head[r:r + 2048].astype(np.float64)
        want[r:r + 2048] = W @ h
        s[r:r + 2048] = np.abs(W) @ np.abs(h)
    return [(want[:, c], n * 2.0 ** -24 * (1 + 2.0 ** -18) * s[:, c] + 1e-30) for c in range(3)]


def assert_within_any(got, cands, what=""):
    """got within the bound of at least one candidate: cands is a list of (want, bound), or -- several outputs checked together,
    got a tuple of them -- a list of tuples of (want, bound).  Returns the largest err / bound of the best candidate."""
    if not isinstance(got, tuple):
        got, cands = (got,), [(c,) for c in cands]
    best, msg = np.inf, ""
    for c in cands:
        ratios = []
        for gv, (want, bound) in zip(got, c):
            gv = np.asarray(gv, np.float64).reshape(np.shape(want))
            assert np.isfinite(gv).all(), f"{what}: non-finite output"
            ratios.append(np.abs(gv - want) / bound)
        j = int(np.argmax([r.max() for r in ratios]))
        if ratios[j].max() < best:
            best, r, (want, bound) = float(ratios[j].max()), ratios[j], c[j]
            i = np.unravel_index(np.argmax(r), r.shape)
            msg = (f"output {j}: {(r > 1).sum()} / {r.size} outside; worst at {i}: err / bound {r[i]:.3g} (bound {bound[i]:.3g}, "
                   f"want {want[i]:.4g}; rms bound / rms want {np.sqrt(np.mean(bound ** 2) / max(np.mean(want ** 2), 1e-300)):.2e})")
    assert best <= 1.0, f"{what}: no norm candidate fits: {msg}"
    return best
