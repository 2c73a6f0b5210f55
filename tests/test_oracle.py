"""CPU tests of the oracle itself: internal consistency (C restatement vs independent numpy restatement), the
known-answer vector from SURVEY.md 8c, the committed golden fixtures, and -- when oracle/_ref exists -- the
reference's own rep_penalty.cpp."""
import os

import numpy as np
import pytest

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_half_conversions(oracle):
    lib = oracle.lib()
    vals = np.arange(0, 65536, dtype=np.uint32).astype(np.uint16)
    f = vals.view(np.float16).astype(np.float32)
    for u in list(range(0, 65536, 97)) + [0, 1, 0x3ff, 0x400, 0x7bff, 0x8001, 0xfbff]:
        x = np.uint16(u).view(np.float16)
        if np.isnan(x):
            continue
        assert lib.orc_h2f(int(u)) == np.float32(x)
        assert lib.orc_f2h(float(np.float32(x))) == u
    rng = np.random.default_rng(0)
    d = rng.standard_normal(20000) * np.exp(rng.uniform(-20, 12, 20000))
    got = np.array([lib.orc_d2h(float(v)) for v in d], dtype=np.uint16)
    with np.errstate(over="ignore"):
        want = d.astype(np.float16).view(np.uint16)
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("K,N,gs", [(256, 64, 32), (512, 128, 128), (256, 32, 256)])
def test_dequant_matches_numpy(oracle, K, N, gs):
    qw, qz, sc, _ = oracle.synth_q4(K, N, gs, seed=K + N)
    w_c = oracle.dequant_f64(qw, qz, sc)
    w_np = oracle.dequant_numpy(qw, qz, sc)
    np.testing.assert_array_equal(w_c, w_np)
    # reconstruct_kernel: one fp16 multiply of an exact integer -> equals numpy's fp16 product
    q_minus_z = np.rint(w_np / sc.astype(np.float64).repeat(gs, 0)).astype(np.float16)
    np.testing.assert_array_equal(oracle.reconstruct_f16(qw, qz, sc), q_minus_z * sc.repeat(gs, 0))


def test_act_order_pipeline(oracle):
    K, N, gs = 512, 64, 64
    qw, qz, sc, g_idx = oracle.synth_q4(K, N, gs, act_order=True, seed=5)
    x = oracle.synth_x(3, K)
    x_map = oracle.make_x_map(g_idx, K // gs)
    assert sorted(x_map.tolist()) == list(range(K))
    assert (np.diff(g_idx[x_map]) >= 0).all()                      # rows sorted by group
    for g in range(K // gs):                                        # stable inside a group
        rows = x_map[g * gs:(g + 1) * gs]
        assert (np.diff(rows.astype(np.int64)) > 0).all()
    # direct math in the original row order
    shifts = np.arange(8, dtype=np.uint32) * 4
    q = ((qw.view(np.uint32)[:, None, :] >> shifts[None, :, None]) & 0xF).reshape(K, N).astype(np.int64)
    z = ((qz.view(np.uint32)[:, :, None] >> shifts[None, None, :]) & 0xF).reshape(K // gs, N).astype(np.int64) + 1
    W = sc.astype(np.float64)[g_idx] * (q - z[g_idx])
    want = x.astype(np.float64) @ W
    got = oracle.ref64_with_act_order(x, qw, qz, sc, g_idx)
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
    np.testing.assert_array_equal(oracle.column_remap(x, x_map), x[:, x_map])


def test_cpu_baseline_port(oracle):
    qw, qz, sc, _ = oracle.synth_q4(1024, 256, 128, seed=2)
    x = oracle.synth_x(2, 1024)
    ref = oracle.q4_matmul_f64(x, qw, qz, sc)
    got = oracle.q4_matmul_cpu_f32(x, qw, qz, sc).astype(np.float64)
    assert np.abs(got - ref).max() <= 2e-3 * np.abs(ref).max()


def test_rep_penalty_known_answer(oracle):
    # generated from the reference binary during the survey (SURVEY.md 8c)
    m = oracle.rep_penalty(16, [[5, 7, 7, 9]], 1.15, 2, 2)
    want = np.ones(16, dtype=np.float32)
    want[5], want[7], want[9] = np.float32(1.0750000477), np.float32(1.1499999762), np.float32(1.1499999762)
    np.testing.assert_array_equal(m, want)


def test_rep_penalty_golden(oracle):
    g = np.load(os.path.join(GOLD, "rep_penalty_ref.npz"))
    n = int(g["n_cases"])
    for i in range(n):
        vocab, pmax, sustain, decay = int(g[f"vocab_{i}"]), float(g[f"pmax_{i}"]), int(g[f"sustain_{i}"]), int(g[f"decay_{i}"])
        seq, logits = g[f"seq_{i}"], g[f"logits_{i}"]
        np.testing.assert_array_equal(oracle.rep_penalty(vocab, seq, pmax, sustain, decay), g[f"mask_{i}"])
        np.testing.assert_array_equal(oracle.apply_rep_penalty(seq[None], pmax, sustain, decay, logits[None])[0], g[f"applied_{i}"])


def test_rep_penalty_against_compiled_reference(oracle):
    """25 random cases against the reference's own rep_penalty.cpp (its outputs stored by oracle/gen_golden_cpu.py)."""
    g = np.load(os.path.join(GOLD, "rep_penalty_ref.npz"))
    rng = np.random.default_rng(1)
    for i in range(25):
        vocab = int(rng.integers(8, 2000)); n = int(rng.integers(1, 400))
        seq = rng.integers(0, vocab, size=n)
        pmax = float(rng.uniform(1.0, 1.5)); sustain = int(rng.integers(-1, 300)); decay = int(rng.integers(0, 300))
        np.testing.assert_array_equal(oracle.rep_penalty(vocab, seq, pmax, sustain, decay), g[f"rand_mask_{i}"])
        lg = rng.standard_normal((1, vocab)).astype(np.float32)
        np.testing.assert_array_equal(oracle.apply_rep_penalty(seq[None], pmax, sustain, decay, lg), g[f"rand_applied_{i}"])


def test_rope_rotation_property(oracle):
    """rotate-half RoPE preserves the norm of each (l, r) pair up to fp16 rounding."""
    hd, heads, T = 128, 4, 5
    rng = np.random.default_rng(3)
    x = rng.standard_normal((1, T * heads, hd)).astype(np.float16)
    inv = 1.0 / (10000 ** (np.arange(0, hd, 2) / hd))
    ang = np.outer(np.arange(64), inv)
    emb = np.concatenate([ang, ang], -1)
    sin, cos = np.sin(emb).astype(np.float16), np.cos(emb).astype(np.float16)
    y = oracle.rope(x, sin, cos, 1, T * heads, hd, heads, 7).astype(np.float64)
    xf = x.astype(np.float64)
    n0 = xf[..., :64] ** 2 + xf[..., 64:] ** 2
    n1 = y[..., :64] ** 2 + y[..., 64:] ** 2
    np.testing.assert_allclose(n1, n0, rtol=2e-2, atol=2e-3)
    # position 0 with past_len 0 is the identity (cos=1, sin=0)
    y0 = oracle.rope(x[:, :heads], sin, cos, 1, heads, hd, heads, 0)
    np.testing.assert_array_equal(y0, x[:, :heads])


def test_decode_attn_against_torch_fixture(oracle):
    """oracle.decode_attn_f64 against the reference's attention tensor program run with torch on the CPU
    (tests/golden/decode_attn_torch.npz, generated by oracle/gen_golden_attn.py)."""
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "decode_attn_torch.npz"))
    for i in range(int(g["n_cases"])):
        heads, kvh, hd, seq, max_seq = (int(v) for v in g[f"shape_{i}"])
        kc = np.zeros((kvh, max_seq, hd), np.float16); vc = np.zeros_like(kc)
        kc[:, :seq], vc[:, :seq] = g[f"kc_{i}"], g[f"vc_{i}"]
        exact = oracle.decode_attn_f64(g[f"q_{i}"], kc, vc, heads, kvh, hd, seq, max_seq)
        np.testing.assert_allclose(exact, g[f"f32_{i}"], rtol=0, atol=3e-6 * max(1.0, np.abs(exact).max()) + 2e-6)
        # the fp16 branch: same rounding points, torch accumulates its fp16 GEMMs in fp32 -> agree to an fp16 ulp or so
        r16 = oracle.decode_attn_f64(g[f"q_{i}"], kc, vc, heads, kvh, hd, seq, max_seq, fp16_steps=True)
        scale = max(1.0, np.abs(exact).max())
        assert np.abs(r16 - g[f"f16_{i}"]).max() <= 3e-3 * scale
        assert np.abs(r16 - exact).max() <= 5e-3 * scale


@pytest.mark.parametrize("K,N,gs", [(1024, 64, 128), (2048, 32, 32), (512, 96, 512)])
def test_int16_group_quantisation_of_x_error_bound(oracle, K, N, gs):
    """The decode kernel's arithmetic restated in numpy (q4_gemv.cu: x carried per quantisation group as a 16-bit integer
    with its own scale, exact integer dot products against the raw nibbles, zero point folded in as zp * sum(x_q), groups
    combined in fp32 with the fp16 scales): the claimed bound -- within 1e-4 of the output rms of the exact result for
    groupsize <= 128 -- holds on the synthetic tensors the parity tests use."""
    qw, qz, sc, _ = oracle.synth_q4(K, N, gs, seed=K + N)
    x = oracle.synth_x(3, K, seed=5)
    exact = oracle.q4_matmul_f64(x, qw, qz, sc)
    q = ((qw.view(np.uint32)[:, None, :] >> (4 * np.arange(8, dtype=np.uint32))[None, :, None]) & 15).reshape(K, N).astype(np.int64)
    z = ((qz.view(np.uint32)[:, :, None] >> (4 * np.arange(8, dtype=np.uint32))[None, None, :]) & 15).reshape(K // gs, N).astype(np.int64) + 1
    out = np.zeros((3, N), dtype=np.float32)
    for g in range(K // gs):
        xs = x[:, g * gs:(g + 1) * gs].astype(np.float32)
        mx = np.abs(xs).max(axis=1, keepdims=True)
        inv = np.where(mx > 0, np.float32(32767.0) / mx, 0).astype(np.float32)
        xq = np.rint(xs * inv).astype(np.int64)                              # |x_q| <= 32767
        dot = xq @ q[g * gs:(g + 1) * gs] - xq.sum(axis=1, keepdims=True) * z[g][None, :]       # exact integers
        assert np.abs(dot).max() < 2 ** 31
        sx = (mx * np.float32(1.0 / 32767.0)).astype(np.float32)
        out += (sc[g].astype(np.float32)[None, :] * sx) * dot.astype(np.float32)
    rms = np.sqrt(np.mean(exact ** 2))
    # below the fp16 rounding of the result (2^-11) in every case; < 1e-4 for the usual group sizes
    assert np.abs(out - exact).max() <= (1e-4 if gs <= 128 else 4e-4) * rms
