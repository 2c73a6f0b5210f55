"""CPU proof that helpers.quant_error_bound bounds the x quantisation of the two decode GEMVs, on every input generator.

Both quantisers are emulated in numpy step by step: the segments a launch forms (the quantisation group cut at the 128-k ring
stage; q4_gemv also cuts at a random cluster slice and staging chunk and splits sums by the stage parity of the two k-warps), the
fp32 x * (Q / absmax) rounded half-to-even as __float2int_rn does, the two byte planes, the exact int32 segment value of seg_flush
(checked to stay inside int32) and the fp32 folding of the segments.  The emulated error against float64 must lie within B."""
import zlib

import numpy as np
import pytest

from helpers import (QUANT_Q, X_KINDS, gen_x, outlier_channels, quant_error_bound, synth_q4_ckpt, synth_q4_saturated)

INT32_MAX = 2**31 - 1
STAGE_K = 128
f32 = np.float32


def _unpack(oracle, qw, qz, sc):
    """nibbles q [K, N], z + 1 [G, N], scales [G, N] fp32."""
    K8, N = qw.shape
    G = qz.shape[0]
    sh = np.arange(8, dtype=np.uint32) * 4
    q = ((qw.view(np.uint32)[:, None, :] >> sh[None, :, None]) & 0xF).reshape(K8 * 8, N).astype(np.int64)
    z = ((qz.view(np.uint32)[:, :, None] >> sh[None, None, :]) & 0xF).reshape(G, N).astype(np.int64) + 1
    return q, z, sc.astype(f32)


def _quantise(xs, Q):
    """One segment of one token: (x_q int64, x scale fp32) as quantise_row / the segment table compute them."""
    mx = f32(np.abs(xs.astype(f32)).max()) if xs.size else f32(0)
    inv = f32(Q) / mx if mx > 0 else f32(0)
    xq = np.rint(xs.astype(f32) * inv).astype(np.int64)
    return xq, f32(mx * f32(1.0 / Q))


def emulate_gemv(xg, q, z1, sc, M_pass, rng, chunk_stages=None, cs=None):
    """q4_gemv_kernel on the gathered x [M, K]: returns (fp16 result, largest |val| of any seg_flush)."""
    M, K = xg.shape
    G = sc.shape[0]
    gs = K // G
    spt = -(-K // STAGE_K)
    win = min(gs, STAGE_K)                               # segment: the group, cut at the ring stage
    chunk_k = min(16384 // (2 * M_pass), 31 * win)
    host_chunk = min(chunk_k // STAGE_K, spt)
    chunk_stages = chunk_stages or int(rng.integers(1, host_chunk + 1))
    cs = cs or int(rng.integers(1, min(8, spt) + 1))
    Q = QUANT_Q["gemv"]
    out = np.zeros((M, q.shape[1]), f32)
    vmax = 0
    for rank in range(cs):
        sg0, sg1 = rank * spt // cs, (rank + 1) * spt // cs
        acc = np.zeros((2, M, q.shape[1]), f32)            # the two k-warps
        for c0 in range(sg0, sg1, chunk_stages):
            c1 = min(sg1, c0 + chunk_stages)
            k_lo, k_hi = c0 * STAGE_K, min(c1 * STAGE_K, K)
            for s_lo in range(k_lo, k_hi, win):
                s_hi, g = min(k_hi, s_lo + win), s_lo // gs
                wz = q[s_lo:s_hi] - z1[g]                        # q - zp, zp = z + 1
                for m in range(M):
                    xq, sx = _quantise(xg[m, s_lo:s_hi], Q)
                    assert np.abs(xq).max(initial=0) <= Q
                    hi, lo = xq >> 8, xq & 0xFF                  # signed high byte, unsigned low byte
                    assert ((hi >= -128) & (hi <= 127)).all() and (256 * hi + lo == xq).all()
                    par = ((np.arange(s_lo, s_hi) // STAGE_K - sg0) & 1)
                    for p in (0, 1):
                        sel = par == p
                        if not sel.any():
                            continue
                        val = xq[sel] @ wz[sel]                  # 256 * ia + ib - zp * sum x_q, exact
                        vmax = max(vmax, int(np.abs(val).max()))
                        acc[p, m] = f32(sc[g] * sx) * val.astype(f32) + acc[p, m]
        out += acc[0] + acc[1]
    return out.astype(np.float16), vmax


def emulate_step(xg, q, z1, sc):
    """decode_step_kernel's GEMV on the gathered x: segments = group x 128-k stage, both x bytes signed."""
    M, K = xg.shape
    G = sc.shape[0]
    gs = K // G
    win = min(gs, STAGE_K)
    Q = QUANT_Q["step"]
    out = np.zeros((M, q.shape[1]), f32)
    for s_lo in range(0, K, win):
        s_hi = min(K, s_lo + win)
        g = s_lo // gs
        wz = q[s_lo:s_hi] - z1[g]
        for m in range(M):
            xq, sx = _quantise(xg[m, s_lo:s_hi], Q)
            a = (xq + 128) >> 8
            b = ((xq & 0xFF) ^ 0x80) - 0x80                     # sign-extended low byte
            assert ((a >= -128) & (a <= 127)).all() and (256 * a + b == xq).all()
            val = xq @ wz
            assert np.abs(val).max() <= INT32_MAX
            out[m] = f32(sc[g] * sx) * val.astype(f32) + out[m]
    return out.astype(np.float16)


def _case(oracle, kind, M, K, N, gs, act, wkind, seed):
    ch = outlier_channels(K, gs, seed % 5)
    x = gen_x(kind, M, K, seed=seed, channels=ch, gs=gs)
    if wkind == "ckpt":
        qw, qz, sc, g_idx = synth_q4_ckpt(K, N, gs, act, seed=seed, scale=1e-3 if kind == "big" else 1.0)
    else:
        qw, qz, sc, g_idx = synth_q4_saturated(K, N, gs, sign=-1 if wkind == "sat-" else 1, act=act, seed=seed,
                                               scales=np.full((1 if gs is None else K // gs, N), 1e-5) if kind == "big" else None)
    x_map = None
    if g_idx is not None:
        x_map = oracle.make_x_map(g_idx, qz.shape[0])
        qw = oracle.make_sequential(qw, x_map)
    return x, qw, qz, sc, x_map


CASES = [(kind, M, K, N, gs, act, w)
         for kind in X_KINDS
         for (M, K, N, gs, act, w) in [(1, 1024, 64, None, False, "ckpt"), (3, 1024, 64, 128, True, "ckpt"),
                                       (2, 2048, 32, 512, False, "ckpt"), (1, 640, 32, 32, False, "sat-"),
                                       (2, 1152, 32, None, True, "sat+"), (4, 1024, 32, 256, False, "ckpt")]]


@pytest.mark.parametrize("kind,M,K,N,gs,act,wkind", CASES)
def test_emulated_kernels_within_bound(oracle, kind, M, K, N, gs, act, wkind):
    seed = zlib.crc32(repr((kind, M, K, N, gs, act, wkind)).encode()) % 1000
    x, qw, qz, sc, x_map = _case(oracle, kind, M, K, N, gs, act, wkind, seed)
    q, z1, scf = _unpack(oracle, qw, qz, sc)
    xg = x if x_map is None else x[:, x_map.astype(np.int64)]
    rng = np.random.default_rng(seed)
    for kk in ("gemv", "step"):
        B, ref = quant_error_bound(oracle, x, qw, qz, sc, x_map, kind=kk)
        assert np.isfinite(ref).all() and np.abs(ref).max() < 65504, kind
        runs = [emulate_gemv(xg, q, z1, scf, M, rng)[0] for _ in range(3)] if kk == "gemv" else [emulate_step(xg, q, z1, scf)]
        for got in runs:
            err = np.abs(got.astype(np.float64) - ref)
            assert (err <= B).all(), (kk, kind, float((err / B).max()))
            if kind == "const":
                # x_q = +-Q exactly: the only error left is fp32 and the final fp16 rounding
                s = np.abs(xg.astype(np.float64)) @ np.abs(oracle.dequant_f64(qw, qz, sc))
                assert (err <= 2.0 ** -10 * np.abs(ref) + K * 2.0 ** -24 * s + 2.0 ** -24).all()


@pytest.mark.parametrize("gs", [32, 128, 256, None])
def test_bound_is_not_vacuous(oracle, gs):
    """On Gaussian x at K = 1024 the rms of B is below 2e-3 of the output rms (REL_TOL-sized): a kernel error of the size of fp16
    accumulation, or a wrong segment scale, would break it.  B is a worst-case sum, so it grows as sqrt(K) relative to the output;
    the kernels' actual error does not (it is a sum of independent roundings)."""
    K = 1024
    x = gen_x("gauss", 64, K, seed=K)
    qw, qz, sc, _ = synth_q4_ckpt(K, 256, gs, seed=gs or 1)
    for kk in ("gemv", "step"):
        B, ref = quant_error_bound(oracle, x, qw, qz, sc, kind=kk)
        r = np.sqrt(np.mean(B ** 2)) / np.sqrt(np.mean(ref ** 2))
        assert r < 2e-3, (kk, r)


@pytest.mark.parametrize("M", [1, 2, 8])
def test_int32_headroom_of_seg_flush(oracle, M):
    """Constant x and saturated weights: every x_q is Q and every q - zp is -16, so a segment's |val| = 16 Q * (its k).  A segment
    never spans a 128-k stage, so |val| <= 16 * 32767 * 128 = 67,106,816, 32x inside int32, whatever the chunk (with one group,
    a segment as long as a k-warp's share of a 8192-k chunk would have come 65,535 short of INT32_MAX)."""
    K = 16384
    x = np.ones((M, K), np.float16)
    qw, qz, sc, _ = synth_q4_saturated(K, 8, None, sign=-1)
    q, z1, scf = _unpack(oracle, qw, qz, sc)
    for chunk_stages in (31, 128):
        got, vmax = emulate_gemv(x, q, z1, scf, M, np.random.default_rng(0), chunk_stages=chunk_stages, cs=1)
        assert vmax == 16 * 32767 * STAGE_K
    want = -16.0 * K * sc.astype(np.float64)
    assert (np.abs(got.astype(np.float64) - want) <= 2.0 ** -11 * np.abs(want)).all()


def test_step_high_byte_needs_q_32639():
    """decode_step splits x_q = 256 a + b with both bytes signed, a = (x_q + 128) >> 8: Q = 32639 is the largest Q with a in s8."""
    for Q, fits in ((32639, True), (32640, False), (32767, False)):
        a = (Q + 128) >> 8
        assert (a <= 127) == fits, Q
