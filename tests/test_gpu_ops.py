"""GPU parity of the small ops and the fused decoder blocks, through the C ABI and through the pybind shim."""
import numpy as np
import pytest

from helpers import RefLib, assert_close_ref64, to_cuda, ulp_diff_f16
from stack_harness import sincos

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("rows,dim", [(1, 4096), (3, 5120), (17, 6656), (2, 100)])
def test_rms_norm(oracle, rows, dim):
    from exllama_b200 import capi
    rng = np.random.default_rng(rows + dim)
    x = rng.standard_normal((rows, dim)).astype(np.float16)
    w = (1 + 0.1 * rng.standard_normal(dim)).astype(np.float16)
    want, rm = oracle.rms_norm(x, w, 1e-6)
    got = capi.rms_norm(to_cuda(x), to_cuda(w), 1e-6).cpu().numpy()
    # fp32 summation order + rsqrtf approximation can move the fp16 row factor by one ulp -> allow 2 ulp on outputs
    assert ulp_diff_f16(got, want).max() <= 2
    assert (ulp_diff_f16(got, want) == 0).mean() > 0.5 or rows * dim < 1000
    # in-place aliasing (cuda_ext.py:148-152)
    tx = to_cuda(x.copy())
    capi.rms_norm(tx, to_cuda(w), 1e-6, out=tx)
    np.testing.assert_array_equal(tx.cpu().numpy(), got)


@pytest.mark.parametrize("bsz,q_len,heads,hd,past", [(1, 1, 32, 128, 0), (1, 1, 32, 128, 777), (2, 5, 8, 128, 3), (1, 7, 4, 64, 10)])
def test_rope_bit_exact(oracle, bsz, q_len, heads, hd, past):
    from exllama_b200 import capi
    rng = np.random.default_rng(7)
    x = rng.standard_normal((bsz, q_len, heads * hd)).astype(np.float16)
    sin, cos = sincos(2048, hd)
    want = oracle.rope(x.reshape(bsz, q_len * heads, hd), sin, cos, bsz, q_len * heads, hd, heads, past).reshape(x.shape)
    tx = to_cuda(x.copy())
    capi.rope_(tx, to_cuda(sin), to_cuda(cos), past, heads, hd)
    np.testing.assert_array_equal(tx.cpu().numpy().view(np.uint16), want.view(np.uint16))


def test_silu_mul(oracle):
    from exllama_b200 import capi
    rng = np.random.default_rng(9)
    x = (rng.standard_normal((2, 11008)) * 2).astype(np.float16)
    y = rng.standard_normal((2, 11008)).astype(np.float16)
    want = oracle.silu_mul(x, y)
    tx = to_cuda(x.copy())
    capi.silu_mul_(tx, to_cuda(y))
    got = tx.cpu().numpy()
    # hexp / hrcp are approximate on the GPU: a few fp16 ulps against the correctly rounded restatement
    d = ulp_diff_f16(got, want)
    assert d.max() <= 8 and np.mean(d <= 2) > 0.95, (d.max(), np.mean(d <= 2))


def test_update_cache_and_column_remap(oracle):
    import torch
    from exllama_b200 import capi
    rng = np.random.default_rng(5)
    kvh, hd, q_len, max_seq, past = 8, 128, 3, 64, 11
    k = rng.standard_normal((1, q_len, kvh * hd)).astype(np.float16)
    v = rng.standard_normal((1, q_len, kvh * hd)).astype(np.float16)
    kc = rng.standard_normal((1, kvh, max_seq, hd)).astype(np.float16)
    vc = rng.standard_normal((1, kvh, max_seq, hd)).astype(np.float16)
    wk, wv = oracle.update_cache(k, v, kc, vc, hd, kvh, q_len, max_seq, past)
    tkc, tvc = to_cuda(kc.copy(), vc.copy())
    capi.update_cache(to_cuda(k), to_cuda(v), tkc, tvc, hd, kvh, q_len, max_seq, past)
    np.testing.assert_array_equal(tkc.cpu().numpy(), wk)
    np.testing.assert_array_equal(tvc.cpu().numpy(), wv)
    x = rng.standard_normal((19, 512)).astype(np.float16)
    perm = rng.permutation(512).astype(np.uint32)
    got = capi.column_remap(to_cuda(x), torch.from_numpy(perm.view(np.int32)).cuda()).cpu().numpy()
    np.testing.assert_array_equal(got, x[:, perm])


def test_half_matmul(oracle):
    import torch
    from exllama_b200 import capi
    rng = np.random.default_rng(6)
    x = rng.standard_normal((5, 512)).astype(np.float16)
    w = (rng.standard_normal((512, 64)) * 0.1).astype(np.float16)
    ref = oracle.half_matmul_f64(x, w)
    assert_close_ref64(capi.half_matmul_cublas(to_cuda(x), to_cuda(w)).cpu().numpy(), ref, what="hm cublas")
    out = torch.zeros((5, 64), dtype=torch.float16, device="cuda")
    capi.half_matmul(to_cuda(x), to_cuda(w), out)
    assert_close_ref64(out.cpu().numpy(), ref, what="hm custom")
    acc = rng.standard_normal((5, 64)).astype(np.float16)
    o2 = to_cuda(acc.copy())
    capi.half_matmul_cublas(to_cuda(x), to_cuda(w), out=o2, no_zero=True)
    assert_close_ref64(o2.cpu().numpy(), oracle.half_matmul_f64(x, w, acc_in=acc), what="hm cublas acc")


# ---------------------------------------------------------------------------------------------------
# fused decoder blocks vs the unfused sequence restated with the oracle
# ---------------------------------------------------------------------------------------------------

def _layer(oracle, hidden, inter, gs, act, seed):
    names = [("q", hidden, hidden), ("k", hidden, hidden), ("v", hidden, hidden), ("o", hidden, hidden),
             ("gate", hidden, inter), ("up", hidden, inter), ("down", inter, hidden)]
    t = {}
    for i, (n, K, N) in enumerate(names):
        t[n] = oracle.synth_q4(K, N, gs, act_order=act, seed=seed + i)
    return t


def _oracle_mm(oracle, x, t):
    return oracle.ref64_with_act_order(x, *t)


@pytest.mark.parametrize("act", [False, True])
@pytest.mark.parametrize("q_len,past", [(1, 0), (1, 37), (3, 5)])
def test_q4_attn_block(oracle, act, q_len, past):
    import torch
    from exllama_b200 import capi
    hidden, heads, hd, gs, max_seq = 1024, 8, 128, 128, 64
    t = _layer(oracle, hidden, 2048, gs, act, seed=100)
    rng = np.random.default_rng(1)
    x = rng.standard_normal((1, q_len, hidden)).astype(np.float16)
    w = (1 + 0.1 * rng.standard_normal(hidden)).astype(np.float16)
    sin, cos = sincos(max_seq, hd)
    kc = np.zeros((1, heads, max_seq, hd), np.float16); vc = np.zeros_like(kc)

    # oracle sequence: norm -> q,k,v -> fp16 -> rope(q,k) -> cache (q4_attn.cu:130-165)
    xn, _ = oracle.rms_norm(x.reshape(q_len, hidden), w, 1e-6)
    q64, k64, v64 = (_oracle_mm(oracle, xn, t[n]) for n in ("q", "k", "v"))

    def mk(n):
        qw, qz, sc, g = t[n]
        tq, tz, ts = to_cuda(qw.copy(), qz, sc)
        return capi.Q4(tq, tz, ts, None if g is None else torch.from_numpy(g))
    Q, Kp, V = mk("q"), mk("k"), mk("v")
    tq = torch.empty((1, q_len, hidden), dtype=torch.float16, device="cuda"); tk = torch.empty_like(tq); tv = torch.empty_like(tq)
    tkc, tvc = to_cuda(kc.copy(), vc.copy())
    capi.q4_attn(to_cuda(x), to_cuda(w), 1e-6, tq, tk, tv, Q, Kp, V, to_cuda(sin), to_cuda(cos), q_len, past, heads, heads, hd, tkc, tvc, max_seq)
    torch.cuda.synchronize()

    # v is a plain projection
    assert_close_ref64(tv.cpu().numpy().reshape(q_len, hidden), v64, rel=3e-3, rms=3e-3, what="v")
    # q,k: apply the oracle's rope to OUR pre-rope fp16 values is not observable; instead rope the fp16-rounded ref64
    for name, got, r64 in (("q", tq, q64), ("k", tk, k64)):
        pre = r64.astype(np.float16).reshape(1, q_len * heads, hd)
        want = oracle.rope(pre, sin, cos, 1, q_len * heads, hd, heads, past).reshape(q_len, hidden).astype(np.float64)
        assert_close_ref64(got.cpu().numpy().reshape(q_len, hidden), want, rel=4e-3, rms=4e-3, what=name)
    # cache rows equal the returned k / v states, everything else untouched
    gk = tkc.cpu().numpy(); gv = tvc.cpu().numpy()
    ks = tk.cpu().numpy().reshape(q_len, heads, hd); vs = tv.cpu().numpy().reshape(q_len, heads, hd)
    for tt in range(q_len):
        np.testing.assert_array_equal(gk[0, :, past + tt], ks[tt])
        np.testing.assert_array_equal(gv[0, :, past + tt], vs[tt])
    mask = np.ones(max_seq, bool); mask[past:past + q_len] = False
    assert not gk[0][:, mask].any() and not gv[0][:, mask].any()


@pytest.mark.parametrize("act", [False, True])
@pytest.mark.parametrize("rows", [1, 2, 5])
def test_q4_mlp_and_attn2_block(oracle, act, rows):
    import torch
    from exllama_b200 import capi
    hidden, inter, gs = 1024, 2816, 128
    t = _layer(oracle, hidden, inter, gs, act, seed=200)
    rng = np.random.default_rng(2)
    x = (rng.standard_normal((rows, hidden))).astype(np.float16)
    w = (1 + 0.1 * rng.standard_normal(hidden)).astype(np.float16)

    def mk(n):
        qw, qz, sc, g = t[n]
        tq, tz, ts = to_cuda(qw.copy(), qz, sc)
        return capi.Q4(tq, tz, ts, None if g is None else torch.from_numpy(g))

    # q4_attn_2: x += attn . o_proj
    attn = rng.standard_normal((rows, hidden)).astype(np.float16)
    tx = to_cuda(x.copy())
    capi.q4_attn_2(tx, to_cuda(attn), mk("o"))
    want = oracle.ref64_with_act_order(attn, *t["o"], acc_in=x)
    assert_close_ref64(tx.cpu().numpy(), want, what="attn_2")

    # q4_mlp: x += down(silu(gate(n)) * up(n)), n = norm(x)   (q4_mlp.cu:118-197)
    xn, _ = oracle.rms_norm(x, w, 1e-6)
    g16 = _oracle_mm(oracle, xn, t["gate"]).astype(np.float16)
    u16 = _oracle_mm(oracle, xn, t["up"]).astype(np.float16)
    act16 = oracle.silu_mul(g16, u16)
    want = oracle.ref64_with_act_order(act16, *t["down"], acc_in=x)
    tx = to_cuda(x.copy())
    capi.q4_mlp(tx, to_cuda(w), 1e-6, mk("gate"), mk("up"), mk("down"))
    torch.cuda.synchronize()
    # intermediate fp16 roundings (gate/up -> fp16 -> approximate silu) differ by an ulp here and there: the
    # error budget through the down projection is a few 1e-3 of the output rms
    assert_close_ref64(tx.cpu().numpy(), want, rel=6e-3, rms=6e-3, what="mlp")


def test_pybind_surface_end_to_end(oracle):
    """The reference-facing plugin API (cuda_ext.ext_* and exllama_ext.*) on torch tensors."""
    import torch
    from exllama_b200 import cuda_ext
    K, N, gs = 1024, 512, 128
    qw, qz, sc, g_idx = oracle.synth_q4(K, N, gs, act_order=True, seed=77)
    tq, tz, ts = to_cuda(qw.copy(), qz, sc)
    h = cuda_ext.ext_make_q4(tq, tz, ts, torch.from_numpy(g_idx), 0)
    for M in (1, 4, 40):
        x = oracle.synth_x(M, K, seed=M)
        out = cuda_ext.ext_q4_matmul(to_cuda(x).view(1, M, K), h, N)
        assert out.shape == (1, M, N)
        assert_close_ref64(out.view(M, N).cpu().numpy(), oracle.ref64_with_act_order(x, qw, qz, sc, g_idx), what=f"ext_q4_matmul M={M}")
    x = oracle.synth_x(3, K)
    w = np.ones(K, np.float16)
    got = cuda_ext.ext_rms_norm(to_cuda(x), to_cuda(w), 1e-6).cpu().numpy()
    want, _ = oracle.rms_norm(x, w, 1e-6)
    assert ulp_diff_f16(got, want).max() <= 2
    with pytest.raises(RuntimeError, match="x and w have incompatible shapes"):
        cuda_ext.ext_q4_matmul(to_cuda(oracle.synth_x(1, K // 2)), h, N)
    # LoRA entry point: out = (x A) B + x W
    A = (np.random.default_rng(0).standard_normal((K, 16)) * 0.05).astype(np.float16)
    B = (np.random.default_rng(1).standard_normal((16, N)) * 0.05).astype(np.float16)
    x = oracle.synth_x(2, K, seed=9)
    out = cuda_ext.ext_q4_matmul(to_cuda(x), h, N, to_cuda(A), to_cuda(B)).cpu().numpy()
    xa = oracle.half_matmul_f64(x, A).astype(np.float16)
    lora = oracle.half_matmul_f64(xa, B).astype(np.float16)
    want = oracle.ref64_with_act_order(x, qw, qz, sc, g_idx, acc_in=lora)
    assert_close_ref64(out, want, rel=4e-3, rms=4e-3, what="lora")


# ---- decode attention over the KV cache (SURVEY.md 8f-1; model.py:372-409) --------------------------------------------------
@pytest.mark.parametrize("heads,kv_heads,seq,max_seq", [
    (32, 32, 1, 2048), (32, 32, 255, 2048), (32, 32, 257, 2048), (32, 32, 1921, 2048), (4, 4, 2048, 2048),
    (8, 2, 300, 512), (64, 8, 1000, 1024), (2, 1, 3001, 4096), (40, 40, 777, 2048),
    (8, 8, 1025, 2048), (8, 2, 1300, 2048), (32, 32, 1537, 2048), (64, 8, 1792, 2048), (8, 8, 4096, 4096)])
def test_decode_attn(oracle, heads, kv_heads, seq, max_seq):
    import torch
    from exllama_b200 import capi
    hd = 128
    rng = np.random.default_rng(heads * 7 + seq)
    q = rng.standard_normal(heads * hd).astype(np.float16)
    kc = rng.standard_normal((kv_heads, max_seq, hd)).astype(np.float16)
    vc = rng.standard_normal((kv_heads, max_seq, hd)).astype(np.float16)
    # a few dominant keys so the softmax is not flat (exercises the running-max rescale across splits / sub-blocks)
    for h in range(kv_heads):
        kc[h, rng.integers(0, seq)] *= 4
    # rows past the context are never read (a weight-0 read of a NaN row would still poison the sum)
    kc[:, seq:] = np.nan; vc[:, seq:] = np.nan
    want = oracle.decode_attn_f64(q, kc, vc, heads, kv_heads, hd, seq, max_seq)
    tq, tk, tv = to_cuda(q, kc, vc)
    got = capi.decode_attn(tq, tk, tv, heads, kv_heads, hd, seq, max_seq).cpu().numpy()
    # fp32 arithmetic, fp16 output: the final rounding (2^-11) dominates
    assert_close_ref64(got, want, rel=1.5e-3, rms=1.5e-3, what="decode_attn")
    # and it is closer to the exact answer than the reference's regular-attention branch with its fp16 rounding points
    ref16 = oracle.decode_attn_f64(q, kc, vc, heads, kv_heads, hd, seq, max_seq, fp16_steps=True)
    assert np.abs(got - want).max() <= np.abs(ref16 - want).max() + 2e-3 * np.abs(want).max()
    # against the torch ops of model.py:395-409 on the same cache (what the kernel replaces)
    rep = heads // kv_heads
    qq = tq.view(1, 1, heads, hd).transpose(1, 2)
    keys = tk[None, :, :seq].repeat_interleave(rep, dim=1)
    vals = tv[None, :, :seq].repeat_interleave(rep, dim=1)
    w = torch.matmul(qq, keys.transpose(2, 3))
    w /= np.sqrt(hd)
    w = torch.nn.functional.softmax(w, dim=-1, dtype=torch.float16)
    tref = torch.matmul(w, vals).transpose(1, 2).reshape(-1).float().cpu().numpy()
    assert np.abs(got.astype(np.float64) - tref).max() <= 4e-3 * max(1.0, np.abs(want).max())


def test_decode_attn_errors():
    from exllama_b200 import capi
    import torch
    q = torch.zeros(4 * 64, dtype=torch.float16, device="cuda")
    kc = torch.zeros((4, 16, 64), dtype=torch.float16, device="cuda")
    with pytest.raises(RuntimeError, match="head_dim"):
        capi.decode_attn(q, kc, kc, 4, 4, 64, 1, 16)
    q = torch.zeros(4 * 128, dtype=torch.float16, device="cuda")
    kc = torch.zeros((4, 16, 128), dtype=torch.float16, device="cuda")
    with pytest.raises(RuntimeError, match="seq"):
        capi.decode_attn(q, kc, kc, 4, 4, 128, 17, 16)
    with pytest.raises(RuntimeError, match="head counts"):
        capi.decode_attn(q, kc, kc, 4, 3, 128, 1, 16)
