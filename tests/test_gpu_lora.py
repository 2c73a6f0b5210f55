"""LoRA adapters: the per-op entry points (q4_attn, q4_attn_2, q4_mlp with lora tensors) and the persistent decode step
(exl_decode_plan_create_lora).

The per-op kernels are pinned to the float64 oracle composed with the reference's rounding points (fp16(x . A), fp16(. B), then
+= x . W).  The fused step is checked against the same oracle composition for the whole token, and against the per-op path, with the
tolerances of tests/test_gpu_decode_step.py (the fused step skips the second rounding, fp16(t . B): well inside them).  Every case also
checks that the adapter matters: the logits move by at least 20x the logit tolerance against a plan without the adapter.  Test
adapters are strong (alpha = 8 r: the LoRA term is about twice a projection's own output) and the input state small, so that an
adapter on q and v shows in the logits even when the softmax over a long synthetic context is flat.
"""
import numpy as np
import pytest

from helpers import assert_close_ref64, oracle_decode_step, oracle_mm

pytestmark = pytest.mark.gpu

PROJ = ("q", "k", "v", "o", "gate", "up", "down")
TARGETS = {"qv": ("q", "v"), "all": PROJ}
X_SCALE = 0.05


def _mk_stack(hidden=1024, inter=2816, layers=2, heads=8, kv_heads=8, gs=128, max_seq=256, batch=1, vocab=2048, seed=3, act=False):
    import torch
    from exllama_b200.stack import DecodeStack, LlamaShape
    shape = LlamaShape("synthetic-lora", hidden, inter, layers, heads, vocab=vocab, kv_heads=kv_heads)
    st = DecodeStack(shape, groupsize=gs, act_order=act, device="cuda:0", max_seq=max_seq, seed=seed, batch=batch)
    g = torch.Generator(device="cuda"); g.manual_seed(seed + 100)
    for kc, vc in zip(st.key_cache, st.value_cache):
        kc.copy_((torch.randn(kc.shape, device="cuda", generator=g) * 0.5).half())
        vc.copy_((torch.randn(vc.shape, device="cuda", generator=g) * 0.5).half())
    return st


def _add(st, rank, targets, layers=None, seed=1):
    return st.add_lora(rank, targets=TARGETS[targets], layers=layers, alpha=8 * rank, seed=seed)


def _snap(st):
    return [(kc.clone(), vc.clone()) for kc, vc in zip(st.key_cache, st.value_cache)]


def _restore(st, snap):
    for (kc, vc), (k0, v0) in zip(zip(st.key_cache, st.value_cache), snap):
        kc.copy_(k0); vc.copy_(v0)


def _np(t):
    return t.cpu().numpy()


def _per_op(st, snap, xs, pasts):
    logits, rows = [], []
    for b, past in enumerate(pasts):
        logits.append(st.decode_step(xs[b:b + 1].clone(), past, seq=b).clone())
        rows.append([(kc[b, :, past].clone(), vc[b, :, past].clone()) for kc, vc in zip(st.key_cache, st.value_cache)])
    _restore(st, snap)
    return logits, rows


def _plain_logits(st, snap, xs, pasts):
    """The same stack's plan without the adapter: its logits [bsz, vocab] (caches restored)."""
    from exllama_b200 import capi
    saved, plan, xo, lg = st.lora, st.dplan, st._plan_xout, st._plan_logits
    st.lora = None
    st.make_plan()
    out = st.decode_step_fused_batch(xs, pasts).clone() if st.batch > 1 else st.decode_step_fused(xs[:1], pasts[0]).clone().view(1, -1)
    st.dplan.close()
    st.lora, st.dplan, st._plan_xout, st._plan_logits = saved, plan, xo, lg
    _restore(st, snap)
    assert isinstance(plan, capi.DecodePlan)
    return out


def _assert_adapter_matters(got, plain, what, rel=1.5e-2):
    """max |logits - logits without the adapter| >= 20 x the logit tolerance's rms term."""
    got = np.asarray(got, np.float64); plain = np.asarray(plain, np.float64)
    tol = rel * np.sqrt(np.mean(got * got))
    d = np.abs(got - plain).max()
    assert d >= 20 * tol, f"{what}: the adapter moves the logits by {d:.4g}, less than 20 x {tol:.4g}"


def _check_step(oracle, st, xs, pasts, what):
    """Fused step with the stack's adapter vs the oracle and the per-op path, for every sequence; the new K/V rows; adapter matters."""
    import torch
    bsz = len(pasts)
    snap = _snap(st)
    ref_logits, ref_rows = _per_op(st, snap, xs, pasts)
    plain = _plain_logits(st, snap, xs, pasts)
    logits = (st.decode_step_fused_batch(xs, pasts) if st.batch > 1 else st.decode_step_fused(xs[:1], pasts[0]).view(1, -1)).cpu().numpy()
    torch.cuda.synchronize()
    got_x = st._plan_xout.view(-1, st.shape.hidden)[:bsz].cpu().numpy()
    for b in range(bsz):
        want_x, want_logits, rows = oracle_decode_step(oracle, st, snap, _np(xs[b]), pasts[b], b)
        w = f"{what} seq {b} (ctx {pasts[b]})"
        assert_close_ref64(got_x[b], want_x.reshape(-1).astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} final hidden vs oracle")
        assert_close_ref64(logits[b], want_logits.reshape(-1), rel=1.5e-2, rms=1.5e-2, what=f"{w} logits vs oracle")
        assert_close_ref64(logits[b], _np(ref_logits[b]).reshape(-1).astype(np.float64), rel=1.5e-2, rms=1.5e-2, what=f"{w} logits vs per-op")
        for i, (kc, vc) in enumerate(zip(st.key_cache, st.value_cache)):
            k_new, v_new = _np(kc[b, :, pasts[b]]), _np(vc[b, :, pasts[b]])
            assert_close_ref64(k_new, rows[i][0].astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} layer {i} new k vs oracle")
            assert_close_ref64(v_new, rows[i][1].astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} layer {i} new v vs oracle")
            assert_close_ref64(k_new, _np(ref_rows[b][i][0]).astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} layer {i} new k vs per-op")
            assert_close_ref64(v_new, _np(ref_rows[b][i][1]).astype(np.float64), rel=1e-2, rms=1e-2, what=f"{w} layer {i} new v vs per-op")
        _assert_adapter_matters(logits[b], _np(plain[b]), w)
    _restore(st, snap)


def _xs(bsz, hidden, seed):
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    return (torch.randn((bsz, 1, hidden), device="cuda", generator=g) * X_SCALE).half()


# ---- per-op entry points with LoRA tensors (no reference-kernel goldens exist for them: the oracle is the pin) ----------------------
@pytest.mark.parametrize("kv", [8, 2])
@pytest.mark.parametrize("act", [False, True])
@pytest.mark.parametrize("rank", [8, 32])
def test_per_op_blocks_vs_oracle(oracle, rank, act, kv):
    import torch
    from exllama_b200 import cuda_ext
    ext = cuda_ext.exllama_ext
    st = _mk_stack(layers=1, kv_heads=kv, max_seq=64, act=act, seed=40 + rank + kv)
    _add(st, rank, "all", seed=rank)
    s, L, past = st.shape, st.layers[0], 9
    hd, heads = s.head_dim, s.heads
    x = (torch.randn((1, 1, s.hidden), device="cuda") * 0.5).half()
    x0 = _np(x).reshape(1, -1).copy()
    kc0, vc0 = _np(st.key_cache[0][0]).copy(), _np(st.value_cache[0][0]).copy()
    q = torch.empty((1, 1, heads * hd), dtype=torch.float16, device="cuda")
    k = torch.empty((1, 1, kv * hd), dtype=torch.float16, device="cuda"); v = torch.empty_like(k)
    ab = lambda n: st.lora[0][n]
    lt = st._lora_temp(0, PROJ, 1)
    ext.q4_attn(x, L.ln1, s.eps, q, k, v, L.q.q4, L.k.q4, L.v.q4, st.sin, st.cos, 1, past, heads, kv, hd, st.key_cache[0], st.value_cache[0],
                st.max_seq, *ab("q"), *ab("k"), *ab("v"), lt)
    sin = st.sin.view(-1, hd).cpu().numpy(); cos = st.cos.view(-1, hd).cpu().numpy()
    xn, _ = oracle.rms_norm(x0, _np(L.ln1), s.eps)
    wq, wk, wv = (oracle_mm(oracle, xn, getattr(L, n), ab(n)).astype(np.float16) for n in ("q", "k", "v"))
    wq = oracle.rope(wq.reshape(1, heads, hd), sin, cos, 1, heads, hd, heads, past).reshape(-1)
    wk = oracle.rope(wk.reshape(1, kv, hd), sin, cos, 1, kv, hd, kv, past).reshape(-1)
    tol = dict(rel=6e-3, rms=6e-3)
    assert_close_ref64(_np(q).reshape(-1), wq.astype(np.float64), what="q4_attn q", **tol)
    assert_close_ref64(_np(k).reshape(-1), wk.astype(np.float64), what="q4_attn k", **tol)
    assert_close_ref64(_np(v).reshape(-1), wv.reshape(-1).astype(np.float64), what="q4_attn v", **tol)
    assert_close_ref64(_np(st.key_cache[0][0, :, past]).reshape(-1), wk.astype(np.float64), what="k cache row", **tol)
    kc0[:, past] = _np(st.key_cache[0][0, :, past]); vc0[:, past] = _np(st.value_cache[0][0, :, past])
    assert np.array_equal(_np(st.key_cache[0][0]), kc0) and np.array_equal(_np(st.value_cache[0][0]), vc0)
    # q4_attn_2: x += (attn . A) . B + attn . W
    attn = (torch.randn((1, heads * hd), device="cuda") * 0.5).half()
    x2 = x.view(1, -1).clone()
    ext.q4_attn_2(x2, attn, L.o.q4, *ab("o"), lt)
    want = oracle_mm(oracle, _np(attn), L.o, ab("o"), acc=x0)
    assert_close_ref64(_np(x2), want, what="q4_attn_2", **tol)
    # q4_mlp: x += down(silu(gate(n)) * up(n)), every projection with its adapter
    x3 = x.view(1, -1).clone()
    ext.q4_mlp(x3, L.ln2, s.eps, L.gate.q4, L.up.q4, L.down.q4, *ab("gate"), *ab("up"), *ab("down"), lt)
    xn, _ = oracle.rms_norm(x0, _np(L.ln2), s.eps)
    a = oracle.silu_mul(oracle_mm(oracle, xn, L.gate, ab("gate")).astype(np.float16), oracle_mm(oracle, xn, L.up, ab("up")).astype(np.float16))
    want = oracle_mm(oracle, a, L.down, ab("down"), acc=x0)
    assert_close_ref64(_np(x3), want, what="q4_mlp", **tol)
    st.close()


# ---- the fused step --------------------------------------------------------------------------------------------------------------
# (kv heads, groupsize, rank, targets, past_len, act-order, adapted layers)
CASES = [
    (8, 128, 8, "qv", 0, False, None), (8, 128, 16, "all", 1, False, None), (2, 32, 64, "all", 16, False, None),
    (2, 128, 128, "qv", 37, False, None), (8, 32, 128, "all", 200, False, None), (2, 128, 16, "qv", 200, False, None),
    (8, 128, 16, "all", 37, True, None), (8, 32, 64, "qv", 200, True, None), (2, 128, 32, "all", 16, True, None),
    (2, 32, 8, "all", 1, True, None), (8, 128, 16, "all", 37, False, [0]), (2, 128, 64, "qv", 0, False, [0]),
]


@pytest.mark.parametrize("kv,gs,rank,targets,past,act,layers", CASES)
def test_fused_step_vs_oracle_and_per_op(oracle, kv, gs, rank, targets, past, act, layers):
    st = _mk_stack(kv_heads=kv, gs=gs, act=act, seed=3 + kv + gs + rank)
    _add(st, rank, targets, layers=layers, seed=rank + past)
    st.make_plan()
    info = st.dplan.info()
    n_ad = len(layers) if layers is not None else 2
    assert info["barriers_per_step"] == 1 + (5 + int(act)) * 2 + n_ad * (1 if targets == "qv" else 4), info      # q, v: both in the QKV phase
    _check_step(oracle, st, _xs(1, 1024, past + rank), [past], f"kv {kv} g{gs} r{rank} {targets} act {act} layers {layers}")
    st.dplan.close(); st.close()


@pytest.mark.parametrize("kv,bsz,rank,targets", [(8, 2, 16, "all"), (2, 3, 64, "qv"), (2, 4, 128, "all"), (8, 4, 8, "qv")])
def test_batched_fused_step(oracle, kv, bsz, rank, targets):
    """Batch 2-4 at ragged contexts, the same adapter for every sequence."""
    st = _mk_stack(kv_heads=kv, batch=4, seed=50 + bsz + kv)
    _add(st, rank, targets, seed=bsz)
    st.make_plan()
    _check_step(oracle, st, _xs(bsz, 1024, 7 * bsz), [0, 200, 16, 37][:bsz], f"batch {bsz} kv {kv} r{rank} {targets}")
    st.dplan.close(); st.close()


def test_sequence_and_graph(oracle):
    """Five consecutive tokens of four sequences, then CUDA-graph replay of the last launch."""
    import torch
    st = _mk_stack(layers=3, kv_heads=2, max_seq=128, batch=4, seed=5)
    _add(st, 16, "all")
    st.make_plan()
    xs = [_xs(4, 1024, 9 + t) for t in range(5)]
    starts = [40, 3, 90, 17]
    snap = _snap(st)
    ref = [[st.decode_step(x[b:b + 1].clone(), starts[b] + t, seq=b).clone() for b in range(4)] for t, x in enumerate(xs)]
    _restore(st, snap)
    got = [st.decode_step_fused_batch(x, [p + t for p in starts]).clone() for t, x in enumerate(xs)]
    torch.cuda.synchronize()
    for t in range(5):
        for b in range(4):
            assert_close_ref64(_np(got[t][b]), _np(ref[t][b]).reshape(-1).astype(np.float64), rel=2e-2, rms=2e-2, what=f"token {t} seq {b}")
    x, last = xs[-1], [p + 4 for p in starts]
    side = torch.cuda.Stream(); side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        st.decode_step_fused_batch(x, last)
    torch.cuda.current_stream().wait_stream(side); torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        st.decode_step_fused_batch(x, last)
    for _ in range(3):
        gr.replay()
    torch.cuda.synchronize()
    # fp32 red.add order differs from launch to launch, and t is rounded to fp16 after its sum: a little more spread than without LoRA
    assert_close_ref64(_np(st._plan_logits), _np(got[-1]).astype(np.float64), rel=5e-3, rms=5e-3, what="graph replay")
    st.dplan.close(); st.close()


def test_short_context_after_a_long_one(oracle):
    """One LoRA plan: a long context (every attention partial slot written), then short ones; each matches the per-op path."""
    import torch
    from exllama_b200 import capi
    st = _mk_stack(kv_heads=8, max_seq=512, seed=7)
    _add(st, 32, "all")
    st.make_plan()
    snap = _snap(st)
    for t, past in enumerate([400, 3, 17, 0, 300, 1]):
        x = _xs(1, 1024, 21 + t)
        ref = st.decode_step(x.clone(), past).clone()
        _restore(st, snap)
        n0 = capi.launch_count()
        got = st.decode_step_fused(x, past).clone()
        torch.cuda.synchronize()
        assert capi.launch_count() - n0 in (1, 2)
        _restore(st, snap)
        assert_close_ref64(_np(got).reshape(-1), _np(ref).reshape(-1).astype(np.float64), rel=1.5e-2, rms=1.5e-2, what=f"ctx {past}")
    st.dplan.close(); st.close()


@pytest.mark.parametrize("name,bsz,ctx", [("7b", 1, 1920), ("7b", 4, 1920), ("70b", 2, 1920)])
def test_full_shapes_vs_per_op(oracle, name, bsz, ctx):
    """Llama 7B (r 16 on all seven, batch 1 and 4) and Llama-2 70B (r 16 on all seven, batch 2), 2 layers, against the per-op path."""
    import torch
    from exllama_b200.shapes import GQA_SHAPES, SHAPES
    s = {**SHAPES, **GQA_SHAPES}[name]
    st = _mk_stack(s.hidden, s.inter, 2, s.heads, s.kv_heads, 128, 2048, batch=bsz, vocab=s.vocab, seed=17)
    _add(st, 16, "all")
    st.make_plan()
    xs = _xs(bsz, s.hidden, 23)
    past = [ctx - 37 * b for b in range(bsz)]
    snap = _snap(st)
    ref, _ = _per_op(st, snap, xs, past)
    got = st.decode_step_fused_batch(xs, past) if bsz > 1 else st.decode_step_fused(xs, past[0]).view(1, -1)
    torch.cuda.synchronize()
    assert torch.isfinite(got).all()
    for b in range(bsz):
        assert_close_ref64(_np(got[b]), _np(ref[b]).reshape(-1).astype(np.float64), rel=1.5e-2, rms=1.5e-2, what=f"{name} seq {b} logits")
    st.dplan.close(); st.close()


def test_no_adapter_plan_is_the_batch_plan(oracle):
    """exl_decode_plan_create_lora with no adapter (NULL, or every rank 0) is exl_decode_plan_create_batch's plan: the same plan info
    and kernel, so the results differ only as two launches of one plan do (the order of fp32 red.add); that spread is measured here
    on the batch plan itself and the no-adapter plans must stay inside it."""
    import torch
    from exllama_b200 import capi
    st = _mk_stack(kv_heads=2, batch=2, seed=31)
    hs = [[L.q.q4, L.k.q4, L.v.q4, L.o.q4, L.gate.q4, L.up.q4, L.down.q4] for L in st.layers]
    args = (hs, [L.ln1 for L in st.layers], [L.ln2 for L in st.layers], st.key_cache, st.value_cache, st.sin, st.cos, 8, 128, st.max_seq, 1e-6)
    kw = dict(final_norm=st.norm, lm_head=st.lm_head, num_kv_heads=2, max_batch=2)
    xs = _xs(2, 1024, 3)
    snap = _snap(st)
    outs, infos = [], []
    for lora in ("batch", "batch", [None, None], [(None,) * 7, (None,) * 7]):
        plan = capi.DecodePlan(*args, **kw) if lora == "batch" else capi.DecodePlan(*args, **kw, lora=lora)
        xo = torch.empty((2, 1024), dtype=torch.float16, device="cuda")
        outs.append((plan.step_batch(xs, [37, 5], x_out=xo).clone(), xo.clone()))
        torch.cuda.synchronize()
        infos.append(plan.info())
        plan.close()
        _restore(st, snap)
    spread_x = (outs[1][1].float() - outs[0][1].float()).abs().max().item()
    for (lg, xo), info in zip(outs[2:], infos[2:]):
        assert info == infos[0]
        assert (xo.float() - outs[0][1].float()).abs().max().item() <= max(2 * spread_x, 2e-3), spread_x
        assert_close_ref64(_np(lg), _np(outs[0][0]).astype(np.float64), rel=2e-3, rms=2e-3, what="logits")
    st.close()


def test_rejected_arguments(oracle):
    """Every EXL_ERR_ARG case of exl_decode_plan_create_lora, each naming the per-op path."""
    import ctypes as C
    import torch
    from exllama_b200 import capi
    st = _mk_stack(layers=2, kv_heads=8, max_seq=64, seed=2)
    _add(st, 16, "qv")
    hs = [[L.q.q4, L.k.q4, L.v.q4, L.o.q4, L.gate.q4, L.up.q4, L.down.q4] for L in st.layers]
    args = (hs, [L.ln1 for L in st.layers], [L.ln2 for L in st.layers], st.key_cache, st.value_cache, st.sin, st.cos, 8, 128, st.max_seq, 1e-6)
    good = st._plan_lora()
    with pytest.raises(capi.ExlError, match=r"error 1: .*tensor parallelism.*per-op path"):
        capi.DecodePlan(*args, tp_rank=0, tp_world=2, lora=good)
    A, B = st.lora[0]["q"]
    for r in (12, 136):
        bad = [(( torch.zeros((1024, r), dtype=torch.float16, device="cuda"), torch.zeros((r, 1024), dtype=torch.float16, device="cuda")),) + (None,) * 6, None]
        with pytest.raises(capi.ExlError, match=r"error 1: .*rank %d.*multiples of 8 up to 128.*per-op path" % r):
            capi.DecodePlan(*args, lora=bad)
    flat = torch.zeros(1024 * 16 + 8, dtype=torch.float16, device="cuda")
    mis = flat[1:1 + 1024 * 16].view(1024, 16)                       # 2-byte aligned
    with pytest.raises(capi.ExlError, match=r"error 1: .*16-byte aligned.*per-op path"):
        capi.DecodePlan(*args, lora=[((mis, B),) + (None,) * 6, None])
    st.close()


def test_rejected_arguments_c_abi(oracle):
    """The layer-count and NULL-pointer cases straight through the C ABI (DecodePlan never builds them)."""
    import ctypes as C
    import torch
    from exllama_b200 import capi
    st = _mk_stack(layers=2, kv_heads=8, max_seq=64, seed=2)
    _add(st, 16, "qv")
    hs = [[L.q.q4, L.k.q4, L.v.q4, L.o.q4, L.gate.q4, L.up.q4, L.down.q4] for L in st.layers]
    A, B = st.lora[0]["q"]
    n = 2
    def call(n_layers, a_ptr, b_ptr, rank0):
        lo = capi._DecodeLora()
        lo.n_layers = n_layers
        pa = (capi.vp * (7 * n))(*([a_ptr] + [None] * (7 * n - 1)))
        pb = (capi.vp * (7 * n))(*([b_ptr] + [None] * (7 * n - 1)))
        rk = (capi.i32 * (7 * n))(*([rank0] + [0] * (7 * n - 1)))
        lo.a, lo.b, lo.rank = C.cast(pa, C.POINTER(capi.vp)), C.cast(pb, C.POINTER(capi.vp)), C.cast(rk, C.POINTER(capi.i32))
        d = _desc(st, hs)
        h = capi.vp()
        rc = capi.lib().exl_decode_plan_create_lora(C.byref(d[0]), 1, C.byref(lo), C.byref(h))
        msg = capi.lib().exl_last_error().decode()
        if rc == 0:
            capi.lib().exl_decode_plan_destroy(h)
        return rc, msg
    rc, msg = call(1, A.data_ptr(), B.data_ptr(), 16)
    assert rc == 1 and "adapter has 1 layers, the model 2" in msg, msg
    rc, msg = call(2, None, B.data_ptr(), 16)
    assert rc == 1 and "NULL A or B" in msg and "per-op path" in msg, msg
    rc, msg = call(2, A.data_ptr(), None, 16)
    assert rc == 1 and "NULL A or B" in msg and "per-op path" in msg, msg
    rc, msg = call(2, A.data_ptr(), B.data_ptr(), 16)
    assert rc == 0, msg
    st.close()


def _desc(st, hs):
    """exl_decode_desc of a single-sequence plan over the stack, with the arrays it points to (kept alive by the returned tuple)."""
    import ctypes as C
    from exllama_b200 import capi
    n = len(hs)
    mats = (capi.vp * (7 * n))(*[int(h) if not isinstance(h, C.c_void_p) else h.value for hs_ in hs for h in hs_])
    arr = lambda ts: (capi.vp * n)(*[t.data_ptr() for t in ts])
    keep = [arr([L.ln1 for L in st.layers]), arr([L.ln2 for L in st.layers]), arr(st.key_cache), arr(st.value_cache)]
    d = capi._DecodeDesc()
    d.n_layers, d.num_heads, d.head_dim, d.max_seq_len, d.vocab, d.rms_eps = n, st.shape.heads, 128, st.max_seq, 0, 1e-6
    d.mats = C.cast(mats, C.POINTER(capi.vp))
    d.ln1, d.ln2, d.key_cache, d.value_cache = (C.cast(x, C.POINTER(capi.vp)) for x in keep)
    d.sin, d.cos = st.sin.data_ptr(), st.cos.data_ptr()
    d.num_kv_heads = st.shape.kv_heads
    return d, mats, keep
