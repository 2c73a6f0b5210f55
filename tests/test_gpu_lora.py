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

from helpers import assert_close_ref64, oracle_mm
from stack_harness import (check_fused_step, check_reset_after_long_context, check_sequence_and_graph, lib_state,  # noqa: F401
                           fused_step, restore, snapshot, stacks)

pytestmark = pytest.mark.gpu

PROJ = ("q", "k", "v", "o", "gate", "up", "down")
TARGETS = {"qv": ("q", "v"), "all": PROJ}
X_SCALE = 0.05


def _add(st, rank, targets, layers=None, seed=1):
    return st.add_lora(rank, targets=TARGETS[targets], layers=layers, alpha=8 * rank, seed=seed)


def _np(t):
    return t.cpu().numpy()


def _plain_logits(st, snap, xs, pasts):
    """The same stack's plan without the adapter: its logits [bsz, vocab] (caches restored)."""
    from exllama_b200 import capi
    saved, plan, xo, lg = st.lora, st.dplan, st._plan_xout, st._plan_logits
    st.lora = None
    st.make_plan()
    out = fused_step(st, xs, pasts).clone()
    st.dplan.close()
    st.lora, st.dplan, st._plan_xout, st._plan_logits = saved, plan, xo, lg
    restore(st, snap)
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
    plain = _plain_logits(st, snapshot(st), xs, pasts)
    logits, _, _ = check_fused_step(oracle, st, xs, pasts, what)
    for b in range(len(pasts)):
        _assert_adapter_matters(logits[b], _np(plain[b]), f"{what} seq {b} (ctx {pasts[b]})")


def _xs(bsz, hidden, seed):
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    return (torch.randn((bsz, 1, hidden), device="cuda", generator=g) * X_SCALE).half()


# ---- per-op entry points with LoRA tensors (no reference-kernel goldens exist for them: the oracle is the pin) ----------------------
@pytest.mark.parametrize("kv", [8, 2])
@pytest.mark.parametrize("act", [False, True])
@pytest.mark.parametrize("rank", [8, 32])
def test_per_op_blocks_vs_oracle(oracle, stacks, rank, act, kv):
    import torch
    from exllama_b200 import cuda_ext
    ext = cuda_ext.exllama_ext
    st = stacks(layers=1, kv_heads=kv, max_seq=64, act=act, seed=40 + rank + kv)
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


# ---- the fused step --------------------------------------------------------------------------------------------------------------
# (kv heads, groupsize, rank, targets, past_len, act-order, adapted layers)
CASES = [
    (8, 128, 8, "qv", 0, False, None), (8, 128, 16, "all", 1, False, None), (2, 32, 64, "all", 16, False, None),
    (2, 128, 128, "qv", 37, False, None), (8, 32, 128, "all", 200, False, None), (2, 128, 16, "qv", 200, False, None),
    (8, 128, 16, "all", 37, True, None), (8, 32, 64, "qv", 200, True, None), (2, 128, 32, "all", 16, True, None),
    (2, 32, 8, "all", 1, True, None), (8, 128, 16, "all", 37, False, [0]), (2, 128, 64, "qv", 0, False, [0]),
]


@pytest.mark.parametrize("kv,gs,rank,targets,past,act,layers", CASES)
def test_fused_step_vs_oracle_and_per_op(oracle, stacks, kv, gs, rank, targets, past, act, layers):
    st = stacks(kv_heads=kv, gs=gs, act=act, seed=3 + kv + gs + rank)
    _add(st, rank, targets, layers=layers, seed=rank + past)
    st.make_plan()
    info = st.dplan.info()
    n_ad = len(layers) if layers is not None else 2
    assert info["barriers_per_step"] == 1 + (5 + int(act)) * 2 + n_ad * (1 if targets == "qv" else 4), info      # q, v: both in the QKV phase
    _check_step(oracle, st, _xs(1, 1024, past + rank), [past], f"kv {kv} g{gs} r{rank} {targets} act {act} layers {layers}")


@pytest.mark.parametrize("kv,bsz,rank,targets", [(8, 2, 16, "all"), (2, 3, 64, "qv"), (2, 4, 128, "all"), (8, 4, 8, "qv")])
def test_batched_fused_step(oracle, stacks, kv, bsz, rank, targets):
    """Batch 2-4 at ragged contexts, the same adapter for every sequence."""
    st = stacks(kv_heads=kv, batch=4, seed=50 + bsz + kv)
    _add(st, rank, targets, seed=bsz)
    st.make_plan()
    _check_step(oracle, st, _xs(bsz, 1024, 7 * bsz), [0, 200, 16, 37][:bsz], f"batch {bsz} kv {kv} r{rank} {targets}")


def test_sequence_and_graph(oracle, stacks):
    """Five consecutive tokens of four sequences, then CUDA-graph replay of the last launch."""
    st = stacks(layers=3, kv_heads=2, max_seq=128, batch=4, seed=5)
    _add(st, 16, "all")
    st.make_plan()
    # fp32 red.add order differs from launch to launch, and t is rounded to fp16 after its sum: a little more spread than without LoRA
    check_sequence_and_graph(st, [_xs(4, 1024, 9 + t) for t in range(5)], [40, 3, 90, 17], replay_tol=5e-3)


def test_short_context_after_a_long_one(oracle, stacks):
    """One LoRA plan: a long context (every attention partial slot written), then short ones; the table reset launches exactly where
    att_needs_reset says, and each context matches the per-op path."""
    st = stacks(kv_heads=8, max_seq=512, seed=7)
    _add(st, 32, "all")
    st.make_plan()
    contexts = [[400], [3], [17], [0], [300], [1]]
    check_reset_after_long_context(st, [_xs(1, 1024, 21 + t) for t in range(len(contexts))], contexts)


@pytest.mark.parametrize("name,bsz,ctx", [("7b", 1, 1920), ("7b", 4, 1920), ("70b", 2, 1920)])
def test_full_shapes_vs_per_op(oracle, stacks, name, bsz, ctx):
    """Llama 7B (r 16 on all seven, batch 1 and 4) and Llama-2 70B (r 16 on all seven, batch 2), 2 layers, against the per-op path."""
    from exllama_b200.shapes import GQA_SHAPES, SHAPES
    s = {**SHAPES, **GQA_SHAPES}[name]
    st = stacks(hidden=s.hidden, inter=s.inter, heads=s.heads, kv_heads=s.kv_heads, max_seq=2048, batch=bsz, vocab=s.vocab, seed=17)
    _add(st, 16, "all")
    st.make_plan()
    check_fused_step(None, st, _xs(bsz, s.hidden, 23), [ctx - 37 * b for b in range(bsz)], name)


def test_no_adapter_plan_is_the_batch_plan(oracle, stacks):
    """exl_decode_plan_create_lora with no adapter (NULL, or every rank 0) is exl_decode_plan_create_batch's plan: the same plan info
    and kernel, so the results differ only as two launches of one plan do (the order of fp32 red.add); that spread is measured here
    on the batch plan itself and the no-adapter plans must stay inside it."""
    import torch
    from exllama_b200 import capi
    st = stacks(kv_heads=2, batch=2, seed=31)
    hs = [[L.q.q4, L.k.q4, L.v.q4, L.o.q4, L.gate.q4, L.up.q4, L.down.q4] for L in st.layers]
    args = (hs, [L.ln1 for L in st.layers], [L.ln2 for L in st.layers], st.key_cache, st.value_cache, st.sin, st.cos, 8, 128, st.max_seq, 1e-6)
    kw = dict(final_norm=st.norm, lm_head=st.lm_head, num_kv_heads=2, max_batch=2)
    xs = _xs(2, 1024, 3)
    snap = snapshot(st)
    outs, infos = [], []
    for lora in ("batch", "batch", [None, None], [(None,) * 7, (None,) * 7]):
        plan = capi.DecodePlan(*args, **kw) if lora == "batch" else capi.DecodePlan(*args, **kw, lora=lora)
        xo = torch.empty((2, 1024), dtype=torch.float16, device="cuda")
        outs.append((plan.step_batch(xs, [37, 5], x_out=xo).clone(), xo.clone()))
        torch.cuda.synchronize()
        infos.append(plan.info())
        plan.close()
        restore(st, snap)
    spread_x = (outs[1][1].float() - outs[0][1].float()).abs().max().item()
    for (lg, xo), info in zip(outs[2:], infos[2:]):
        assert info == infos[0]
        assert (xo.float() - outs[0][1].float()).abs().max().item() <= max(2 * spread_x, 2e-3), spread_x
        assert_close_ref64(_np(lg), _np(outs[0][0]).astype(np.float64), rel=2e-3, rms=2e-3, what="logits")


def test_rejected_arguments(oracle, stacks):
    """Every EXL_ERR_ARG case of exl_decode_plan_create_lora, each naming the per-op path."""
    import ctypes as C
    import torch
    from exllama_b200 import capi
    st = stacks(layers=2, kv_heads=8, max_seq=64, seed=2)
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


def test_rejected_arguments_c_abi(oracle, stacks):
    """The layer-count and NULL-pointer cases straight through the C ABI (DecodePlan never builds them)."""
    import ctypes as C
    from exllama_b200 import capi
    st = stacks(layers=2, kv_heads=8, max_seq=64, seed=2)
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
