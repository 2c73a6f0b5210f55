"""float64 oracles of prefill over an existing KV cache (test infrastructure, shared by test_prefill_attn_oracle.py and
test_gpu_prefill_attn.py).

prefill_attn_f64 composes oracle.decode_attn_f64 -- pinned to the reference's single-query program by
tests/golden/decode_attn_torch.npz -- over the rows of a chunk: token t of the chunk is one decode query at context
past_len + t + 1.  oracle_prefill restates DecodeStack.prefill of one sequence at any past_len with prefill's rounding points."""
import numpy as np

from helpers import adapter_of, oracle_mm


def prefill_attn_f64(oracle, q, key_cache, value_cache, heads, kv_heads, past_len, max_seq, head_dim=128):
    """q [q_len, heads, hd] fp16, caches [kv_heads, max_seq, hd] fp16 (rows [past_len, past_len + q_len) hold the chunk) ->
    float64 [q_len, heads, hd]."""
    q_len = q.shape[0]
    out = np.empty((q_len, heads, head_dim), dtype=np.float64)
    kc, vc = np.ascontiguousarray(key_cache), np.ascontiguousarray(value_cache)
    for t in range(q_len):
        qt = np.ascontiguousarray(q[t].reshape(-1))
        out[t] = oracle.decode_attn_f64(qt, kc, vc, heads, kv_heads, head_dim, past_len + t + 1, max_seq).reshape(heads, head_dim)
    return out


def _np(t):
    return t.cpu().numpy()


def _add16(a, b):
    return (a.astype(np.float64) + b.astype(np.float64)).astype(np.float16)


def oracle_prefill(oracle, st, caches, x, past_len, seq, M):
    """float64/fp16 restatement of DecodeStack.prefill of one sequence x [T, hidden] fp16 at past_len into cache sequence seq.

    caches: per layer (key_cache, value_cache) tensors AFTER the prefill (attention reads rows [0, past_len + t] of them, as the
    kernel does, so each layer's attention is checked on the rows the stack wrote).  M (rows of every q4 call, bsz * T) picks the
    GEMM route: fp16-rounded weights above 48 rows (wgmma), exact products at or below (skinny).  Returns (logits [T, vocab]
    float64, per layer (k, v) new cache rows [kv_heads, T, hd] fp16)."""
    s = st.shape
    hd, H, KV = s.head_dim, s.heads, s.kv_heads
    T = x.shape[0]
    sin = _np(st.sin).reshape(-1, hd); cos = _np(st.cos).reshape(-1, hd)
    mm = lambda xin, i, n: oracle_mm(oracle, xin, getattr(st.layers[i], n), adapter_of(st, i, n), recons=M > 48).astype(np.float16)
    rows = []
    for i, L in enumerate(st.layers):
        xn, _ = oracle.rms_norm(x, _np(L.ln1), s.eps)
        q, k, v = (mm(xn, i, n) for n in ("q", "k", "v"))
        q = oracle.rope(q.reshape(1, T * H, hd), sin, cos, 1, T * H, hd, H, past_len).reshape(T, H, hd)
        k = oracle.rope(k.reshape(1, T * KV, hd), sin, cos, 1, T * KV, hd, KV, past_len).reshape(T, KV, hd)
        v = v.reshape(T, KV, hd)
        rows.append((k.transpose(1, 0, 2), v.transpose(1, 0, 2)))
        kc, vc = _np(caches[i][0][seq]), _np(caches[i][1][seq])
        attn = prefill_attn_f64(oracle, q, kc, vc, H, KV, past_len, st.max_seq, hd).astype(np.float16).reshape(T, H * hd)
        x = _add16(x, mm(attn, i, "o"))
        xn, _ = oracle.rms_norm(x, _np(L.ln2), s.eps)
        g, u = mm(xn, i, "gate"), mm(xn, i, "up")
        g64 = g.astype(np.float64)
        act = (g64 / (1.0 + np.exp(-g64))).astype(np.float16)               # torch's fp16 silu: one rounding
        act = (act.astype(np.float64) * u.astype(np.float64)).astype(np.float16)
        x = _add16(x, mm(act, i, "down"))
    hn, _ = oracle.rms_norm(x, _np(st.norm), s.eps)
    return hn.astype(np.float64) @ _np(st.lm_head).astype(np.float64).T, rows
