"""ctypes/numpy front-end of the CPU oracle (oracle/gptq_oracle.c) and of the
reference-compiled libraries under oracle/_ref/.

TEST INFRASTRUCTURE ONLY: importable from tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs.  The product package
(exllama_b200/) never imports this module.

All fp16 tensors are numpy float16 arrays (or uint16 bit views); packed GPTQ
tensors are int32/uint32 arrays laid out as the reference expects
(exllama_ext/exllama_ext.cpp:166-176):
    qweight [K/8, N] int32, qzeros [G, N/8] int32, scales [G, N] fp16, g_idx [K] int32.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_REF_CPU = None

_vp = C.c_void_p
_i = C.c_int
_f = C.c_float


def build(force: bool = False) -> None:
    """Compile liboracle.so, and oracle/_ref/* when EXLLAMA_REFERENCE names a checkout of the reference."""
    so = os.path.join(_HERE, "liboracle.so")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(os.path.join(_HERE, "gptq_oracle.c")):
        subprocess.check_call(["make", "-C", _HERE, os.path.join(_HERE, "liboracle.so")], stdout=subprocess.DEVNULL)
    ref = os.environ.get("EXLLAMA_REFERENCE")
    if ref and os.path.isdir(os.path.join(ref, "exllama_ext")):
        subprocess.check_call(["make", "-C", _HERE, "ref", "REF=" + ref], stdout=subprocess.DEVNULL)


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(so):
            build()
        _LIB = C.CDLL(so)
        _LIB.orc_h2f.restype = C.c_float
        _LIB.orc_h2f.argtypes = [C.c_uint16]
        _LIB.orc_f2h.restype = C.c_uint16
        _LIB.orc_f2h.argtypes = [C.c_float]
        _LIB.orc_d2h.restype = C.c_uint16
        _LIB.orc_d2h.argtypes = [C.c_double]
        _LIB.orc_num_threads.restype = C.c_int
    return _LIB


def ref_cpu_lib():
    """The reference's own rep_penalty.cpp compiled into oracle/_ref/ (None if absent)."""
    global _REF_CPU
    if _REF_CPU is None:
        so = os.path.join(_HERE, "_ref", "librep_penalty_ref.so")
        if not os.path.exists(so):
            return None
        _REF_CPU = C.CDLL(so)
    return _REF_CPU


def ref_cuda_lib_path():
    so = os.path.join(_HERE, "_ref", "libexllama_ref.so")
    return so if os.path.exists(so) else None


def _p(a: np.ndarray | None):
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"], "oracle needs contiguous arrays"
    return a.ctypes.data_as(_vp)


def _h(a: np.ndarray) -> np.ndarray:
    """fp16 array -> contiguous uint16 bit view."""
    a = np.ascontiguousarray(a)
    assert a.dtype == np.float16
    return a.view(np.uint16)


def _u32(a: np.ndarray) -> np.ndarray:
    a = np.ascontiguousarray(a)
    assert a.dtype in (np.int32, np.uint32)
    return a.view(np.uint32)


# ---------------------------------------------------------------------------
# act-order
# ---------------------------------------------------------------------------

def make_x_map(g_idx: np.ndarray, groups: int) -> np.ndarray:
    g = _u32(g_idx)
    out = np.empty(g.shape[0], dtype=np.uint32)
    lib().orc_make_x_map(_p(g), _i(g.shape[0]), _i(groups), _p(out))
    return out


def make_sequential(qweight: np.ndarray, x_map: np.ndarray) -> np.ndarray:
    qw = _u32(qweight)
    out = np.empty_like(qw)
    lib().orc_make_sequential(_p(qw), _p(out), _p(_u32(x_map)), _i(qw.shape[0] * 8), _i(qw.shape[1]))
    return out.view(qweight.dtype)


def column_remap(x: np.ndarray, x_map: np.ndarray) -> np.ndarray:
    xb = _h(x)
    out = np.empty_like(xb)
    lib().orc_column_remap(_p(xb), _p(out), _i(x.shape[0]), _i(x.shape[1]), _p(_u32(x_map)))
    return out.view(np.float16)


# ---------------------------------------------------------------------------
# dequant / matmul
# ---------------------------------------------------------------------------

def reconstruct_f16(qweight, qzeros, scales) -> np.ndarray:
    qw, qz, sc = _u32(qweight), _u32(qzeros), _h(scales)
    K, N, G = qw.shape[0] * 8, qw.shape[1], qz.shape[0]
    out = np.empty((K, N), dtype=np.uint16)
    lib().orc_reconstruct_f16(_p(qw), _p(qz), _p(sc), _i(K), _i(N), _i(G), _p(out))
    return out.view(np.float16)


def dequant_f64(qweight, qzeros, scales) -> np.ndarray:
    qw, qz, sc = _u32(qweight), _u32(qzeros), _h(scales)
    K, N, G = qw.shape[0] * 8, qw.shape[1], qz.shape[0]
    out = np.empty((K, N), dtype=np.float64)
    lib().orc_dequant_f64(_p(qw), _p(qz), _p(sc), _i(K), _i(N), _i(G), _p(out))
    return out


def dequant_numpy(qweight, qzeros, scales) -> np.ndarray:
    """Independent pure-numpy restatement of W = scale * (q - (z + 1)) (q4_matrix.cu:196-208)."""
    qw, qz = _u32(qweight), _u32(qzeros)
    K8, N = qw.shape
    G = qz.shape[0]
    shifts = (np.arange(8, dtype=np.uint32) * 4)
    q = ((qw[:, None, :] >> shifts[None, :, None]) & 0xF).reshape(K8 * 8, N).astype(np.int64)
    z = ((qz[:, :, None] >> shifts[None, None, :]) & 0xF).reshape(G, N).astype(np.int64) + 1
    gs = (K8 * 8) // G
    grp = np.arange(K8 * 8) // gs
    return scales.astype(np.float64)[grp] * (q - z[grp]).astype(np.float64)


def q4_matmul_f64(x, qweight, qzeros, scales, x_map=None, acc_in=None, recons=False) -> np.ndarray:
    """Exact float64 contraction (ref64).  recons=True contracts against the fp16-rounded
    reconstructed weights (prefill flavour)."""
    qw, qz, sc, xb = _u32(qweight), _u32(qzeros), _h(scales), _h(x)
    M, K = x.shape
    N, G = qw.shape[1], qz.shape[0]
    assert qw.shape[0] * 8 == K
    out = np.empty((M, N), dtype=np.float64)
    fn = lib().orc_q4_matmul_recons_f64 if recons else lib().orc_q4_matmul_f64
    fn(_p(xb), _i(M), _i(K), _i(N), _p(qw), _p(qz), _p(sc), _i(G),
       _p(_u32(x_map)) if x_map is not None else None,
       _p(_h(acc_in)) if acc_in is not None else None, _p(out))
    return out


def q4_matmul_cpu_f32(x, qweight, qzeros, scales, x_map=None) -> np.ndarray:
    """The timed CPU baseline ("port"): dequant + fp32 GEMV on all host threads."""
    qw, qz, sc, xb = _u32(qweight), _u32(qzeros), _h(scales), _h(x)
    M, K = x.shape
    N, G = qw.shape[1], qz.shape[0]
    out = np.empty((M, N), dtype=np.uint16)
    lib().orc_q4_matmul_cpu_f32(_p(xb), _i(M), _i(K), _i(N), _p(qw), _p(qz), _p(sc), _i(G),
                                _p(_u32(x_map)) if x_map is not None else None, _p(out))
    return out.view(np.float16)


def num_threads() -> int:
    return int(lib().orc_num_threads())


def set_num_threads(n: int) -> None:
    lib().orc_set_num_threads(_i(int(n)))


def half_matmul_f64(x, w, acc_in=None) -> np.ndarray:
    M, K = x.shape
    N = w.shape[1]
    out = np.empty((M, N), dtype=np.float64)
    lib().orc_half_matmul_f64(_p(_h(x)), _p(_h(w)), _i(M), _i(K), _i(N),
                              _p(_h(acc_in)) if acc_in is not None else None, _p(out))
    return out


# ---------------------------------------------------------------------------
# small fused ops
# ---------------------------------------------------------------------------

def rms_norm(x, w, eps: float):
    xb = _h(x)
    rows, dim = x.shape
    out = np.empty_like(xb)
    rm = np.empty(rows, dtype=np.uint16)
    lib().orc_rms_norm(_p(xb), _p(_h(w)), _p(out), _f(eps), _i(rows), _i(dim), _p(rm))
    return out.view(np.float16), rm.view(np.float16)


def rope(x, sin, cos, bsz, rows_per_batch, head_dim, num_heads, past_len) -> np.ndarray:
    xb = _h(x).copy()
    lib().orc_rope(_p(xb), _p(_h(sin)), _p(_h(cos)), _i(bsz), _i(rows_per_batch), _i(head_dim),
                   _i(num_heads), _i(past_len))
    return xb.view(np.float16).reshape(x.shape)


def silu_mul(x, y) -> np.ndarray:
    xb = _h(x).copy()
    lib().orc_silu_mul(_p(xb), _p(_h(y)), _i(x.size))
    return xb.view(np.float16).reshape(x.shape)


def update_cache(key, value, key_cache, value_cache, head_dim, kvh, q_len, max_seq, past_len):
    kc, vc = _h(key_cache).copy(), _h(value_cache).copy()
    lib().orc_update_cache(_p(_h(key)), _p(_h(value)), _p(kc), _p(vc), _i(head_dim), _i(kvh), _i(q_len),
                           _i(max_seq), _i(past_len))
    return kc.view(np.float16).reshape(key_cache.shape), vc.view(np.float16).reshape(value_cache.shape)


def decode_attn_f64(q, key_cache, value_cache, heads, kv_heads, head_dim, seq, max_seq, fp16_steps=False) -> np.ndarray:
    """model.py:372-409 for one token; q [heads*hd] fp16, caches [kv_heads, max_seq, hd] fp16 -> float64 [heads*hd]."""
    out = np.zeros(heads * head_dim, dtype=np.float64)
    lib().orc_decode_attn(_p(_h(q)), _p(_h(key_cache)), _p(_h(value_cache)), _p(out), _i(heads), _i(kv_heads), _i(head_dim),
                          _i(seq), _i(max_seq), _i(1 if fp16_steps else 0))
    return out


def rep_penalty(vocab_size, sequence, penalty_max, sustain, decay, use_ref=False) -> np.ndarray:
    seq = np.ascontiguousarray(sequence, dtype=np.int64).reshape(-1).view(np.uint64)
    mask = np.empty(vocab_size, dtype=np.float32)
    if use_ref:
        ref_cpu_lib().ref_rep_penalty(_i(vocab_size), _p(seq), _p(mask), _f(penalty_max), _i(sustain), _i(decay),
                                      _i(seq.shape[0]))
    else:
        lib().orc_rep_penalty(_i(vocab_size), _p(seq), _p(mask), _f(penalty_max), _i(sustain), _i(decay),
                              _i(seq.shape[0]))
    return mask


def apply_rep_penalty(sequence, penalty_max, sustain, decay, logits, use_ref=False) -> np.ndarray:
    seq = np.ascontiguousarray(sequence, dtype=np.int64).view(np.uint64)
    lg = np.ascontiguousarray(logits, dtype=np.float32).copy()
    bsz, vocab = lg.shape
    seq = seq.reshape(bsz, -1)
    fn = ref_cpu_lib().ref_apply_rep_penalty if use_ref else lib().orc_apply_rep_penalty
    for b in range(bsz):
        fn(_i(vocab), _p(np.ascontiguousarray(seq[b])), _f(penalty_max), _i(sustain), _i(decay),
           _i(seq.shape[1]), C.c_void_p(lg[b].ctypes.data))
    return lg


# ---------------------------------------------------------------------------
# synthetic GPTQ tensors (SURVEY.md section 8d)
# ---------------------------------------------------------------------------

def synth_q4(K: int, N: int, groupsize: int, act_order: bool = False, seed: int = 0):
    """Seeded synthetic GPTQ tensor set: uniform nibbles, scales in [0.002, 0.02)."""
    rng = np.random.default_rng(seed)
    G = K // groupsize
    qweight = rng.integers(0, 2**32, size=(K // 8, N), dtype=np.uint32).view(np.int32)
    qzeros = rng.integers(0, 2**32, size=(G, N // 8), dtype=np.uint32).view(np.int32)
    scales = (rng.random((G, N), dtype=np.float32) * 0.018 + 0.002).astype(np.float16)
    g_idx = None
    if act_order:
        perm = rng.permutation(K)
        g_idx = np.empty(K, dtype=np.int32)
        g_idx[perm] = (np.arange(K) // groupsize).astype(np.int32)
    return qweight, qzeros, scales, g_idx


def synth_x(M: int, K: int, seed: int = 1) -> np.ndarray:
    rng = np.random.default_rng(seed)
    return rng.standard_normal((M, K), dtype=np.float32).astype(np.float16)


def ref64_with_act_order(x, qweight, qzeros, scales, g_idx, acc_in=None, recons=False):
    """ref64 of the full make_q4 + q4_matmul pipeline for an act-order tensor: the oracle's own
    make_x_map/make_sequential followed by the contraction with the x gather."""
    G = qzeros.shape[0]
    if g_idx is None:
        return q4_matmul_f64(x, qweight, qzeros, scales, None, acc_in, recons)
    x_map = make_x_map(g_idx, G)
    qseq = make_sequential(qweight, x_map)
    return q4_matmul_f64(x, qseq, qzeros, scales, x_map, acc_in, recons)
