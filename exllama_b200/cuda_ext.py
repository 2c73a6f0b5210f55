"""Drop-in mirror of the reference's cuda_ext.py (cuda_ext.py:43-167).

Same public names -- `exllama_ext` (the extension module, reached by model.py as cuda_ext.exllama_ext.*),
`none_tensor`, `ext_make_q4`, `ext_q4_matmul`, `ext_half_matmul`, `ext_rope_`, `ext_rms_norm`, `ext_rms_norm_`,
`ext_rep_penalty_mask_cpu`, `ext_apply_rep_penalty_mask_cpu` -- with the same argument meaning, so the
reference's model.py / generator.py / test_benchmark_inference.py run unchanged with this module on
sys.path in place of the original (see INTEGRATION.md).

Differences from the reference shim: the extension is built ahead of time in-tree for sm_90a
(exllama_b200/_build.py) instead of JIT-compiled with no arch flags (cuda_ext.py:43-64), and it is loaded by
file path (the reference's `from exllama_ext import ...` no longer resolves under torch >= 2.11, SURVEY.md 8c).
There is no fallback: a missing extension raises ImportError.
"""
import importlib.util
import os
import sys

import torch

_here = os.path.dirname(os.path.abspath(__file__))
_ext_path = os.path.join(_here, "exllama_ext.so")

if not os.path.exists(_ext_path):
    if os.environ.get("EXL_B200_NO_BUILD"):
        raise ImportError(f"{_ext_path} not built (python -m exllama_b200._build); no CPU fallback exists")
    from . import _build
    _build.build_ext()

_spec = importlib.util.spec_from_file_location("exllama_ext", _ext_path)
exllama_ext = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(exllama_ext)
sys.modules.setdefault("exllama_ext", exllama_ext)

make_q4 = exllama_ext.make_q4
q4_matmul = exllama_ext.q4_matmul
q4_matmul_lora = exllama_ext.q4_matmul_lora
half_matmul = exllama_ext.half_matmul
half_matmul_cublas = exllama_ext.half_matmul_cublas
rms_norm = exllama_ext.rms_norm
rope_ = exllama_ext.rope_
rep_penalty = exllama_ext.rep_penalty
apply_rep_penalty = exllama_ext.apply_rep_penalty

# Dummy tensor to pass instead of None (cuda_ext.py:82)
none_tensor = torch.empty((1, 1), device="meta")


def ext_make_q4(qweight, qzeros, scales, g_idx, device):
    """Construct a Q4 matrix, return its handle (cuda_ext.py:87-93)."""
    return make_q4(qweight, qzeros, scales, g_idx if g_idx is not None else none_tensor, device)


def ext_q4_matmul(x, q4, q4_width, lora_A=None, lora_B=None):
    """x @ q4 (cuda_ext.py:98-110)."""
    outshape = x.shape[:-1] + (q4_width,)
    x = x.view(-1, x.shape[-1])
    output = torch.empty((x.shape[0], q4_width), dtype=torch.float16, device=x.device)
    if lora_A is None:
        q4_matmul(x, q4, output)
    else:
        lora_temp = torch.empty((x.shape[0], lora_A.shape[1]), dtype=torch.float16, device=x.device)
        q4_matmul_lora(x, q4, output, lora_A, lora_B, lora_temp)
    return output.view(outshape)


def ext_half_matmul(x, w, cublas=False):
    """x @ w for half tensors (cuda_ext.py:115-127)."""
    outshape = x.shape[:-1] + (w.shape[1],)
    x = x.view(-1, x.shape[-1])
    if cublas:
        output = torch.empty((x.shape[0], w.shape[1]), dtype=torch.float16, device=x.device)
        half_matmul_cublas(x, w, output)
    else:
        output = torch.zeros((x.shape[0], w.shape[1]), dtype=torch.float16, device=x.device)
        half_matmul(x, w, output)
    return output.view(outshape)


def ext_rope_(x, sin, cos, past_len, num_heads, head_dim):
    """In-place RoPE (cuda_ext.py:132-134)."""
    rope_(x, sin, cos, past_len, num_heads, head_dim)


def ext_rms_norm(x, w, epsilon):
    """x * w / sqrt(row_mean(x * x) + epsilon) (cuda_ext.py:139-146)."""
    outshape = x.shape
    x = x.view(-1, x.shape[-1])
    output = torch.empty_like(x)
    rms_norm(x, w, output, epsilon)
    return output.view(outshape)


def ext_rms_norm_(x, w, epsilon):
    """In-place variant (cuda_ext.py:148-152)."""
    x = x.view(-1, x.shape[-1])
    rms_norm(x, w, x, epsilon)


def ext_rep_penalty_mask_cpu(vocab_size, sequence, penalty_max, sustain, decay):
    """Repetition-penalty mask on the CPU (cuda_ext.py:157-161)."""
    rep_mask = torch.empty(vocab_size, dtype=torch.float32)
    rep_penalty(sequence, rep_mask, penalty_max, sustain, decay)
    return rep_mask


def ext_apply_rep_penalty_mask_cpu(sequence, penalty_max, sustain, decay, logits):
    """Apply the repetition penalty to logits in place (cuda_ext.py:164-166)."""
    apply_rep_penalty(sequence, penalty_max, sustain, decay, logits)
