"""Generates tests/golden/ref_gpu_gqa.npz: outputs of the REFERENCE's own q4_attn (oracle/_ref/libexllama_ref.so, built by build()
with EXLLAMA_REFERENCE naming the reference checkout) with grouped-query attention (kv_heads < heads), on the seeded inputs of
tests/test_gpu_gqa.py, so that that test compares exl_q4_attn with the reference without the reference being present.
The reference runs with concurrent_streams off (the shim's default), its default path (q4_attn.cu:150-165).  Only the cases with
kv_heads % 4 == 0 (test_gpu_gqa.REF_CASES): the reference's update_cache_kernel writes 4 KV heads per thread (q4_attn.cu:17,50-71)
and runs past the end of a cache with fewer.  Needs an sm_90 GPU.
    python oracle/gen_golden_ref_gpu_gqa.py [OUT.npz]
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import torch  # noqa: E402

from helpers import RefLib, to_cuda  # noqa: E402
from oracle import oracle as O  # noqa: E402
from stack_harness import sincos  # noqa: E402
import test_gpu_gqa as TG  # noqa: E402

out = {}
f16 = lambda *s: torch.zeros(s, dtype=torch.float16, device="cuda")  # noqa: E731

ref = RefLib()
ref.prepare_buffers(inter=4096, max_rows=64, dq_numel=8)
hd, max_seq = 128, TG.MAX_SEQ_OP
for heads, kv, q_len, past, act in TG.REF_CASES:
    hidden = heads * hd
    t, x, w = TG.q4_attn_inputs(O, heads, kv, q_len, act)
    hq, hk, hv = (ref.make_q4(*to_cuda(qw.copy(), qz, sc), g) for (qw, qz, sc, g) in (t["q"], t["k"], t["v"]))
    ts, tc = to_cuda(*sincos(max_seq, hd))
    tx, q, k, v = to_cuda(x), f16(1, q_len, hidden), f16(1, q_len, kv * hd), f16(1, q_len, kv * hd)
    kc, vc = f16(1, kv, max_seq, hd), f16(1, kv, max_seq, hd)
    torch.cuda.synchronize()
    ref.lib.ref_q4_attn(*[a.data_ptr() if torch.is_tensor(a) else a for a in
                          (tx, to_cuda(w), 1e-6, q, k, v, hq, hk, hv, ts, tc, 1, q_len, hidden, hd, heads, kv, past, kc, vc, max_seq, 0)])
    ref.sync()
    key = TG.q4_attn_key(heads, kv, q_len, past, act)
    for n, a in zip(("q", "k", "v", "kc", "vc"), (q, k, v, kc, vc)):
        out[f"{key}_{n}"] = a.cpu().numpy()

out["device"] = np.array(torch.cuda.get_device_name(0))
path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "ref_gpu_gqa.npz")
np.savez_compressed(path, **out)
print("wrote", path, len(out) - 1, "arrays")
