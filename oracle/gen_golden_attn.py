"""Generates tests/golden/decode_attn_torch.npz: the regular-attention branch of the reference
(the reference's model.py:383-409: repeat_kv, matmul, /= sqrt(head_dim), softmax, matmul, transpose) executed with
torch on the CPU, once in float32 (softmax dtype float32) and once with the reference's fp16 rounding points, on small
seeded inputs.  The statements below are the reference's tensor program restated on views of the same shapes; the
fixture pins oracle.decode_attn_f64 (both modes).  Run in the build container:  python oracle/gen_golden_attn.py"""
import math
import os

import numpy as np
import torch

rng = np.random.default_rng(20260923)
cases = [(4, 4, 128, 37, 64), (4, 2, 128, 150, 256), (2, 1, 128, 1, 16), (2, 1, 128, 260, 512)]
out = {"n_cases": len(cases)}
for i, (heads, kvh, hd, seq, max_seq) in enumerate(cases):
    q = rng.standard_normal(heads * hd).astype(np.float16)
    kc = rng.standard_normal((1, kvh, max_seq, hd)).astype(np.float16)
    vc = rng.standard_normal((1, kvh, max_seq, hd)).astype(np.float16)
    res = {}
    for mode, dt in (("f32", torch.float32), ("f16", torch.float16)):
        query = torch.from_numpy(q).to(dt).view(1, 1, heads, hd).transpose(1, 2)
        keys = torch.from_numpy(kc).to(dt).narrow(2, 0, seq)
        vals = torch.from_numpy(vc).to(dt).narrow(2, 0, seq)
        n_rep = heads // kvh
        if n_rep > 1:     # repeat_kv
            keys = keys[:, :, None, :, :].expand(1, kvh, n_rep, seq, hd).reshape(1, heads, seq, hd)
            vals = vals[:, :, None, :, :].expand(1, kvh, n_rep, seq, hd).reshape(1, heads, seq, hd)
        w = torch.matmul(query, keys.transpose(2, 3))
        w /= math.sqrt(hd)
        w = torch.nn.functional.softmax(w, dim=-1, dtype=dt)
        o = torch.matmul(w, vals).transpose(1, 2).reshape(heads * hd)
        res[mode] = o.float().numpy()
    out[f"shape_{i}"] = np.array([heads, kvh, hd, seq, max_seq])
    out[f"q_{i}"], out[f"kc_{i}"], out[f"vc_{i}"] = q, kc[0, :, :seq].copy(), vc[0, :, :seq].copy()
    out[f"f32_{i}"], out[f"f16_{i}"] = res["f32"], res["f16"]
path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "decode_attn_torch.npz")
np.savez_compressed(path, **out)
print("wrote", path, os.path.getsize(path))
