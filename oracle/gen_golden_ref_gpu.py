"""Generates tests/golden/ref_gpu.npz: outputs of the REFERENCE's own CUDA kernels (oracle/_ref/libexllama_ref.so, built by
`make -C oracle ref REF=<reference checkout>`) on the seeded inputs of tests/test_gpu_ref_pin.py and tests/test_gpu_q4_matmul.py,
so that those tests compare this repo's kernels with the reference without the reference being present.
Needs an sm_90 GPU.  Large outputs are stored as a fixed column sample (helpers.golden_cols).
    python oracle/gen_golden_ref_gpu.py [OUT.npz]
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import torch  # noqa: E402

from helpers import RefLib, golden_cols, to_cuda  # noqa: E402
from oracle import oracle as O  # noqa: E402
from stack_harness import sincos  # noqa: E402
import test_gpu_q4_matmul as TQ  # noqa: E402
import test_gpu_ref_pin as TP  # noqa: E402

out = {}
cols = lambda a: np.ascontiguousarray(a[..., golden_cols(a.shape[-1], a.shape[-1])])  # noqa: E731
f16 = lambda *s: torch.zeros(s, dtype=torch.float16, device="cuda")  # noqa: E731


def call(fn, *args):
    torch.cuda.synchronize()
    fn(*[a.data_ptr() if torch.is_tensor(a) else a for a in args])
    ref.sync()


def handle(t):
    qw, qz, sc, g = t
    return ref.make_q4(*to_cuda(qw.copy(), qz, sc), g)


# ---------------------------------------------------------------- test_gpu_ref_pin.py
ref = RefLib()
ref.prepare_buffers(inter=11008, max_rows=64, dq_numel=8)
for rows, dim in [(1, 4096), (1, 5120), (3, 6656), (7, 8192), (17, 4096)]:
    rng = np.random.default_rng(rows * 31 + dim)
    x = rng.standard_normal((rows, dim)).astype(np.float16)
    w = (1 + 0.1 * rng.standard_normal(dim)).astype(np.float16)
    t = f16(rows, dim)
    call(ref.lib.ref_rms_norm, to_cuda(x), to_cuda(w), t, 1e-6, rows, dim, 0)
    out[f"rms_norm_{rows}_{dim}"] = cols(t.cpu().numpy())
for bsz, q_len, heads, hd, past in [(1, 1, 32, 128, 0), (1, 1, 40, 128, 1919), (1, 5, 8, 128, 3), (2, 3, 4, 128, 100)]:
    x = np.random.default_rng(17 + past).standard_normal((bsz, q_len, heads * hd)).astype(np.float16)
    t = to_cuda(x)
    call(ref.lib.ref_rope, t, *to_cuda(*sincos(2048, hd)), bsz, q_len * heads, hd, heads, past)
    out[f"rope_{bsz}_{q_len}_{heads}_{hd}_{past}"] = t.cpu().numpy()
rng = np.random.default_rng(3)
for M, K in ((1, 4096), (7, 5120), (33, 6656)):
    x = rng.standard_normal((M, K)).astype(np.float16)
    perm = rng.permutation(K).astype(np.uint32)
    t = f16(M, K)
    call(ref.lib.ref_column_remap, to_cuda(x), t, M, K, torch.from_numpy(perm.view(np.int32)).cuda())
    out[f"column_remap_{M}_{K}"] = cols(t.cpu().numpy())
rng = np.random.default_rng(4)
for M, K, N in ((1, 4096, 16), (5, 512, 64), (16, 64, 4096)):
    x = rng.standard_normal((M, K)).astype(np.float16)
    w = (rng.standard_normal((K, N)) * 0.1).astype(np.float16)
    t = f16(M, N)
    call(ref.lib.ref_half_matmul_cublas, to_cuda(x), to_cuda(w), t, M, K, N, 0)
    out[f"hgemm_{M}_{K}_{N}"] = cols(t.cpu().numpy())
for act in (False, True):
    for q_len, past in [(1, 0), (1, 37), (2, 5)]:
        hidden, heads, hd, gs, max_seq = 1024, 8, 128, 128, 64
        t = TP._layer(O, hidden, 2048, gs, act, seed=300)
        rng = np.random.default_rng(11)
        x = rng.standard_normal((1, q_len, hidden)).astype(np.float16)
        w = (1 + 0.1 * rng.standard_normal(hidden)).astype(np.float16)
        ts, tc = to_cuda(*sincos(max_seq, hd))
        hq, hk, hv = (handle(t[n]) for n in ("q", "k", "v"))
        tx, q, k, v = to_cuda(x), f16(1, q_len, hidden), f16(1, q_len, hidden), f16(1, q_len, hidden)
        kc, vc = f16(1, heads, max_seq, hd), f16(1, heads, max_seq, hd)
        call(ref.lib.ref_q4_attn, tx, to_cuda(w), 1e-6, q, k, v, hq, hk, hv, ts, tc, 1, q_len, hidden, hd, heads, heads, past, kc, vc, max_seq, 0)
        for n, a in zip(("q", "k", "v", "kc", "vc", "x"), (q, k, v, kc, vc, tx)):
            out[f"q4_attn_{q_len}_{past}_{int(act)}_{n}"] = a.cpu().numpy()
for act in (False, True):
    for rows in (1, 2):
        hidden = 1024
        t = TP._layer(O, hidden, 2816, 128, act, seed=400)
        rng = np.random.default_rng(12)
        x = rng.standard_normal((rows, hidden)).astype(np.float16)
        attn = rng.standard_normal((rows, hidden)).astype(np.float16)
        w = (1 + 0.1 * rng.standard_normal(hidden)).astype(np.float16)
        ho, hg, hu, hdn = (handle(t[n]) for n in ("o", "gate", "up", "down"))
        xr = to_cuda(x)
        call(ref.lib.ref_q4_attn_2, xr, to_cuda(attn), ho, rows)
        out[f"q4_attn_2_{rows}_{int(act)}"] = xr.cpu().numpy()
        xr = to_cuda(x)
        call(ref.lib.ref_q4_mlp, xr, to_cuda(w), 1e-6, hg, hu, hdn, rows, hidden, 0)
        out[f"q4_mlp_{rows}_{int(act)}"] = xr.cpu().numpy()
qw, qz, sc, _ = O.synth_q4(4096, 4096, 128, seed=5)
h, tx = handle((qw, qz, sc, None)), to_cuda(O.synth_x(1, 4096, seed=6))
out["spread_runs"] = np.stack([ref.q4_matmul(tx, h, 4096, mode=0).cpu().numpy() for _ in range(3)])

# ---------------------------------------------------------------- test_gpu_q4_matmul.py
ref = RefLib()
ref.prepare_buffers(inter=11008, max_rows=256, dq_numel=4096 * 11008)
for M, K, N, gs, act in [(1, 4096, 4096, 128, False), (1, 4096, 11008, 128, False), (4, 5120, 5120, 128, True), (7, 2048, 6656, 32, True)]:
    qw, qz, sc, g_idx = TQ._mk(O, K, N, gs, act, seed=41)
    tq, tz, ts = to_cuda(qw.copy(), qz, sc)
    h = ref.make_q4(tq, tz, ts, g_idx)
    key = f"decode_{M}_{K}_{N}_{gs}_{int(act)}"
    out[key] = cols(ref.q4_matmul(to_cuda(O.synth_x(M, K, seed=7)), h, N, mode=0).cpu().numpy())
    if act:      # the reference's sequential qweight (make_q4 rewrites it in place): the first 32 columns of the sample
        out[key + "_qweight"] = np.ascontiguousarray(tq.cpu().numpy()[:, golden_cols(N, N)[:32]])
qw, qz, sc, _ = TQ._mk(O, 4096, 4096, 128, False, seed=43)
h = handle((qw, qz, sc, None))
out["recons_64_4096_4096"] = cols(ref.q4_matmul(to_cuda(O.synth_x(64, 4096, seed=8)), h, 4096, mode=1).cpu().numpy())

out["device"] = np.array(torch.cuda.get_device_name(0))
path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "ref_gpu.npz")
np.savez_compressed(path, **out)
print("wrote", path)
