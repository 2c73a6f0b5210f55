"""Generates tests/golden/rep_penalty_ref.npz by running the REFERENCE's own rep_penalty.cpp
(compiled into oracle/_ref/librep_penalty_ref.so by `make -C oracle ref REF=<reference checkout>`).
Run in the build container:  python oracle/gen_golden_cpu.py"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import oracle as O  # noqa: E402

assert O.ref_cpu_lib() is not None, "build oracle/_ref first (make -C oracle ref REF=<reference checkout>)"
rng = np.random.default_rng(20260922)
cases = [(16, 4, 1.15, 2, 2), (64, 40, 1.2, 8, 16), (1000, 300, 1.3, 64, 128), (50, 10, 1.25, -1, 0),
         (50, 7, 1.1, 0, 5), (4096, 512, 1.18, 256, 256), (100, 1, 1.5, 0, 0), (100, 30, 1.0, 10, 10)]
out = {"n_cases": len(cases)}
for i, (vocab, n, pmax, sustain, decay) in enumerate(cases):
    seq = rng.integers(0, vocab, size=n).astype(np.int64)
    if i == 0:
        seq = np.array([5, 7, 7, 9], dtype=np.int64)
    logits = rng.standard_normal(vocab).astype(np.float32)
    out[f"vocab_{i}"], out[f"pmax_{i}"], out[f"sustain_{i}"], out[f"decay_{i}"] = vocab, pmax, sustain, decay
    out[f"seq_{i}"], out[f"logits_{i}"] = seq, logits
    out[f"mask_{i}"] = O.rep_penalty(vocab, seq, pmax, sustain, decay, use_ref=True)
    out[f"applied_{i}"] = O.apply_rep_penalty(seq[None], pmax, sustain, decay, logits[None], use_ref=True)[0]
# tests/test_oracle.py::test_rep_penalty_against_compiled_reference: 25 random cases, inputs redrawn from the same seed by the test
rng = np.random.default_rng(1)
for i in range(25):
    vocab = int(rng.integers(8, 2000)); n = int(rng.integers(1, 400))
    seq = rng.integers(0, vocab, size=n)
    pmax = float(rng.uniform(1.0, 1.5)); sustain = int(rng.integers(-1, 300)); decay = int(rng.integers(0, 300))
    out[f"rand_mask_{i}"] = O.rep_penalty(vocab, seq, pmax, sustain, decay, use_ref=True)
    lg = rng.standard_normal((1, vocab)).astype(np.float32)
    out[f"rand_applied_{i}"] = O.apply_rep_penalty(seq[None], pmax, sustain, decay, lg, use_ref=True)
path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "rep_penalty_ref.npz")
np.savez_compressed(path, **out)
print("wrote", path)
