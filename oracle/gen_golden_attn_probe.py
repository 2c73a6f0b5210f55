"""tests/golden/attn_probe_n1.npz: what the attention-probe helpers (tests/helpers.py plant_probe, probe_expectation) compute for
one token on the CPU cases of tests/test_attn_probe_oracle.py -- want, bound, a digest of the planted caches and the plants.  It was
written by the one-token helpers, before they took n tokens; tests/test_multi_probe_oracle.py holds the n-token helpers to it bit
for bit.  Rerun only on purpose (a deliberate change of the one-token probe):

    python oracle/gen_golden_attn_probe.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def main():
    from oracle import oracle as O
    from test_multi_probe_oracle import n1_record
    O.lib()
    out = n1_record(O)
    np.savez(os.path.join(ROOT, "tests", "golden", "attn_probe_n1.npz"), **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
