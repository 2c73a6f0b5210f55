"""CPU side of tests/test_gpu_decode_grid.py: every case of its table stands on a proven schedule, and the table reaches every grid regime.

For each case, the checker of its plan kind (tests/decode_sched_check*.cpp: ds_check, ds_check_gqa, ds_check_batch, ds_check_multi,
ds_check_lora) proves the schedule at the case's grid over every context of its cache.  tests/decode_grid_regimes.cpp then names the
code paths each launch of the case reaches at that grid, from decode_step_sched.h alone; the union over the table must hold all of them,
so that a case dropped from the table, or a grid changed, cannot quietly leave a path of the kernel unrun:
  * a QKV range crossing q|k or k|v, and a GU range crossing gate|up (the producer's matrix switch inside one range);
  * QKV, GU and DOWN ranges longer than one tile's K stages (the CTA quantises every K stage of x);
  * ATT limited by the grid (grid < cap x KV heads), and ATT limited by the per-head cap (the rest of the grid sits it out);
  * the attention partial table reset before a launch, and no reset;
  * batched plans with compact x staging (batch_xstages < spt_max) and with full staging;
  * an odd grid, and grid == heads (the smallest grid a plan takes).
"""
import ctypes
import os
import subprocess

import pytest

from test_gpu_decode_grid import CASES, NATIVE_SMS, dims

HERE = os.path.dirname(os.path.abspath(__file__))
SMEM_OPTIN = 232448          # cudaDevAttrMaxSharedMemoryPerBlockOptin on sm_90 (227 KB)
REGIMES = ["qkv crosses q|k or k|v", "gu crosses gate|up", "qkv range > spt", "gu range > spt", "down range > spt",
           "att limited by the grid", "att limited by the cap", "reset", "compact x staging", "full x staging"]
EXTRA = ["no reset", "odd grid", "grid == heads"]
PROJ = ("q", "k", "v", "o", "gate", "up", "down")


def _so(tmp_path_factory, src):
    so = str(tmp_path_factory.mktemp("grid") / (os.path.splitext(src)[0] + ".so"))
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wall", "-Werror", os.path.join(HERE, src), "-o", so])
    return ctypes.CDLL(so)


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    """(the multi-token checker's library, which holds ds_check / _gqa / _batch / _multi, the LoRA checker's, the regimes')"""
    tail = [ctypes.c_longlong, ctypes.c_char_p, ctypes.c_int, ctypes.POINTER(ctypes.c_longlong), ctypes.POINTER(ctypes.c_int)]
    chk = _so(tmp_path_factory, "decode_sched_check_multi.cpp")
    chk.ds_check.argtypes = [ctypes.c_int] * 9 + tail
    chk.ds_check_gqa.argtypes = [ctypes.c_int] * 10 + tail
    chk.ds_check_batch.argtypes = [ctypes.c_int] * 11 + tail
    chk.ds_check_multi.argtypes = [ctypes.c_int] * 12 + tail
    chk.ds_max_batch.argtypes = [ctypes.c_int] * 6 + [ctypes.c_longlong, ctypes.c_int]
    chk.ds_max_tokens.argtypes = [ctypes.c_int] * 5 + [ctypes.c_longlong, ctypes.c_int]
    lora = _so(tmp_path_factory, "decode_sched_check_lora.cpp")
    lora.ds_check_lora.argtypes = [ctypes.c_int] * 8 + [ctypes.POINTER(ctypes.c_int), ctypes.c_longlong, ctypes.c_char_p, ctypes.c_int,
                                                        ctypes.POINTER(ctypes.c_longlong)]
    rg = _so(tmp_path_factory, "decode_grid_regimes.cpp")
    rg.dg_regimes.argtypes = [ctypes.c_int] * 9 + [ctypes.POINTER(ctypes.c_int)]
    return chk, lora, rg


def _kind(case):
    return "multi" if case.max_tokens else ("batch" if dims(case)[7] > 1 else "one")


def _layers(case):
    return case.stack.get("layers", 2)


def prove(libs, case):
    """Run the checker(s) of the case's plan kind at its grid over every context of its cache; returns [(checker, rc, message)]."""
    chk, lora, _ = libs
    H, HQ, I, heads, kv, vocab, act, max_batch, max_seq = dims(case)
    grid = case.grid or NATIVE_SMS
    out = []

    def run(name, fn, *args):
        msg = ctypes.create_string_buffer(512)
        rc = fn(*args, SMEM_OPTIN, msg, len(msg), ctypes.byref(ctypes.c_longlong()), ctypes.byref(ctypes.c_int()))
        out.append((name, rc, msg.value.decode()))
    kind = _kind(case)
    if kind == "multi":
        assert chk.ds_max_tokens(H, HQ, I, heads, kv, SMEM_OPTIN, grid) >= case.max_tokens
        for k in sorted({k for k, _ in case.launches}):
            run(f"ds_check_multi k {k}", chk.ds_check_multi, H, HQ, I, heads, kv, vocab, grid, k, case.max_tokens, 0, max_seq - k, max_seq)
    elif kind == "batch":
        assert chk.ds_max_batch(H, HQ, I, heads, kv, int(act), SMEM_OPTIN, grid) >= max_batch
        for bsz in sorted({len(p) for p in case.launches}):
            run(f"ds_check_batch bsz {bsz}", chk.ds_check_batch, H, HQ, I, heads, kv, vocab, grid, bsz, max_batch, 0, max_seq - 1)
    elif kv == heads:
        run("ds_check", chk.ds_check, H, HQ, I, heads, vocab, grid, 0, max_seq - 1, int(act))
    else:
        run("ds_check_gqa", chk.ds_check_gqa, H, HQ, I, heads, kv, vocab, grid, 0, max_seq - 1, int(act))
    if case.lora:
        n = _layers(case)
        targets = PROJ if case.lora[1] == "all" else case.lora[1]
        rank = (ctypes.c_int * (7 * n))(*[case.lora[0] if p in targets else 0 for _ in range(n) for p in PROJ])
        msg = ctypes.create_string_buffer(512)
        rc = lora.ds_check_lora(H, HQ, I, heads, kv, grid, max_batch, n, rank, SMEM_OPTIN, msg, len(msg), ctypes.byref(ctypes.c_longlong()))
        out.append(("ds_check_lora", rc, msg.value.decode()))
    return out


def regimes(libs, case):
    """The named regimes the case's launches reach at its grid."""
    rg = libs[2]
    H, HQ, I, heads, kv, vocab, act, max_batch, max_seq = dims(case)
    grid = case.grid or NATIVE_SMS
    kind = _kind(case)
    got = set()
    for launch in case.launches:
        if kind == "multi":
            code, nb, past = 2, launch[0], launch[1]
        elif kind == "batch":
            code, nb, past = 1, len(launch), max(launch)
        else:
            code, nb, past = 0, 1, launch[0]
        flags = (ctypes.c_int * len(REGIMES))()
        assert rg.dg_regimes(H, HQ, I, heads, kv, grid, code, nb, past, flags) == len(REGIMES)
        got |= {name for name, f in zip(REGIMES, flags) if f}
        if not flags[REGIMES.index("reset")]:
            got.add("no reset")
    if grid % 2:
        got.add("odd grid")
    if grid == heads:
        got.add("grid == heads")
    return got


@pytest.mark.parametrize("case", [pytest.param(c, id=c.id) for c in CASES])
def test_case_schedule_is_proven(libs, case):
    for name, rc, msg in prove(libs, case):
        assert rc == 0, f"{case.id}: {name} at grid {case.grid or NATIVE_SMS}: {msg}"


def test_table_reaches_every_regime(libs, capsys):
    reached = {}
    for c in CASES:
        for r in regimes(libs, c):
            reached.setdefault(r, []).append(c.id)
    with capsys.disabled():
        print()
        for r in REGIMES + EXTRA:
            print(f"  {r:>24}: {len(reached.get(r, []))} cases, e.g. {reached.get(r, ['-'])[:3]}")
    missing = [r for r in REGIMES + EXTRA if r not in reached]
    assert not missing, missing


def test_regimes_named_in_the_table():
    """Spot checks of the partitions the table is built on (decode_step_sched.h by hand): on the standard stack grid 8 crosses q|k at
    unit 64 (CTA 2 owns [48, 72)), grid 9 crosses gate|up at unit 176 (CTA 4 owns [156, 195)); 132 and 114 put a CTA boundary on
    both; 13B's QKV ranges at 114 CTAs are 42-43 units long against 40 K stages per tile."""
    def share(U, c, G):
        return U * c // G
    assert share(192, 2, 8) < 64 < share(192, 3, 8)
    assert share(352, 4, 9) < 176 < share(352, 5, 9)
    for G in (132, 114):
        assert any(share(352, c, G) == 176 for c in range(G + 1)) and any(share(192, c, G) == 64 for c in range(G + 1))
    U13 = 3 * 40 * 40
    assert {share(U13, c + 1, 114) - share(U13, c, 114) for c in range(114)} == {42, 43}


def test_batch_rejection_at_grid_31(libs):
    """test_gpu_decode_grid.py's rejected batch: 4 x 8 virtual heads need 32 CTAs, so grid 31 takes 3 sequences."""
    chk = libs[0]
    assert chk.ds_max_batch(1024, 1024, 2816, 8, 8, 0, SMEM_OPTIN, 31) == 3
