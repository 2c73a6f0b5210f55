"""CPU proof of the LoRA schedule of the persistent decode kernel (exl_decode_plan_create_lora).

tests/decode_sched_check_lora.cpp (which includes the batch, GQA and multi-head checkers) compiles exllama_b200/csrc/decode_step_sched.h
-- the header decode_step.cu includes -- with g++.  For 7B, 13B, 33B, 65B and 70B at batch 1 and at each one's largest batch, for ranks
8, 16, 64 and 128, with adapters on {q, v} and on all seven projections, it proves: every (adapted matrix, K stage) unit of every LA
step is owned by exactly one CTA, balanced to +-1; every tile of every adapted matrix gets its B term exactly once (and no other tile
one); >= 2 ring stages fit; the extra barriers are one per adapted phase of every layer.  Without an adapter the plan is ds_plan_batch's
(and at batch 1 ds_plan_gqa's) exactly.  It also checks the ctypes mirror of struct exl_decode_lora against the C layout.
"""
import ctypes
import os
import subprocess

import pytest

from exllama_b200.shapes import GQA_SHAPES, SHAPES

HERE = os.path.dirname(os.path.abspath(__file__))
SMEM_OPTIN = 232448          # cudaDevAttrMaxSharedMemoryPerBlockOptin on sm_90 (227 KB)
SMS = 132                    # H100 SXM
ALL = {**SHAPES, **GQA_SHAPES}
MAX_BATCH = {"7b": 4, "13b": 3, "33b": 2, "65b": 2, "70b": 2}      # tests/test_batch_schedule.py pins this table
PROJ = ("q", "k", "v", "o", "gate", "up", "down")
TARGETS = {"qv": ("q", "v"), "all": PROJ}
I32P = ctypes.POINTER(ctypes.c_int)


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("sched_lora") / "libdecode_sched_check_lora.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wall", "-Werror",
                           os.path.join(HERE, "decode_sched_check_lora.cpp"), "-o", so])
    lib = ctypes.CDLL(so)
    lib.ds_check_lora.restype = ctypes.c_int
    lib.ds_check_lora.argtypes = [ctypes.c_int] * 8 + [I32P, ctypes.c_longlong, ctypes.c_char_p, ctypes.c_int, ctypes.POINTER(ctypes.c_longlong)]
    plan_tail = [ctypes.c_longlong, I32P, ctypes.POINTER(ctypes.c_longlong), I32P]
    lib.ds_plan_batch.restype = lib.ds_plan_gqa.restype = lib.ds_plan_lora.restype = ctypes.c_int
    lib.ds_plan_gqa.argtypes = [ctypes.c_int] * 7 + plan_tail
    lib.ds_plan_batch.argtypes = [ctypes.c_int] * 7 + plan_tail + [I32P]
    lib.ds_plan_lora.argtypes = [ctypes.c_int] * 8 + [I32P] + plan_tail + [I32P, ctypes.POINTER(ctypes.c_longlong)]
    lib.ds_lora_layout.restype = None
    lib.ds_lora_layout.argtypes = [ctypes.POINTER(ctypes.c_longlong)]
    return lib


def ranks(n_layers, rank, targets, layers=None):
    r = [0] * (7 * n_layers)
    for l in (range(n_layers) if layers is None else layers):
        for t in targets:
            r[l * 7 + PROJ.index(t)] = rank
    return (ctypes.c_int * len(r))(*r)


def check(lib, s, max_batch, n_layers, rk, grid=SMS):
    msg = ctypes.create_string_buffer(512)
    bar = ctypes.c_longlong()
    rc = lib.ds_check_lora(s.hidden, s.heads * 128, s.inter, s.heads, s.kv_heads, grid, max_batch, n_layers, rk, SMEM_OPTIN, msg, len(msg),
                           ctypes.byref(bar))
    return rc, msg.value.decode(), bar.value


def plan_lora(lib, s, max_batch, n_layers, rk, grid=SMS):
    d, m, sl, x, b = ctypes.c_int(), ctypes.c_longlong(), ctypes.c_int(), ctypes.c_int(), ctypes.c_longlong()
    rc = lib.ds_plan_lora(s.hidden, s.heads * 128, s.inter, s.heads, s.kv_heads, grid, max_batch, n_layers, rk, SMEM_OPTIN,
                          ctypes.byref(d), ctypes.byref(m), ctypes.byref(sl), ctypes.byref(x), ctypes.byref(b))
    return rc, d.value, m.value, sl.value, x.value, b.value


def barriers_formula(n_layers, rank, targets, layers=None):
    """exl_decode_plan_info's extra term: one barrier per adapted phase (QKV, O, GU, DOWN) of every adapted layer."""
    phase = {"q": 0, "k": 0, "v": 0, "o": 1, "gate": 2, "up": 2, "down": 3}
    per_layer = len({phase[t] for t in targets}) if rank else 0
    return per_layer * (n_layers if layers is None else len(layers))


@pytest.mark.parametrize("targets", list(TARGETS))
@pytest.mark.parametrize("rank", [8, 16, 64, 128])
@pytest.mark.parametrize("name", list(MAX_BATCH))
def test_full_shapes(lib, name, rank, targets):
    s = ALL[name]
    n_layers = 2                                                    # the schedule does not depend on the layer
    rk = ranks(n_layers, rank, TARGETS[targets])
    for mb in sorted({1, MAX_BATCH[name]}):
        rc, msg, bar = check(lib, s, mb, n_layers, rk)
        assert rc == 0, f"{name} r{rank} {targets} batch {mb}: {msg}"
        assert bar == barriers_formula(n_layers, rank, TARGETS[targets])
        base = plan_lora(lib, s, mb, n_layers, ranks(n_layers, 0, ()))
        got = plan_lora(lib, s, mb, n_layers, rk)
        assert got[0] == 0 and got[1] >= 2 and got[:5] == base[:5], (got, base)      # the adapter adds no shared memory
        assert got[5] == bar


@pytest.mark.parametrize("name", list(MAX_BATCH))
def test_every_rank_the_kernel_takes(lib, name):
    """Every multiple of 8 up to 128 on all seven projections, on layer 0 only (no barrier on layer 1); and a rank the kernel does not take
    is caught."""
    s = ALL[name]
    for rank in range(8, 129, 8):
        rc, msg, bar = check(lib, s, MAX_BATCH[name], 2, ranks(2, rank, PROJ, layers=[0]))
        assert rc == 0, f"{name} r{rank}: {msg}"
        assert bar == barriers_formula(2, rank, PROJ, layers=[0]) == 4
    for bad in (4, 12, 136, -8):
        rc, msg, _ = check(lib, s, 1, 1, ranks(1, bad, ("q",)))
        assert rc == 1 and "L5" in msg, msg


@pytest.mark.parametrize("name", list(MAX_BATCH))
def test_no_adapter_is_the_plain_plan(lib, name):
    """All ranks 0: no extra barrier, and exactly ds_plan_batch's plan (ds_plan_gqa's at batch 1)."""
    s = ALL[name]
    for mb in sorted({1, MAX_BATCH[name]}):
        rc, depth, smem, slots, xst, bar = plan_lora(lib, s, mb, 3, ranks(3, 0, ()))
        d, m, sl, x = ctypes.c_int(), ctypes.c_longlong(), ctypes.c_int(), ctypes.c_int()
        assert lib.ds_plan_batch(s.hidden, s.heads * 128, s.inter, s.heads, s.kv_heads, SMS, mb, SMEM_OPTIN, ctypes.byref(d), ctypes.byref(m),
                                 ctypes.byref(sl), ctypes.byref(x)) == 0
        assert (rc, depth, smem, slots, xst, bar) == (0, d.value, m.value, sl.value, x.value, 0)
        if mb == 1:
            assert lib.ds_plan_gqa(s.hidden, s.heads * 128, s.inter, s.heads, s.kv_heads, SMS, 0, SMEM_OPTIN, ctypes.byref(d), ctypes.byref(m),
                                   ctypes.byref(sl)) == 0
            assert (depth, smem, slots) == (d.value, m.value, sl.value)
        assert check(lib, s, mb, 3, ranks(3, 0, ()))[::2] == (0, 0)


@pytest.mark.parametrize("H,I,heads,kv", [(1024, 2816, 8, 8), (1024, 2816, 8, 2), (2048, 5632, 16, 2)])
def test_small_shapes(lib, H, I, heads, kv):
    """The shapes of tests/test_gpu_lora.py, every batch, {q, v} and all seven, a few grids."""
    from exllama_b200.shapes import LlamaShape
    s = LlamaShape("small", H, I, 2, heads, vocab=2048, kv_heads=kv)
    for grid in (SMS, 100, 17):
        for mb in (1, 2, 3, 4):
            for targets in TARGETS.values():
                rc, msg, _ = check(lib, s, mb, 2, ranks(2, 32, targets), grid=grid)
                assert rc == 0, f"{(H, I, heads, kv, grid, mb, targets)}: {msg}"


def test_ctypes_layout_matches_c(lib):
    from exllama_b200.capi import _DecodeLora
    out = (ctypes.c_longlong * 5)()
    lib.ds_lora_layout(out)
    assert list(out) == [ctypes.sizeof(_DecodeLora)] + [getattr(_DecodeLora, f).offset for f in ("n_layers", "a", "b", "rank")]
