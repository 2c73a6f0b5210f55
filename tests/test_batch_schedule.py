"""CPU proof of the persistent decode kernel's schedule for batched decode (1 .. 4 sequences per launch, each at its own context).

tests/decode_sched_check_batch.cpp (which includes the GQA and multi-head checkers) compiles exllama_b200/csrc/decode_step_sched.h --
the header decode_step.cu includes -- with g++.  Its ds_check_batch entry point checks, for bsz sequences on a plan made for
max_batch of them and at every longest context: partition and balance of every phase, cta_of as the inverse of range_lo, at most 2
virtual heads per CTA in ATT, unique partial slots over the virtual query heads that the combine reads only where they were written
(unless att_needs_reset holds for the longest context), lm_head coverage, every CTA's K stages inside the compacted per-sequence
staging, and >= 2 ring stages.  The attention schedule depends on the longest context alone (shorter sequences own empty units past
their end), so this covers every mix of contexts.
"""
import ctypes
import os
import subprocess

import pytest

from exllama_b200.shapes import GQA_SHAPES, SHAPES
from helpers import att_needs_reset

HERE = os.path.dirname(os.path.abspath(__file__))
SMEM_OPTIN = 232448          # cudaDevAttrMaxSharedMemoryPerBlockOptin on sm_90 (227 KB)
SMS = 132                    # H100 SXM
ALL = {**SHAPES, **GQA_SHAPES}


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("sched_batch") / "libdecode_sched_check_batch.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wall", "-Werror",
                           os.path.join(HERE, "decode_sched_check_batch.cpp"), "-o", so])
    lib = ctypes.CDLL(so)
    tail = [ctypes.c_longlong, ctypes.c_char_p, ctypes.c_int, ctypes.POINTER(ctypes.c_longlong), ctypes.POINTER(ctypes.c_int)]
    lib.ds_check_gqa.restype = lib.ds_check_batch.restype = ctypes.c_int
    lib.ds_check_gqa.argtypes = [ctypes.c_int] * 10 + tail
    lib.ds_check_batch.argtypes = [ctypes.c_int] * 11 + tail
    plan_tail = [ctypes.c_longlong, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_longlong), ctypes.POINTER(ctypes.c_int)]
    lib.ds_plan_gqa.restype = lib.ds_plan_batch.restype = ctypes.c_int
    lib.ds_plan_gqa.argtypes = [ctypes.c_int] * 7 + plan_tail
    lib.ds_plan_batch.argtypes = [ctypes.c_int] * 7 + plan_tail + [ctypes.POINTER(ctypes.c_int)]
    lib.ds_max_batch.restype = ctypes.c_int
    lib.ds_max_batch.argtypes = [ctypes.c_int] * 6 + [ctypes.c_longlong, ctypes.c_int]
    return lib


def check(lib, H, I, heads, kv, vocab, bsz, max_batch, past_lo, past_hi, grid=SMS):
    msg = ctypes.create_string_buffer(512)
    gaps, resets = ctypes.c_longlong(), ctypes.c_int()
    rc = lib.ds_check_batch(H, heads * 128, I, heads, kv, vocab, grid, bsz, max_batch, past_lo, past_hi, SMEM_OPTIN, msg, len(msg),
                            ctypes.byref(gaps), ctypes.byref(resets))
    return rc, msg.value.decode(), gaps.value, resets.value


def check_gqa(lib, H, I, heads, kv, vocab, past_lo, past_hi, grid=SMS):
    msg = ctypes.create_string_buffer(512)
    gaps, resets = ctypes.c_longlong(), ctypes.c_int()
    rc = lib.ds_check_gqa(H, heads * 128, I, heads, kv, vocab, grid, past_lo, past_hi, 0, SMEM_OPTIN, msg, len(msg),
                          ctypes.byref(gaps), ctypes.byref(resets))
    return rc, msg.value.decode(), gaps.value, resets.value


def plan(lib, H, I, heads, kv, max_batch, grid=SMS):
    depth, smem, slots, xst = ctypes.c_int(), ctypes.c_longlong(), ctypes.c_int(), ctypes.c_int()
    rc = lib.ds_plan_batch(H, heads * 128, I, heads, kv, grid, max_batch, SMEM_OPTIN, ctypes.byref(depth), ctypes.byref(smem),
                           ctypes.byref(slots), ctypes.byref(xst))
    return rc, depth.value, smem.value, slots.value, xst.value


def max_batch(lib, s, act=False, grid=SMS):
    return lib.ds_max_batch(s.hidden, s.heads * 128, s.inter, s.heads, s.kv_heads, int(act), SMEM_OPTIN, grid)


# what max_batch_for says at 132 SMs and 227 KB: shared memory limits 33B, 65B and 70B; 13B is held at 3 by 3 x 40 heads <= 132 CTAs
MAX_BATCH = {"7b": 4, "13b": 3, "33b": 2, "65b": 2, "70b": 2}


def test_max_batch_table(lib):
    assert {k: max_batch(lib, s) for k, s in ALL.items()} == MAX_BATCH
    for s in ALL.values():
        assert max_batch(lib, s, act=True) == 1                       # act-order plans take one sequence
    assert max_batch(lib, SHAPES["13b"], grid=160) == 4               # the segment rule, not shared memory, holds 13B back


@pytest.mark.parametrize("name", list(MAX_BATCH))
def test_full_shapes_at_max_batch(lib, name):
    """Every batch size up to the shape's largest, on a plan for the largest, at every longest context of a 4096-row cache."""
    s = ALL[name]
    mb = MAX_BATCH[name]
    rc, depth, smem, slots, xst = plan(lib, s.hidden, s.inter, s.heads, s.kv_heads, mb)
    assert rc == 0 and depth >= 2 and smem + 2048 <= SMEM_OPTIN, (depth, smem)
    assert xst <= max(s.hidden, s.heads * 128, s.inter) // 128
    for bsz in range(1, mb + 1):
        rc, msg, _, _ = check(lib, s.hidden, s.inter, s.heads, s.kv_heads, s.vocab, bsz, mb, 0, 4095)
        assert rc == 0, f"{name} bsz {bsz}: {msg}"
    rc, msg, _, _ = check(lib, s.hidden, s.inter, s.heads, s.kv_heads, s.vocab, mb, mb + 1, 0, 64) if mb < 4 else (1, "P7", 0, 0)
    assert rc == 1 and ("P7" in msg or "P3" in msg), msg                # one more sequence does not fit


SMALL = [(1024, 2816, 8, 8), (1024, 2816, 8, 2), (1024, 2816, 8, 1), (1024, 2816, 8, 4), (2048, 5632, 16, 2), (2048, 5632, 16, 16)]


@pytest.mark.parametrize("H,I,heads,kv", SMALL)
def test_small_shapes_every_batch(lib, H, I, heads, kv):
    for bsz in (1, 2, 3, 4):
        for vocab in (0, 512):
            rc, msg, _, _ = check(lib, H, I, heads, kv, vocab, bsz, 4, 0, 300)
            assert rc == 0, f"{(H, I, heads, kv, vocab, bsz)}: {msg}"


@pytest.mark.parametrize("name", list(MAX_BATCH))
def test_batch1_is_the_single_sequence_schedule(lib, name):
    """A plan for one sequence through the batch entry points: exactly ds_plan_gqa's plan, and the same proof outcome (gaps and
    resets) as ds_check_gqa."""
    s = ALL[name]
    rc, depth, smem, slots, xst = plan(lib, s.hidden, s.inter, s.heads, s.kv_heads, 1)
    d, m, sl = ctypes.c_int(), ctypes.c_longlong(), ctypes.c_int()
    assert lib.ds_plan_gqa(s.hidden, s.heads * 128, s.inter, s.heads, s.kv_heads, SMS, 0, SMEM_OPTIN, ctypes.byref(d), ctypes.byref(m), ctypes.byref(sl)) == 0
    assert (rc, depth, smem, slots, xst) == (0, d.value, m.value, sl.value, 0)
    assert check(lib, s.hidden, s.inter, s.heads, s.kv_heads, s.vocab, 1, 1, 0, 600) == check_gqa(lib, s.hidden, s.inter, s.heads, s.kv_heads, s.vocab, 0, 600)


@pytest.mark.parametrize("H,I,heads,kv", SMALL)
def test_batch1_small_shapes_match(lib, H, I, heads, kv):
    assert check(lib, H, I, heads, kv, 512, 1, 1, 0, 300) == check_gqa(lib, H, I, heads, kv, 512, 0, 300)


@pytest.mark.parametrize("heads,kv,bsz", [(8, 8, 2), (8, 2, 3), (8, 2, 4), (64, 8, 2)])
def test_reset_over_virtual_heads(lib, heads, kv, bsz):
    """The table is reset exactly where the predicate (longest context) holds, and nowhere past the short contexts."""
    H, I = (1024, 2816) if heads == 8 else (8192, 28672)
    rc, msg, gaps, resets = check(lib, H, I, heads, kv, 512, bsz, bsz, 0, 1023)
    assert rc == 0, msg
    assert resets == sum(att_needs_reset(heads, kv, p, SMS, bsz) for p in range(1024)) and resets > 0
    last = max(p for p in range(1024) if att_needs_reset(heads, kv, p, SMS, bsz))
    rc, msg, gaps, resets = check(lib, H, I, heads, kv, 512, bsz, bsz, last + 1, 1023)
    assert rc == 0 and gaps == 0 and resets == 0


def test_rejects_what_does_not_fit(lib):
    s = SHAPES["13b"]
    rc, msg, _, _ = check(lib, s.hidden, s.inter, s.heads, s.kv_heads, s.vocab, 1, 4, 0, 4)
    assert rc == 1 and "P3" in msg                                   # 4 x 40 heads > 132 CTAs
    rc, msg, _, _ = check(lib, 1024, 2816, 8, 8, 512, 3, 2, 0, 4)
    assert rc == 1 and "batch" in msg                                # bsz > max_batch
    assert plan(lib, 1024, 2816, 8, 8, 5)[0] == 1
