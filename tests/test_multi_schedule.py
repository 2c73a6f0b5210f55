"""CPU proof of the persistent decode kernel's schedule for multi-token steps (1 .. 4 consecutive tokens of one sequence per launch).

tests/decode_sched_check_multi.cpp (which includes the batch, GQA and multi-head checkers) compiles exllama_b200/csrc/decode_step_sched.h --
the header decode_step.cu includes -- with g++.  Its ds_check_multi entry point checks, for k tokens on a plan made for max_tokens of them
and at every context past_len with past_len + k inside a 4096-row cache: partition and balance of ATT over the real KV heads, cta_of as
the inverse of range_lo, at most 2 KV heads per CTA, exactly one tail owner per KV head, unique partial slots over the k * heads virtual
query heads that the combine reads only where they were written unless att_needs_reset_multi holds -- and a gap exactly where it holds --,
the GEMV and HEAD schedules equal to the batch's at nb = k, and >= 2 ring stages.
"""
import ctypes
import os
import subprocess

import pytest

from exllama_b200.shapes import GQA_SHAPES, SHAPES

HERE = os.path.dirname(os.path.abspath(__file__))
SMEM_OPTIN = 232448          # cudaDevAttrMaxSharedMemoryPerBlockOptin on sm_90 (227 KB)
SMS = 132                    # H100 SXM
MAX_SEQ = 4096
ALL = {**SHAPES, **GQA_SHAPES}


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("sched_multi") / "libdecode_sched_check_multi.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wall", "-Werror",
                           os.path.join(HERE, "decode_sched_check_multi.cpp"), "-o", so])
    lib = ctypes.CDLL(so)
    tail = [ctypes.c_longlong, ctypes.c_char_p, ctypes.c_int, ctypes.POINTER(ctypes.c_longlong), ctypes.POINTER(ctypes.c_int)]
    lib.ds_check_multi.restype = ctypes.c_int
    lib.ds_check_multi.argtypes = [ctypes.c_int] * 12 + tail
    lib.ds_plan_multi.restype = ctypes.c_int
    lib.ds_plan_multi.argtypes = [ctypes.c_int] * 7 + [ctypes.c_longlong, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_longlong),
                                                       ctypes.POINTER(ctypes.c_int)]
    lib.ds_max_tokens.restype = lib.ds_max_batch.restype = ctypes.c_int
    lib.ds_max_tokens.argtypes = [ctypes.c_int] * 5 + [ctypes.c_longlong, ctypes.c_int]
    lib.ds_max_batch.argtypes = [ctypes.c_int] * 6 + [ctypes.c_longlong, ctypes.c_int]
    lib.ds_att_needs_reset_multi.restype = ctypes.c_int
    lib.ds_att_needs_reset_multi.argtypes = [ctypes.c_int] * 4
    return lib


def check(lib, H, I, heads, kv, vocab, k, max_tokens, past_lo, past_hi, grid=SMS):
    msg = ctypes.create_string_buffer(512)
    gaps, resets = ctypes.c_longlong(), ctypes.c_int()
    rc = lib.ds_check_multi(H, heads * 128, I, heads, kv, vocab, grid, k, max_tokens, past_lo, past_hi, MAX_SEQ, SMEM_OPTIN, msg, len(msg),
                            ctypes.byref(gaps), ctypes.byref(resets))
    return rc, msg.value.decode(), gaps.value, resets.value


def max_tokens(lib, s, grid=SMS):
    return lib.ds_max_tokens(s.hidden, s.heads * 128, s.inter, s.heads, s.kv_heads, SMEM_OPTIN, grid)


def plan(lib, s, k, grid=SMS):
    depth, smem, slots = ctypes.c_int(), ctypes.c_longlong(), ctypes.c_int()
    rc = lib.ds_plan_multi(s.hidden, s.heads * 128, s.inter, s.heads, s.kv_heads, grid, k, SMEM_OPTIN, ctypes.byref(depth), ctypes.byref(smem),
                           ctypes.byref(slots))
    return rc, depth.value, smem.value, slots.value


# what max_tokens_for says at 132 SMs and 227 KB.  The history is shared, so 13B and 33B are not held back by their head counts as
# their batches are (shared memory holds 33B at 3 and 65B at 2);
# 70B's n_rep 8 query vectors per KV head and token need ~97 KB of attention scratch at 2 tokens, which does not fit beside the ring
MAX_TOKENS = {"7b": 4, "13b": 4, "33b": 3, "65b": 2, "70b": 1}
MAX_BATCH = {"7b": 4, "13b": 3, "33b": 2, "65b": 2, "70b": 2}        # test_batch_schedule.py's table: unchanged


def test_max_tokens_table(lib):
    assert {k: max_tokens(lib, s) for k, s in ALL.items()} == MAX_TOKENS
    assert {k: lib.ds_max_batch(s.hidden, s.heads * 128, s.inter, s.heads, s.kv_heads, 0, SMEM_OPTIN, SMS) for k, s in ALL.items()} == MAX_BATCH


@pytest.mark.parametrize("name", list(MAX_TOKENS))
def test_full_shapes_every_token_count(lib, name):
    """Every k up to the shape's largest, on a plan for the largest, at every context of a 4096-row cache."""
    s = ALL[name]
    mt = MAX_TOKENS[name]
    rc, depth, smem, slots = plan(lib, s, mt)
    assert rc == 0 and depth >= 2 and smem + 2048 <= SMEM_OPTIN, (depth, smem)
    for k in range(1, mt + 1):
        rc, msg, _, _ = check(lib, s.hidden, s.inter, s.heads, s.kv_heads, s.vocab, k, mt, 0, MAX_SEQ)
        assert rc == 0, f"{name} k {k}: {msg}"
    if mt < 4:
        rc, msg, _, _ = check(lib, s.hidden, s.inter, s.heads, s.kv_heads, s.vocab, mt + 1, mt + 1, 0, 64)
        assert rc == 1 and "P7" in msg, msg                             # one more token does not fit


SMALL = [(1024, 2816, 8, 8), (1024, 2816, 8, 2), (1024, 2816, 8, 1), (1024, 2816, 8, 4), (2048, 5632, 16, 2), (2048, 5632, 16, 16)]


@pytest.mark.parametrize("H,I,heads,kv", SMALL)
def test_small_shapes_every_token_count(lib, H, I, heads, kv):
    top = lib.ds_max_tokens(H, heads * 128, I, heads, kv, SMEM_OPTIN, SMS)
    assert top == (4 if heads // kv <= 4 else 2)          # n_rep * max_tokens query vectors per KV head share the staging area
    for mt in (1, top):
        for k in range(1, mt + 1):
            for vocab in (0, 512):
                rc, msg, _, _ = check(lib, H, I, heads, kv, vocab, k, mt, 0, MAX_SEQ)
                assert rc == 0, f"{(H, I, heads, kv, vocab, k, mt)}: {msg}"


@pytest.mark.parametrize("heads,kv", [(8, 8), (8, 2), (64, 8)])
def test_reset_where_the_predicate_holds(lib, heads, kv):
    """Short contexts leave CTAs idle inside a KV head's range: the proof counts the contexts with a gap, which are exactly those where
    the predicate holds, and none past the last of them."""
    H, I = (1024, 2816) if heads == 8 else (8192, 28672)
    rc, msg, gaps, resets = check(lib, H, I, heads, kv, 512, 1, 1, 0, 1023)
    assert rc == 0, msg
    want = [p for p in range(1024) if lib.ds_att_needs_reset_multi(heads, kv, p, SMS)]
    assert resets == len(want) and resets > 0 and gaps > 0
    rc, msg, gaps, resets = check(lib, H, I, heads, kv, 512, 1, 1, want[-1] + 1, 1023)
    assert rc == 0 and gaps == 0 and resets == 0


def test_rejects_what_does_not_fit(lib):
    s = GQA_SHAPES["70b"] if "70b" in GQA_SHAPES else ALL["70b"]
    rc, msg, _, _ = check(lib, s.hidden, s.inter, s.heads, s.kv_heads, s.vocab, 2, 2, 0, 4)
    assert rc == 1 and "P7" in msg                                    # 2 x 8 query vectors per KV head: the scratch does not fit
    rc, msg, _, _ = check(lib, 1024, 2816, 8, 8, 512, 3, 2, 0, 4)
    assert rc == 1 and "tokens" in msg                                # k > max_tokens
    assert plan(lib, ALL["7b"], 5)[0] == 1
