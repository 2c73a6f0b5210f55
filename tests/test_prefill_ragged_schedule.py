"""CPU proof of the ragged prefill attention work list (exllama_b200/csrc/prefill_attn_sched.h).

prefill_attn.cu includes the header; tests/prefill_ragged_check.cpp compiles the same header with g++ and checks, for every n_seq
1 .. 64 and q_len mixes on both sides of the 64 / n_rep-token query-tile edge at n_rep 1, 2, 4 and 8: every (sequence, KV group,
row tile) is computed by exactly one CTA, no CTA is empty, the grid is sum_i kv_heads * ceil(q_len[i] * n_rep / 64), the
sequences run in non-increasing past_len + q_len order with each sequence's row tiles from the last; and the uniform description
exl_prefill_attn launches is today's (kv_heads * bsz, row tiles) grid tile for tile.
"""
import ctypes
import os
import random
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
MAX_SEQ = 64


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("pa_sched") / "libprefill_ragged_check.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wall", "-Werror",
                           os.path.join(HERE, "prefill_ragged_check.cpp"), "-o", so])
    lib = ctypes.CDLL(so)
    ip = ctypes.POINTER(ctypes.c_int)
    lib.pr_check_ragged.restype = ctypes.c_int
    lib.pr_check_ragged.argtypes = [ctypes.c_int, ip, ip, ip, ctypes.c_int, ctypes.c_int, ctypes.c_char_p, ctypes.c_int]
    lib.pr_check_uniform.restype = ctypes.c_int
    lib.pr_check_uniform.argtypes = [ctypes.c_int] * 5 + [ctypes.c_char_p, ctypes.c_int]
    return lib


def check_ragged(lib, q_lens, past_lens, cache_seqs, kv_heads, n_rep):
    n = len(q_lens)
    arr = lambda a: (ctypes.c_int * n)(*a)
    msg = ctypes.create_string_buffer(256)
    rc = lib.pr_check_ragged(n, arr(q_lens), arr(past_lens), arr(cache_seqs), kv_heads, n_rep, msg, len(msg))
    assert rc == 0, f"{msg.value.decode()}: q_lens {q_lens} past_lens {past_lens} cache_seqs {cache_seqs} kv {kv_heads} n_rep {n_rep}"


def edge_lens(n_rep):
    """q_lens on both sides of the query-tile edge (64 / n_rep tokens) and of twice it."""
    e = 64 // n_rep
    return sorted({1, max(1, e - 1), e, e + 1, 2 * e - 1, 2 * e, 2 * e + 1})


@pytest.mark.parametrize("n_rep", [1, 2, 4, 8])
def test_every_n_seq_up_to_the_cap(lib, n_rep):
    rng = random.Random(n_rep)
    lens = edge_lens(n_rep)
    for n in range(1, MAX_SEQ + 1):
        for trial in range(3):
            q_lens = [rng.choice(lens) if trial < 2 else rng.randint(1, 300) for _ in range(n)]
            past_lens = [rng.choice([0, 0, 1, 37, 200, rng.randint(0, 2000)]) for _ in range(n)]
            cache_seqs = rng.sample(range(n + 7), n)
            check_ragged(lib, q_lens, past_lens, cache_seqs, rng.choice([1, 2, 8]), n_rep)


@pytest.mark.parametrize("n_rep", [1, 2, 4, 8])
def test_equal_costs_and_single_sequences(lib, n_rep):
    """Ties in past_len + q_len (the sort must keep every sequence) and every edge length alone."""
    e = 64 // n_rep
    check_ragged(lib, [e, e + 1, e - 1 if e > 1 else 1, e], [1, 0, 2, 1], [3, 0, 2, 1], 8, n_rep)
    check_ragged(lib, [5] * MAX_SEQ, [0] * MAX_SEQ, list(range(MAX_SEQ))[::-1], 4, n_rep)
    for ql in edge_lens(n_rep):
        check_ragged(lib, [ql], [0], [0], 8, n_rep)


@pytest.mark.parametrize("n_rep", [1, 2, 4, 8])
def test_uniform_description_is_todays_grid(lib, n_rep):
    msg = ctypes.create_string_buffer(256)
    for bsz in (1, 2, 3, 4, 17, MAX_SEQ, 100):
        for q_len in edge_lens(n_rep) + [257]:
            for kv_heads in (1, 8):
                rc = lib.pr_check_uniform(bsz, q_len, 37, kv_heads, n_rep, msg, len(msg))
                assert rc == 0, f"{msg.value.decode()}: bsz {bsz} q_len {q_len} kv {kv_heads} n_rep {n_rep}"
