"""CPU proof of the persistent decode kernel's schedule under grouped-query attention (kv_heads < heads).

tests/decode_sched_check_gqa.cpp (which includes the multi-head checker, tests/decode_sched_check.cpp) compiles
exllama_b200/csrc/decode_step_sched.h -- the header decode_step.cu includes -- with g++.
Its ds_check_gqa / ds_plan_gqa entry points check, for a shape with kv_heads KV heads: the QKV tiles of three matrices of unequal
width and their accumulator columns [HQ | HKV | HKV], attention units of (KV head, 16-position chunk), the partial-slot table of
every query head (its CTA range is that of its KV head), the act-order staging slots, lm_head coverage and the shared-memory plan
with the attention scratch on the x staging area.  Also: the Python shapes and the ctypes mirror of exl_decode_desc.
"""
import ctypes
import os
import subprocess

import pytest

from exllama_b200.shapes import GQA_SHAPES, SHAPES, LlamaShape

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SMEM_OPTIN = 232448          # cudaDevAttrMaxSharedMemoryPerBlockOptin on sm_90 (227 KB)
SMS = 132                    # H100 SXM


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("sched_gqa") / "libdecode_sched_check.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wall", "-Werror",
                           os.path.join(HERE, "decode_sched_check_gqa.cpp"), "-o", so])
    lib = ctypes.CDLL(so)
    tail = [ctypes.c_longlong, ctypes.c_char_p, ctypes.c_int, ctypes.POINTER(ctypes.c_longlong), ctypes.POINTER(ctypes.c_int)]
    lib.ds_check.restype = lib.ds_check_gqa.restype = ctypes.c_int
    lib.ds_check.argtypes = [ctypes.c_int] * 9 + tail
    lib.ds_check_gqa.argtypes = [ctypes.c_int] * 10 + tail
    plan_tail = [ctypes.c_longlong, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_longlong), ctypes.POINTER(ctypes.c_int)]
    lib.ds_plan.restype = lib.ds_plan_gqa.restype = ctypes.c_int
    lib.ds_plan.argtypes = [ctypes.c_int] * 6 + plan_tail
    lib.ds_plan_gqa.argtypes = [ctypes.c_int] * 7 + plan_tail
    return lib


def check(lib, H, I, heads, kv_heads, vocab, grid, past_lo, past_hi, act):
    msg = ctypes.create_string_buffer(512)
    gaps, resets = ctypes.c_longlong(), ctypes.c_int()
    rc = lib.ds_check_gqa(H, heads * 128, I, heads, kv_heads, vocab, grid, past_lo, past_hi, int(act), SMEM_OPTIN, msg, len(msg),
                          ctypes.byref(gaps), ctypes.byref(resets))
    return rc, msg.value.decode(), gaps.value, resets.value


def plan(lib, H, I, heads, kv_heads, act, grid=SMS):
    depth, smem, slots = ctypes.c_int(), ctypes.c_longlong(), ctypes.c_int()
    rc = lib.ds_plan_gqa(H, heads * 128, I, heads, kv_heads, grid, int(act), SMEM_OPTIN, ctypes.byref(depth), ctypes.byref(smem), ctypes.byref(slots))
    return rc, depth.value, smem.value, slots.value


S70 = GQA_SHAPES["70b"]


def test_70b_every_context_length(lib):
    rc, msg, _, _ = check(lib, S70.hidden, S70.inter, S70.heads, S70.kv_heads, S70.vocab, SMS, 0, 4095, act=False)
    assert rc == 0, msg


@pytest.mark.parametrize("grid", [64, 100])
def test_70b_other_grids(lib, grid):
    rc, msg, _, _ = check(lib, S70.hidden, S70.inter, S70.heads, S70.kv_heads, S70.vocab, grid, 0, 600, act=False)
    assert rc == 0, f"grid {grid}: {msg}"


def test_70b_act_order(lib):
    rc, msg, _, _ = check(lib, S70.hidden, S70.inter, S70.heads, S70.kv_heads, S70.vocab, SMS, 0, 4095, act=True)
    assert rc == 0, msg


TINY = [(1024, 2816, 8, 1), (1024, 2816, 8, 2), (1024, 2816, 8, 4), (2048, 5632, 16, 2)]


@pytest.mark.parametrize("act", [False, True])
@pytest.mark.parametrize("H,I,heads,kv", TINY)
def test_tiny_gqa_shapes(lib, H, I, heads, kv, act):
    # partition, cta_of inverse, slot table of every query head, <= 2 matrices per act-order range, lm_head coverage, ATT units
    # == kv_heads * max(1, ceil(ctx / 16)), combine reads only written slots unless the table is reset -- at every context
    for vocab in (0, 512):
        rc, msg, _, _ = check(lib, H, I, heads, kv, vocab, SMS, 0, 300, act)
        assert rc == 0, f"{(H, I, heads, kv, vocab, act)}: {msg}"


def test_70b_reset_confined_to_short_contexts(lib):
    """Under GQA 16 CTAs share a KV head (128 of 132 CTAs for 70B).  Stale partial slots exist only while the attention units are
    fewer than those CTAs, and there the host resets the table; from then on nothing extra is launched."""
    G = min(SMS, S70.kv_heads * 16)
    want = sum(1 for past in range(4096) if (past + 15) // 16 >= 2 and S70.kv_heads * ((past + 15) // 16) < G)
    assert want == 224                                   # contexts 17 .. 240
    rc, msg, gaps, resets = check(lib, S70.hidden, S70.inter, S70.heads, S70.kv_heads, S70.vocab, SMS, 0, 4095, False)
    assert rc == 0, msg
    assert gaps > 0 and resets == want
    rc, msg, gaps, resets = check(lib, S70.hidden, S70.inter, S70.heads, S70.kv_heads, S70.vocab, SMS, 241, 4095, False)
    assert rc == 0 and gaps == 0 and resets == 0


@pytest.mark.parametrize("act", [False, True])
def test_70b_plan_fits(lib, act):
    rc, depth, smem, slots = plan(lib, S70.hidden, S70.inter, S70.heads, S70.kv_heads, act)
    assert rc == 0
    assert depth >= 2, depth
    assert smem + 2048 <= SMEM_OPTIN
    assert slots == 16 + 2


@pytest.mark.parametrize("name", ["7b", "13b", "33b", "65b"])
def test_mha_entry_points_unchanged(lib, name):
    """kv_heads == heads through the GQA entry points is exactly the multi-head schedule and plan."""
    s = SHAPES[name]
    for act in (False, True):
        a = plan(lib, s.hidden, s.inter, s.heads, s.heads, act)
        depth, smem, slots = ctypes.c_int(), ctypes.c_longlong(), ctypes.c_int()
        lib.ds_plan(s.hidden, s.hidden, s.inter, s.heads, SMS, int(act), SMEM_OPTIN, ctypes.byref(depth), ctypes.byref(smem), ctypes.byref(slots))
        assert a == (0, depth.value, smem.value, slots.value)
        msg = ctypes.create_string_buffer(512)
        gaps, resets = ctypes.c_longlong(), ctypes.c_int()
        rc = lib.ds_check(s.hidden, s.hidden, s.inter, s.heads, s.vocab, SMS, 0, 300, int(act), SMEM_OPTIN, msg, len(msg), ctypes.byref(gaps), ctypes.byref(resets))
        assert check(lib, s.hidden, s.inter, s.heads, s.heads, s.vocab, SMS, 0, 300, act) == (rc, msg.value.decode(), gaps.value, resets.value)


def test_rejects_bad_kv_heads(lib):
    rc, msg, _, _ = check(lib, 1024, 2816, 8, 3, 512, SMS, 0, 4, False)        # heads % kv_heads != 0
    assert rc == 1 and "kv_heads" in msg
    rc, msg, _, _ = check(lib, 1024, 2816, 8, 16, 512, SMS, 0, 4, False)       # more KV heads than heads
    assert rc == 1 and "kv_heads" in msg
    assert plan(lib, 1024, 2816, 8, 3, False)[0] == 1
    with pytest.raises(ValueError):
        LlamaShape("bad", 1024, 2816, 2, 8, kv_heads=3)


def test_shapes():
    assert LlamaShape("x", 1024, 2816, 2, 8).kv_heads == 8
    assert LlamaShape("x", 1024, 2816, 2, 8, vocab=2048).kv_heads == 8
    want = {"7b": ("llama-7b", 4096, 11008, 32, 32), "13b": ("llama-13b", 5120, 13824, 40, 40),
            "33b": ("llama-33b", 6656, 17920, 60, 52), "65b": ("llama-65b", 8192, 22016, 80, 64)}
    assert list(SHAPES) == list(want)
    for k, (name, hidden, inter, layers, heads) in want.items():
        s = SHAPES[k]
        assert (s.name, s.hidden, s.inter, s.layers, s.heads, s.head_dim, s.vocab, s.eps, s.kv_heads) == \
            (name, hidden, inter, layers, heads, 128, 32000, 1e-6, heads)
    assert "70b" not in SHAPES
    assert (S70.hidden, S70.inter, S70.layers, S70.heads, S70.kv_heads, S70.eps) == (8192, 28672, 80, 64, 8, 1e-5)


def test_decode_desc_layout_matches_c(tmp_path):
    """ctypes' _DecodeDesc has the size of the C struct and num_kv_heads where C puts it (appended as the last field)."""
    from exllama_b200.capi import _DecodeDesc
    src = tmp_path / "probe.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "exl_b200.h"\n'
                   'int main(void) { printf("%zu %zu\\n", sizeof(exl_decode_desc), offsetof(exl_decode_desc, num_kv_heads)); return 0; }\n')
    exe = tmp_path / "probe"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    size, off = map(int, subprocess.check_output([str(exe)]).split())
    assert ctypes.sizeof(_DecodeDesc) == size
    assert _DecodeDesc.num_kv_heads.offset == off
    assert _DecodeDesc._fields_[-1][0] == "num_kv_heads"
