"""CPU checks of token log-probabilities (exl_token_logprobs):

- oracle/logprob_oracle.py against scipy.special.log_softmax: logprob, lse, greedy with its tie rule, the NaN rules, and the torch
  program it is compared with on the GPU;
- the work list of token_logprob_kernel (exllama_b200/csrc/logprob_sched.h), compiled with g++ (tests/logprob_sched_check.cpp):
  every (row tile, vocab tile) computed exactly once, partial slots unique and inside the work size, every slot written read by the
  combine, for T 1 .. 4096 and V 1 .. 152064 at several SM counts;
- the C entry points reject bad arguments and fail loudly without a GPU (no CPU fallback).
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


def _inputs(T, H, V, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    hn = torch.randn((T, H), generator=g).half()
    lm = (torch.randn((V, H), generator=g) * 0.05).half()
    y = torch.randint(0, V, (T,), generator=g)
    return hn, lm, y


@pytest.mark.parametrize("T,H,V", [(1, 64, 1), (3, 64, 7), (17, 128, 300), (40, 192, 1000)])
def test_oracle_matches_scipy(T, H, V):
    import torch
    from scipy.special import log_softmax
    from oracle.logprob_oracle import logprobs64
    hn, lm, y = _inputs(T, H, V, seed=T + V)
    o = logprobs64(hn, lm, y)
    logits = hn.double().numpy() @ lm.double().numpy().T
    ls = log_softmax(logits, axis=1)
    np.testing.assert_allclose(o["logprob"].numpy(), ls[np.arange(T), y.numpy()], rtol=0, atol=1e-12)
    np.testing.assert_allclose(o["lse"].numpy(), logits[:, 0] - ls[:, 0], rtol=0, atol=1e-12)
    np.testing.assert_array_equal(o["greedy"].numpy(), logits.argmax(axis=1))
    assert bool((o["bound"] > 0).all()) and bool((o["gbound"] > 0).all())
    # the bound covers a float32 evaluation of the same sums
    f32 = torch.from_numpy((hn.float() @ lm.float().t()).numpy())
    assert bool(((f32.double() - torch.from_numpy(logits)).abs().max(dim=1).values <= o["gbound"] / 2).all())


def test_oracle_tie_rule_and_undefined_rows():
    import torch
    from oracle.logprob_oracle import logprobs64
    hn, lm, y = _inputs(6, 64, 50, seed=1)
    lm[9] = lm[31] = lm[44] = (hn[0].float() * 0.5).half()           # three equal maxima of row 0
    y[1], y[2] = -1, 50                                               # targets outside [0, V)
    hn[3, 5] = float("nan"); hn[4, 0] = float("inf")
    o = logprobs64(hn, lm, y)
    assert int(o["greedy"][0]) == 9 and float(o["margin"][0]) == 0.0
    assert torch.isnan(o["logprob"][1:5]).all() and torch.isfinite(o["logprob"][[0, 5]]).all()
    assert o["greedy"][3] == -1 and o["greedy"][4] == -1 and o["greedy"][1] >= 0 and o["greedy"][2] >= 0


def test_torch_program_is_the_reference_rule():
    import torch
    from oracle.logprob_oracle import logprobs64, torch_program
    hn, lm, y = _inputs(8, 128, 333, seed=2)
    o = logprobs64(hn, lm, y)
    got = torch_program(hn.float(), lm.float(), y).double()
    assert float((got - o["logprob"]).abs().max()) < 1e-4


@pytest.fixture(scope="module")
def sched(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("lp_sched") / "liblogprob_sched_check.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wall", "-Werror",
                           os.path.join(HERE, "logprob_sched_check.cpp"), "-o", so])
    lib = C.CDLL(so)
    lib.lp_check.restype = C.c_int
    lib.lp_check.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_longlong), C.c_char_p, C.c_int]
    return lib


def _check(lib, T, V, sms):
    msg = C.create_string_buffer(256)
    wb = C.c_longlong()
    rc = lib.lp_check(T, V, sms, C.byref(wb), msg, len(msg))
    assert rc == 0, f"{msg.value.decode()}: T {T} V {V} sms {sms}"
    return wb.value


TS = [1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512, 1000, 1920, 2048, 4095, 4096]
VS = [1, 2, 255, 256, 257, 511, 513, 32000, 32001, 32016, 32768, 128256, 151936, 152064]


@pytest.mark.parametrize("sms", [132, 114, 1, 7])
def test_schedule_covers_every_tile_once(sched, sms):
    for T in TS:
        for V in VS:
            wb = _check(sched, T, V, sms)
            chunks = wb // (16 * T)
            assert wb == 16 * T * chunks and 1 <= chunks <= -(-V // 256)


def test_schedule_random_shapes(sched):
    rng = np.random.default_rng(5)
    for _ in range(300):
        _check(sched, int(rng.integers(1, 4097)), int(rng.integers(1, 152065)), int(rng.choice([132, 114, 66, 3])))


def test_schedule_shape_of_the_launch(sched):
    """One wave of one CTA per SM whenever the row tiles fit, every lm_head tile shared by all row tiles of its chunk's CTAs."""
    # T 1920 (15 row tiles) at vocab 32000 (125 tiles) on 132 SMs: 8 chunks, 120 CTAs; T 4096: 32 row tiles, 4 chunks
    assert _check(sched, 1920, 32000, 132) == 16 * 1920 * 8
    assert _check(sched, 4096, 32000, 132) == 16 * 4096 * 4
    assert _check(sched, 1, 32000, 132) == 16 * 1 * 125
    assert _check(sched, 17000, 32000, 132) == 16 * 17000 * 1


def test_entry_points_reject_arguments_and_need_a_gpu():
    import torch
    from exllama_b200 import capi
    lib = capi.lib()
    p = C.c_void_p(1 << 20)                     # 16-byte aligned, never dereferenced
    odd = C.c_void_p((1 << 20) + 2)
    args = lambda **kw: [kw.get("hn", p), kw.get("T", 4), kw.get("H", 128), kw.get("lm", p), kw.get("V", 100), kw.get("y", p),
                         kw.get("lp", p), kw.get("g", p), kw.get("w", p), kw.get("wb", 1 << 20), None]
    for bad in (dict(T=0), dict(V=0), dict(H=100), dict(H=0), dict(hn=None), dict(lm=None), dict(y=None), dict(lp=None), dict(g=None),
                dict(w=None), dict(hn=odd), dict(lm=odd), dict(y=odd), dict(lp=odd), dict(g=odd), dict(w=odd)):
        assert lib.exl_token_logprobs(*args(**bad)) == 1, bad
    n = C.c_int64()
    assert lib.exl_token_logprobs_work_size(0, 10, 0, C.byref(n)) == 1
    assert lib.exl_token_logprobs_work_size(1, 0, 0, C.byref(n)) == 1
    if torch.cuda.is_available():
        pytest.skip("GPU present: the no-GPU case does not apply")
    rc = lib.exl_token_logprobs(*args())
    assert rc != 0 and b"no CPU fallback" in lib.exl_last_error()
    rc = lib.exl_token_logprobs_work_size(4, 100, 0, C.byref(n))
    assert rc != 0 and b"no CPU fallback" in lib.exl_last_error()
