"""The whole-token persistent kernel (csrc/decode_step.cu) against (a) the oracle composition of the reference's decode
path -- rms_norm, q4_matmul, rope, cache update, attention, residual adds, silu*mul, final norm, lm_head, each restated
from the reference file:line the oracle cites -- and (b) this repo's own per-op kernels driven as model.py drives them
(DecodeStack.decode_step), on the same seeded synthetic GPTQ stack."""
import numpy as np
import pytest

from stack_harness import (check_fused_step, check_reset_after_long_context, check_sequence_and_graph, lib_state,  # noqa: F401
                           stacks)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("gs,act", [(128, False), (32, False), (256, False), (128, True), (32, True)])
@pytest.mark.parametrize("past", [0, 1, 16, 37, 200])
def test_fused_step_vs_oracle_and_per_op_path(oracle, stacks, gs, act, past):
    import torch
    st = stacks(gs=gs, act=act)
    st.make_plan()
    info = st.dplan.info()
    assert info["grid"] >= 100 and info["ring_stages"] >= 8, info
    rng = np.random.default_rng(past + gs)
    x = (rng.standard_normal(st.shape.hidden) * 0.5).astype(np.float16)
    check_fused_step(oracle, st, torch.from_numpy(x).cuda().view(1, 1, -1), [past], f"g{gs} act {act}")


def test_fused_step_sequence_and_graph(oracle, stacks):
    """Five consecutive tokens (barrier generation, accumulator clean-up and the cache rows carry over between launches),
    then the same launch replayed from a CUDA graph: bit-identical KV rows are not required (fp32 atomics), logits agree."""
    import torch
    st = stacks(layers=3, max_seq=128, seed=5)
    st.make_plan()
    g = torch.Generator(device="cuda"); g.manual_seed(9)
    xs = [(torch.randn((1, 1, 1024), device="cuda", generator=g) * 0.5).half() for _ in range(5)]
    check_sequence_and_graph(st, xs, [40])


def test_fused_step_short_context_after_long_one(oracle, stacks):
    """ONE plan: a long context first (every slot of the attention-partial table gets written), then short contexts where some CTAs
    inside a head's CTA range own no attention unit (tests/test_decode_schedule.py: the hazard the CPU schedule proof found).
    Partials of the long context must not leak into the short contexts' softmax combine: exl_decode_step resets the table first."""
    import torch
    st = stacks(seed=7)
    st.make_plan()
    g = torch.Generator(device="cuda"); g.manual_seed(21)
    # 8 heads -> 56 CTAs take part in the attention phase; 16-position chunks: contexts 17 .. 96 leave some of them idle
    contexts = [[200], [37], [17], [100], [49], [3], [96], [200]]
    xs = [(torch.randn((1, 1, 1024), device="cuda", generator=g) * 0.5).half() for _ in contexts]
    check_reset_after_long_context(st, xs, contexts)


def test_fused_step_7b_shape_long_context(oracle, stacks):
    """BASELINE shape (hidden 4096, inter 11008, 32 heads, vocab 32000) at ctx 1920, 2 layers: against the per-op path."""
    import torch
    st = stacks(hidden=4096, inter=11008, heads=32, max_seq=2048, vocab=32000, seed=11)
    st.make_plan()
    x = (torch.randn((1, 1, 4096), device="cuda") * 0.5).half()
    check_fused_step(None, st, x, [1920], "7B shape")


def test_fused_step_act_order_13b_shape(oracle, stacks):
    """BASELINE config 3 shape (hidden 5120, inter 13824, 40 heads, act-order), 2 layers at ctx 1920: against the per-op path."""
    import torch
    st = stacks(hidden=5120, inter=13824, heads=40, max_seq=2048, vocab=32000, seed=13, act=True)
    st.make_plan()
    x = (torch.randn((1, 1, 5120), device="cuda") * 0.5).half()
    check_fused_step(None, st, x, [1920], "13B shape, act-order")
