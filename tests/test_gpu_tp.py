"""Tensor-parallel GPU parity (needs >= 2 GPUs on one machine; skipped otherwise).
tools/tp_check.py under torchrun: identical full GPTQ tensors on every rank -> column / row shards ->
(a) q4_attn_2_tp / q4_mlp_tp + NCCL all-reduce and (b) the fused GEMV + NVLink one-shot all-reduce kernels, both against
the single-rank float64 oracle; (b) additionally bitwise identical on every rank, over 60 back-to-back launches and 30
CUDA-graph replays, with zero flag time-outs."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gpus():
    import torch
    return torch.cuda.device_count()


@pytest.mark.parametrize("world", [2, 4])
def test_tp_check_under_torchrun(world):
    if _gpus() < world:
        pytest.skip(f"needs {world} GPUs")
    env = dict(os.environ); env.pop("OMP_NUM_THREADS", None)
    p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
                        "--master-port", str(29600 + world), os.path.join(ROOT, "tools", "tp_check.py")],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600, env=env, cwd=ROOT)
    tail = p.stdout[-3000:]
    assert p.returncode == 0, tail
    assert f"tp_check world={world}" in p.stdout and "-> OK" in p.stdout, tail


@pytest.mark.parametrize("world", [2])
def test_tp_fused_decode_step_under_torchrun(world):
    """csrc/decode_step.cu with tp_world > 1 (peer-memory reductions + cross-GPU barrier inside the kernel) against the per-op
    tensor-parallel path on the same sharded stack (tools/tp_step_check.py)."""
    if _gpus() < world:
        pytest.skip(f"needs {world} GPUs")
    env = dict(os.environ); env.pop("OMP_NUM_THREADS", None)
    p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
                        "--master-port", str(29700 + world), os.path.join(ROOT, "tools", "tp_step_check.py"), "--layers", "3"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600, env=env, cwd=ROOT)
    tail = p.stdout[-3000:]
    assert p.returncode == 0, tail
    assert f"tp_step_check world={world} -> OK" in p.stdout, tail
