"""Llama shapes of the BASELINE configs (SURVEY.md section 8).  Torch-free on purpose: bench.py's `--impl reference`
arm imports this and nothing else of the package, so that arm loads none of this repo's native code."""
from dataclasses import dataclass
from typing import Optional


@dataclass
class LlamaShape:
    name: str
    hidden: int
    inter: int
    layers: int
    heads: int
    head_dim: int = 128
    vocab: int = 32000
    eps: float = 1e-6
    kv_heads: Optional[int] = None      # grouped-query attention (config num_key_value_heads, model.py:62-67); None: = heads

    def __post_init__(self):
        if self.kv_heads is None:
            self.kv_heads = self.heads
        if self.kv_heads < 1 or self.heads % self.kv_heads:
            raise ValueError(f"{self.name}: kv_heads ({self.kv_heads}) must divide heads ({self.heads})")


SHAPES = {
    "7b": LlamaShape("llama-7b", 4096, 11008, 32, 32),
    "13b": LlamaShape("llama-13b", 5120, 13824, 40, 40),
    "33b": LlamaShape("llama-33b", 6656, 17920, 60, 52),
    "65b": LlamaShape("llama-65b", 8192, 22016, 80, 64),
}

# Grouped-query attention models.  Kept out of SHAPES: bench.py's roofline counts KV bytes and its CPU-baseline k/v projections
# as if kv_heads == heads, so bench.py --model 70b would print a wrong roofline.  tools/step_bench.py and tools/step_trace.py
# accept these names.
GQA_SHAPES = {
    "70b": LlamaShape("llama-2-70b", 8192, 28672, 80, 64, kv_heads=8, eps=1e-5),
}


def q4_bytes(K, N, gs, M=1, act=False, accumulate=False):
    """Algorithmic bytes of one q4_matmul (SURVEY.md 8d)."""
    return K * N // 2 + 2 * (K // gs) * N + 4 * (K // gs) * (N // 8) + 2 * M * K + 2 * M * N * (2 if accumulate else 1) + (4 * K if act else 0)
