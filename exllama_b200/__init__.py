"""exllama_b200 -- H100 (sm_90a) implementation of the exllama_ext operator surface.

Layout:
  csrc/            hand-written CUDA kernels + the C ABI (include/exl_b200.h) + the pybind shim
  capi.py          ctypes binding of libexl_b200.so (raw pointers; used by tests and bench)
  cuda_ext.py      drop-in mirror of the reference's cuda_ext.py (same ext_* wrappers, same module attributes)
  tp.py            tensor-parallel sharding of GPTQ tensors + the per-projection all-reduce
  _build.py        in-tree build of libexl_b200.so and the `exllama_ext` torch extension
"""
__version__ = "0.1.0"
