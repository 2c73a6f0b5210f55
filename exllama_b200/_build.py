"""In-tree build of the native pieces (sm_90a only).

  libexl_b200.so      : nvcc, all kernels + the C ABI, no torch dependency
  exllama_ext*.so     : torch C++ extension (pybind shim, g++ only) linked against libexl_b200.so

Both land next to this file, so the package imports straight from the source tree.
"""
from __future__ import annotations

import os
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_SO = os.path.join(HERE, "libexl_b200.so")
EXT_SO = os.path.join(HERE, "exllama_ext.so")

CU_SOURCES = ["capi.cu", "q4_gemv.cu", "q4_matrix.cu", "elementwise.cu", "half_matmul.cu", "q4_gemm_tc.cu", "decode_attn.cu", "decode_step.cu",
              "prefill_attn.cu", "sample.cu", "logprob.cu", "beam.cu"]
HEADERS = ["exl_common.cuh", "sample_select.cuh", "decode_step_sched.h", "prefill_attn_sched.h", "logprob_sched.h",
           os.path.join("..", "..", "include", "exl_b200.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = "arch=compute_90a,code=sm_90a"          # H100 (Hopper): wgmma, TMA, clusters
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-gencode", ARCH,
              "-Xcompiler", "-fPIC"]


def _newer(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build_lib(force: bool = False, verbose: bool = False) -> str:
    srcs = [os.path.join(CSRC, s) for s in CU_SOURCES]
    deps = srcs + [os.path.join(CSRC, h) for h in HEADERS]
    if force or _newer(LIB_SO, deps):
        objs = []
        procs = []
        os.makedirs(os.path.join(HERE, "_obj"), exist_ok=True)
        for s in srcs:
            o = os.path.join(HERE, "_obj", os.path.basename(s) + ".o")
            objs.append(o)
            if force or _newer(o, [s] + deps[len(srcs):]):
                cmd = [NVCC] + NVCC_FLAGS + ["-c", s, "-o", o]
                if verbose:
                    print(" ".join(cmd))
                procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        for cmd, p in procs:
            out, _ = p.communicate()
            if p.returncode != 0:
                raise RuntimeError("nvcc failed: " + " ".join(cmd) + "\n" + out.decode())
        cmd = [NVCC, "-shared", "-gencode", ARCH, "-o", LIB_SO] + objs + ["-lcublas"]
        subprocess.check_call(cmd)
    return LIB_SO


def build_ext(force: bool = False, verbose: bool = False) -> str:
    """The pybind shim is plain C++ (no kernels): compile with g++ against torch headers."""
    build_lib(force=force, verbose=verbose)
    src = os.path.join(CSRC, "pybind_shim.cpp")
    if not (force or _newer(EXT_SO, [src, os.path.join(HERE, "..", "include", "exl_b200.h")])):
        return EXT_SO
    import torch  # noqa: F401
    from torch.utils import cpp_extension as ce
    inc = ce.include_paths() + [sysconfig.get_paths()["include"], "/usr/local/cuda/include"]
    torch_lib = os.path.join(os.path.dirname(torch.__file__), "lib")
    cmd = ["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-DTORCH_EXTENSION_NAME=exllama_ext",
           "-DTORCH_API_INCLUDE_EXTENSION_H", "-D_GLIBCXX_USE_CXX11_ABI=" + str(int(torch._C._GLIBCXX_USE_CXX11_ABI))]
    for i in inc:
        cmd += ["-isystem", i]
    cmd += [src, "-o", EXT_SO, "-L" + HERE, "-lexl_b200", "-L" + torch_lib, "-lc10", "-lc10_cuda", "-ltorch_cpu",
            "-ltorch_cuda", "-ltorch", "-ltorch_python", "-Wl,-rpath,$ORIGIN", "-Wl,-rpath," + torch_lib]
    if verbose:
        print(" ".join(cmd))
    subprocess.check_call(cmd)
    return EXT_SO


def build_all(force: bool = False, verbose: bool = False) -> None:
    build_lib(force, verbose)
    build_ext(force, verbose)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose=True)
    print("built", LIB_SO, EXT_SO)
