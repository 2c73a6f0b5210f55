#!/usr/bin/env python
"""Stage the UNMODIFIED reference for the drop-in run (VERDICT r1 item 4, SURVEY.md 8d "model level").

A GPU machine need not have the reference checkout, so the reference's Python files, its extension sources and its sample dataset
are copied verbatim into the git-ignored `baseline/_ref/exllama/` (it travels with the working tree, it never enters the
history), and its extension is built ahead of time, from those copies, into
`baseline/_ref/exllama_ext_ref.so` with exactly the flags cuda_ext.py:43-64 passes plus the sm_90a gencode
(the reference passes no arch flags; on the GPU box torch would add the detected arch itself).

Run with the reference checkout:  EXLLAMA_REFERENCE=<path> python tools/stage_reference.py
"""
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("EXLLAMA_REFERENCE", "")
DST = os.path.join(ROOT, "baseline", "_ref", "exllama")
EXT_SO = os.path.join(ROOT, "baseline", "_ref", "exllama_ext_ref.so")

PY_FILES = ["model.py", "tokenizer.py", "generator.py", "alt_generator.py", "lora.py", "perplexity.py", "model_init.py", "globals.py",
            "cuda_ext.py", "test_benchmark_inference.py"]


def stage(force=False):
    if not os.path.isdir(REF):
        print(f"stage_reference: EXLLAMA_REFERENCE={REF!r} is not a reference checkout -- using what is already staged", file=sys.stderr)
        return os.path.exists(EXT_SO)
    os.makedirs(DST, exist_ok=True)
    for f in PY_FILES:
        shutil.copy2(os.path.join(REF, f), os.path.join(DST, f))
    for d in ("exllama_ext", "datasets"):
        dst = os.path.join(DST, d)
        if os.path.isdir(dst):
            shutil.rmtree(dst)
        shutil.copytree(os.path.join(REF, d), dst)
    srcs = ["exllama_ext/exllama_ext.cpp", "exllama_ext/cuda_buffers.cu", "exllama_ext/cuda_func/q4_matrix.cu",
            "exllama_ext/cuda_func/q4_matmul.cu", "exllama_ext/cuda_func/column_remap.cu", "exllama_ext/cuda_func/rms_norm.cu",
            "exllama_ext/cuda_func/rope.cu", "exllama_ext/cuda_func/half_matmul.cu", "exllama_ext/cuda_func/q4_attn.cu",
            "exllama_ext/cuda_func/q4_mlp.cu", "exllama_ext/cpu_func/rep_penalty.cpp"]       # cuda_ext.py:45-57
    newest = max(os.path.getmtime(os.path.join(DST, s)) for s in srcs)
    if not force and os.path.exists(EXT_SO) and os.path.getmtime(EXT_SO) >= newest:
        return True
    import torch
    from torch.utils import cpp_extension as ce
    build_dir = os.path.join(ROOT, "baseline", "_ref", "ext_build")
    os.makedirs(build_dir, exist_ok=True)
    import sysconfig
    inc = ce.include_paths("cuda") + [sysconfig.get_paths()["include"], os.path.join(DST, "exllama_ext")]
    abi = "-D_GLIBCXX_USE_CXX11_ABI=" + str(int(torch._C._GLIBCXX_USE_CXX11_ABI))
    common = ["-DTORCH_EXTENSION_NAME=exllama_ext", "-DTORCH_API_INCLUDE_EXTENSION_H", abi, "-std=c++17"]
    objs, procs = [], []
    for s in srcs:
        src = os.path.join(DST, s)
        obj = os.path.join(build_dir, os.path.basename(s) + ".o")
        objs.append(obj)
        if s.endswith(".cu"):
            cmd = ["nvcc", "-O3", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr",
                   "-D__CUDA_NO_HALF_OPERATORS__", "-D__CUDA_NO_HALF_CONVERSIONS__", "-D__CUDA_NO_BFLOAT16_CONVERSIONS__",
                   "-D__CUDA_NO_HALF2_OPERATORS__", "-Xcompiler", "-fPIC"] + common + sum((["-isystem", i] for i in inc), []) + ["-c", src, "-o", obj]
        else:
            cmd = ["g++", "-O3", "-fPIC"] + common + sum((["-isystem", i] for i in inc), []) + ["-c", src, "-o", obj]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError("reference extension build failed: " + " ".join(cmd) + "\n" + out.decode())
    torch_lib = os.path.join(os.path.dirname(torch.__file__), "lib")
    cuda_lib = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "lib64")
    subprocess.check_call(["g++", "-shared", "-o", EXT_SO] + objs + ["-L" + torch_lib, "-L" + cuda_lib, "-lc10", "-lc10_cuda", "-ltorch_cpu",
                           "-ltorch_cuda", "-ltorch", "-ltorch_python", "-lcudart", "-lcublas", "-Wl,-rpath," + torch_lib])
    return True


if __name__ == "__main__":
    ok = stage(force="--force" in sys.argv)
    print("staged" if ok else "not staged", DST, EXT_SO)
