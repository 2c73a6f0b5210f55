#!/usr/bin/env python
"""Drop-in demonstration (VERDICT r1 item 4 / row N1): run the reference's UNCHANGED test_benchmark_inference.py
(test_benchmark_inference.py:161-222: `-p` perf and `-ppl` perplexity) on a synthetic model directory,
once over the reference's own extension and once over this repo's, and compare what it prints.

    python tools/run_dropin.py --model-dir /tmp/synth7b [--exts ref,ours] [--out dropin.json] [-- extra args]

The reference's files are the verbatim copies staged by tools/stage_reference.py under baseline/_ref/exllama/ (a GPU machine
need not have the reference checkout).  Nothing in them is edited; the harness only prepares the interpreter before running the script:
  ours : sys.modules["cuda_ext"] = exllama_b200.cuda_ext            (INTEGRATION.md 1a)
  ref  : the pre-built reference extension is registered as `exllama_ext` and torch.utils.cpp_extension.load is made to
         return it, so the reference's cuda_ext.py imports unchanged without a 40 s JIT compile (and without
         tripping over torch >= 2.11 no longer leaving JIT modules importable by name, SURVEY.md 8c caveat 1).
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFDIR = os.path.join(ROOT, "baseline", "_ref", "exllama")
REF_SO = os.path.join(ROOT, "baseline", "_ref", "exllama_ext_ref.so")


def child(ext, script_args):
    import importlib.util
    import runpy
    sys.path.insert(0, ROOT)
    sys.path.insert(0, REFDIR)
    os.chdir(REFDIR)                       # the script opens datasets/... relative to its own directory
    import torch  # noqa: F401
    if ext == "ours":
        import exllama_b200.cuda_ext as ce
        sys.modules["cuda_ext"] = ce
    else:
        spec = importlib.util.spec_from_file_location("exllama_ext", REF_SO)
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
        sys.modules["exllama_ext"] = m
        import torch.utils.cpp_extension as cpp
        cpp.load = lambda *a, **k: m
    sys.argv = ["test_benchmark_inference.py"] + script_args
    runpy.run_path(os.path.join(REFDIR, "test_benchmark_inference.py"), run_name="__main__")
    if ext == "ours":
        from exllama_b200 import capi
        print(f" ** exl_b200 launches: {capi.launch_count()} last_q4_path: {capi.last_q4_path()}")


def parse(out):
    speeds = [float(x) for x in re.findall(r"\*\* Speed: ([0-9.]+) tokens/second", out)]
    ppl = re.findall(r"\*\* Perplexity[^:]*: ([0-9.eE+-]+|nan|inf)", out)
    r = {"prompt_tok_s": speeds[0] if len(speeds) > 0 else None,
         "gen_tok_s_ctx1920": speeds[1] if len(speeds) > 1 else None,
         "gen_tok_s_ctx4": speeds[2] if len(speeds) > 2 else None,
         "perplexity": float(ppl[0]) if ppl else None}
    m = re.search(r"exl_b200 launches: (\d+) last_q4_path: (\w+)", out)
    if m:
        r["exl_b200_launches"] = int(m.group(1)); r["last_q4_path"] = m.group(2)
    return r


def main():
    if "--child" in sys.argv:
        i = sys.argv.index("--child")
        return child(sys.argv[i + 1], sys.argv[i + 2:])
    ap = argparse.ArgumentParser()
    ap.add_argument("--model-dir", required=True)
    ap.add_argument("--exts", default="ref,ours")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "dropin.json"))
    ap.add_argument("--length", type=int, default=2048)
    ap.add_argument("--ppl-chunks", type=int, default=None, help="default: the script's own default (100)")
    ap.add_argument("--no-ppl", action="store_true")
    ap.add_argument("--tag", default="")
    ap.add_argument("rest", nargs="*")
    args = ap.parse_args()
    script_args = ["-d", args.model_dir, "-p", "-l", str(args.length)] + ([] if args.no_ppl else ["-ppl"])
    if args.ppl_chunks:
        script_args += ["-ppl_cn", str(args.ppl_chunks)]
    script_args += args.rest
    res = {"script": "test_benchmark_inference.py (unchanged, baseline/_ref/exllama)", "args": script_args, "tag": args.tag}
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    for ext in args.exts.split(","):
        t0 = time.time()
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", ext] + script_args, stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, text=True)
        log = os.path.splitext(args.out)[0] + f"_{ext}.log"
        open(log, "w").write(p.stdout)
        r = parse(p.stdout)
        r["returncode"] = p.returncode; r["wall_s"] = round(time.time() - t0, 1)
        if p.returncode != 0:
            r["tail"] = p.stdout[-1500:]
        res[ext] = r
        print(ext, json.dumps(r), flush=True)
    if res.get("ref", {}).get("perplexity") and res.get("ours", {}).get("perplexity"):
        a, b = res["ref"]["perplexity"], res["ours"]["perplexity"]
        res["ppl_rel_diff"] = abs(a - b) / abs(a)
        for k in ("prompt_tok_s", "gen_tok_s_ctx1920", "gen_tok_s_ctx4"):
            if res["ref"].get(k) and res["ours"].get(k):
                res["speedup_" + k] = round(res["ours"][k] / res["ref"][k], 3)
    json.dump(res, open(args.out, "w"), indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
