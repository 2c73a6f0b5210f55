"""Kernel timeline of one graph-replayed decode step (CUPTI through torch.profiler): start, duration and the gap to the
previous kernel for every launch of a few layers, plus per-kernel totals.  Diagnostic only (CUPTI adds overhead).
Caution: the second time this ran on the GPU box it produced no output for 300 s and was killed by its timeout (cause not
established; kineto + graph-launched cluster/PDL kernels is an unusual mix) -- always run it under `timeout`."""
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from exllama_b200.stack import SHAPES, DecodeStack  # noqa: E402

shape = SHAPES["7b"]
stack = DecodeStack(shape, max_seq=2048)
if "--torch-attn" in sys.argv:
    stack.fused_decode_attn = False
hidden0 = (torch.randn((1, 1, shape.hidden), device="cuda") * 0.5).half()
hidden = hidden0.clone()
for kc, vc in zip(stack.key_cache, stack.value_cache):
    kc.normal_(0, 0.5); vc.normal_(0, 0.5)


def step():
    hidden.copy_(hidden0)
    return stack.decode_step(hidden, 1920)


for _ in range(3):
    step()
torch.cuda.synchronize()
g = torch.cuda.CUDAGraph()
with torch.cuda.graph(g):
    step()
for _ in range(3):
    g.replay()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    g.replay()
    torch.cuda.synchronize()
path = os.path.join(tempfile.mkdtemp(), "timeline_trace.json")
print("trace", path)
prof.export_chrome_trace(path)
ev = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel"]
ev.sort(key=lambda e: e["ts"])
t0 = ev[0]["ts"]
print("kernels", len(ev), "span_us", round(ev[-1]["ts"] + ev[-1]["dur"] - t0, 1))
prev_end = None
tot = {}
for i, e in enumerate(ev):
    name = e["name"][:60]
    gap = (e["ts"] - prev_end) if prev_end is not None else 0.0
    tot.setdefault(name, [0, 0.0, 0.0])
    tot[name][0] += 1; tot[name][1] += e["dur"]; tot[name][2] += gap
    if 5 * 8 <= i < 5 * 8 + 12:
        print(f"{e['ts'] - t0:9.2f} dur {e['dur']:7.2f} gap {gap:6.2f}  {name}")
    prev_end = max(prev_end or 0, e["ts"] + e["dur"])
import statistics
byname = {}
starts = {}
for i, e in enumerate(ev):
    byname.setdefault(e["name"][:60], []).append(e["dur"])
    if i + 1 < len(ev):
        starts.setdefault(e["name"][:60], []).append(ev[i + 1]["ts"] - e["ts"])
for k, v in byname.items():
    if len(v) >= 32:
        st = starts[k]
        print(k[:50], "dur min/med/max", round(min(v), 1), round(statistics.median(v), 1), round(max(v), 1),
              "| start-to-next-start min/med/max", round(min(st), 1), round(statistics.median(st), 1), round(max(st), 1))
        print("   ", [round(x, 1) for x in st[:40]])
print()
for k, (n, d, gp) in sorted(tot.items(), key=lambda kv: -kv[1][1]):
    print(f"{n:4d} x  dur {d / n:7.2f} us  gap-before {gp / n:6.2f} us  {k}")
os.remove(path)
