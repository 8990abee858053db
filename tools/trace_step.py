"""Kernel timeline of steady-state fold steps (torch.profiler / CUPTI): prints every kernel of two steps with stream, start
and duration, plus the union of busy intervals.  Development aid."""
import json
import os
import sys
import tempfile

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench

if len(sys.argv) > 1:
    bench.LIVE_SLOT_FRACTION = float(sys.argv[1])
wl = bench.FoldStepGPU(0, 1, latency_sms=int(sys.argv[2]) if len(sys.argv) > 2 else 0, workload=sys.argv[3] if len(sys.argv) > 3 else "fib")
wl.start(True)
for _ in range(4):
    wl.step(False)
wl.drain()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    for _ in range(4):
        wl.step(False)
    wl.drain()
    torch.cuda.synchronize()
trace = os.path.join(tempfile.mkdtemp(), "trace.json")
prof.export_chrome_trace(trace)
ev = json.load(open(trace))["traceEvents"]
ks = [e for e in ev if e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset") and "ts" in e]
ks.sort(key=lambda e: e["ts"])
t0 = ks[0]["ts"]
busy, cur_end = 0.0, None
for e in ks:
    s, d = e["ts"], e["dur"]
    if cur_end is None or s > cur_end:
        busy += d
        cur_end = s + d
    elif s + d > cur_end:
        busy += s + d - cur_end
        cur_end = s + d
span = ks[-1]["ts"] + ks[-1]["dur"] - t0
print(f"kernels {len(ks)} span {span/1e3:.3f} ms busy(union) {busy/1e3:.3f} ms  sum {sum(e['dur'] for e in ks)/1e3:.3f} ms")
lim = t0 + span / 2
for e in ks:
    if e["ts"] > lim:
        break
    name = e["name"].split("<")[0].replace("void lurk::", "").replace("lurk::", "")[:34]
    print(f"{(e['ts']-t0)/1e3:9.3f} +{e['dur']/1e3:7.3f} ms  s{e['args'].get('stream','?'):>3}  {name}")
