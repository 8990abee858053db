"""Kernel timeline of the fold step's critical chain (torch.profiler / CUPTI, profiler on, so every time is inflated a little).

For one steady-state step of each circuit it prints:
  - the kernels of stage B's chain on the chain's stream (cross term .. fold_axpy) with start and duration;
  - the tail of commit(T): every kernel from the end of its bucket accumulation to the start of the challenge kernel;
  - the tail of commit(W2 - D): every kernel from the end of its bucket accumulation to its last kernel (the device result);
  - the step period (challenge start to challenge start) and the launches per step the fold context counts.

Usage: python tools/msm_tail_timeline.py [steps_profiled]   (development aid; needs an H100)"""
import json
import os
import re
import subprocess
import sys
import tempfile

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench


def short(name):
    name = name.replace("void ", "").replace("lurk::", "")
    base = name.split("(")[0]
    m = re.match(r"([A-Za-z0-9_]+)(<(.*)>)?", base)
    if not m:
        return base[:60]
    args = m.group(3) or ""
    args = re.sub(r"Fp<(\w+)Params>", r"\1", args)
    return f"{m.group(1)}<{args}>" if args else m.group(1)


def first_targ(name):
    m = re.search(r"<([^,>]*)", name)
    return m.group(1) if m else ""


def device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def main():
    nprof = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    wl = bench.FoldStepGPU(0, 1)
    wl.start(True)
    for _ in range(4):
        wl.step(False)
    wl.drain()
    torch.cuda.synchronize()
    launches = [(f"{k} (curve {i.curve})", i.ctx.stats()) for k, i in enumerate(wl.inst)]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(nprof):
            wl.step(False)
        wl.drain()
        torch.cuda.synchronize()
    trace = os.path.join(tempfile.mkdtemp(), "trace.json")
    prof.export_chrome_trace(trace)
    ev = json.load(open(trace))["traceEvents"]
    ks = [e for e in ev if e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy") and "ts" in e]
    ks.sort(key=lambda e: e["ts"])
    for e in ks:
        e["end"] = e["ts"] + e["dur"]
        e["stream"] = e["args"].get("stream", -1)
    print(f"device: {device_info()}")
    print(f"profiled steps: {nprof}, kernels + copies in the window: {len(ks)}")
    for k, st in launches:
        print(f"circuit {k}: launches per step {st['launches_a'] + st['launches_b']} (stage A {st['launches_a']}, stage B {st['launches_b']})")

    chals = [e for e in ks if "fold_challenge_kernel" in e["name"]]
    by_curve = {}
    for c in chals:
        by_curve.setdefault(short(c["name"]), []).append(c)
    for curve, cs in by_curve.items():
        if len(cs) < 2:
            continue
        C = cs[len(cs) // 2]                 # a step with neighbours on both sides
        t0 = C["ts"]
        period = (cs[-1]["ts"] - cs[0]["ts"]) / (len(cs) - 1)
        print(f"\n=== {curve}: step period (challenge to challenge) {period / 1e3:.3f} ms")
        same = [e for e in ks if e["stream"] == C["stream"]]
        cross = [e for e in same if "cross_term" in e["name"] and e["ts"] < t0]
        axpy = [e for e in same if "fold_axpy" in e["name"] and e["ts"] > t0]
        if cross and axpy:
            a, b = cross[-1], axpy[0]
            print(f"stage B chain on stream {C['stream']} (t = 0 at the cross term's start), {(b['end'] - a['ts']) / 1e3:.3f} ms:")
            prev = None
            for e in same:
                if a["ts"] <= e["ts"] <= b["ts"]:
                    gap = "" if prev is None else f"gap {(e['ts'] - prev) / 1e3:6.3f}"
                    print(f"  {(e['ts'] - a['ts']) / 1e3:8.3f} +{e['dur'] / 1e3:7.3f} ms  {gap:>12}  {short(e['name'])}")
                    prev = e["end"]
        accT = [e for e in same if "msm_accumulate_kernel" in e["name"] and e["ts"] < t0]
        if not accT:
            print("no commit(T) accumulation on the chain's stream")
            continue
        A = accT[-1]
        tail = t0 - A["end"]
        print(f"commit(T) tail: end of accumulation -> start of challenge = {tail / 1e3:.3f} ms "
              f"({100 * tail / period:.1f} % of the step); accumulation {A['dur'] / 1e3:.3f} ms; challenge {C['dur'] / 1e3:.3f} ms")
        for e in ks:
            if A["end"] <= e["ts"] < t0 and e["stream"] == C["stream"]:
                print(f"  +{(e['ts'] - A['end']) / 1e3:7.3f} dur {e['dur'] / 1e3:7.3f} ms  {short(e['name'])}")
        fb = first_targ(A["name"])
        accW = [e for e in ks if "msm_accumulate_kernel" in e["name"] and first_targ(e["name"]) == fb and e["stream"] != C["stream"]
                and e["end"] < t0]
        if not accW:
            print("no commit(W2 - D) accumulation found before the challenge")
            continue
        W = accW[-1]
        wk = [e for e in ks if e["stream"] == W["stream"] and e["ts"] >= W["end"]]
        # the commitment's own tail: the kernels up to the next stream activity that is not MSM work
        tailk = []
        for e in wk:
            if not e["name"].startswith("void lurk::msm_"):
                break
            if "msm_count_kernel" in e["name"] or "msm_hist_smem_kernel" in e["name"]:   # the next commitment's sort
                break
            tailk.append(e)
        if tailk:
            wt = tailk[-1]["end"] - W["end"]
            print(f"commit(W2 - D) tail on stream {W['stream']}: end of accumulation -> end of its last kernel = {wt / 1e3:.3f} ms; "
                  f"accumulation {W['dur'] / 1e3:.3f} ms")
            for e in tailk:
                print(f"  +{(e['ts'] - W['end']) / 1e3:7.3f} dur {e['dur'] / 1e3:7.3f} ms  {short(e['name'])}")


if __name__ == "__main__":
    main()
