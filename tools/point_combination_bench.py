#!/usr/bin/env python3
"""Host lurk_point_combination against lurk_point_combination_batch (csrc/pointcomb.cu) at the verifiers' shapes, one JSON object per line.

Shapes: the joint commitment over 2 and 4 points (BN254 G1); HyperKZG's P over l + 4 points for l = 21 and 23 and its Q over 3 (BN254 G1),
and the two as the two groups of one batch call; the inner-product argument's Q over 2 log n + 2 points for log n = 14 (Grumpkin) and 21
(Pallas); and a sweep of group sizes on BN254 G1 and Grumpkin for the host / device threshold of point_combination_groups.  Per shape
the host call and the batch call alternate; each call is timed with a host clock that ends in a stream synchronise (the batch call
synchronises its stream itself); best, worst and median of --steady calls after --warmup.  A second, separate pass runs each batch shape
under torch.profiler and reports the kernel's device time (mean over the launches).  Device name and power limit are read in the same
run.  Usage: point_combination_bench.py [--steady N] [--warmup N] [--out FILE]"""
import argparse
import json
import os
import random
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import compress_ctx_bench as ccb  # noqa: E402  (device info, curve points)
import lurk_beta_b200 as L  # noqa: E402
from oracle import spec  # noqa: E402

OUT = None


def emit(line):
    print(line, flush=True)
    if OUT:
        OUT.write(line + "\n")
        OUT.flush()


def group(curve, k, seed):
    """k random points of `curve` (96-byte header form) and k random scalars, canonical bytes"""
    r = spec.FIELD_MODULUS[spec.CURVES[curve]["scalar"]]
    rng = random.Random(seed)
    pts = ccb.points(curve, k, 7000 + seed)
    pb = np.concatenate([L.compress._point(P) for P in pts])
    sb = L.compress._fes([rng.randrange(r) for _ in range(k)])
    return pb, sb


def host_call(curve, pb, sb):
    out = np.zeros(96, dtype=np.uint8)
    L._capi.check(L._capi.lib().lurk_point_combination(curve, L._capi.np_ptr(pb), L._capi.np_ptr(sb), len(pb) // 96, L.FMT_CANONICAL,
                                                       L._capi.np_ptr(out)))
    return out


def stat(v):
    return {"best_ms": round(min(v), 3), "worst_ms": round(max(v), 3), "median_ms": round(float(np.median(v)), 3), "n": len(v)}


def shapes():
    out = [("joint commitment, 2 points", 0, [2]), ("joint commitment, 4 points", 0, [4]),
           ("HyperKZG P, l = 21 (l + 4 points)", 0, [25]), ("HyperKZG P, l = 23 (l + 4 points)", 0, [27]), ("HyperKZG Q (3 points)", 0, [3]),
           ("HyperKZG P and Q in one call, l = 21", 0, [25, 3]),
           ("IPA Q, 2^14 key (2 * 14 + 2 points)", 1, [30]), ("IPA Q, 2^21 key (2 * 21 + 2 points)", 2, [44])]
    for curve in (0, 1):
        for k in (2, 3, 4, 5, 6, 8, 10, 12, 16, 130):
            out.append((f"sweep, {k} points", curve, [k]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steady", type=int, default=20, help="timed calls per shape and side")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append the lines to this file")
    a = ap.parse_args()
    global OUT
    OUT = open(a.out, "a") if a.out else None
    info = ccb.device_info()
    stream = torch.cuda.Stream()
    runs = []
    for name, curve, counts in shapes():
        groups = [group(curve, k, 10 * i + k) for i, k in enumerate(counts)]
        want = [host_call(curve, pb, sb) for pb, sb in groups]
        got = L.compress.point_combination_batch(curve, groups, stream=stream.cuda_stream)
        assert all(np.array_equal(got[g], want[g]) for g in range(len(groups))), name
        t_host, t_dev = [], []
        for i in range(a.warmup + a.steady):              # the two sides alternate
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for pb, sb in groups:
                host_call(curve, pb, sb)
            t1 = time.perf_counter()
            L.compress.point_combination_batch(curve, groups, stream=stream.cuda_stream)
            stream.synchronize()
            t2 = time.perf_counter()
            if i >= a.warmup:
                t_host.append((t1 - t0) * 1e3)
                t_dev.append((t2 - t1) * 1e3)
        runs.append((name, curve, counts, groups))
        emit(json.dumps({"op": "point combination, " + name, "curve": curve, "terms": counts, "host_lurk_point_combination": stat(t_host),
                         "device_lurk_point_combination_batch": stat(t_dev),
                         "note": "host clock per call ending in a stream synchronise, alternating host / device, after %d warm-up calls; host: "
                                 "one lurk_point_combination per group" % a.warmup, **info}))
    # kernel time, a separate pass
    from torch.profiler import ProfilerActivity, profile
    for name, curve, counts, groups in runs:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(10):
                L.compress.point_combination_batch(curve, groups, stream=stream.cuda_stream)
            torch.cuda.synchronize()
        ev = [e for e in prof.events() if "point_comb_kernel" in e.name and e.device_type == torch.autograd.DeviceType.CUDA]
        us = [getattr(e, "device_time", None) or e.cuda_time for e in ev]
        emit(json.dumps({"op": "point_comb_kernel, " + name, "curve": curve, "terms": counts, "launches": len(us),
                         "kernel_mean_ms": round(float(np.mean(us)) / 1e3, 3) if us else None,
                         "kernel_min_ms": round(float(np.min(us)) / 1e3, 3) if us else None,
                         "note": "torch.profiler device time of the kernel, 10 launches, separate from the timed pass", **info}))


if __name__ == "__main__":
    main()
