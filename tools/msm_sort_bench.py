"""Device time of a fold commitment's digit sort (csrc/msm_impl.cuh), shared-memory histograms against the global-atomics kernels
(LURK_MSM_SORT=legacy), alternating launch by launch in one process on the lengths the fold step at fib rc = 100 commits:

  T       1 114 100 scalars, 34 % non-zero, window 16 (the fold context's table for commit(T))
  W2 - D    911 900 scalars, 36 % non-zero, window 16 (commit(W2 - D); the vector is generated already reduced by D, so the second
            32-byte load and the subtraction the fold context's sort performs for it are NOT in these numbers)

The time is the span between the CUDA events the commitment context records before the sort's first kernel (or memset) and after its last kernel
(lurk_msm_ctx_last_sort_ms).  Algorithmic bytes: each of the two passes reads every 32-byte scalar, the scatter writes 4 bytes per
non-zero digit (counted as windows x non-zero scalars, an upper bound); the bound is those bytes at the H100 SXM data sheet's 3.35 TB/s.

Usage: python tools/msm_sort_bench.py [launches] >> profiles/h100_msm_sort.jsonl   (needs an H100; one JSON line per shape)"""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lurk_beta_b200 as L

CURVE, FIELD, WINDOW = L.CURVE_BN254_G1, L.FIELD_BN254_FR, 16
SHAPES = [("T", 1_114_100, 0.34), ("W2-D", 911_900, 0.36)]
HBM_BYTES_PER_S = 3.35e12


def device_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30).stdout.strip().splitlines()
    return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()


def scalars(n, nonzero, seed):
    rng = np.random.default_rng(seed)
    raw = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    raw[:, 31] &= 0x0f                                        # < 2^252: reduced
    raw[rng.random(n) >= nonzero] = 0
    live = int(raw.any(axis=1).sum())
    d = torch.from_numpy(raw.reshape(-1)).cuda()
    L._capi.check(L._capi.lib().lurk_convert_dev(FIELD, C.c_void_p(d.data_ptr()), n, L.FMT_MONTGOMERY, C.c_void_p(d.data_ptr()), None))
    return d, live


def main():
    if not torch.cuda.is_available():
        sys.exit("msm_sort_bench.py measures on a GPU and none is present")
    launches = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    dev = device_info()
    for k, (name, n, frac) in enumerate(SHAPES):
        ck = L.CommitmentKey.setup(CURVE, b"ck", n).precompute(WINDOW)
        ck.set_profiling(True)
        d, live = scalars(n, frac, seed=k)
        ms, point = {"smem": [], "legacy": []}, {}
        for it in range(launches + 5):                        # five warm-up rounds
            for sort in ("legacy", "smem"):
                if sort == "legacy":
                    os.environ["LURK_MSM_SORT"] = "legacy"
                else:
                    os.environ.pop("LURK_MSM_SORT", None)
                out = ck.commit_device(d.data_ptr(), n)
                assert point.setdefault(sort, out.tobytes()) == out.tobytes()
                if it >= 5:
                    ms[sort].append(ck.last_sort_ms())
        os.environ.pop("LURK_MSM_SORT", None)
        assert point["smem"] == point["legacy"], "the two sorts disagree"
        nwin = 254 // WINDOW + 1
        nbytes = n * 64 + 4 * live * nwin
        rec = {"tool": "msm_sort_bench", "device": dev, "shape": name, "n": n, "nonzero_scalars": live, "window": WINDOW, "launches": launches,
               "algorithmic_bytes": nbytes, "bound_ms_at_3.35TBps": round(1e3 * nbytes / HBM_BYTES_PER_S, 4)}
        for sort, v in ms.items():
            mean = float(np.mean(v))
            rec[sort] = {"mean_ms": round(mean, 4), "min_ms": round(float(np.min(v)), 4), "max_ms": round(float(np.max(v)), 4),
                         "GBps": round(nbytes / mean / 1e6, 1), "share_of_bandwidth_bound": round(nbytes / HBM_BYTES_PER_S / (mean * 1e-3), 3)}
        rec["speedup"] = round(rec["legacy"]["mean_ms"] / rec["smem"]["mean_ms"], 2)
        print(json.dumps(rec), flush=True)
        ck.close()


if __name__ == "__main__":
    main()
