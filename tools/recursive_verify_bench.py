#!/usr/bin/env python3
"""The recursive verifier (lurk_recursive_verify_dev / lurk_recursive_verify: RecursiveSNARK::verify's is_sat checks), one JSON object per
line.

  workloads:       Nova fib rc = 100 (primary + bench.SECONDARY: r_U_primary, r_U_secondary, l_u_secondary) and SuperNova trie_nivc (the
                   rc = 400 Lurk circuit and the trie lookup on one BN254 key, then bench.SECONDARY's two).  Running instances: random W and X
                   with u = 0 and E = (A z)∘(B z) (formed on the device with lurk_spmv_csr_dev and lurk_cross_term_dev), so they hold
                   and every MSM is over dense scalars; the fresh secondary instance: random free columns and X, u = 1, its glue columns
                   derived from their defining rows as bench.py derives them, so it holds too.  Commitments come from the same keys.
  whole call:      wall clock ending in a device synchronise, best and spread of 7 steady calls, _dev and host form (Montgomery host
                   arrays, no conversion), and the split: r1cs_sat_kernel's device time (torch.profiler, one call) against the rest.
  kernel:          r1cs_sat_kernel against the spmv3_kernel + relaxed_residual_kernel pair it replaced, both as check_running launches
                   them on bench.py's fold workload after real folds (same grid, kept products in use), torch.profiler device time per
                   call, processes of this tree and of --parent-tree (a built checkout of the commit before the change) alternating;
                   algorithmic bytes 68 per non-zero (value, column, z gather) + 56 per row (three row_ptr entries, E) over the 3.35 TB/s
                   data-sheet bound; the 3 x rows x 32 B of scratch the old check needed.
  shape setup:     lurk_spartan_ctx_create_verifier against lurk_spartan_ctx_create, wall clock and device bytes (torch.cuda.mem_get_info
                   around creation).
  CPU baseline:    the oracle's OpenMP spmv (three matrices) + msm (W and E) on all host threads, one run, fib primary; a port, not the
                   Rust verifier.
Device name and power limit are read in the same run.  Usage: recursive_verify_bench.py [--out FILE] [--skip-trie] [--parent-tree DIR]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
import lurk_beta_b200 as L  # noqa: E402
from spartan_ctx_bench import HBM_BYTES_PER_S, device_info, timed  # noqa: E402

OUT = None


def emit(obj):
    line = json.dumps(obj)
    print(line, flush=True)
    if OUT:
        OUT.write(line + "\n")
        OUT.flush()


def rand_elems(n, rng):
    a = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    a[:, 31] &= 0x0f
    return a.reshape(-1)


def to_mont(field, t):
    L._capi.check(L._capi.lib().lurk_convert_dev(field, C.c_void_p(t.data_ptr()), t.numel() // 32, L.FMT_MONTGOMERY, C.c_void_p(t.data_ptr()), None))
    return t


def point(buf, mont_curve=None):
    """a 96-byte point -> (x, y) of canonical ints or None; mont_curve: the bytes are Montgomery coordinates on that curve"""
    if not buf[64:].any():
        return None
    x, y = (int.from_bytes(buf[32 * k:32 * k + 32].tobytes(), "little") for k in range(2))
    if mont_curve is not None:
        pb = int.from_bytes(L.spartan.field_modulus(mont_curve ^ 1), "little")      # the base field of curve k is field k ^ 1
        rinv = pow(1 << 256, -1, pb)
        x, y = x * rinv % pb, y * rinv % pb
    return x, y


class Circuit:
    """one shape: its matrices, both kinds of Spartan context (with creation time and bytes), and instances on its key"""

    def __init__(self, name, field, mats, n_w, ck):
        self.name, self.field, self.mats, self.n_w, self.ck = name, field, mats, n_w, ck
        self.rows = len(mats[0][0]) - 1
        self.nnz = [int(m[0][-1]) for m in mats]
        self.setup = {}
        for kind, verifier_only in (("full", False), ("verifier_only", True)):
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            free0 = torch.cuda.mem_get_info()[0]
            ctx, ms = timed(lambda: L.spartan.SpartanContext(field, mats, n_w, 2, verifier_only=verifier_only))
            torch.cuda.synchronize()
            self.setup[kind] = {"create_ms": round(ms, 1), "device_bytes": free0 - torch.cuda.mem_get_info()[0]}
            setattr(self, kind, ctx)
        # the three CSRs alone: row_ptr (8 B per row), column (4 B) and value (32 B) per non-zero
        self.setup["csr_bytes_from_shape"] = 3 * 8 * (self.rows + 1) + 36 * sum(self.nnz)

    def commit(self, t, n):
        return point(self.ck.commit_device(t.data_ptr(), n), mont_curve=self.field)      # LURK_CURVE_k's scalar field is LURK_FIELD_k

    def products(self, dz):
        """(A z)∘(B z) on the device: lurk_spmv_csr_dev for A z and B z, lurk_cross_term_dev with u1 = u2 = 0 for the product"""
        f = self.field
        prod = []
        for rp, col, val in self.mats[:2]:
            d_rp, d_col = torch.from_numpy(np.ascontiguousarray(rp, dtype=np.uint64).view(np.uint8)).cuda(), torch.from_numpy(np.ascontiguousarray(col, dtype=np.uint32).view(np.uint8)).cuda()
            d_val = to_mont(f, torch.from_numpy(np.ascontiguousarray(val, dtype=np.uint8).reshape(-1)).cuda())
            y = torch.empty(self.rows * 32, dtype=torch.uint8, device="cuda")
            L._capi.check(L._capi.lib().lurk_spmv_csr_dev(f, C.c_void_p(d_rp.data_ptr()), C.c_void_p(d_col.data_ptr()), C.c_void_p(d_val.data_ptr()),
                                                          self.rows, C.c_void_p(dz.data_ptr()), C.c_void_p(y.data_ptr()), None))
            prod.append(y)
        zero = torch.zeros(self.rows * 32, dtype=torch.uint8, device="cuda")
        E = torch.empty(self.rows * 32, dtype=torch.uint8, device="cuda")
        z32 = L._capi.np_ptr(np.zeros(32, dtype=np.uint8))
        p = lambda t: C.c_void_p(t.data_ptr())
        L._capi.check(L._capi.lib().lurk_cross_term_dev(f, p(prod[0]), p(zero), p(zero), p(zero), p(prod[1]), p(zero), z32, z32, self.rows, p(E), None))
        torch.cuda.synchronize()
        return E

    def running(self, seed):
        """a relaxed instance that holds: random W, X, u = 0, E = (A z)∘(B z); (z, E, comm_W, comm_E) on the device"""
        rng = np.random.default_rng(seed)
        f = self.field
        z = np.concatenate([rand_elems(self.n_w, rng), np.zeros(32, dtype=np.uint8), rand_elems(2, rng)])
        dz = to_mont(f, torch.from_numpy(z).cuda())
        E = self.products(dz)
        return dict(z=dz, E=E, comm_W=self.commit(dz, self.n_w), comm_E=self.commit(E, self.rows))

    def fresh(self, seed, free, prod_rows):
        """a strict instance that holds: random free columns and X, u = 1, each glue column g (W[free + g]) set to (A z)(B z) of its
        defining row prod_rows[g], as bench.py derives the glue of its fresh instances"""
        rng = np.random.default_rng(seed)
        one = np.zeros(32, dtype=np.uint8)
        one[0] = 1
        z = np.concatenate([rand_elems(free, rng), np.zeros((self.n_w - free) * 32, dtype=np.uint8), one, rand_elems(2, rng)])
        dz = to_mont(self.field, torch.from_numpy(z).cuda())
        glue = self.products(dz).view(self.rows, 32)[torch.from_numpy(np.asarray(prod_rows, dtype=np.int64)).cuda()]
        dz.view(-1, 32)[free:free + len(prod_rows)] = glue
        torch.cuda.synchronize()
        return dict(z=dz, E=None, comm_W=self.commit(dz, self.n_w), comm_E=None)


def instances(plan, shape="verifier_only"):
    return [dict(shape=getattr(c, shape), ck=c.ck, z=i["z"].data_ptr(), E=None if i["E"] is None else i["E"].data_ptr(), comm_W=i["comm_W"],
                 comm_E=i["comm_E"]) for c, i in plan]


def host_instances(plan):
    out = []
    for c, i in plan:
        out.append(dict(shape=c.verifier_only, ck=c.ck, z=i["z"].cpu().numpy(), E=None if i["E"] is None else i["E"].cpu().numpy(), comm_W=i["comm_W"],
                        comm_E=i["comm_E"]))
    return out


def steady(fn, k=7):
    fn()                                     # warm-up
    ts = []
    out = None
    for _ in range(k):
        out, t = timed(fn)
        ts.append(t)
    return out, min(ts), max(ts)


def workload(name, plan, info):
    from torch.profiler import ProfilerActivity, profile
    dev = instances(plan)
    (ok, verdicts), best, worst = steady(lambda: L.recursive_verify(dev))
    host = host_instances(plan)
    (hok, hverdicts), hbest, hworst = steady(lambda: L.recursive_verify(host, fmt=L.FMT_MONTGOMERY, device=False))
    assert (ok, verdicts) == (hok, hverdicts), "the host and the device form disagree"
    assert L.recursive_verify(instances(plan, "full")) == (ok, verdicts), "a full and a verifier-only shape disagree"
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        L.recursive_verify(dev)
        torch.cuda.synchronize()
    sat_us = sum(k.device_time_total for k in prof.key_averages() if "r1cs_sat_kernel" in k.key)
    emit(dict({"op": f"lurk_recursive_verify, {name}", "instances": [c.name for c, _ in plan], "accepted": ok,
               "bad_rows": [v["bad_rows"] for v in verdicts], "commitments_ok": [v["comm_W_ok"] and v["comm_E_ok"] for v in verdicts],
               "dev_call_ms": {"best": round(best, 2), "worst": round(worst, 2)}, "host_call_ms": {"best": round(hbest, 2), "worst": round(hworst, 2)},
               "r1cs_pass_device_ms": round(sat_us / 1e3, 2), "rest_of_dev_call_ms": round(best - sat_us / 1e3, 2),
               "source": "wall clock ending in a device synchronise, best / worst of 7 steady calls after one warm-up; r1cs pass: torch.profiler, "
                         "sum of the r1cs_sat_kernel launches of one call (the instances of different keys overlap, so pass + rest can exceed "
                         "the call); rest = commitments, range checks, stream fork / join"}, **info))


# Run in a child process with a source tree first on sys.path (this one, or a checkout of the commit before r1cs_sat_kernel): the fold
# context's check_running on bench.py's workload after real folds, its R1CS kernels timed by torch.profiler.  The same workload, the same
# grid (8 CTAs of 256 per SM at most) and the same kept products in both trees; only the kernels differ.
CHECK_RUNNING_SCRIPT = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import numpy as np, torch, bench
from torch.profiler import ProfilerActivity, profile
wl = bench.FoldStepGPU(0, 1, workload=sys.argv[2])
wl.start(staged=True)
for _ in range(2):
    wl.step(staged=True)
wl.drain()
inst = wl.inst[0]
assert inst.ctx.check_running() == (0, True, True)
reps = int(sys.argv[3])
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(reps):
        inst.ctx.check_running()
    torch.cuda.synchronize()
out = {"rows": int(inst.nT), "nnz": [int(m[0][-1]) for m in inst.mats]}
for k in prof.key_averages():
    for name in ("r1cs_sat_kernel", "spmv3_kernel", "relaxed_residual_kernel"):
        if name in k.key:
            out[name] = out.get(name, 0.0) + k.device_time_total / reps
print("RESULT " + json.dumps(out))
"""


def check_running_kernels(tree, workload, reps):
    import subprocess
    out = subprocess.run([sys.executable, "-c", CHECK_RUNNING_SCRIPT, tree, workload, str(reps)], cwd=tree, capture_output=True, text=True,
                         check=True).stdout
    return json.loads(next(l for l in out.splitlines() if l.startswith("RESULT "))[7:])


def kernel_line(name, workload, parent, info, rounds=2, reps=10):
    """r1cs_sat_kernel against the pair it replaced (spmv3_kernel + relaxed_residual_kernel), both inside check_running, alternating
    processes of this tree and of `parent` (a built checkout of the commit before the change; without it the pair is not measured)"""
    new, old = [], []
    for _ in range(rounds):
        new.append(check_running_kernels(ROOT, workload, reps))
        if parent:
            old.append(check_running_kernels(parent, workload, reps))
    best = lambda runs, keys: min(sum(r[k] for k in keys) for r in runs) if runs and all(k in runs[0] for k in keys) else None
    new_us = best(new, ["r1cs_sat_kernel"])
    pair_us = best(old, ["spmv3_kernel", "relaxed_residual_kernel"])
    rows, nnz = new[0]["rows"], new[0]["nnz"]
    nbytes = 68 * sum(nnz) + 56 * rows
    line = {"op": f"check_running's R1CS kernels, {name}", "rows": rows, "nnz": nnz, "algorithmic_bytes": nbytes,
            "datasheet_bound_us": round(nbytes / HBM_BYTES_PER_S * 1e6, 1),
            "r1cs_sat_kernel_us": round(new_us, 1) if new_us else "not measured",
            "r1cs_sat_kernel_us_per_process": [round(r["r1cs_sat_kernel"], 1) for r in new],
            "pair_us": round(pair_us, 1) if pair_us else "not measured",
            "pair_us_per_process": [{k: round(r[k], 1) for k in ("spmv3_kernel", "relaxed_residual_kernel") if k in r} for r in old] or "not measured",
            "scratch_bytes": {"r1cs_sat_kernel": 16, "spmv3 + relaxed_residual": 3 * rows * 32},
            "source": f"torch.profiler, CUDA activities, device time per check_running call, mean over {reps} calls per process, best of {rounds} "
                      "processes per tree, the trees alternating; bench.py's workload after real folds (kept products in use), grid 8 CTAs of 256 "
                      "per SM at most in both"}
    if new_us:
        line["share_of_hbm_bound"] = round(nbytes / HBM_BYTES_PER_S / (new_us * 1e-6), 3)
    emit(dict(line, **info))


def cpu_line(c, inst, info):
    from oracle import capi as oracle
    th = bench.host_threads()
    z = inst["z"].clone()
    E = inst["E"].clone()
    for t in (z, E):
        L._capi.check(L._capi.lib().lurk_convert_dev(c.field, C.c_void_p(t.data_ptr()), t.numel() // 32, L.FMT_CANONICAL, C.c_void_p(t.data_ptr()), None))
    z, E = z.cpu().numpy(), E.cpu().numpy()
    bases = L.synthetic_bases(c.field, max(c.n_w, c.rows))
    t0 = time.perf_counter()
    for rp, col, val in c.mats:
        oracle.spmv(c.field, rp, col, val, z, nthreads=th)
    t1 = time.perf_counter()
    cw = oracle.msm(c.field, bases, z[:32 * c.n_w], nthreads=th)
    ce = oracle.msm(c.field, bases, E, nthreads=th)
    t2 = time.perf_counter()
    assert point(cw) == inst["comm_W"] and point(ce) == inst["comm_E"], "the CPU port and the GPU key disagree"
    emit(dict({"op": f"CPU baseline (OpenMP port: oracle spmv x3 + msm x2), {c.name}", "threads": th, "spmv_ms": round((t1 - t0) * 1e3, 1),
               "msm_ms": round((t2 - t1) * 1e3, 1), "note": "one run; a port of the checks, not Arecibo's Rust verifier"}, **info))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also append the lines to this file")
    ap.add_argument("--skip-trie", action="store_true")
    ap.add_argument("--parent-tree", default=None, help="a checkout of the commit before r1cs_sat_kernel with its library built: times the "
                                                         "spmv3_kernel + relaxed_residual_kernel pair check_running launched there")
    args = ap.parse_args()
    global OUT
    OUT = open(args.out, "a") if args.out else None
    info = device_info()
    sec = bench.SECONDARY
    smats, sn_w, _, s_prod = bench.step_circuit(3, 1, slot_elems=sec["free"], glue=sec["glue"], cons=sec["cons"])
    mats, n_w, _, _ = bench.step_circuit(1, 100)
    rows = len(mats[0][0]) - 1
    ck0 = L.CommitmentKey(0, L.synthetic_bases(0, max(n_w, rows)))
    ck1 = L.CommitmentKey(1, L.synthetic_bases(1, max(sn_w, len(smats[0][0]) - 1)))
    prim = Circuit("fib rc=100 primary (BN254 Fr)", 0, mats, n_w, ck0)
    secc = Circuit("secondary circuit (bench.SECONDARY, BN254 Fq)", 1, smats, sn_w, ck1)
    for c in (prim, secc):
        emit(dict({"op": f"shape setup, {c.name}", "rows": c.rows, "nnz": c.nnz, **c.setup,
                   "source": "wall clock around creation ending in a device synchronise; bytes from torch.cuda.mem_get_info around it"}, **info))
    kernel_line("fib rc=100 primary (BN254 Fr)", "fib", args.parent_tree, info)
    p_inst = prim.running(1)
    plan = [(prim, p_inst), (secc, secc.running(2)), (secc, secc.fresh(3, sec["free"], s_prod))]
    workload("Nova fib rc=100 + bench.SECONDARY", plan, info)
    cpu_line(prim, p_inst, info)
    del plan, p_inst, prim, ck0
    torch.cuda.empty_cache()
    if args.skip_trie:
        return
    mats0, n_w0, _, _ = bench.step_circuit(1, 400)
    _, slot_elems = bench.slot_offsets(1, 0, bench.TRIE_LOOKUP["slots"], bench.TRIE_LOOKUP["bd"], 0)
    mats1, n_w1, _, _ = bench.step_circuit(2, 1, slot_elems=slot_elems, glue=bench.TRIE_LOOKUP["glue"], cons=bench.TRIE_LOOKUP["cons"])
    need = max(n_w0, len(mats0[0][0]) - 1, n_w1, len(mats1[0][0]) - 1)
    ckt = L.CommitmentKey(0, L.synthetic_bases(0, need))
    lurk = Circuit("trie_nivc Lurk rc=400 circuit (BN254 Fr)", 0, mats0, n_w0, ckt)
    trie = Circuit("trie_nivc trie lookup (BN254 Fr)", 0, mats1, n_w1, ckt)
    for c in (lurk, trie):
        emit(dict({"op": f"shape setup, {c.name}", "rows": c.rows, "nnz": c.nnz, **c.setup,
                   "source": "wall clock around creation ending in a device synchronise; bytes from torch.cuda.mem_get_info around it"}, **info))
    kernel_line("trie_nivc Lurk rc=400 circuit (BN254 Fr)", "trie_nivc", args.parent_tree, info)
    plan = [(lurk, lurk.running(4)), (trie, trie.running(5)), (secc, secc.running(2)), (secc, secc.fresh(3, sec["free"], s_prod))]
    workload("SuperNova trie_nivc (Lurk rc=400 + trie lookup) + bench.SECONDARY", plan, info)


if __name__ == "__main__":
    main()
