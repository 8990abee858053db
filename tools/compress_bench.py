#!/usr/bin/env python3
"""Composed GPU time of `compress` (reference src/proof/nova.rs:341-356 / supernova.rs:293-317).

Default: the primary circuit of a fib rc = 100 proof -- the R1CS shape of bench.py's synthetic step circuit (1 114 100 constraints -> 2^21
rows, 911 900 variables -> 2^20) -- in two compositions, run alternately: RelaxedR1CSSNARK::prove + two HyperKZG openings (W at ry[1:], E at
rx; the first JSON line, as before), and Arecibo's: the same prove, batch_eval_reduce of both claims and ONE opening of the joint polynomial.
--nivc: SuperNova's BatchedRelaxedR1CSSNARK::prove at the trie_nivc shapes (bench.py's rc = 400 Lurk circuit and TRIE_LOOKUP coprocessor)
+ batch_eval_reduce + one opening.
Random z / E (the prover's cost does not depend on satisfiability; tests/test_gpu_spartan_chain.py and tests/test_gpu_spartan_batched.py
check real folded instances against the verifier at small sizes).  One JSON object per line; wall-clock per phase with a device
synchronise.  The challenge function is a Python stand-in (sha256), so every sum-check phase includes one Python callback per round.
poly_combine_kernel's device time comes from torch.profiler (CUDA activities) in a separate pass after the timed runs, next to its
algorithmic bytes 32 (sum_i 2^n_i + 2^m) and the bound those bytes give at the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (the step-circuit generator and the trie_nivc shapes)
import lurk_beta_b200 as L  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def challenge(label, data):
    return int.from_bytes(hashlib.sha256(repr((label, data)).encode()).digest()[:30], "little")


def pcs_challenge(r, m):
    return challenge("pcs", (r, bytes(m[:64])))


def rand_mont(n, seed):
    rng = np.random.default_rng(seed)
    raw = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    raw[:, 31] &= 0x1f
    return torch.from_numpy(raw.reshape(-1)).cuda()


def device_info():
    limit = None
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30)
        limit = float(out.stdout.strip().splitlines()[0])
    except Exception:           # no nvidia-smi: the limit is reported as unknown
        pass
    return {"device": torch.cuda.get_device_name(), "power_limit_w": limit}


def kzg_key(n_key):
    g = L.synthetic_bases(0, 1, start=9)
    gi = (int.from_bytes(g[:32].tobytes(), "little"), int.from_bytes(g[32:].tobytes(), "little"))
    t0 = time.perf_counter()
    ck = L.CommitmentKey.powers_of_tau(0, gi, 987654321987654321, n_key)
    torch.cuda.synchronize()
    key_ms = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    ck.precompute()          # the fixed-base window table of the key (what the fold's commit(W) uses as well); short vectors bypass it
    torch.cuda.synchronize()
    return ck, key_ms, (time.perf_counter() - t0) * 1e3


def combine_profile(claims, reps=10):
    """device time of poly_combine_kernel over `reps` reductions of `claims`, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    nv = [c[1] for c in claims]
    m = max(nv)
    joint = torch.empty((1 << m) * 32, dtype=torch.uint8, device="cuda")
    cb = lambda r, msg: challenge("batch_eval", (r, bytes(msg[:64])))
    L.spartan.batch_eval_reduce(0, claims, cb, joint.data_ptr())          # warm-up
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            L.spartan.batch_eval_reduce(0, claims, cb, joint.data_ptr())
        torch.cuda.synchronize()
    rows = [k for k in prof.key_averages() if "poly_combine_kernel" in k.key]
    nbytes = 32 * (sum(1 << n for n in nv) + (1 << m))
    launches = sum(k.count for k in rows)
    if not launches:
        return {"kernel": "poly_combine_kernel", "device_time_us": "not measured", "algorithmic_bytes": nbytes}
    t = sum(k.device_time_total for k in rows) / launches * 1e-6
    return {"kernel": "poly_combine_kernel", "launches": launches, "device_time_us": round(t * 1e6, 1), "algorithmic_bytes": nbytes,
            "achieved_TBps": round(nbytes / t / 1e12, 3), "datasheet_bound_us": round(nbytes / HBM_BYTES_PER_S * 1e6, 1),
            "share_of_datasheet_bound": round(nbytes / HBM_BYTES_PER_S / t, 3), "source": "torch.profiler, CUDA activities"}


def nova(rc):
    t0 = time.perf_counter()
    mats, n_w, rows, _ = bench.step_circuit(1, rc)
    prover = L.spartan.RelaxedR1CSProver(0, mats, n_w, 2)
    torch.cuda.synchronize()
    setup_s = time.perf_counter() - t0
    nnz = [int(m[0][-1]) for m in mats]
    dW, dE = rand_mont(n_w, 1), rand_mont(rows, 2)
    z = prover.pad_z(dW, 12345, [6, 7])
    n_key = max(prover.num_vars, 1 << prover.log_rows)
    ck, key_ms, table_ms = kzg_key(n_key)
    nvb = prover.num_vars.bit_length() - 1
    best = {"two": None, "one": None}
    for rep in range(3):
        for kind in ("two", "one"):                          # the two compositions alternate
            timings = {}
            t0 = time.perf_counter()
            proof = prover.prove(z, dE, 12345, challenge, timings)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            if kind == "two":
                L.spartan.hyperkzg_prove(0, ck, z.data_ptr(), proof["ry"][1:], pcs_challenge)
                torch.cuda.synchronize()
                t2 = time.perf_counter()
                L.spartan.hyperkzg_prove(0, ck, proof["E_padded"].data_ptr(), proof["rx"], pcs_challenge)
                torch.cuda.synchronize()
                t3 = time.perf_counter()
                timings["open W (HyperKZG, 2^%d)" % nvb] = (t2 - t1) * 1e3
                timings["open E (HyperKZG, 2^%d)" % prover.log_rows] = (t3 - t2) * 1e3
            else:
                claims = [(z.data_ptr(), nvb, proof["ry"][1:], proof["eval_W"]), (proof["E_padded"].data_ptr(), prover.log_rows, proof["rx"], proof["claims"][3])]
                _, r, _, _, _, joint = L.spartan.batch_eval_reduce(0, claims, lambda rr, msg: challenge("batch_eval", (rr, bytes(msg[:64]))))
                torch.cuda.synchronize()
                t2 = time.perf_counter()
                L.spartan.hyperkzg_prove(0, ck, joint.data_ptr(), r, pcs_challenge)
                torch.cuda.synchronize()
                t3 = time.perf_counter()
                timings["batch_eval_reduce (2^%d + 2^%d -> 2^%d)" % (nvb, prover.log_rows, len(r))] = (t2 - t1) * 1e3
                timings["open joint (HyperKZG, 2^%d)" % len(r)] = (t3 - t2) * 1e3
            total = (t3 - t0) * 1e3
            if best[kind] is None or total < best[kind][0]:
                best[kind] = (total, timings)
    shape = {"rc": rc, "constraints": rows, "variables": n_w, "nnz": nnz, "rows_padded_log2": prover.log_rows, "vars_padded_log2": nvb}
    setup = {"matrices_to_device_and_transposes_s": round(setup_s, 2), "powers_of_tau_key_ms": round(key_ms, 1), "key_points": n_key,
             "fixed_base_table_ms": round(table_ms, 1)}
    note = "best of 3; per-phase wall-clock with a device synchronise; Python stand-in transcript"
    print(json.dumps(dict({"op": "compress, primary circuit, GPU half (RelaxedR1CSSNARK::prove + 2 HyperKZG openings)"}, **shape,
                          total_ms=round(best["two"][0], 2), phases_ms={k: round(v, 3) for k, v in best["two"][1].items()}, setup=setup, note=note)),
          flush=True)
    claims = [(z.data_ptr(), nvb, [1] * nvb, 0), (proof["E_padded"].data_ptr(), prover.log_rows, [1] * prover.log_rows, 0)]
    print(json.dumps(dict({"op": "compress, primary circuit, GPU half (RelaxedR1CSSNARK::prove + batch_eval_reduce + 1 HyperKZG opening)"}, **shape,
                          total_ms=round(best["one"][0], 2), phases_ms={k: round(v, 3) for k, v in best["one"][1].items()},
                          combine=combine_profile(claims), note=note + "; run alternately with the two-opening composition", **device_info())),
          flush=True)


def supernova(rc):
    t0 = time.perf_counter()
    mats0, n_w0, rows0, _ = bench.step_circuit(1, rc)
    _, slot_elems = bench.slot_offsets(1, 0, bench.TRIE_LOOKUP["slots"], bench.TRIE_LOOKUP["bd"], 0)
    mats1, n_w1, rows1, _ = bench.step_circuit(2, 1, slot_elems=slot_elems, glue=bench.TRIE_LOOKUP["glue"], cons=bench.TRIE_LOOKUP["cons"])
    prover = L.spartan.BatchedRelaxedR1CSProver(0, [(mats0, n_w0, 2), (mats1, n_w1, 2)])
    torch.cuda.synchronize()
    setup_s = time.perf_counter() - t0
    insts = []
    for i, (n_w, rows) in enumerate(((n_w0, rows0), (n_w1, rows1))):
        insts.append((prover.pad_z(i, rand_mont(n_w, 1 + 2 * i), 12345 + i, [6, 7]), rand_mont(rows, 2 + 2 * i), 12345 + i))
    m = max(max(pr.num_vars.bit_length() - 1, pr.log_rows) for pr in prover.provers)
    ck, key_ms, table_ms = kzg_key(1 << m)
    best = None
    for rep in range(3):
        timings = {}
        t0 = time.perf_counter()
        proof = prover.prove(insts, challenge, timings)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        L.spartan.hyperkzg_prove(0, ck, proof["joint"].data_ptr(), proof["r"], pcs_challenge)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        timings["open joint (HyperKZG, 2^%d)" % len(proof["r"])] = (t2 - t1) * 1e3
        if best is None or (t2 - t0) * 1e3 < best[0]:
            best = ((t2 - t0) * 1e3, timings)
    claims = [(inst[0].data_ptr(), pr.num_vars.bit_length() - 1, [1] * (pr.num_vars.bit_length() - 1), 0) for inst, pr in zip(insts, prover.provers)]
    claims += [(e.data_ptr(), pr.log_rows, [1] * pr.log_rows, 0) for e, pr in zip(proof["E_padded"], prover.provers)]
    circuits = [{"name": name, "constraints": rows, "variables": n_w, "rows_padded_log2": pr.log_rows, "vars_padded_log2": pr.num_vars.bit_length() - 1}
                for name, rows, n_w, pr in (("lurk rc=%d" % rc, rows0, n_w0, prover.provers[0]), ("trie lookup", rows1, n_w1, prover.provers[1]))]
    print(json.dumps({"op": "compress, SuperNova primary circuits, GPU half (BatchedRelaxedR1CSSNARK::prove + batch_eval_reduce + 1 HyperKZG opening)",
                      "circuits": circuits, "total_ms": round(best[0], 2), "phases_ms": {k: round(v, 3) for k, v in best[1].items()},
                      "combine": combine_profile(claims),
                      "setup": {"matrices_to_device_and_transposes_s": round(setup_s, 2), "powers_of_tau_key_ms": round(key_ms, 1), "key_points": 1 << m,
                                "fixed_base_table_ms": round(table_ms, 1)},
                      "note": "best of 3; per-phase wall-clock with a device synchronise; Python stand-in transcript", **device_info()}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rc", type=int, default=None, help="frames of the Lurk step circuit (default: 100, or 400 with --nivc)")
    ap.add_argument("--nivc", action="store_true", help="SuperNova's batched SNARK at the trie_nivc shapes")
    a = ap.parse_args()
    if a.nivc:
        supernova(a.rc or 400)
    else:
        nova(a.rc or 100)


if __name__ == "__main__":
    main()
