#!/usr/bin/env python3
"""The Spartan prover context (lurk_spartan_ctx_*, csrc/spartan.cu) against the Python compositions it replaces, one JSON object per line.

  fib:        the primary circuit of a fib rc = 100 proof (bench.step_circuit: 2^21 rows, 2^20 variables), plain RelaxedR1CSSNARK;
  trie_nivc:  SuperNova's batched SNARK over bench.py's rc = 400 Lurk circuit and the TRIE_LOOKUP coprocessor;
  secondary:  bench.SECONDARY on BN254 Fq (the Grumpkin half of CompressedSNARK::prove).
For each: setup (the context against RelaxedR1CSProver's padded_and_transposed + DeviceCSR path), prove time (context against the Python
composition prove + batch_eval_reduce, alternating, best of 3, wall-clock with a device synchronise, the same Python stand-in transcript);
for fib, the eval table's device time from torch.profiler (sp_eval_table_kernel against the 3 transposed SpMV + 2 AXPY kernels) with
algorithmic bytes from nnz; and the primary and secondary proofs run from two host threads at once against one after the other.
Random z / E: the prover's cost does not depend on satisfiability.  Device name and power limit are read in the same run."""
import hashlib
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import lurk_beta_b200 as L  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def challenge(label, data):
    return int.from_bytes(hashlib.sha256(repr((label, data)).encode()).digest()[:30], "little")


def device_info():
    limit = None
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30)
        limit = float(out.stdout.strip().splitlines()[0])
    except Exception:           # no nvidia-smi: the limit is reported as unknown
        pass
    return {"device": torch.cuda.get_device_name(), "power_limit_w": limit}


def rand_mont(n, seed):
    rng = np.random.default_rng(seed)
    raw = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    raw[:, 31] &= 0x1f
    return torch.from_numpy(raw.reshape(-1)).cuda()


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def setup(field, circuits):
    """(contexts, Python provers, ms of each setup); circuits: [(mats, n_w)]"""
    ctxs, t_ctx = timed(lambda: [L.spartan.SpartanContext(field, mats, n_w, 2) for mats, n_w in circuits])
    provers, t_py = timed(lambda: [L.spartan.RelaxedR1CSProver(field, mats, n_w, 2) for mats, n_w in circuits])
    return ctxs, provers, t_ctx, t_py


def python_plain(field, prover, zp, dE, u):
    p = prover.p
    proof = prover.prove(zp, dE, u, challenge)
    nvb = prover.num_vars.bit_length() - 1
    claims = [(zp.data_ptr(), nvb, proof["ry"][1:], proof["eval_W"]), (proof["E_padded"].data_ptr(), prover.log_rows, proof["rx"], proof["claims"][3])]
    return L.spartan.batch_eval_reduce(field, claims, lambda r, m: challenge("batch_eval", (r, [int.from_bytes(m[i:i + 32], "little") for i in range(0, len(m), 32)])) % p)


def plain_inputs(prover, seed):
    n_w, rows = prover.n_w, prover.rows
    W, E = rand_mont(n_w, seed), rand_mont(rows, seed + 1)
    u, X = 12345, [6, 7]
    z = torch.cat([W, torch.from_numpy(np.concatenate([L.spartan._fe(x * (1 << 256) % prover.p) for x in [u] + X])).cuda()])
    return z, E, prover.pad_z(W, u, X), u


def compare_plain(name, field, mats, n_w):
    ctxs, provers, t_ctx, t_py = setup(field, [(mats, n_w)])
    ctx, prover = ctxs[0], provers[0]
    z, E, zp, u = plain_inputs(prover, 1)
    best = {"context": None, "python": None}
    for _ in range(3):
        for kind in ("context", "python"):
            _, t = timed(lambda: ctx.prove(z.data_ptr(), E.data_ptr(), challenge) if kind == "context" else python_plain(field, prover, zp, E, u))
            best[kind] = t if best[kind] is None else min(best[kind], t)
    nnz = [int(m[0][-1]) for m in mats]
    line = {"op": f"Spartan prove, {name}", "field": field, "constraints": prover.rows, "variables": n_w, "nnz": nnz,
            "rows_padded_log2": prover.log_rows, "vars_padded_log2": prover.num_vars.bit_length() - 1,
            "setup_ms": {"context": round(t_ctx, 1), "python_padded_and_transposed": round(t_py, 1)},
            "prove_ms": {"context": round(best["context"], 2), "python_composition": round(best["python"], 2)},
            "note": "prove = RelaxedR1CSSNARK::prove + batch_eval_reduce([W, E]); best of 3, alternating; Python stand-in transcript"}
    return ctx, prover, (z, E), line


def table_profile(ctx, prover, reps=10):
    """device time of the eval table: sp_eval_table_kernel against the transposed SpMVs (spmv_kernel + spmv_long_kernel) and the AXPYs"""
    from torch.profiler import ProfilerActivity, profile
    f = ctx.field
    eq = rand_mont(1 << ctx.log_rows, 9)
    nz = 2 * ctx.num_vars
    out = torch.empty(nz * 32, dtype=torch.uint8, device="cuda")
    ys = [torch.empty(nz * 32, dtype=torch.uint8, device="cuda") for _ in range(3)]

    def old():
        for M, y in zip(prover.MT, ys):
            M.mv(f, eq.data_ptr(), y.data_ptr())
        prover._axpy(ys[0], ys[1], 5, out)
        prover._axpy(out, ys[2], 25, out)
    ctx.eval_table(eq.data_ptr(), 5, out.data_ptr())
    old()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            ctx.eval_table(eq.data_ptr(), 5, out.data_ptr())
            old()
        torch.cuda.synchronize()

    def per_call(names):
        rows = [k for k in prof.key_averages() if any(n in k.key for n in names)]
        return sum(k.device_time_total for k in rows) / reps if rows else None
    new_us, old_us = per_call(["sp_eval_table_kernel"]), per_call(["spmv_kernel", "spmv_long_kernel", "axpy_kernel"])
    tnnz = sum(int(M.col.numel()) for M in prover.MT)
    # per non-zero: value (32) + row index (4) + the eq entry it gathers (32); per output column: row_ptr (8) + output (32)
    nbytes = tnnz * (32 + 4 + 32) + nz * (8 + 32)
    line = {"op": "eval table (compute_eval_table_sparse)", "nnz": tnnz, "columns": nz, "algorithmic_bytes": nbytes,
            "datasheet_bound_us": round(nbytes / HBM_BYTES_PER_S * 1e6, 1), "source": "torch.profiler, CUDA activities, mean of %d" % reps}
    line["fused_kernel_us"] = round(new_us, 1) if new_us else "not measured"
    line["three_spmv_two_axpy_us"] = round(old_us, 1) if old_us else "not measured"
    if new_us:
        line["fused_achieved_TBps"] = round(nbytes / (new_us * 1e-6) / 1e12, 3)
    return line


def concurrent(jobs):
    """jobs: [(ctx, z, E)]; (sequential ms, concurrent ms from one host thread and stream each), best of 3"""
    streams = [torch.cuda.Stream() for _ in jobs]

    def one(i):
        ctx, z, E = jobs[i]
        with torch.cuda.stream(streams[i]):
            ctx.prove(z.data_ptr(), E.data_ptr(), challenge, stream=streams[i].cuda_stream)
        streams[i].synchronize()
    best_seq = best_con = None
    for _ in range(3):
        _, t_seq = timed(lambda: [one(i) for i in range(len(jobs))])

        def both():
            th = [threading.Thread(target=one, args=(i,)) for i in range(len(jobs))]
            for t in th:
                t.start()
            for t in th:
                t.join()
        _, t_con = timed(both)
        best_seq = t_seq if best_seq is None else min(best_seq, t_seq)
        best_con = t_con if best_con is None else min(best_con, t_con)
    return best_seq, best_con


def main():
    info = device_info()
    mats, n_w, _, _ = bench.step_circuit(1, 100)
    ctx, prover, (z, E), line = compare_plain("fib rc=100 primary (BN254 Fr)", 0, mats, n_w)
    print(json.dumps(dict(line, **info)), flush=True)
    print(json.dumps(dict(table_profile(ctx, prover), **info)), flush=True)
    del prover
    sec = bench.SECONDARY
    smats, sn_w, _, _ = bench.step_circuit(3, 1, slot_elems=sec["free"], glue=sec["glue"], cons=sec["cons"])
    sctx, sprover, (sz, sE), sline = compare_plain("secondary circuit (bench.SECONDARY, BN254 Fq)", 1, smats, sn_w)
    print(json.dumps(dict(sline, **info)), flush=True)
    t_seq, t_con = concurrent([(ctx, z, E), (sctx, sz, sE)])
    print(json.dumps(dict({"op": "primary (fib rc=100, BN254 Fr) and secondary (BN254 Fq) proofs", "sequential_ms": round(t_seq, 2),
                           "concurrent_ms": round(t_con, 2), "note": "two host threads, one stream each; best of 3"}, **info)), flush=True)
    del ctx, z, E
    torch.cuda.empty_cache()
    # trie_nivc: the rc = 400 Lurk circuit and the trie-lookup coprocessor, batched
    mats0, n_w0, _, _ = bench.step_circuit(1, 400)
    _, slot_elems = bench.slot_offsets(1, 0, bench.TRIE_LOOKUP["slots"], bench.TRIE_LOOKUP["bd"], 0)
    mats1, n_w1, _, _ = bench.step_circuit(2, 1, slot_elems=slot_elems, glue=bench.TRIE_LOOKUP["glue"], cons=bench.TRIE_LOOKUP["cons"])
    ctxs, t_ctx = timed(lambda: [L.spartan.SpartanContext(0, m, n, 2) for m, n in ((mats0, n_w0), (mats1, n_w1))])
    bprover, t_py = timed(lambda: L.spartan.BatchedRelaxedR1CSProver(0, [(mats0, n_w0, 2), (mats1, n_w1, 2)]))
    dev, py = [], []
    for i, pr in enumerate(bprover.provers):
        zz, ee, zp, u = plain_inputs(pr, 10 + 2 * i)
        dev.append((zz.data_ptr(), ee.data_ptr()))
        py.append((zp, ee, u, zz))
    best = {"context": None, "python": None}
    for _ in range(3):
        for kind in ("context", "python"):
            fn = (lambda: L.spartan.spartan_prove_batch(ctxs, dev, challenge)) if kind == "context" else (lambda: bprover.prove([q[:3] for q in py], challenge))
            _, t = timed(fn)
            best[kind] = t if best[kind] is None else min(best[kind], t)
    print(json.dumps(dict({"op": "Spartan prove, trie_nivc (batched: Lurk rc=400 + trie lookup, BN254 Fr)",
                           "circuits": [{"constraints": pr.rows, "variables": pr.n_w, "rows_padded_log2": pr.log_rows,
                                         "vars_padded_log2": pr.num_vars.bit_length() - 1} for pr in bprover.provers],
                           "setup_ms": {"context": round(t_ctx, 1), "python_padded_and_transposed": round(t_py, 1)},
                           "prove_ms": {"context": round(best["context"], 2), "python_composition": round(best["python"], 2)},
                           "note": "prove = BatchedRelaxedR1CSSNARK::prove incl. batch_eval_reduce; best of 3, alternating; Python stand-in transcript"},
                          **info)), flush=True)


if __name__ == "__main__":
    main()
