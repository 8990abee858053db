#!/usr/bin/env python3
"""The verifier side (lurk_spartan_matrix_evals_dev, lurk_spartan_verify / _batch, lurk_ipa_verify_dev), one JSON object per line.

  matrix evaluations:  sp_matrix_eval_kernel against the composition it avoids (eq(r_x) and eq(r_y) tables -> sp_eval_table_kernel ->
                       inner product), alternating, device time from torch.profiler (mean over the launches), and the fused call alone
                       between CUDA events (mean over 50 calls), on the fib rc = 100 primary, bench.SECONDARY and the trie_nivc circuits;
                       algorithmic bytes 36 per non-zero + 8 per row; the scratch each needs; the OpenMP port of matrices_eval
                       (tests/csrc/matrices_eval_cpu.c) on the host's threads, checked equal, as the CPU baseline.
  whole verifiers:     lurk_spartan_verify (fib primary, secondary) and lurk_spartan_verify_batch (trie_nivc), wall-clock ending in a
                       device synchronise, best of 5, the Python stand-in transcript of tools/spartan_ctx_bench.py.  The instance is the
                       zero witness with u = 0 (it satisfies every R1CS); the verifier's work does not depend on the values.
  IPA verifier:        2^21 bases on Pallas, the secondary's key size on Grumpkin; wall-clock, best of 5, beside the commitment to 2^log_n
                       scalars alone on the same key (the rest is the s pass and the host's side of the check).
Device name and power limit are read in the same run.  Usage: spartan_verify_bench.py [--out FILE]"""
import argparse
import ctypes
import hashlib
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import matrices_eval_cpu  # noqa: E402
import lurk_beta_b200 as L  # noqa: E402
from spartan_ctx_bench import HBM_BYTES_PER_S, challenge, device_info, timed  # noqa: E402


OUT = None


def emit(line):
    print(line, flush=True)
    if OUT:
        OUT.write(line + "\n")
        OUT.flush()


def best_of(fn, k=5):
    out, best = None, None
    for _ in range(k):
        out, t = timed(fn)
        best = t if best is None else min(best, t)
    return out, best


def kernel_profile(ctx, reps=20):
    """sp_matrix_eval_kernel against eq tables + sp_eval_table_kernel + dot_kernel, alternating, device time per evaluation"""
    from torch.profiler import ProfilerActivity, profile
    f, p = ctx.field, ctx.p
    rng = np.random.default_rng(3)
    rx = [int.from_bytes(rng.bytes(32), "little") % p for _ in range(ctx.log_rows)]
    ry = [int.from_bytes(rng.bytes(32), "little") % p for _ in range(ctx.log_vars + 1)]
    nz = 2 * ctx.num_vars
    eq_x = torch.empty((1 << ctx.log_rows) * 32, dtype=torch.uint8, device="cuda")
    eq_y = torch.empty(nz * 32, dtype=torch.uint8, device="cuda")
    tab = torch.empty(nz * 32, dtype=torch.uint8, device="cuda")

    def composition():
        L.spartan.eq_evals(f, rx, eq_x.data_ptr())
        L.spartan.eq_evals(f, ry, eq_y.data_ptr())
        ctx.eval_table(eq_x.data_ptr(), 5, tab.data_ptr())
        return L.spartan.inner_product(f, tab.data_ptr(), eq_y.data_ptr(), nz)
    A, B, C = ctx.matrix_evals(rx, ry)
    assert (A + 5 * B + 25 * C) % p == composition(), "the two paths disagree"
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            ctx.matrix_evals(rx, ry)
            composition()
        torch.cuda.synchronize()

    def per_call(names):
        rows = [k for k in prof.key_averages() if any(n in k.key for n in names)]
        return sum(k.device_time_total for k in rows) / reps if rows else None
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(50):
        ctx.matrix_evals(rx, ry)
    end.record()
    end.synchronize()
    event_us = start.elapsed_time(end) * 1e3 / 50
    t0 = time.perf_counter()
    cpu = matrices_eval_cpu.matrices_eval(p, ctx.mats, ctx.n_w, ctx.num_vars, rx, ry)
    cpu_ms = (time.perf_counter() - t0) * 1e3
    assert cpu == (A, B, C), "the GPU and the CPU port disagree"
    return per_call(["sp_matrix_eval_kernel"]), per_call(["eq_kernel", "sp_eval_table_kernel", "dot_kernel"]), event_us, cpu_ms


def zero_instance(ctx):
    z = torch.zeros((ctx.n_w + 1 + ctx.n_x) * 32, dtype=torch.uint8, device="cuda")
    E = torch.zeros(ctx.rows * 32, dtype=torch.uint8, device="cuda")
    return z, E


def matrix_line(name, field, mats, n_w, info):
    ctx = L.spartan.SpartanContext(field, mats, n_w, 2)
    nnz = [int(m[0][-1]) for m in mats]
    ctx.mats = mats
    new_us, old_us, event_us, cpu_ms = kernel_profile(ctx)
    nbytes = 36 * sum(nnz) + 8 * 3 * ctx.rows
    line = {"op": f"matrix evaluations, {name}", "field": field, "nnz": nnz, "rows": ctx.rows, "rows_padded_log2": ctx.log_rows,
            "vars_padded_log2": ctx.log_vars, "algorithmic_bytes": nbytes, "datasheet_bound_us": round(nbytes / HBM_BYTES_PER_S * 1e6, 1),
            "sp_matrix_eval_kernel_us": round(new_us, 1) if new_us else "not measured",
            "composition_us": round(old_us, 1) if old_us else "not measured",
            "matrix_evals_call_cuda_events_us": round(event_us, 1),
            "cpu_port_ms": round(cpu_ms, 1), "cpu_port_threads": matrices_eval_cpu.threads(),
            "scratch_bytes": {"sp_matrix_eval_kernel": 0, "composition": 32 * ((1 << ctx.log_rows) + 4 * ctx.num_vars)},
            "source": "kernel times: torch.profiler, CUDA activities, mean of 20 alternating launches each; composition = 2 eq_kernel + "
                      "sp_eval_table_kernel + dot_kernel; matrix_evals call: CUDA events around 50 synchronous lurk_spartan_matrix_evals_dev calls "
                      "(kernel + counter reset + host gaps); cpu port: one wall-clock run incl. its eq tables"}
    if new_us:
        line["share_of_hbm_bound"] = round(nbytes / HBM_BYTES_PER_S / (new_us * 1e-6), 3)
    emit(json.dumps(dict(line, **info)))
    return ctx


def verify_line(name, ctx, info):
    z, E = zero_instance(ctx)
    proof = ctx.prove(z.data_ptr(), E.data_ptr(), challenge)
    (ok, _), t = best_of(lambda: ctx.verify(proof, 0, [0] * ctx.n_x, challenge))
    assert ok, "the verifier rejected an honest proof"
    line = {"op": f"lurk_spartan_verify, {name}", "field": ctx.field, "accepted": ok, "verify_ms": round(t, 2),
            "note": "wall-clock ending in a device synchronise, best of 5; Python stand-in transcript; zero witness, u = 0"}
    emit(json.dumps(dict(line, **info)))


def ipa_line(name, curve, log_n, info):
    field = curve                   # the scalar field of curve k is field k (include/lurk_b200.h)
    n = 1 << log_n
    rng = np.random.default_rng(log_n)
    bases = L.synthetic_bases(curve, n + 1)
    ck = L.CommitmentKey(curve, bases[:64 * n])
    gc = tuple(int.from_bytes(bases[64 * n + 32 * k:64 * n + 32 * k + 32].tobytes(), "little") for k in range(2))
    vecs = []
    for _ in range(2):
        raw = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
        raw[:, 31] &= 0x1f
        vecs.append(raw.reshape(-1))
    comm_b = ck.commit(vecs[0])
    comm = (int.from_bytes(comm_b[:32].tobytes(), "little"), int.from_bytes(comm_b[32:64].tobytes(), "little")) if comm_b[64:].any() else None
    a_dev, b_dev = (torch.from_numpy(v).cuda() for v in vecs)
    for t in (a_dev, b_dev):
        L._capi.check(L._capi.lib().lurk_convert_dev(field, ctypes.c_void_p(t.data_ptr()), n, L.FMT_MONTGOMERY, ctypes.c_void_p(t.data_ptr()), None))
    c = L.spartan.inner_product(field, a_dev.data_ptr(), b_dev.data_ptr(), n)
    chal = lambda rnd, msg: 1 + int.from_bytes(hashlib.sha256(bytes([rnd]) + msg).digest()[:16], "little")
    a_work, b_work = a_dev.clone(), b_dev.clone()          # consumed by the prover
    Ls, Rs, a_fin, _ = L.spartan.ipa_prove(curve, ck, gc, a_work.data_ptr(), b_work.data_ptr(), log_n, chal)
    del a_work, b_work
    (ok, _, _), t = best_of(lambda: L.spartan.ipa_verify(curve, ck, gc, comm, c, b_dev.data_ptr(), log_n, Ls, Rs, a_fin, chal))
    assert ok, "the IPA verifier rejected an honest proof"
    _, t_msm = best_of(lambda: ck.commit_device(b_dev.data_ptr(), n))
    line = {"op": f"lurk_ipa_verify_dev, {name}", "curve": curve, "log_n": log_n, "accepted": ok, "verify_ms": round(t, 2),
            "commit_2^log_n_alone_ms": round(t_msm, 2), "rest_ms": round(t - t_msm, 2),
            "note": "wall-clock ending in a device synchronise, best of 5; rest = verify - the commitment alone: the s pass, the host's side of the "
                    "check (Straus over 2 log_n + 2 points, overlapped with the commitment) and a_hat ck_hat after it"}
    emit(json.dumps(dict(line, **info)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also append the lines to this file")
    args = ap.parse_args()
    global OUT
    OUT = open(args.out, "a") if args.out else None
    info = device_info()
    matrices_eval_cpu.lib()                      # compile the CPU port before anything is timed
    mats, n_w, _, _ = bench.step_circuit(1, 100)
    ctx = matrix_line("fib rc=100 primary (BN254 Fr)", 0, mats, n_w, info)
    verify_line("fib rc=100 primary (BN254 Fr)", ctx, info)
    del ctx
    sec = bench.SECONDARY
    smats, sn_w, _, _ = bench.step_circuit(3, 1, slot_elems=sec["free"], glue=sec["glue"], cons=sec["cons"])
    sctx = matrix_line("secondary circuit (bench.SECONDARY, BN254 Fq)", 1, smats, sn_w, info)
    verify_line("secondary circuit (bench.SECONDARY, BN254 Fq)", sctx, info)
    sec_log = max(sctx.log_rows, sctx.log_vars)
    del sctx
    torch.cuda.empty_cache()
    mats0, n_w0, _, _ = bench.step_circuit(1, 400)
    _, slot_elems = bench.slot_offsets(1, 0, bench.TRIE_LOOKUP["slots"], bench.TRIE_LOOKUP["bd"], 0)
    mats1, n_w1, _, _ = bench.step_circuit(2, 1, slot_elems=slot_elems, glue=bench.TRIE_LOOKUP["glue"], cons=bench.TRIE_LOOKUP["cons"])
    c0 = matrix_line("trie_nivc Lurk rc=400 circuit (BN254 Fr)", 0, mats0, n_w0, info)
    c1 = L.spartan.SpartanContext(0, mats1, n_w1, 2)
    zs = [zero_instance(c) for c in (c0, c1)]
    proof = L.spartan.spartan_prove_batch([c0, c1], [(z.data_ptr(), e.data_ptr()) for z, e in zs], challenge)
    (ok, _), t = best_of(lambda: L.spartan.spartan_verify_batch([c0, c1], [(0, [0, 0]), (0, [0, 0])], proof, challenge))
    assert ok, "the batched verifier rejected an honest proof"
    emit(json.dumps(dict({"op": "lurk_spartan_verify_batch, trie_nivc (Lurk rc=400 + trie lookup, BN254 Fr)", "accepted": ok,
                           "verify_ms": round(t, 2), "note": "wall-clock ending in a device synchronise, best of 5; zero witnesses, u = 0"},
                          **info)))
    del c0, c1, zs, proof
    torch.cuda.empty_cache()
    ipa_line("Pallas primary key 2^21", 2, 21, info)
    ipa_line(f"Grumpkin secondary key 2^{sec_log}", 1, sec_log, info)


if __name__ == "__main__":
    main()
