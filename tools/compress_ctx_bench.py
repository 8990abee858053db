#!/usr/bin/env python3
"""Wall-clock of CompressedSNARK::prove's GPU half (reference src/proof/nova.rs:341-356 / supernova.rs:293-317) in three configurations,
run alternately:
  (a) composed:    SpartanContext.prove (or spartan_prove_batch) + the joint commitment on the host + the one-shot opening call
                   (hyperkzg_prove / ipa_prove, which allocate their scratch per call), primary then secondary;
  (b) sequential:  one lurk_compress_prove_dev call with LURK_COMPRESS_SEQUENTIAL;
  (c) concurrent:  one lurk_compress_prove_dev call, the two circuits on two library-owned threads and streams.
(b) and (c) also run with a native C challenge function (built into a temporary directory with gcc) so that the Python interpreter's
share -- one callback per sum-check round, serialised by the GIL across the two threads -- shows separately.  For each compress
configuration the first call on a fresh context (which allocates the arenas) is reported apart from the steady-state calls.

Shapes: the primary circuit of fib rc = 100 (bench.step_circuit: 2^21 rows, 2^20 variables; BN254 + HyperKZG on a powers-of-tau key with
its fixed-base table), or with --nivc SuperNova's batched primary at the trie_nivc shapes (the rc = 400 Lurk circuit and the TRIE_LOOKUP
coprocessor); the secondary is bench.SECONDARY (Grumpkin + IPA) in both.  Random z / E and commitments (the prover's cost does not depend
on satisfiability; tests/test_gpu_compress.py checks real folded instances).  One JSON object per line: best-of and spread (max - min)
per configuration, milliseconds, host clock around calls that end in a device synchronise."""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (the step-circuit generator and the shapes)
import lurk_beta_b200 as L  # noqa: E402
from oracle import spec as ospec  # noqa: E402  (host point arithmetic of the composed joint commitment)

NATIVE_C = r"""
#include <stddef.h>
#include <stdint.h>
int challenge(void *user, int circuit, int phase, int round, const uint8_t *msg, size_t len, uint8_t out[32]) {
    uint64_t h = 1469598103934665603ull ^ (uint64_t)(circuit * 7919 + phase * 131 + round);
    size_t i;
    (void)user;
    for (i = 0; i < len; i++) h = (h ^ msg[i]) * 1099511628211ull;
    for (i = 0; i < 32; i++) out[i] = 0;
    h = (h >> 2) | 1;
    for (i = 0; i < 8; i++) out[i] = (uint8_t)(h >> (8 * i));
    return 0;
}
"""


def native_challenge(tmp):
    src, so = os.path.join(tmp, "chal.c"), os.path.join(tmp, "libchal.so")
    with open(src, "w") as f:
        f.write(NATIVE_C)
    subprocess.check_call(["/usr/bin/gcc", "-O2", "-shared", "-fPIC", src, "-o", so])
    lib = C.CDLL(so)
    return C.cast(lib.challenge, C.c_void_p).value, lib


def challenge(k, label, data):
    return int.from_bytes(hashlib.sha256(repr((k, label, data)).encode()).digest()[:30], "little")


def rand_mont(n, seed):
    rng = np.random.default_rng(seed)
    raw = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    raw[:, 31] &= 0x1f
    return torch.from_numpy(raw.reshape(-1)).cuda()


def points(curve, k, start):
    b = L.synthetic_bases(curve, k, start=start)
    return [(int.from_bytes(b[64 * i:64 * i + 32].tobytes(), "little"), int.from_bytes(b[64 * i + 32:64 * i + 64].tobytes(), "little")) for i in range(k)]


def device_info():
    limit = None
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30)
        limit = float(out.stdout.strip().splitlines()[0])
    except Exception:           # no nvidia-smi: the limit is reported as unknown
        pass
    return {"device": torch.cuda.get_device_name(), "power_limit_w": limit}


def circuit(field, seed, frames, **shape):
    mats, n_w, rows, _ = bench.step_circuit(seed, frames, **shape)
    ctx = L.spartan.SpartanContext(field, mats, n_w, 2)
    z, e = rand_mont(n_w + 3, seed), rand_mont(rows, seed + 1)          # z = (W, u, X) as LURK_FOLD_BUF_Z1 holds it
    return dict(ctx=ctx, z=z, e=e, n_w=n_w, rows=rows)


def composed(k, curve, ctxs, insts, pcs, batched):
    """configuration (a) for one circuit"""
    field = ospec.CURVES[curve]["scalar"]
    p, pb = ospec.FIELD_MODULUS[field], ospec.FIELD_MODULUS[ospec.CURVES[curve]["base"]]
    chal = lambda label, data: challenge(k, label, data)
    if batched:
        got = L.spartan.spartan_prove_batch(ctxs, [(z, e) for z, e, _, _ in insts], chal)
    else:
        got = ctxs[0].prove(insts[0][0], insts[0][1], chal)
    comm = None
    for P, w in zip([x[2] for x in insts] + [x[3] for x in insts], got["weights"]):
        comm = ospec.ec_add(comm, ospec.ec_mul(w, P, pb), pb)
    if pcs[0] == "hyperkzg":
        L.spartan.hyperkzg_prove(curve, pcs[1], got["joint"].data_ptr(), got["r"], lambda rnd, msg: challenge(k, "pcs", (rnd, bytes(msg))) % p)
    else:
        msg = b"".join(int(v).to_bytes(32, "little") for v in (comm[0], comm[1], 1, got["joint_eval"]))
        gc = ospec.ec_mul(challenge(k, "pcs", (0, msg)) % p, pcs[2], pb)
        m = len(got["r"])
        b = torch.empty((1 << m) * 32, dtype=torch.uint8, device="cuda")
        L.spartan.eq_evals(field, got["r"], b.data_ptr())
        L.spartan.ipa_prove(curve, pcs[1], gc, got["joint"].data_ptr(), b.data_ptr(), m, lambda rnd, msg: challenge(k, "pcs", (rnd + 1, bytes(msg))) % p)


def run(nivc, reps, steady):
    t0 = time.perf_counter()
    if nivc:
        _, slot_elems = bench.slot_offsets(1, 0, bench.TRIE_LOOKUP["slots"], bench.TRIE_LOOKUP["bd"], 0)
        prim = [circuit(0, 1, 400), circuit(0, 2, 1, slot_elems=slot_elems, glue=bench.TRIE_LOOKUP["glue"], cons=bench.TRIE_LOOKUP["cons"])]
    else:
        prim = [circuit(0, 1, 100)]
    s = bench.SECONDARY
    sec = circuit(1, 8, 1, slot_elems=s["free"], glue=s["glue"], cons=s["cons"])
    setup_s = time.perf_counter() - t0
    m1 = max(max(c["ctx"].log_rows, c["ctx"].log_vars) for c in prim)
    m2 = max(sec["ctx"].log_rows, sec["ctx"].log_vars)
    g = points(0, 1, 9)[0]
    kck = L.CommitmentKey.powers_of_tau(0, g, 987654321987654321, 1 << m1)
    kck.precompute()
    ipa_ck = L.CommitmentKey(1, L.synthetic_bases(1, 1 << m2, start=1))
    ck_c = points(1, 1, (1 << m2) + 11)[0]
    pcs = [("hyperkzg", kck), ("ipa", ipa_ck, ck_c)]
    cp = points(0, 2 * len(prim), 100)
    cs = points(1, 2, 200)
    pinsts = [(c["z"].data_ptr(), c["e"].data_ptr(), cp[2 * i], cp[2 * i + 1]) for i, c in enumerate(prim)]
    sinst = (sec["z"].data_ptr(), sec["e"].data_ptr(), cs[0], cs[1])
    pctxs = [c["ctx"] for c in prim]
    batched = nivc
    torch.cuda.synchronize()
    tmp = tempfile.mkdtemp(prefix="compress_ctx_bench_")
    native_fn, native_lib = native_challenge(tmp)
    configs = ["composed", "sequential", "concurrent", "sequential_native_cb", "concurrent_native_cb"]
    first = {c: [] for c in configs[1:]}
    steady_t = {c: [] for c in configs}
    held = None
    for rep in range(reps):
        for cfg in configs:                                   # the configurations alternate
            if cfg == "composed":
                for _ in range(steady):
                    t = time.perf_counter()
                    composed(0, 0, pctxs, pinsts, pcs[0], batched)
                    composed(1, 1, [sec["ctx"]], [sinst], pcs[1], False)
                    torch.cuda.synchronize()
                    steady_t[cfg].append((time.perf_counter() - t) * 1e3)
                continue
            kw = dict(sequential=cfg.startswith("sequential"), batched=batched, native=(native_fn, None) if cfg.endswith("native_cb") else None)
            torch.cuda.synchronize()
            t = time.perf_counter()
            cctx = L.CompressContext(pctxs if nivc else pctxs[0], sec["ctx"], pcs[0], pcs[1])
            cctx.prove(pinsts, sinst, challenge, **kw)
            torch.cuda.synchronize()
            first[cfg].append((time.perf_counter() - t) * 1e3)
            for _ in range(steady):
                t = time.perf_counter()
                cctx.prove(pinsts, sinst, challenge, **kw)
                torch.cuda.synchronize()
                steady_t[cfg].append((time.perf_counter() - t) * 1e3)
            held = cctx.info()
            cctx.close()
    stat = lambda v: {"best_ms": round(min(v), 2), "spread_ms": round(max(v) - min(v), 2), "median_ms": round(float(np.median(v)), 2), "n": len(v)}
    out = {"op": "CompressedSNARK::prove, GPU half, primary + secondary" + (" (SuperNova, batched primary)" if nivc else " (Nova)"),
           "primary": [{"rows": c["rows"], "variables": c["n_w"], "rows_padded_log2": c["ctx"].log_rows, "vars_padded_log2": c["ctx"].log_vars} for c in prim],
           "primary_pcs": "HyperKZG (powers-of-tau key, fixed-base table)", "joint_len_primary_log2": m1,
           "secondary": {"rows": sec["rows"], "variables": sec["n_w"], "pcs": "IPA", "joint_len_log2": m2},
           "steady": {c: stat(v) for c, v in steady_t.items()}, "first_call_on_fresh_context": {c: stat(v) for c, v in first.items()},
           "context_device_bytes": held["device_bytes"] if held else None, "setup_s": round(setup_s, 1),
           "note": "best-of / spread over %d alternating rounds x %d steady calls; host clock around calls ending in a device synchronise; "
                   "(a) uses the Python transcript and host point arithmetic for the joint commitment, (b)/(c) the same Python transcript or a "
                   "native C one" % (reps, steady), **device_info()}
    print(json.dumps(out), flush=True)
    del native_lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nivc", action="store_true", help="SuperNova's batched primary at the trie_nivc shapes")
    ap.add_argument("--reps", type=int, default=4, help="alternating rounds of all configurations")
    ap.add_argument("--steady", type=int, default=3, help="steady-state calls per configuration and round")
    a = ap.parse_args()
    run(a.nivc, a.reps, a.steady)


if __name__ == "__main__":
    main()
