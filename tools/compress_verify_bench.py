#!/usr/bin/env python3
"""Wall-clock of CompressedSNARK::verify's GPU half (reference src/proof/nova.rs:358-373 / supernova.rs:304-317) in three configurations,
run alternately, on proofs lurk_compress_prove_dev made:
  (a) composed:    SpartanContext.verify (or spartan_verify_batch) + the joint commitment (lurk_point_combination) + the opening -- IPA:
                   the scale of ck_c, eq(r) and ipa_verify; HyperKZG: the fold check in Python and P, Q with lurk_point_combination --
                   primary then secondary;
  (b) sequential:  one lurk_compress_verify call with LURK_COMPRESS_SEQUENTIAL;
  (c) concurrent:  one lurk_compress_verify call, the secondary on a library thread and a forked stream.
Each runs under the Python transcript and under a native C one (built into a temporary directory with gcc).  The pairing callback does no
work (a native function answering "holds"): its cost is the caller's.  Every timed call must accept.

Also timed on their own: the host point arithmetic of the verifier -- the joint commitment (2n points), IPA's Q Straus (2 + 2m points:
comm, ck_c, L_j, R_j) and HyperKZG's P (m + 4 points) and Q (3 points) -- as lurk_point_combination calls of those sizes.

Shapes as tools/compress_ctx_bench.py: the fib rc = 100 primary (BN254 + HyperKZG on a powers-of-tau key), or with --nivc SuperNova's
batched primary at the trie_nivc shapes; bench.SECONDARY (Grumpkin + IPA) in both.  The instances are random but satisfied: z is random,
E = Az o Bz - u Cz, and the commitments are commit(W), commit(E) on the circuits' keys, so that the verifier runs every check.  One JSON
object per line: best, worst and median per configuration, milliseconds, host clock around calls that end in a device synchronise."""
import argparse
import ctypes as C
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
import compress_ctx_bench as ccb  # noqa: E402  (shapes, transcript, device info)
import lurk_beta_b200 as L  # noqa: E402
from oracle import spec as ospec  # noqa: E402  (the fold check's field arithmetic in the composed path)

NATIVE_PAIRING = r"""
#include <stdint.h>
int pairing(void *user, int circuit, const uint8_t *P, const uint8_t *Q, int *holds) { (void)user; (void)circuit; (void)P; (void)Q; *holds = 1; return 0; }
"""


def native_pairing(tmp):
    src, so = os.path.join(tmp, "pairing.c"), os.path.join(tmp, "libpairing.so")
    with open(src, "w") as f:
        f.write(NATIVE_PAIRING)
    subprocess.check_call(["/usr/bin/gcc", "-O2", "-shared", "-fPIC", src, "-o", so])
    lib = C.CDLL(so)
    return C.cast(lib.pairing, C.c_void_p).value, lib


def canonical(field, t):
    c = t.clone()
    L._capi.check(L._capi.lib().lurk_convert_dev(field, C.c_void_p(c.data_ptr()), c.numel() // 32, L.FMT_CANONICAL, C.c_void_p(c.data_ptr()), None))
    return c.cpu().numpy()


def point_of(b):
    v = [int.from_bytes(b[32 * i:32 * i + 32].tobytes(), "little") for i in range(3)]
    return (v[0], v[1]) if v[2] else None


def circuit(field, seed, frames, **shape):
    """ccb.circuit, keeping the matrices"""
    mats, n_w, rows, _ = ccb.bench.step_circuit(seed, frames, **shape)
    return dict(ctx=L.spartan.SpartanContext(field, mats, n_w, 2), z=ccb.rand_mont(n_w + 3, seed), e=ccb.rand_mont(rows, seed + 1), n_w=n_w, rows=rows,
                mats=mats)


def satisfied(field, c, ck):
    """E = Az o Bz - u Cz for the random z of c, and the instance's (u, X, comm_W, comm_E)"""
    n_w, rows = c["n_w"], c["rows"]
    y = [torch.empty(rows * 32, dtype=torch.uint8, device="cuda") for _ in range(3)]
    for m, (rp, col, val) in enumerate(c["mats"]):
        L.spartan.DeviceCSR(field, rows, rp, col, val).mv(field, c["z"].data_ptr(), y[m].data_ptr())
    zero = torch.zeros(rows * 32, dtype=torch.uint8, device="cuda")
    u_mont = c["z"][32 * n_w:32 * n_w + 32].cpu().numpy()
    L._capi.check(L._capi.lib().lurk_cross_term_dev(field, *[C.c_void_p(t.data_ptr()) for t in (y[0], zero, zero, y[0], y[1], y[2])],
                                                    L._capi.np_ptr(u_mont), L._capi.np_ptr(np.zeros(32, dtype=np.uint8)), rows,
                                                    C.c_void_p(c["e"].data_ptr()), None))
    zc, ec = canonical(field, c["z"]), canonical(field, c["e"])
    ints = lambda b: [int.from_bytes(b[32 * i:32 * i + 32].tobytes(), "little") for i in range(len(b) // 32)]
    return (ints(zc[32 * n_w:32 * n_w + 32])[0], ints(zc[32 * n_w + 32:]), point_of(ck.commit(zc[:32 * n_w])), point_of(ck.commit(ec)))


def combination(curve, pts, scalars):
    buf = np.concatenate([L.compress._point(P) for P in pts])
    out = np.zeros(96, dtype=np.uint8)
    L._capi.check(L._capi.lib().lurk_point_combination(curve, L._capi.np_ptr(buf), L._capi.np_ptr(L.spartan._fes(scalars)), len(pts), L.FMT_CANONICAL,
                                                       L._capi.np_ptr(out)))
    return point_of(out)


def composed(k, curve, ctxs, insts, proof, vk, batched):
    """configuration (a) for one circuit; returns whether it accepts"""
    field = ospec.CURVES[curve]["scalar"]
    p = ospec.FIELD_MODULUS[field]
    chal = lambda label, data: ccb.challenge(k, label, data)
    if batched:
        ok, d = L.spartan.spartan_verify_batch(ctxs, [x[:2] for x in insts], proof, chal)
    else:
        ok, d = ctxs[0].verify(proof, insts[0][0], insts[0][1], chal)
    if not ok:
        return False
    comm = combination(curve, [x[2] for x in insts] + [x[3] for x in insts], d["weights"])
    m = len(d["r"])
    if vk[0] == "ipa":
        msg = L.compress._point(comm).tobytes() + int(d["joint_eval"]).to_bytes(32, "little")
        gc = combination(curve, [vk[2]], [ccb.challenge(k, "pcs", (0, msg)) % p])
        b = torch.empty((1 << m) * 32, dtype=torch.uint8, device="cuda")
        L.spartan.eq_evals(field, d["r"], b.data_ptr())
        return L.spartan.ipa_verify(curve, vk[1], gc, comm, d["joint_eval"], b.data_ptr(), m, proof["L"], proof["R"], proof["a_final"],
                                    lambda rnd, msg: ccb.challenge(k, "pcs", (rnd + 1, bytes(msg))) % p)[0]
    com_b = b"".join(L.compress._point(P).tobytes() for P in proof["com"])
    r = ccb.challenge(k, "pcs", (0, com_b)) % p
    v, x = proof["v"], d["r"]
    Y = list(v[2]) + [d["joint_eval"]]
    if any(2 * r * Y[i + 1] % p != (r * (1 - x[m - 1 - i]) * (v[0][i] + v[1][i]) + x[m - 1 - i] * (v[0][i] - v[1][i])) % p for i in range(m)):
        return False
    q = ccb.challenge(k, "pcs", (1, L.spartan._fes([e for t in v for e in t]).tobytes())) % p
    dd = ccb.challenge(k, "pcs", (2, b"".join(L.compress._point(P).tobytes() for P in proof["w"]))) % p
    u, dt = [r, (-r) % p, r * r % p], [1, dd, dd * dd % p]
    qj = [pow(q, j, p) for j in range(m)]
    bu = sum(dt[t] * qj[j] * v[t][j] for t in range(3) for j in range(m)) % p
    combination(curve, [comm] + list(proof["com"]) + [vk[1]] + list(proof["w"]), [sum(dt) * e % p for e in qj] + [(-bu) % p] +
                [dt[t] * u[t] % p for t in range(3)])
    combination(curve, list(proof["w"]), dt)
    return True                                      # the pairing is the caller's, as in (b) and (c)


def time_host(curve, k, reps=20):
    """lurk_point_combination over k random points of `curve`: best and worst of reps calls, ms"""
    p = ospec.FIELD_MODULUS[ospec.CURVES[curve]["scalar"]]
    pts = ccb.points(curve, k, 5000)
    rng = np.random.default_rng(k)
    sc = [int.from_bytes(rng.bytes(32), "little") % p for _ in range(k)]
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        combination(curve, pts, sc)
        t.append((time.perf_counter() - t0) * 1e3)
    return {"points": k, "best_ms": round(min(t), 3), "worst_ms": round(max(t), 3)}


def run(nivc, reps, steady):
    t0 = time.perf_counter()
    if nivc:
        _, slot_elems = ccb.bench.slot_offsets(1, 0, ccb.bench.TRIE_LOOKUP["slots"], ccb.bench.TRIE_LOOKUP["bd"], 0)
        shapes = [(1, 400, {}), (2, 1, dict(slot_elems=slot_elems, glue=ccb.bench.TRIE_LOOKUP["glue"], cons=ccb.bench.TRIE_LOOKUP["cons"]))]
    else:
        shapes = [(1, 100, {})]
    s = ccb.bench.SECONDARY
    prim = [circuit(0, seed, frames, **kw) for seed, frames, kw in shapes]
    sec = circuit(1, 8, 1, slot_elems=s["free"], glue=s["glue"], cons=s["cons"])
    m1 = max(max(c["ctx"].log_rows, c["ctx"].log_vars) for c in prim)
    m2 = max(sec["ctx"].log_rows, sec["ctx"].log_vars)
    g = ccb.points(0, 1, 9)[0]
    kck = L.CommitmentKey.powers_of_tau(0, g, 987654321987654321, 1 << m1)
    kck.precompute()
    ipa_ck = L.CommitmentKey(1, L.synthetic_bases(1, 1 << m2, start=1))
    ck_c = ccb.points(1, 1, (1 << m2) + 11)[0]
    pinsts = [satisfied(0, c, kck) for c in prim]
    sinst = satisfied(1, sec, ipa_ck)
    pctxs = [c["ctx"] for c in prim]
    cctx = L.CompressContext(pctxs if nivc else pctxs[0], sec["ctx"], ("hyperkzg", kck), ("ipa", ipa_ck, ck_c))
    proof = cctx.prove([(c["z"].data_ptr(), c["e"].data_ptr(), x[2], x[3]) for c, x in zip(prim, pinsts)],
                       (sec["z"].data_ptr(), sec["e"].data_ptr(), sinst[2], sinst[3]), ccb.challenge, batched=nivc)
    cctx.close()
    setup_s = time.perf_counter() - t0
    vk = [("hyperkzg", g), ("ipa", ipa_ck, ck_c)]
    tmp = tempfile.mkdtemp(prefix="compress_verify_bench_")
    chal_fn, chal_lib = ccb.native_challenge(tmp)
    pair_fn, pair_lib = native_pairing(tmp)
    # the native transcript's proof: made under the same C function, so that it verifies under it
    cctx = L.CompressContext(pctxs if nivc else pctxs[0], sec["ctx"], ("hyperkzg", kck), ("ipa", ipa_ck, ck_c))
    proof_native = cctx.prove([(c["z"].data_ptr(), c["e"].data_ptr(), x[2], x[3]) for c, x in zip(prim, pinsts)],
                              (sec["z"].data_ptr(), sec["e"].data_ptr(), sinst[2], sinst[3]), None, batched=nivc, native=(chal_fn, None))
    cctx.close()
    torch.cuda.synchronize()
    configs = ["composed", "sequential", "concurrent", "sequential_native_cb", "concurrent_native_cb"]
    times = {c: [] for c in configs}
    accepted = {c: True for c in configs}
    for rep in range(reps + 1):                                 # round 0 warms every configuration up and is not counted
        for cfg in configs:                                     # the configurations alternate
            for _ in range(steady):
                torch.cuda.synchronize()
                t = time.perf_counter()
                if cfg == "composed":
                    ok = composed(0, 0, pctxs, pinsts, proof[0], vk[0], nivc) and composed(1, 1, [sec["ctx"]], [sinst], proof[1], vk[1], False)
                else:
                    nat = cfg.endswith("native_cb")
                    ok, _ = L.compress_verify(pctxs if nivc else pctxs[0], sec["ctx"], vk[0], vk[1], pinsts, sinst, proof_native if nat else proof,
                                              ccb.challenge, batched=nivc, sequential=cfg.startswith("sequential"),
                                              native=(chal_fn, None) if nat else None, native_pairing=pair_fn)
                torch.cuda.synchronize()
                if rep:
                    times[cfg].append((time.perf_counter() - t) * 1e3)
                    accepted[cfg] &= bool(ok)
    stat = lambda v: {"best_ms": round(min(v), 2), "worst_ms": round(max(v), 2), "median_ms": round(float(np.median(v)), 2), "n": len(v)}
    n = len(prim)
    host = {"joint_commitment_primary": time_host(0, 2 * n), "joint_commitment_secondary": time_host(1, 2),
            "ipa_Q_straus_secondary": time_host(1, 2 + 2 * m2), "hyperkzg_P_primary": time_host(0, m1 + 4), "hyperkzg_Q_primary": time_host(0, 3)}
    out = {"op": "CompressedSNARK::verify, GPU half, primary + secondary" + (" (SuperNova, batched primary)" if nivc else " (Nova)"),
           "primary": [{"rows": c["rows"], "variables": c["n_w"], "rows_padded_log2": c["ctx"].log_rows, "vars_padded_log2": c["ctx"].log_vars} for c in prim],
           "primary_pcs": "HyperKZG (pairing left to a no-op callback)", "joint_len_primary_log2": m1,
           "secondary": {"rows": sec["rows"], "variables": sec["n_w"], "pcs": "IPA", "joint_len_log2": m2},
           "steady": {c: stat(v) for c, v in times.items()}, "accepted": accepted, "host_point_arithmetic": host, "setup_s": round(setup_s, 1),
           "note": "best / worst / median over %d alternating rounds x %d calls after one warm-up round; host clock around calls ending in a device "
                   "synchronise; (a) uses the Python transcript, (b)/(c) the Python one or a native C one" % (reps, steady), **ccb.device_info()}
    print(json.dumps(out), flush=True)
    del chal_lib, pair_lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nivc", action="store_true", help="SuperNova's batched primary at the trie_nivc shapes")
    ap.add_argument("--reps", type=int, default=4, help="alternating rounds of all configurations")
    ap.add_argument("--steady", type=int, default=2, help="calls per configuration and round")
    a = ap.parse_args()
    run(a.nivc, a.reps, a.steady)


if __name__ == "__main__":
    main()
