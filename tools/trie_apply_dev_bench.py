"""The trie store's two forms side by side: lurk_trie_ctx_apply (operations in host memory, planned on the host) and
lurk_trie_ctx_apply_dev (operations in device memory, planned on the GPU), through trie.DeviceTrie.apply / apply_dev.

Writes profiles/h100_trie_apply_dev.jsonl (one JSON object per line), with the card's name and power limit read in
the same run.

  python tools/trie_apply_dev_bench.py [--out profiles/h100_trie_apply_dev.jsonl] [--quick]

Workloads of tools/trie_apply_bench.py (BN254 Fr, H = 85): random-key inserts at 10^3, 10^4 and 10^5 operations,
shared-prefix inserts and the 50/50 insert / lookup mix at 10^5.  Both forms run in this process, alternating, each
timed batch on a fresh context warmed by one untimed batch of the same shape.  Before any timing, both forms apply the
same batch and their results, proofs and node counts must be equal.
Timing, per call: the host clock around the call (both forms end in a stream synchronise, so the window holds all of
its work) and CUDA events on the call's stream.  The host form's window includes its Python packing of the operations
(ints -> arrays), which is also timed on its own (pack_ms); the device form's inputs are CUDA tensors made before its
window starts.
Breakdown: one more 10^5 random-key batch through apply_dev under torch.profiler, device time summed per kernel group:
the planner (validate, pointer jumping, ranks, order keys, lcp, and its CUB scan and 32-bit key-value sorts) against
the levels (walk, level kernel, the arity-8 digest launch, registration, their CUB scan and 64-bit key sorts, finish).
"""
import argparse
import json
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

H = 85
PLANNER = ("first_continuer_kernel", "validate_kernel", "jump_kernel", "chain_rank_kernel", "order_key_kernel", "lcp_kernel")


def device_ops(torch, ops):
    """(kinds, prev, roots, keys, values) CUDA tensors of ops"""
    from lurk_beta_b200.field import pack
    n = len(ops)
    col = lambda k: torch.from_numpy(pack([int(o[k]) for o in ops]).reshape(n, 32)).cuda()
    return (torch.tensor([o[0] for o in ops], dtype=torch.int32, device="cuda"), torch.tensor([o[1] for o in ops], dtype=torch.int64, device="cuda"),
            col(2), col(3), col(4))


def pack_ms(ops):
    """the host form's packing of the operations on its own (what DeviceTrie.apply does before the library call)"""
    from lurk_beta_b200.field import pack
    t0 = time.perf_counter()
    np.array([o[0] for o in ops], dtype=np.int32)
    np.array([o[1] for o in ops], dtype=np.int64)
    for k in (2, 3, 4):
        pack([int(o[k]) for o in ops])
    return (time.perf_counter() - t0) * 1e3


def group_of(name):
    if any(k in name for k in PLANNER):
        return "plan_kernels"
    if "RadixSort" in name:
        # the planner sorts 32-bit keys with 32-bit values; the levels sort 64-bit keys alone
        return "level_cub_sort" if ("unsigned long" in name or "NullType" in name) else "plan_cub_sort"
    if "Scan" in name:
        return "cub_scan"
    for needle, group in (("poseidon", "level_poseidon8_digests"), ("level_kernel", "level_kernel"), ("walk_kernel", "level_walk"),
                          ("claim_kernel", "level_register"), ("publish_kernel", "level_register"), ("finish_kernel", "level_finish"),
                          ("group_flags", "level_other"), ("sort_keys_kernel", "level_other"), ("Memcpy", "copies"), ("Memset", "copies")):
        if needle in name:
            return group
    return "other_kernels"


def breakdown(L, torch, ops_for, p, rng):
    from torch.profiler import ProfilerActivity, profile
    K = 100_000
    dt = L.DeviceTrie(0, H, capacity=2 * H * K + 4 * H + 16)
    root = dt.empty_root()
    dt.apply_dev(*device_ops(torch, ops_for("random", K, p, rng, root)))
    args = device_ops(torch, ops_for("random", K, p, rng, root))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dt.apply_dev(*args)
        b.record()
        b.synchronize()
    span = a.elapsed_time(b)
    groups, names = {}, {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us:
            g = group_of(e.key)
            groups[g] = groups.get(g, 0.0) + us / 1e3
            if g.startswith("plan"):
                names[e.key[:80]] = us / 1e3
    dt.close()
    plan = sum(v for g, v in groups.items() if g.startswith("plan"))
    return dict(kind="breakdown", form="apply_dev", workload="random", ops=K, span_ms=span, device_ms_by_group=groups,
                device_ms_total=sum(groups.values()), plan_device_ms=plan, plan_kernels_ms=names,
                note="torch.profiler CUDA activity in a run of its own; cub_scan holds the planner's one scan of n flags and "
                     "the levels' H scans of m flags")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_trie_apply_dev.jsonl"))
    ap.add_argument("--quick", action="store_true")
    args = ap.parse_args()
    import torch
    import lurk_beta_b200 as L
    from oracle import spec
    from trie_apply_bench import ops_for
    from trie_witness_bench import card

    p = spec.FIELD_MODULUS[0]
    rows = [dict(kind="setup", **card(), note="per call: host clock (both forms end in a synchronise) and CUDA events on the call's stream; "
                                               "apply's window includes its Python packing, apply_dev's inputs are on the device first")]
    rng = random.Random(1)
    work = [("random", 1000), ("random", 10_000)] if args.quick else [("random", 1000), ("random", 10_000), ("random", 100_000),
                                                                       ("shared", 100_000), ("mix", 100_000)]
    st = torch.cuda.current_stream()

    def fresh(kind, K):
        dt = L.DeviceTrie(0, H, capacity=2 * H * K + 4 * H + 16)   # room for the warm-up batch and the timed one
        root = dt.empty_root()
        return dt, root

    for kind, K in work:
        # equal outputs first: the same batch through both forms on twin contexts
        a_dt, root = fresh(kind, K)
        b_dt, _ = fresh(kind, K)
        ops = ops_for(kind, K, p, rng, root)
        ra, la, ia = a_dt.apply(ops)
        rb, lb, ib = b_dt.apply_dev(*device_ops(torch, ops))
        torch.cuda.synchronize()
        equal = (np.array_equal(np.frombuffer(b"".join(int(r).to_bytes(32, "little") for r in ra), dtype=np.uint8), rb.cpu().numpy().reshape(-1))
                 and torch.equal(la.reshape(-1), lb.reshape(-1)) and torch.equal(ia.reshape(-1), ib.reshape(-1)) and a_dt.node_count == b_dt.node_count)
        assert equal, f"{kind} {K}: apply and apply_dev differ"
        del ra, la, ia, rb, lb, ib
        a_dt.close(), b_dt.close()
        torch.cuda.empty_cache()

        reps = 3 if K < 100_000 else 2
        t = {"apply": dict(host_ms=[], device_ms=[]), "apply_dev": dict(host_ms=[], device_ms=[])}
        packs = []
        for _ in range(reps):
            for form in ("apply", "apply_dev"):
                dt, root = fresh(kind, K)
                warm = ops_for(kind, K, p, rng, root)
                if form == "apply":
                    dt.apply(warm)
                else:
                    dt.apply_dev(*device_ops(torch, warm))
                ops = ops_for(kind, K, p, rng, root)
                dev_args = device_ops(torch, ops) if form == "apply_dev" else None
                if form == "apply":
                    packs.append(pack_ms(ops))
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                e0.record(st)
                out = dt.apply(ops) if form == "apply" else dt.apply_dev(*dev_args)
                e1.record(st)
                e1.synchronize()
                t[form]["host_ms"].append((time.perf_counter() - t0) * 1e3)
                t[form]["device_ms"].append(e0.elapsed_time(e1))
                del out, dev_args
                dt.close()
                torch.cuda.empty_cache()
        inserts = sum(1 for o in ops if o[0] == 1)
        rows.append(dict(kind="compare", workload=kind, ops=K, inserts=inserts, lookups=K - inserts, outputs_equal=True,
                         apply=t["apply"], apply_dev=t["apply_dev"], apply_pack_ms=packs,
                         apply_best_host_ms=min(t["apply"]["host_ms"]), apply_dev_best_host_ms=min(t["apply_dev"]["host_ms"]),
                         gpu=rows[0]["gpu"], power_limit=rows[0]["power_limit"]))
        print(json.dumps(rows[-1]), flush=True)
    if not args.quick:
        rows.append(breakdown(L, torch, ops_for, p, rng))
        print(json.dumps(rows[-1]), flush=True)
    rows.append(dict(kind="setup_end", **card()))
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
