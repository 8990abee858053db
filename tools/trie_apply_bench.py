"""Trie operations applied on the GPU (csrc/trie_store.cu, trie.DeviceTrie): device time per batch, arity-8 hashes per
second, and the bytes that cross PCIe against the host-packed `insert_inputs` / `lookup_inputs` path.

Writes profiles/h100_trie_apply.jsonl (one JSON object per line), with the card's name and power limit read in the
same run.

  python tools/trie_apply_bench.py [--out profiles/h100_trie_apply.jsonl] [--quick]

BN254 Fr, H = 85 (StandardTrie), K = 10^3, 10^4 and 10^5 operations in one chain from the empty root:
  random   inserts of random keys;
  shared   inserts of keys that share all but their lowest 12 bits (4 chunks), so the paths overlap down to depth 81;
  mix      a 50/50 mix of inserts of random keys and lookups of earlier keys at the chain's latest version.
Every timed batch runs on a fresh context that has first applied one untimed batch of the same shape with other keys
and values, so the context's scratch is allocated, its store is not empty, and the timed batch's nodes are new.
Timing: CUDA events on the call's stream around lurk_trie_ctx_apply, which includes the host's argument check and key
sort (the start event is recorded before them) and ends when the call returns; and the host clock around the call.
Breakdown: one more such batch of 10^5 random-key inserts under torch.profiler, device time summed per kernel group
(the arity-8 digest launch, the level kernel, the walk, registration, CUB's scan and sort, the rest, and copies).
Hashes = H x inserts per batch.  PCIe bytes: this path sends, per operation, its 64-byte descriptor and root, key and
value (32 bytes each), plus 6 bytes per insert for the key order, and reads back 32 bytes of result; the host-packed
path sends 32 x (2 + 8H) bytes per lookup and 32 x (3 + 16H) per insert to lurk_trie_witness_batch_dev.

CPU baseline: the oracle's C arity-8 Poseidon (oracle.capi.poseidon_hash_batch) over a sample of random preimages on 1
and on all host threads; hashes per second, so the time a sequential Trie::insert loop spends hashing is H x inserts
over that rate.
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


def ops_for(kind, K, p, rng, root):
    ops = []
    keys = []
    stem = rng.randrange(p >> 12) << 12
    for i in range(K):
        prev = -1 if i == 0 else i - 1
        if kind == "mix" and i % 2 == 1:
            ops.append((0, i - 1, 0, rng.choice(keys), 0))    # lookups name the latest insert, i - 1
            continue
        if kind == "mix" and i > 1:
            prev = i - 2
        key = stem + rng.randrange(1 << 12) if kind == "shared" else rng.randrange(p)
        keys.append(key)
        ops.append((1, prev, root, key, rng.randrange(p)))
    return ops


GROUPS = (("poseidon", "poseidon8_digests"), ("level_kernel", "level_kernel"), ("walk_kernel", "walk_kernel"),
          ("claim_kernel", "register"), ("publish_kernel", "register"), ("Scan", "cub_scan"), ("RadixSort", "cub_sort"),
          ("Memcpy", "copies"), ("Memset", "copies"))


def group_of(name):
    for needle, group in GROUPS:
        if needle in name:
            return group
    return "other_kernels"


def breakdown(L, torch, ops_for, p, rng):
    from torch.profiler import ProfilerActivity, profile
    K = 100_000
    dt = L.DeviceTrie(0, H, capacity=2 * H * K + 4 * H + 16)
    root = dt.empty_root()
    dt.apply(ops_for("random", K, p, rng, root))
    ops = ops_for("random", K, p, rng, root)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dt.apply(ops)
        b.record()
        b.synchronize()
    span = a.elapsed_time(b)
    groups = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us:
            g = group_of(e.key)
            groups[g] = groups.get(g, 0.0) + us / 1e3
    dt.close()
    return dict(kind="breakdown", workload="random", ops=K, span_ms=span, device_ms_by_group=groups,
                device_ms_total=sum(groups.values()), note="torch.profiler CUDA activity; the span includes host planning and launch gaps")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_trie_apply.jsonl"))
    ap.add_argument("--quick", action="store_true")
    args = ap.parse_args()
    import torch
    import lurk_beta_b200 as L
    from oracle import capi as oracle
    from oracle import spec
    from trie_witness_bench import card

    p = spec.FIELD_MODULUS[0]
    rows = [dict(kind="setup", **card(), note="device: CUDA events around lurk_trie_ctx_apply (host planning included); host: wall clock")]
    rng = random.Random(1)
    sizes = (1000, 10_000) if args.quick else (1000, 10_000, 100_000)
    for kind in ("random", "shared", "mix"):
        for K in sizes:
            reps = 3 if K < 100_000 else 2
            st = torch.cuda.current_stream()
            dev_ms, host_ms, nodes = [], [], []
            for _ in range(reps):
                dt = L.DeviceTrie(0, H, capacity=2 * H * K + 4 * H + 16)   # room for the warm-up batch and the timed one
                root = dt.empty_root()
                dt.apply(ops_for(kind, K, p, rng, root))
                ops = ops_for(kind, K, p, rng, root)
                inserts = sum(1 for o in ops if o[0] == 1)
                lookups = K - inserts
                before = dt.node_count
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                a.record(st)
                res, lk, ins = dt.apply(ops)
                b.record(st)
                b.synchronize()
                host_ms.append((time.perf_counter() - t0) * 1e3)
                dev_ms.append(a.elapsed_time(b))
                nodes.append(dt.node_count - before)
                del lk, ins
                dt.close()
                torch.cuda.empty_cache()
            hashes = H * inserts
            ours = K * (64 + 96 + 32) + 6 * inserts
            packed = 32 * ((2 + 8 * H) * lookups + (3 + 16 * H) * inserts)
            rows.append(dict(kind="apply", workload=kind, ops=K, inserts=inserts, lookups=lookups, new_nodes=nodes,
                             device_ms=dev_ms, host_ms=host_ms, hashes=hashes,
                             hashes_per_s_first=hashes / (dev_ms[0] / 1e3), hashes_per_s_best=hashes / (min(dev_ms) / 1e3),
                             pcie_bytes=ours, pcie_bytes_host_packed=packed, gpu=rows[0]["gpu"], power_limit=rows[0]["power_limit"]))
            print(json.dumps(rows[-1]), flush=True)
    if not args.quick:
        rows.append(breakdown(L, torch, ops_for, p, rng))
        print(json.dumps(rows[-1]), flush=True)
    n = 20_000 if args.quick else 200_000
    pre_rng = random.Random(2)
    pre = np.frombuffer(b"".join(pre_rng.randrange(p).to_bytes(32, "little") for _ in range(8 * n)), dtype=np.uint8).copy()
    for threads in sorted({1, oracle.threads()}):
        t0 = time.perf_counter()
        oracle.poseidon_hash_batch(0, 8, pre, nthreads=threads)
        s = time.perf_counter() - t0
        rows.append(dict(kind="cpu_poseidon8", threads=threads, hashes=n, seconds=s, hashes_per_s=n / s, host_cpus=os.cpu_count()))
        print(json.dumps(rows[-1]), flush=True)
    rows.append(dict(kind="setup_end", **card()))
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
