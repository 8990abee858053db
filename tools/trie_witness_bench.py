"""Trie coprocessor witness on the GPU (csrc/trie.cu): kernel time and write bandwidth, and the fold step of the lookup and
insert circuits with their blocks written by the device batch against the same blocks taken through the glue buffer.

Writes profiles/h100_trie_witness.jsonl (one JSON object per line), with the card's name and power limit read in the
same run.

  python tools/trie_witness_bench.py [--out profiles/h100_trie_witness.jsonl] [--quick]

Kernel: BN254 Fr, H = 85 (StandardTrie), lookup and insert, 1, 100 and 10 000 calls (one call is what a NIVC coprocessor
step runs); CUDA events around repeated launches of lurk_trie_witness_batch_dev / _scatter_dev (both launches of a
batch).  Bytes = count * 32 B * (block length + inputs).  10 000 inserts (21.8 GB of blocks) use the scatter form with
offsets that wrap around a 16 GB buffer: the same bytes reach HBM, later calls overwrite earlier ones.

Fold step: one frame per step whose R1CS is the oracle's constraints of one H = 85 call (tests/trie_gadget_oracle.py)
plus its 4 glue columns (root, key, value, not_dummy), BN254.  "glue": the host writes the whole block into the glue
buffer and it is copied to the device every step; "device": a trie batch of one call writes the block from the call's
inputs.  The two alternate in the same process, staged inputs, host clock around a step ending in a device synchronise.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_TBS = 3.35
H = 85


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, sm = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return dict(gpu=name, power_limit=power, sm_max_clock=sm)


def kernel_rows(L, torch, quick):
    lib = L._capi.lib()
    rng = np.random.default_rng(1)
    cap_bytes = 16 << 30
    out = torch.empty(cap_bytes, dtype=torch.uint8, device="cuda")
    rows = []
    for op in (L.TRIE_LOOKUP, L.TRIE_INSERT):
        blk = L.trie_witness_block(0, op, H)
        n_in = 3 + 16 * H if op == L.TRIE_INSERT else 2 + 8 * H
        for count in ((1, 100) if quick else (1, 100, 10_000)):
            x = rng.integers(0, 256, size=(count * n_in, 32), dtype=np.uint8)
            x[:, 31] &= 0x0F                                     # < p
            d_in = torch.from_numpy(x.reshape(-1)).cuda()
            fits = count * blk * 32 <= cap_bytes
            offs = (np.arange(count, dtype=np.int64) % (cap_bytes // (blk * 32))) * blk
            d_off = torch.from_numpy(offs).cuda()

            def launch():
                if fits:
                    L._capi.check(lib.lurk_trie_witness_batch_dev(0, op, H, d_in.data_ptr(), count, out.data_ptr(), 1, None))
                else:
                    L._capi.check(lib.lurk_trie_witness_scatter_dev(0, op, H, d_in.data_ptr(), count, d_off.data_ptr(), out.data_ptr(), 1, None))

            launch()
            torch.cuda.synchronize()
            reps = 5 if count >= 10_000 else 50
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                launch()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / reps
            nbytes = count * 32 * (blk + n_in)
            rows.append(dict(kind="kernel", field=0, op="insert" if op else "lookup", height=H, count=count, block_elems=blk, bytes=nbytes,
                             ms=round(ms, 4), achieved_tbs=round(nbytes / (ms / 1e3) / 1e12, 4),
                             form="batch_dev" if fits else "scatter_dev (offsets wrap in 16 GB)"))
            print(json.dumps(rows[-1]), flush=True)
    del out
    torch.cuda.empty_cache()
    return rows


def fold_rows(L, torch, samples):
    import trie_gadget_oracle as T
    from oracle import nifs
    curve, field, glue = 0, 0, 4
    p = T.spec.FIELD_MODULUS[field]
    rows = []
    for op in (T.LOOKUP, T.INSERT):
        blk = L.trie_witness_block(field, op, H)
        n_w, n_x = glue + blk, 2
        mats = [nifs.rows_to_csr(m) for m in T.r1cs_rows(field, op, H, glue, 0, 1, 3, n_w)]
        ck = L.CommitmentKey(curve, L.synthetic_bases(curve, max(n_w, len(mats[0][0]) - 1)))
        trie = L.StandardTrie()
        rng = random.Random(op)
        key = rng.randrange(p)
        if op == T.INSERT:
            root = trie.root
            proof, _ = trie.prove_insert(key, 456)
            ins = L.insert_inputs(root, key, 456, proof)
        else:
            trie.insert(key, 456)
            ins = L.lookup_inputs(trie.root, key, trie.prove_lookup(key))
        block = L.trie_witness_batch(field, op, H, L.field.pack(ins))
        g = L.field.pack([ins[0], key, 456 if op == T.INSERT else 0, 1])
        X2 = L.field.pack([7, 9])
        ro = np.zeros((24, 32), dtype=np.uint8)
        ro[4], ro[5] = X2[:32], X2[32:]
        variants = {}
        for name in ("glue", "device"):
            ctx = L.NovaFoldContext(curve, ck, n_w, n_x, mats, depth=2)
            if name == "device":
                bi = ctx.add_trie_batch(op, H, [glue])
                ctx.set_spans([(0, glue, n_w, 1)])
            else:
                ctx.set_spans([(0, n_w, n_w, 1)])
            for b in range(2):
                ctx.host_buffer(b, -1)[:] = g if name == "device" else np.concatenate([g, block])
                ctx.host_buffer(b, -2)[:] = X2
                ctx.host_buffer(b, -3)[:] = ro.reshape(-1)
                if name == "device":
                    ctx.host_buffer(b, bi)[:] = L.field.pack(ins)
            variants[name] = ctx

        def step(ctx, i):
            b = i % 2
            ctx.stage_a(b)
            if i == 0:
                ctx.init_running(b)
            else:
                ctx.stage_b_launch(b)
            ctx.collect(b)

        counts = {k: 0 for k in variants}
        for name, ctx in variants.items():
            for _ in range(3):
                step(ctx, counts[name])
                counts[name] += 1
        times = {k: [] for k in variants}
        for _ in range(samples):
            for name, ctx in variants.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                step(ctx, counts[name])
                ctx.sync()
                torch.cuda.synchronize()
                times[name].append((time.perf_counter() - t0) * 1e3)
                counts[name] += 1
        for name, ctx in variants.items():
            ms = sorted(times[name])
            st = ctx.stats()
            bad, okw, oke = ctx.check_running()
            rows.append(dict(kind="fold_step", variant=name, op="insert" if op else "lookup", height=H, n_w=n_w, rows=len(mats[0][0]) - 1,
                             samples=len(ms), ms_per_step_median=round(ms[len(ms) // 2], 3), ms_per_step_p10=round(ms[len(ms) // 10], 3),
                             ms_per_step_p90=round(ms[(9 * len(ms)) // 10], 3), ms_per_step_min=round(ms[0], 3), ms_per_step_max=round(ms[-1], 3),
                             launches_a=st["launches_a"], launches_b=st["launches_b"],
                             running_instance_check=dict(bad_rows=int(bad), comm_W_ok=okw, comm_E_ok=oke)))
            print(json.dumps(rows[-1]), flush=True)
            ctx.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_trie_witness.jsonl"))
    ap.add_argument("--quick", action="store_true", help="1 and 100 calls only, fewer fold samples")
    args = ap.parse_args()
    import torch
    import lurk_beta_b200 as L
    if L._capi.lib().lurk_device_count() < 1:
        sys.exit("needs a CUDA device")
    head = dict(kind="setup", **card(), hbm_datasheet_tbs=HBM_TBS, note="kernel: CUDA events; fold step: host clock around a step ending in a device synchronise")
    print(json.dumps(head), flush=True)
    rows = [head] + kernel_rows(L, torch, args.quick) + fold_rows(L, torch, samples=10 if args.quick else 40)
    rows.append(dict(kind="setup_end", **card()))
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
