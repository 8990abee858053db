"""SHA-256 coprocessor witness on the GPU (csrc/sha256.cu): kernel write bandwidth, and the sha256_ivc fold step with the
gadget's columns written by the device batch against the same step taking them through the glue buffer.

Writes profiles/h100_sha256_witness.jsonl (one JSON object per line), with the card's name and power limit read in the
same run.

  python tools/sha256_witness_bench.py [--out profiles/h100_sha256_witness.jsonl] [--quick]

Kernel: per field, n in {1, 2, 4} and count in {10, 1 000, 100 000}; CUDA events around repeated launches.  Algorithmic
bytes = count * (32 B * block length + 64 n B of inputs); the kernel is bound by those HBM writes, reported against
3.35 TB/s (H100 SXM data sheet).  Counts whose blocks do not fit into the output buffer (100 000 calls are 145-400 GB)
use the scatter form with block offsets that wrap around a 16 GB buffer: the same bytes reach HBM, later calls overwrite
earlier ones.

Fold step: bench.py's sha256_ivc shape (rc = 10 frames, BN254 primary + Grumpkin secondary, SHA256_FRAME) with the
frame's boolean columns sized to one n = 1 block.  "glue": the host writes them into the glue buffer and they are copied
to the device every step (today's path); "device": the glue span stops before them and a SHA-256 batch of one call per
frame writes them on the device from 2 inputs per frame.  The two alternate in the same process, staged inputs (the
end-to-end step: host-to-device copies included).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBS = 3.35


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
    counts = (10, 1000) if quick else (10, 1000, 100_000)
    for field in (0, 1, 2, 3):
        for n in (1, 2, 4):
            blk = L.witness_block(field, n)
            for count in counts:
                x = rng.integers(0, 256, size=(count * 2 * n, 32), dtype=np.uint8)
                x[:, 31] &= 0x0F                                     # < p on every field
                d_in = torch.from_numpy(x.reshape(-1)).cuda()
                fits = count * blk * 32 <= cap_bytes
                offs = (np.arange(count, dtype=np.int64) % (cap_bytes // (blk * 32))) * blk
                d_off = torch.from_numpy(offs).cuda()

                def launch():
                    if fits:
                        L._capi.check(lib.lurk_sha256_witness_batch_dev(field, n, d_in.data_ptr(), count, out.data_ptr(), 1, None))
                    else:
                        L._capi.check(lib.lurk_sha256_witness_scatter_dev(field, n, d_in.data_ptr(), count, d_off.data_ptr(), out.data_ptr(), 1, None))

                launch()
                torch.cuda.synchronize()
                reps = 3 if count * blk > 2e9 else (10 if count * blk > 1e8 else 50)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(reps):
                    launch()
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / reps
                nbytes = count * (32 * blk + 64 * n)
                rows.append(dict(kind="kernel", field=field, n=n, count=count, block_elems=blk, bytes=nbytes, ms=round(ms, 4),
                                 achieved_tbs=round(nbytes / (ms / 1e3) / 1e12, 3), share_of_hbm=round(nbytes / (ms / 1e3) / 1e12 / HBM_TBS, 3),
                                 form="batch_dev" if fits else "scatter_dev (offsets wrap in 16 GB)"))
                print(json.dumps(rows[-1]), flush=True)
    del out
    torch.cuda.empty_cache()
    return rows


def fold_rows(L, torch, rounds, steps):
    import bench
    blk = L.witness_block(0, 1)
    bench.SHA256_FRAME = dict(bench.SHA256_FRAME, bits=blk)      # one n = 1 block per frame in both variants
    variants = {}
    for name in ("glue", "device"):
        wl = bench.FoldStepGPU(0, 1, workload="sha256_ivc", rc=10)
        if name == "device":
            inst = wl.inst[0]
            ctx, frames, per = inst.ctx, inst.frames, inst.per
            first = inst.slot_elems + inst.glue
            saved = [ctx.host_buffer(b, L._capi.FOLD_BUF_GLUE).reshape(frames, -1)[:, :inst.glue * 32].copy() for b in range(2)]
            ctx.set_spans([(inst.slot_elems, inst.glue, per, frames)])
            idx = ctx.add_sha256_batch(1, [f * per + first for f in range(frames)])
            rng = np.random.default_rng(3)
            for b in range(2):
                ctx.host_buffer(b, L._capi.FOLD_BUF_GLUE)[:] = saved[b].reshape(-1)
                x = rng.integers(0, 256, size=(frames * 2, 32), dtype=np.uint8)
                x[:, 31] &= 0x0F
                ctx.host_buffer(b, idx)[:] = x.reshape(-1)
            wl.h2d_bytes = sum(i.ctx.host_buffer(0, w).size for i in wl.inst for w in range(len(i.ctx.batches))) + \
                sum(i.ctx.host_buffer(0, w).size for i in wl.inst for w in (-1, -2, -3))
        wl.start(staged=True)
        for _ in range(3):
            wl.step(True)
        wl.drain()
        variants[name] = wl
    samples = {k: [] for k in variants}
    for r in range(rounds):
        for name, wl in variants.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                wl.step(True)
            wl.drain()
            torch.cuda.synchronize()
            samples[name].append((time.perf_counter() - t0) * 1e3 / steps)
    rows = []
    for name, wl in variants.items():
        ms = sorted(samples[name])
        st = wl.inst[0].ctx.stats()
        bad, okw, oke = wl.inst[0].ctx.check_running()
        rows.append(dict(kind="fold_step", variant=name, workload="sha256_ivc", rc=10, block_elems=blk, steps_per_sample=steps,
                         ms_per_step_median=round(ms[len(ms) // 2], 3), ms_per_step_min=round(ms[0], 3), ms_per_step_max=round(ms[-1], 3),
                         samples=len(ms), h2d_bytes_per_step=int(wl.h2d_bytes), launches_a=st["launches_a"], launches_b=st["launches_b"],
                         running_instance_check=dict(bad_rows=int(bad), comm_W_ok=okw, comm_E_ok=oke)))
        if name == "device":
            # bench.py's synthetic shape puts a booleanity row on every column of the bits region; the block's last two
            # elements (pack_bits' element, ExprTag::Num) are not bits, so 2 rows per frame do not hold
            rows[-1]["running_instance_check"]["expected_bad_rows"] = 2 * wl.inst[0].frames
        print(json.dumps(rows[-1]), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_sha256_witness.jsonl"))
    ap.add_argument("--quick", action="store_true", help="counts 10 and 1 000 only, fewer fold samples")
    args = ap.parse_args()
    import torch
    import lurk_beta_b200 as L
    if L._capi.lib().lurk_device_count() < 1:
        sys.exit("needs a CUDA device")
    head = dict(kind="setup", **card(), hbm_datasheet_tbs=HBM_TBS, note="kernel: CUDA events; fold step: host clock around steps ending in a device synchronise")
    print(json.dumps(head), flush=True)
    rows = [head] + kernel_rows(L, torch, args.quick) + fold_rows(L, torch, rounds=3 if args.quick else 8, steps=5)
    head2 = dict(kind="setup_end", **card())
    rows.append(head2)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
