#!/usr/bin/env python3
"""Measurements of the individual BASELINE.json configurations and of the HBM-bound helper kernels (one JSON object per
line).  bench.py stays the contract for the headline metric; this produces the per-kernel evidence.
  single process:  python tools/config_benches.py
  N GPUs:          python -m torch.distributed.run --nproc-per-node N ... tools/config_benches.py --only msm24"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lurk_beta_b200 as L

lib = L._capi.lib()
chk = L._capi.check
PEAK = 6568.0
try:
    PEAK = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:
    pass


def rand_elements(rng, count, shape="uniform"):
    raw = rng.integers(0, 256, size=(count, 32), dtype=np.uint8)
    raw[:, 31] &= 0x1f
    if shape == "witness":
        u = rng.random(count)
        small = u < 0.4
        raw[small] = 0
        raw[small, 0] = rng.integers(0, 2, size=int(small.sum()), dtype=np.uint8)
        raw[(u >= 0.4) & (u < 0.5), 2:] = 0
    elif shape == "lem":
        even = np.arange(count) % 2 == 0
        raw[even, 2:] = 0
    return raw.reshape(-1)


def dev_time(fn, reps=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return min(ts), sorted(ts)[len(ts) // 2]


def emit(**kw):
    print(json.dumps(kw), flush=True)


def poseidon_config2():
    rng = np.random.default_rng(22)
    n = 1 << 22
    for field, fname in ((0, "bn254_fr"), (2, "pallas_fq")):
        for arity in (8, 4):
            host = rand_elements(rng, n * arity, "lem")
            pre = torch.from_numpy(host).cuda()
            out = torch.empty(n * 32, dtype=torch.uint8, device="cuda")
            best, med = dev_time(lambda: chk(lib.lurk_poseidon_hash_batch_dev(field, arity, pre.data_ptr(), n, out.data_ptr(), 0, None)))
            hout = np.zeros(n * 32, dtype=np.uint8)
            t0 = time.perf_counter()
            chk(lib.lurk_poseidon_hash_batch(field, arity, L._capi.np_ptr(host), n, L._capi.np_ptr(hout)))
            e2e = time.perf_counter() - t0
            alg = n * (arity + 1) * 32
            emit(config="2: Poseidon batch hash of 2^22 preimages", field=fname, arity=arity, n=n, ms=round(med, 3), ms_best=round(best, 3),
                 mhash_per_s=round(n / med / 1e3, 2), algorithmic_gb_s=round(alg / med / 1e6, 2), hbm_frac=round(alg / med / 1e6 / PEAK, 5),
                 e2e_host_buffers_ms=round(e2e * 1e3, 1), bound="FMA-heavy (IMAD.WIDE) pipe")
            del pre, out


def poseidon_witness(logn=22):
    """K3 at scale (BASELINE.md 3(ii)): the Poseidon *witness* expansion, 32 A in and 32 (A + 3 (8 t + R_P) + 1) out per slot"""
    rng = np.random.default_rng(23)
    n = 1 << logn
    field = 0
    for arity in (8, 4):
        blk = lib.lurk_poseidon_witness_block(field, arity)
        pre = torch.from_numpy(rand_elements(rng, n * arity, "lem")).cuda()
        out = torch.empty(n * blk * 32, dtype=torch.uint8, device="cuda")
        best, med = dev_time(lambda: chk(lib.lurk_poseidon_witness_batch_dev(field, arity, pre.data_ptr(), n, out.data_ptr(), 1, None)), reps=3, warm=1)
        alg = n * (arity * 32 + blk * 32)
        emit(config=f"2/K3: Poseidon slot witnesses of 2^{logn} preimages", field="bn254_fr", arity=arity, n=n, block_elems=int(blk), ms=round(med, 3),
             mwitness_per_s=round(n / med / 1e3, 2), algorithmic_gb_s=round(alg / med / 1e6, 2), hbm_frac=round(alg / med / 1e6 / PEAK, 5),
             output_gb=round(n * blk * 32 / 1e9, 2), bound="FMA-heavy (IMAD.WIDE) pipe; stores 12.9 KB / 9.5 KB per sponge")
        del pre, out
        torch.cuda.empty_cache()


def msm_config3(logn=24, curve=2):
    import torch.distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if world > 1:
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        if not dist.is_initialized():
            dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    n = 1 << logn
    lo, hi = L.shard_bounds(n, world, rank)
    t0 = time.perf_counter()
    bases = L.synthetic_bases(curve, hi - lo, start=lo, fmt=L.FMT_MONTGOMERY)
    ck = L.CommitmentKey(curve, bases, fmt=L.FMT_MONTGOMERY)
    del bases
    setup = time.perf_counter() - t0
    rng = np.random.default_rng(24)
    for fixed in (False, True):
        if fixed:
            t0 = time.perf_counter()
            ck.precompute()
            torch.cuda.synchronize()
            pre_s = time.perf_counter() - t0
        for shape in ("uniform", "witness"):
            sc_all = rand_elements(rng, n, shape)
            d_sc = torch.from_numpy(sc_all[32 * lo:32 * hi]).cuda()
            res = {}

            def run():
                part = ck.commit_device(d_sc.data_ptr(), hi - lo, fmt=L.FMT_MONTGOMERY)
                if world > 1:
                    mine = torch.from_numpy(part).cuda()
                    allp = torch.empty(96 * world, dtype=torch.uint8, device="cuda")
                    dist.all_gather_into_tensor(allp, mine)
                    part = L.point_sum(curve, allp.cpu().numpy(), fmt=L.FMT_MONTGOMERY)
                res["pt"] = part
            if world > 1:
                dist.barrier()
            best, med = dev_time(run, reps=5, warm=2)
            t = torch.tensor([med], device="cuda")
            if world > 1:
                dist.all_reduce(t, op=dist.ReduceOp.MAX)
            med = float(t.item())
            host_ms = None
            if world == 1:
                hs = sc_all
                ck.commit(hs, fmt=L.FMT_MONTGOMERY)
                t1 = time.perf_counter()
                ck.commit(hs, fmt=L.FMT_MONTGOMERY)
                host_ms = round((time.perf_counter() - t1) * 1e3, 2)
            if rank == 0:
                emit(e2e_host_scalars_ms=host_ms, config=f"3: Pedersen MSM 2^{logn} bases", curve=["bn254_g1", "grumpkin", "pallas", "vesta"][curve], n=n, n_gpus=world,
                     scalars=shape, fixed_base_table=fixed, ms=round(med, 3), mterms_per_s=round(n / med / 1e3, 2),
                     algorithmic_gb_s=round(n * 96 / med / 1e6, 2), hbm_frac=round(n * 96 / med / 1e6 / PEAK, 5), key_setup_s=round(setup, 1),
                     table_build_s=round(pre_s, 2) if fixed else None, result_x_prefix=bytes(res["pt"][:8]).hex(),
                     exchange="all_gather of 96-byte partial points + local adds" if world > 1 else None)
            del d_sc


def hbm_kernels():
    rng = np.random.default_rng(5)
    field = 0
    n = 1 << 24
    a = torch.from_numpy(rand_elements(rng, n)).cuda()
    b = torch.from_numpy(rand_elements(rng, n)).cuda()
    out = torch.empty_like(a)
    r = rand_elements(rng, 1)
    best, med = dev_time(lambda: chk(lib.lurk_axpy_dev(field, a.data_ptr(), b.data_ptr(), L._capi.np_ptr(r), n, out.data_ptr(), None)))
    emit(kernel="axpy_kernel", n=n, ms=round(med, 4), gb_s=round(n * 96 / med / 1e6, 1), hbm_frac=round(n * 96 / med / 1e6 / PEAK, 3), bound="hbm")
    u = rand_elements(rng, 1)
    vs = [a, b, out, a, b, out]
    t = torch.empty_like(a)
    best, med = dev_time(lambda: chk(lib.lurk_cross_term_dev(field, *[x.data_ptr() for x in vs], L._capi.np_ptr(u), L._capi.np_ptr(u), n, t.data_ptr(), None)))
    emit(kernel="cross_term_kernel", n=n, ms=round(med, 4), gb_s=round(n * 224 / med / 1e6, 1), hbm_frac=round(n * 224 / med / 1e6 / PEAK, 3),
         bound="hbm (3 distinct input arrays aliased twice here: L2 helps)")
    for logn in (20, 24):
        m = 1 << logn
        d = a[:m * 32].clone()
        best, med = dev_time(lambda: chk(lib.lurk_ntt_dev(field, d.data_ptr(), logn, 0, None)))
        passes = 1 + (max(0, logn - 10) + 1) // 2 + 1      # tile pass, radix-4 passes, copy back
        emit(kernel="ntt", field="bn254_fr", log_n=logn, ms=round(med, 4), algorithmic_gb_s=round(m * 64 / med / 1e6, 1),
             hbm_frac=round(m * 64 / med / 1e6 / PEAK, 4), global_passes=passes, moved_gb_s=round(m * 64 * passes / med / 1e6, 1))
    rows, cols = 1_114_100, 911_903
    nnz_per = rng.integers(1, 4, size=rows)
    rp = np.concatenate([[0], np.cumsum(nnz_per)]).astype(np.uint64)
    col = rng.integers(0, cols, size=int(rp[-1])).astype(np.uint32)
    val = torch.from_numpy(rand_elements(rng, int(rp[-1]))).cuda()
    d_rp, d_col = torch.from_numpy(rp).cuda(), torch.from_numpy(col).cuda()
    y = torch.empty(rows * 32, dtype=torch.uint8, device="cuda")
    best, med = dev_time(lambda: chk(lib.lurk_spmv_csr_dev(field, d_rp.data_ptr(), d_col.data_ptr(), val.data_ptr(), rows, a.data_ptr(), y.data_ptr(), None)))
    bytes_moved = int(rp[-1]) * (32 + 4 + 32) + rows * (8 + 32)
    emit(kernel="spmv_kernel", rows=rows, nnz=int(rp[-1]), ms=round(med, 4), gb_s=round(bytes_moved / med / 1e6, 1),
         hbm_frac=round(bytes_moved / med / 1e6 / PEAK, 3), bound="hbm / gather")


def dag():
    rng = np.random.default_rng(9)
    node_t = np.dtype([("kind", "u1"), ("reserved", "u1"), ("tag", "<u2", (4,)), ("child", "<u4", (4,))], align=True)
    field = 0
    for label, n, n_atoms, back in (("wide random DAG", 1 << 20, 1 << 12, 1 << 18), ("single chain (depth = n)", 2000, 16, 1)):
        atoms = rand_elements(rng, n_atoms)
        nodes = np.zeros(n, dtype=node_t)
        nodes["kind"] = 2
        nodes["tag"][:, :2] = rng.integers(0, 16, size=(n, 2))
        hi = n_atoms + np.arange(n, dtype=np.int64)
        ch = np.maximum(hi[:, None] - rng.integers(1, back + 1, size=(n, 2)), 0)
        if back == 1:
            ch[:, 1] = rng.integers(0, n_atoms, size=n)
        nodes["child"][:, :2] = ch
        out = np.zeros(n * 32, dtype=np.uint8)
        chk(lib.lurk_dag_hash(field, L._capi.np_ptr(nodes), n, L._capi.np_ptr(atoms), n_atoms, L._capi.np_ptr(out)))
        t0 = time.perf_counter()
        chk(lib.lurk_dag_hash(field, L._capi.np_ptr(nodes), n, L._capi.np_ptr(atoms), n_atoms, L._capi.np_ptr(out)))
        dt = time.perf_counter() - t0
        emit(kernel="lurk_dag_hash (host buffers, end to end)", shape=label, nodes=n, ms=round(dt * 1e3, 2), knodes_per_s=round(n / dt / 1e3, 1))


def ck_generate(logn=21):
    """N3: commitment-key generation (DlogGroup::from_label): the map kernel alone on resident uniform bytes, the whole call
    (SHAKE256 on one host thread pipelined against the kernel), and the CPU oracle (pure Python, one core) on a small sample."""
    import ctypes as C
    import hashlib
    n = 1 << logn
    stream = np.frombuffer(hashlib.shake_256(b"ck").digest(32 * n), dtype=np.uint8)
    d_msgs = torch.from_numpy(stream.copy()).cuda()
    out = torch.empty(n * 64, dtype=torch.uint8, device="cuda")
    for curve, cname, exps in ((0, "bn254_g1", "1 batched inversion + 6 square-root passes (s = 1) + 1 inversion"),
                               (1, "grumpkin", "same with s = 28 Tonelli-Shanks"), (2, "pallas", "1 + 4 square-root passes (s = 32) + isogeny + 1"),
                               (3, "vesta", "as pallas")):
        best, med = dev_time(lambda: chk(lib.lurk_hash_to_curve_batch_dev(curve, b"from_uniform_bytes", d_msgs.data_ptr(), 32, n, out.data_ptr(), 1, None)),
                             reps=3, warm=1)
        t0 = time.perf_counter()
        chk(lib.lurk_ck_generate_dev(curve, b"ck", 2, n, C.c_void_p(out.data_ptr()), None))
        torch.cuda.synchronize()
        whole = time.perf_counter() - t0
        t0 = time.perf_counter()
        hashlib.shake_256(b"ck").digest(32 * n)
        xof = time.perf_counter() - t0
        from oracle import h2c, capi as ocapi   # checker / CPU baseline only
        t0 = time.perf_counter()
        h2c.from_label(curve, b"ck", 256)
        orc = (time.perf_counter() - t0) / 256
        th = os.cpu_count() or 1
        nc = 64 * th
        t0 = time.perf_counter()
        ocapi.from_label(curve, b"ck", nc, nthreads=th)
        orc_c = (time.perf_counter() - t0) / nc
        emit(config=f"N3: from_label, 2^{logn} points", curve=cname, n=n, kernel_ms=round(med, 2), mpoints_per_s=round(n / med / 1e3, 2),
             whole_call_ms=round(whole * 1e3, 1), hashlib_xof_ms=round(xof * 1e3, 1), work=exps,
             algorithmic_gb_s=round(n * 96 / med / 1e6, 2), hbm_frac=round(n * 96 / med / 1e6 / PEAK, 5),
             cpu_oracle_python_us_per_point=round(orc * 1e6, 1), cpu_port_c_us_per_point_all_threads=round(orc_c * 1e6, 2), cpu_threads=th,
             cpu_port_c_seconds_for_this_key=round(orc_c * n, 1), bound="FMA-heavy (IMAD.WIDE) pipe: fixed-exponent exponentiations")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="all")
    ap.add_argument("--logn", type=int, default=24)
    a = ap.parse_args()
    if a.only in ("all", "poseidon"):
        poseidon_config2()
    if a.only in ("all", "witness"):
        poseidon_witness(min(a.logn, 22))
    if a.only in ("all", "msm24"):
        msm_config3(a.logn)
    if a.only in ("all", "hbm"):
        hbm_kernels()
    if a.only in ("all", "dag"):
        dag()
    if a.only in ("all", "ckgen"):
        ck_generate(min(a.logn, 21))
