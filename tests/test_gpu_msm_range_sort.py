"""The two-level digit sort of a fixed-base commitment at c <= 16 (csrc/msm_impl.cuh): digits are first partitioned by bucket range
(MSM_RANGE_BUCKETS consecutive buckets), then every range is counting-sorted by bucket in slices of MSM_RSORT_SLICE entries.  Each
case below is committed under the default sort and under the global-atomics one (LURK_MSM_SORT=legacy) in the same process; the two
must agree byte for byte and match the oracle.  The shapes sit on the sort's own boundaries: a range exactly at, one under and one
over a slice, every digit in one range, one hot bucket, a 0/1-heavy witness, CTA and partition-tile edges, and the fold's two
commitment lengths in Montgomery form."""
import ctypes as C

import numpy as np
import pytest

from util import pack, random_elements

pytestmark = pytest.mark.gpu

# csrc/msm_impl.cuh
MSM_RANGE_BUCKETS, MSM_RSORT_SLICE, MSM_PART_SCALARS, MSM_SORT_THREADS = 128, 8192, 2048, 1024
CURVE, WINDOW = 0, 16
N_KEY = 3 * MSM_RSORT_SLICE + 4096          # a read-back commitment takes the c = 16 table from 16 384 scalars on


@pytest.fixture(scope="module")
def key(L, oracle):
    bases = oracle.gen_bases(CURVE, N_KEY)
    ck = L.CommitmentKey(CURVE, bases).precompute(WINDOW)
    yield bases, ck
    ck.close()


def both_sorts(ck, monkeypatch, commit):
    monkeypatch.delenv("LURK_MSM_SORT", raising=False)
    new = commit(ck)
    monkeypatch.setenv("LURK_MSM_SORT", "legacy")
    old = commit(ck)
    monkeypatch.delenv("LURK_MSM_SORT", raising=False)
    assert new.tobytes() == old.tobytes(), "the two sorts disagree"
    return new


def check(key, oracle, monkeypatch, vals):
    bases, ck = key
    sc = pack(vals)
    got = both_sorts(ck, monkeypatch, lambda k: k.commit(sc))
    assert np.array_equal(got, oracle.msm(CURVE, bases[:64 * len(vals)], sc, nthreads=8))


@pytest.mark.parametrize("live", [MSM_RSORT_SLICE - 1, MSM_RSORT_SLICE, MSM_RSORT_SLICE + 1, 3 * MSM_RSORT_SLICE + 1])
@pytest.mark.parametrize("rng_index", [0, (1 << (WINDOW - 1)) // MSM_RANGE_BUCKETS - 1])
def test_one_range_at_the_slice_edges(L, oracle, key, monkeypatch, live, rng_index):
    """`live` scalars with one digit each, all in range `rng_index` (the first or the last), spread over its 128 buckets; the rest of the
    vector is zero.  One slice under, at and over the range sort's slice, and several slices of one range"""
    rng = np.random.default_rng(live + rng_index)
    lo = rng_index * MSM_RANGE_BUCKETS + 1                    # digit magnitude = bucket + 1, positive (<= 2^(c-1)), window 0 only
    vals = [int(v) for v in rng.integers(lo, lo + MSM_RANGE_BUCKETS, size=live)] + [0] * (N_KEY - live)
    check(key, oracle, monkeypatch, [vals[i] for i in rng.permutation(N_KEY)])


@pytest.mark.parametrize("value", [1, 1 << (WINDOW - 1), 0x1234567])
def test_one_hot_bucket(L, oracle, key, monkeypatch, value):
    """every scalar equal: one bucket per window holds all n entries (1: one bucket in all, over four slices of one range)"""
    check(key, oracle, monkeypatch, [value] * N_KEY)


def test_zero_one_heavy_witness(L, oracle, spec, key, monkeypatch):
    bases, ck = key
    for seed in range(2):
        sc = random_elements(spec.CURVES[CURVE]["scalar"], N_KEY, seed=300 + seed, shape="witness")
        got = both_sorts(ck, monkeypatch, lambda k: k.commit(sc))
        assert np.array_equal(got, oracle.msm(CURVE, bases, sc, nthreads=8))
    vals = [1] * (N_KEY // 2) + [0] * (N_KEY // 4) + [2] * (N_KEY - N_KEY // 2 - N_KEY // 4)
    check(key, oracle, monkeypatch, vals)


@pytest.mark.parametrize("n", [16 * MSM_SORT_THREADS + 1, 132 * (MSM_PART_SCALARS + 1)])
def test_cta_and_tile_edges(L, oracle, spec, monkeypatch, n):
    """n one past a multiple of a CTA's threads (one CTA more than 16), and on a 132-SM part CTA ranges of one partition tile and one
    scalar"""
    bases = oracle.gen_bases(CURVE, n)
    ck = L.CommitmentKey(CURVE, bases).precompute(WINDOW)
    try:
        for shape in ("uniform", "witness"):
            sc = random_elements(spec.CURVES[CURVE]["scalar"], n, seed=n, shape=shape)
            got = both_sorts(ck, monkeypatch, lambda k: k.commit(sc))
            assert np.array_equal(got, oracle.msm(CURVE, bases, sc, nthreads=8)), shape
    finally:
        ck.close()


@pytest.mark.parametrize("n,nonzero", [(1_114_100, 0.34), (911_900, 0.36)])
def test_fold_lengths_montgomery(L, monkeypatch, n, nonzero):
    """commit(T) and commit(W2 - D) of the fold step at fib rc = 100: device-resident Montgomery scalars with the fold's share of
    non-zero entries; 2^(c-1) buckets of ~185 entries each.  The two sorts agree, on a second call of the same context too (scratch
    reused).  The fold context's own subtraction of D runs inside the same kernels (test_gpu_fold_shapes covers it)."""
    import torch
    ck = L.CommitmentKey.setup(CURVE, b"range-sort", n).precompute(WINDOW)
    try:
        rng = np.random.default_rng(n)
        raw = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
        raw[:, 31] &= 0x0f
        raw[rng.random(n) >= nonzero] = 0
        d = torch.from_numpy(raw.reshape(-1)).cuda()
        L._capi.check(L._capi.lib().lurk_convert_dev(L.FIELD_BN254_FR, C.c_void_p(d.data_ptr()), n, L.FMT_MONTGOMERY, C.c_void_p(d.data_ptr()), None))
        first = both_sorts(ck, monkeypatch, lambda k: k.commit_device(d.data_ptr(), n))
        assert first.any()
        assert both_sorts(ck, monkeypatch, lambda k: k.commit_device(d.data_ptr(), n)).tobytes() == first.tobytes()
    finally:
        ck.close()
