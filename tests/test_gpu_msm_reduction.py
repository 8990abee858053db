"""The MSM's bucket reduction after the accumulation (csrc/msm_impl.cuh: msm_merge_kernel, msm_merge_long_kernel,
msm_chunk_kernel, msm_bitsum_kernel, msm_slice_sum_kernel, msm_horner_kernel) against the oracle, for bucket distributions
that stress it: dense and sparse vectors, 0/1-heavy witnesses and equal scalars (a few buckets hold every entry, so
thousands of partials go to one bucket and take the long-bucket path), bucket sizes that are exact multiples of the segment length (every
bucket starts at a segment start), single-entry buckets, and sizes around the plan's boundaries.  Each runs in windowed mode
(one bucket set per window, host Horner) and in fixed-base mode (one shared bucket set, device Horner), on BN254 G1 and
Pallas."""
import numpy as np
import pytest

from util import pack, random_elements

pytestmark = pytest.mark.gpu
CURVES = [0, 2]                     # BN254 G1, Pallas
SEG_MULTIPLE = 32                   # every segment length the plan picks (8 .. 32) divides it


def scalars(spec, curve, n, kind, rng):
    field = spec.CURVES[curve]["scalar"]
    p = spec.FIELD_MODULUS[field]
    seed = int(rng.integers(1 << 30))
    if kind == "uniform":
        return random_elements(field, n, seed=seed, shape="uniform")
    if kind == "nonzero34":
        sc = random_elements(field, n, seed=seed, shape="uniform").reshape(n, 32)
        sc[rng.random(n) >= 0.34] = 0
        return sc.reshape(-1)
    if kind == "witness":
        return random_elements(field, n, seed=seed, shape="witness")
    if kind == "bits":              # bit-decomposition slots: almost every entry 0 or 1, a few p - 1
        pick = rng.choice(3, size=n, p=[0.3, 0.68, 0.02])
        return pack([(0, 1, p - 1)[int(k)] for k in pick])
    if kind == "equal":
        v = int.from_bytes(random_elements(field, 1, seed=seed, shape="uniform").tobytes(), "little")
        return pack([v] * n)
    if kind == "seg_multiples":     # window-0 digits only, each bucket's size a multiple of every segment length
        vals, d = [], 1
        sizes = [SEG_MULTIPLE * k for k in (1, 2, 3, 8, 1, 5)]
        while len(vals) < n:
            vals += [d] * min(sizes[d % len(sizes)], n - len(vals))
            d = d % 200 + 1         # digits < 2^8 stay in window 0 for every window width >= 9
        return pack([vals[i] for i in rng.permutation(n)])
    if kind == "single":            # a few dozen terms in a long vector: nearly every bucket holds one entry
        vals = [0] * n
        full = random_elements(field, 60, seed=seed, shape="edge").reshape(60, 32)
        for i, v in zip(rng.choice(n, size=60, replace=False), full):
            vals[int(i)] = int.from_bytes(v.tobytes(), "little")
        return pack(vals)
    raise ValueError(kind)


KINDS = ["uniform", "nonzero34", "witness", "bits", "equal", "seg_multiples", "single"]


@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("fixed", [False, True], ids=["windowed", "fixed"])
def test_reduction_bucket_distributions(L, oracle, spec, curve, fixed):
    n = 1 << 14
    rng = np.random.default_rng(100 + curve + 2 * fixed)
    bases = oracle.gen_bases(curve, n)
    ck = L.CommitmentKey(curve, bases)
    if fixed:
        ck.precompute()
    for kind in KINDS:
        sc = scalars(spec, curve, n, kind, rng)
        assert np.array_equal(ck.commit(sc), oracle.msm(curve, bases, sc, nthreads=8)), kind


def plan_boundary_sizes(L):
    """n around the window-width steps (powers of two) and around the step of the segment length (n * windows = 8 entries
    per thread of the level-1 grid, 1024 threads per SM)"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    nwin = 254 // 10 + 1                     # windowed mode for 2^15 <= n < 2^16: c = 10
    k = 8 * sms * 1024 // nwin
    return [4095, 4096, 4097, 32767, 32769, k - 1, k + 1, 65535, 65537]


@pytest.mark.parametrize("curve", CURVES)
def test_reduction_plan_boundaries(L, oracle, spec, curve):
    rng = np.random.default_rng(7 + curve)
    for n in plan_boundary_sizes(L):
        bases = oracle.gen_bases(curve, n)
        sc = scalars(spec, curve, n, ["uniform", "witness", "equal"][n % 3], rng)
        want = oracle.msm(curve, bases, sc, nthreads=8)
        ck = L.CommitmentKey(curve, bases)
        assert np.array_equal(ck.commit(sc), want), ("windowed", n)
        ck.precompute()
        assert np.array_equal(ck.commit(sc), want), ("fixed", n)


def test_reduction_long_buckets_everywhere(L, oracle, spec):
    """many long buckets: 300 distinct scalars repeated over 2^17 terms put ~440 entries (~20 segment starts) into each of
    thousands of buckets, more than msm_merge_long_kernel launches CTAs for, so they walk the long-bucket list several times"""
    curve, n = 0, 1 << 17
    rng = np.random.default_rng(3)
    bases = oracle.gen_bases(curve, n)
    vals = random_elements(spec.CURVES[curve]["scalar"], 300, seed=4, shape="uniform").reshape(300, 32)
    sc = vals[rng.integers(0, 300, size=n)].reshape(-1)
    want = oracle.msm(curve, bases, sc, nthreads=8)
    ck = L.CommitmentKey(curve, bases)
    assert np.array_equal(ck.commit(sc), want)
    ck.precompute()
    assert np.array_equal(ck.commit(sc), want)
