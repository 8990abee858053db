"""The digit sort of a fixed-base commitment (csrc/msm_impl.cuh): per-CTA shared-memory histograms when one bucket set fits a CTA's
shared memory (window c <= 16), global atomics otherwise or when LURK_MSM_SORT=legacy forces them.  Either sort must give the
oracle's commitment, so the two also agree byte for byte.  The switch is read at every launch, so one process runs both."""
import os
import subprocess
import sys

import numpy as np
import pytest

from util import pack, random_elements

pytestmark = pytest.mark.gpu
SORTS = ["smem", "legacy"]


@pytest.fixture(params=SORTS)
def sort(request, monkeypatch):
    if request.param == "legacy":
        monkeypatch.setenv("LURK_MSM_SORT", "legacy")
    else:
        monkeypatch.delenv("LURK_MSM_SORT", raising=False)
    return request.param


def _key(L, oracle, curve, n, window):
    bases = oracle.gen_bases(curve, n)
    return bases, L.CommitmentKey(curve, bases).precompute(window)


def _launches(ck, sc):
    ck.commit(sc)
    return ck.last_profile()[1]


def test_sort_selection_and_launch_count(L, oracle, spec, monkeypatch):
    """c <= 16 takes the shared-memory sort (one more launch: histogram + columns instead of count); c = 17, a windowed commitment
    and LURK_MSM_SORT=legacy keep the global-atomics kernels"""
    curve, n = 0, 40_000                                     # long enough for the table to be used at c = 17
    bases = oracle.gen_bases(curve, n)
    sc = random_elements(spec.CURVES[curve]["scalar"], n, seed=1)
    monkeypatch.delenv("LURK_MSM_SORT", raising=False)
    plain = _launches(L.CommitmentKey(curve, bases), sc)
    k16, k17 = L.CommitmentKey(curve, bases).precompute(16), L.CommitmentKey(curve, bases).precompute(17)
    new16, old17 = _launches(k16, sc), _launches(k17, sc)
    monkeypatch.setenv("LURK_MSM_SORT", "legacy")
    assert _launches(k16, sc) == new16 - 1 and _launches(k17, sc) == old17
    assert _launches(L.CommitmentKey(curve, bases), sc) == plain
    with pytest.raises(L.LurkError):
        k16.precompute(15)                                    # one table per context


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_sort_all_curves(L, oracle, spec, sort, curve):
    n = 5000
    bases, ck = _key(L, oracle, curve, n, 13)
    for shape in ("uniform", "witness"):
        sc = random_elements(spec.CURVES[curve]["scalar"], n, seed=40 + curve, shape=shape)
        assert np.array_equal(ck.commit(sc), oracle.msm(curve, bases, sc, nthreads=8)), shape


@pytest.mark.parametrize("n,window", [(158, 10), (1025, 12), (132 * 1024 + 7, 16)])
def test_sort_ragged_cta_ranges(L, oracle, spec, sort, n, window):
    """fewer scalars than a CTA has threads (158 is the shortest vector a read-back commitment sends through a table, at the narrowest
    window a table takes; its third takes the windowed path); one scalar more than a CTA's threads; a few scalars more than 132 CTAs
    of 1024 at the fold tables' window, whose histogram is the largest the shared-memory sort takes (128 KB)"""
    curve = 0
    bases, ck = _key(L, oracle, curve, n, window)
    for shape in ("uniform", "witness"):
        sc = random_elements(spec.CURVES[curve]["scalar"], n, seed=n, shape=shape)
        assert np.array_equal(ck.commit(sc), oracle.msm(curve, bases, sc, nthreads=8, naive=(n < 200))), shape
    m = max(1, n // 3)                                        # a shorter vector under the same key: fewer CTAs
    assert np.array_equal(ck.commit(sc[:32 * m]), oracle.msm(curve, bases[:64 * m], sc[:32 * m], nthreads=8, naive=(m < 200)))


def test_sort_degenerate_scalars(L, oracle, spec, sort):
    """all scalars equal: every digit of a window lands in one bucket (a single hot shared-memory counter, and the long-bucket list
    of the merge); all zero; q - 1 and values whose signed digits carry through every window; an identity base"""
    curve, n, c = 0, 20_000, 12
    q = spec.FIELD_MODULUS[spec.CURVES[curve]["scalar"]]
    bases = oracle.gen_bases(curve, n)
    bases[64 * 7:64 * 8] = 0
    ck = L.CommitmentKey(curve, bases).precompute(c)
    half = sum(1 << (c * w + c - 1) for w in range(254 // c))          # every window holds 2^(c-1), the largest positive digit
    carry = sum(((1 << (c - 1)) + 1) << (c * w) for w in range(254 // c))   # every window goes negative and carries into the next
    for vals in ([0x1234567] * n, [0] * n, [q - 1] * n, [q - 1, 1, 0] * (n // 3), [half % q] * n, [carry % q] * n, [(1 << 253) + 12345] * 4097):
        sc = pack(vals)
        assert np.array_equal(ck.commit(sc), oracle.msm(curve, bases[:64 * len(vals)], sc, nthreads=8)), hex(vals[0])
    assert not ck.commit(pack([0] * n)).any()


def test_fold_steps_under_the_legacy_sort():
    """the fold context's commit(W2 - D) (constant part subtracted inside the sort) and commit(T): the fold pipeline's tests pass under
    the default sort in their own file; here they run again with the global-atomics sort, against the same oracle values"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if os.environ.get("LURK_MSM_SORT"):
        pytest.skip("the sort is already forced")
    env = dict(os.environ, LURK_MSM_SORT="legacy")
    out = subprocess.run([sys.executable, "-m", "pytest", os.path.join(root, "tests", "test_gpu_fold_pipeline.py"), "-m", "gpu", "-q", "-x"],
                         capture_output=True, text=True, timeout=1800, cwd=root, env=env)
    assert out.returncode == 0, out.stdout[-3000:]
