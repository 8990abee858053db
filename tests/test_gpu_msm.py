"""GPU parity for S4: Pippenger MSM through the C ABI against the oracle (plain-C Jacobian Pippenger and naive
double-and-add), compared as canonical affine points -- the group law is canonical, so any correct MSM is bit-exact
after normalisation (SURVEY.md 8(c))."""
import numpy as np
import pytest

from util import ints, pack, random_elements

pytestmark = pytest.mark.gpu
CURVES = [0, 1, 2, 3]


def scalars_for(spec, curve, n, seed, shape):
    return random_elements(spec.CURVES[curve]["scalar"], n, seed=seed, shape=shape)


@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("n", [1, 2, 33, 1000])
def test_msm_parity_small(L, oracle, spec, curve, n):
    bases = oracle.gen_bases(curve, n)
    sc = scalars_for(spec, curve, n, seed=n + curve, shape="uniform")
    got = L.CommitmentKey(curve, bases).commit(sc)
    want = oracle.msm(curve, bases, sc, nthreads=4, naive=(n <= 33))
    assert np.array_equal(got, want)


@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("shape", ["uniform", "witness"])
def test_msm_parity_2_16(L, oracle, spec, curve, shape):
    n = 1 << 16
    bases = oracle.gen_bases(curve, n)
    sc = scalars_for(spec, curve, n, seed=11 + curve, shape=shape)
    got = L.CommitmentKey(curve, bases).commit(sc)
    want = oracle.msm(curve, bases, sc, nthreads=8)
    assert np.array_equal(got, want)


def test_msm_edge_scalars_and_identity_bases(L, oracle, spec):
    curve, n = 2, 600
    q = spec.FIELD_MODULUS[spec.CURVES[curve]["scalar"]]
    bases = oracle.gen_bases(curve, n)
    bases[64 * 5:64 * 6] = 0                      # identity base (0, 0) is skipped
    bases[64 * 9:64 * 10] = bases[64 * 8:64 * 9]  # duplicate point: exercises the doubling branch
    ck = L.CommitmentKey(curve, bases)
    for vals in ([0] * n, [1] * n, [q - 1] * n, [2] * n, [q - 1, 1] * (n // 2), [(1 << 254) - 3] * n):
        sc = pack(vals)
        assert np.array_equal(ck.commit(sc), oracle.msm(curve, bases, sc, nthreads=4)), vals[:2]
    # prefix of the key (|W| < |ck|) and empty input
    sc = scalars_for(spec, curve, 100, seed=5, shape="witness")
    assert np.array_equal(ck.commit(sc), oracle.msm(curve, bases[:6400], sc))
    assert not ck.commit(np.zeros(0, dtype=np.uint8)).any()
    # P + (-P) = identity
    two = pack([5, q - 5])
    same = np.concatenate([bases[:64], bases[:64]])
    assert not L.CommitmentKey(curve, same).commit(two).any()


def test_msm_errors(L, oracle, spec):
    curve = 0
    bases = oracle.gen_bases(curve, 4)
    ck = L.CommitmentKey(curve, bases)
    with pytest.raises(L.LurkError):
        ck.commit(pack([1] * 5))                  # more scalars than bases
    with pytest.raises(L.LurkError) as e:
        ck.commit(pack([spec.FIELD_MODULUS[spec.CURVES[curve]["scalar"]]] * 2))
    assert e.value.code == L._capi.ERR_RANGE


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_off_curve_and_unreduced_bases_rejected(L, oracle, spec, curve):
    """a commitment key is validated at upload: coordinates < p and y^2 = x^3 + b ((0, 0) = identity is allowed)"""
    good = oracle.gen_bases(curve, 64)
    good[64 * 7:64 * 8] = 0
    L.CommitmentKey(curve, good)                              # accepted
    bad = good.copy()
    bad[64 * 33 + 32] ^= 1                                    # y of base 33 off by one bit: not on the curve
    with pytest.raises(L.LurkError, match="not on the curve") as e:
        L.CommitmentKey(curve, bad)
    assert e.value.code == L._capi.ERR_RANGE
    bad = good.copy()
    bad[64 * 5:64 * 5 + 32] = pack([spec.FIELD_MODULUS[spec.CURVES[curve]["base"]]])   # x = p
    with pytest.raises(L.LurkError) as e:
        L.CommitmentKey(curve, bad)
    assert e.value.code == L._capi.ERR_RANGE
    # Montgomery-format keys go through the same check
    pb = spec.FIELD_MODULUS[spec.CURVES[curve]["base"]]
    R = (1 << 256) % pb
    gm = pack([x * R % pb for x in ints(good)])
    L.CommitmentKey(curve, gm, fmt=L.FMT_MONTGOMERY)
    gm[64 * 2] ^= 1
    with pytest.raises(L.LurkError, match="not on the curve"):
        L.CommitmentKey(curve, gm, fmt=L.FMT_MONTGOMERY)


def test_msm_montgomery_format(L, oracle, spec):
    curve, n = 0, 500
    C = spec.CURVES[curve]
    pb, q = spec.FIELD_MODULUS[C["base"]], spec.FIELD_MODULUS[C["scalar"]]
    bases = oracle.gen_bases(curve, n)
    sc = scalars_for(spec, curve, n, seed=2, shape="uniform")
    R = 1 << 256
    bm = pack([x * R % pb for x in ints(bases)])
    sm = pack([x * R % q for x in ints(sc)])
    got = L.CommitmentKey(curve, bm, fmt=L.FMT_MONTGOMERY).commit(sm, fmt=L.FMT_MONTGOMERY)
    want = oracle.msm(curve, bases, sc, nthreads=4)
    rinv = pow(R, -1, pb)
    assert [v * rinv % pb for v in ints(got)] == ints(want)


def test_msm_linearity_2_20(L, oracle, spec):
    """size-independent property at a size the oracle cannot check directly quickly: commit is linear,
    commit(a) + commit(b) == commit(a + b), and agrees with the oracle on a 2^14 prefix."""
    curve, n = 0, 1 << 20
    q = spec.FIELD_MODULUS[spec.CURVES[curve]["scalar"]]
    bases = oracle.gen_bases(curve, n)
    ck = L.CommitmentKey(curve, bases)
    a = scalars_for(spec, curve, n, seed=21, shape="witness")
    b = scalars_for(spec, curve, n, seed=22, shape="uniform")
    a64 = a.reshape(-1, 32).view("<u8").astype(object)
    # a + b mod q with python ints on a strided subset would be slow for 2^20; use the oracle's axpy (r = 1)
    ab = oracle.axpy(spec.CURVES[curve]["scalar"], a, b, pack([1]), nthreads=8)
    ca, cb, cab = ck.commit(a), ck.commit(b), ck.commit(ab)
    assert np.array_equal(L.point_sum(curve, np.concatenate([ca, cb])), cab)
    m = 1 << 14
    assert np.array_equal(ck.commit(a[:32 * m]), oracle.msm(curve, bases[:64 * m], a[:32 * m], nthreads=8))


def test_msm_async_launch_finish_and_clone(L, oracle, spec):
    """launch/finish split: two commitments on the same resident key in flight at once (commit(W) and commit(T) of a fold)"""
    import torch
    curve, n = 0, 50_000
    bases = oracle.gen_bases(curve, n)
    a = scalars_for(spec, curve, n, seed=71, shape="witness")
    b = scalars_for(spec, curve, n - 1234, seed=72, shape="uniform")
    ck = L.CommitmentKey(curve, bases)
    ck2 = ck.clone()
    da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    ck.launch_device(da.data_ptr(), n, fmt=L.FMT_CANONICAL, stream=s1.cuda_stream)
    ck2.launch_device(db.data_ptr(), n - 1234, fmt=L.FMT_CANONICAL, stream=s2.cuda_stream)
    with pytest.raises(L.LurkError):
        ck.launch_device(da.data_ptr(), n, fmt=L.FMT_CANONICAL, stream=s1.cuda_stream)     # one launch pending per context
    rb, ra = ck2.finish(), ck.finish()
    assert np.array_equal(ra, oracle.msm(curve, bases, a, nthreads=8))
    assert np.array_equal(rb, oracle.msm(curve, bases[:64 * (n - 1234)], b, nthreads=8))
    with pytest.raises(L.LurkError):
        ck.finish()                                                                         # nothing pending
    ms, launches = ck.last_profile()
    assert launches >= 10


@pytest.mark.parametrize("curve", CURVES)
def test_msm_fixed_base_table_same_results(L, oracle, spec, curve):
    """fixed-base mode (window multiples precomputed, shared bucket set) must not change any result"""
    n = 40_000
    bases = oracle.gen_bases(curve, n)
    bases[64 * 3:64 * 4] = 0                                   # identity base survives the table build
    q = spec.FIELD_MODULUS[spec.CURVES[curve]["scalar"]]
    ck = L.CommitmentKey(curve, bases).precompute()
    for seed, shape in ((1, "uniform"), (2, "witness")):
        sc = scalars_for(spec, curve, n, seed=seed, shape=shape)
        assert np.array_equal(ck.commit(sc), oracle.msm(curve, bases, sc, nthreads=8))
    for vals in ([q - 1] * 257, [1] * 100, [0] * 10, [(1 << 253) + 12345] * 33):
        sc = pack(vals)
        assert np.array_equal(ck.commit(sc), oracle.msm(curve, bases[:64 * len(vals)], sc))
    clone = ck.clone()
    sc = scalars_for(spec, curve, 1000, seed=9, shape="uniform")
    assert np.array_equal(clone.commit(sc), oracle.msm(curve, bases[:64000], sc))


@pytest.mark.parametrize("n", [3, 31, 32, 33, 63, 65, 127, 1023, 1025, 4097, 20011, 65537])
def test_msm_sizes_around_plan_boundaries(L, oracle, spec, n):
    """window width, segment length and the number of partial passes all change with n: sweep sizes around the
    boundaries, plain and fixed-base, scalars with long zero runs in the high windows"""
    curve = [0, 2, 1, 3][n % 4]
    bases = oracle.gen_bases(curve, n)
    sf = spec.CURVES[curve]["scalar"]
    sc = scalars_for(spec, curve, n, seed=n, shape="witness" if n % 2 else "uniform")
    want = oracle.msm(curve, bases, sc, nthreads=8, naive=(n < 40))
    ck = L.CommitmentKey(curve, bases)
    assert np.array_equal(ck.commit(sc), want)
    ck.precompute()
    assert np.array_equal(ck.commit(sc), want)
    m = max(1, n // 3)                                   # a shorter scalar vector on the same (fixed-base) key
    assert np.array_equal(ck.commit(sc[:32 * m]), oracle.msm(curve, bases[:64 * m], sc[:32 * m], nthreads=8, naive=(m < 40)))
