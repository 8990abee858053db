"""lurk_point_combination_batch (csrc/pointcomb.cu): sum_j s_j P_j for independent groups, one CTA per group, checked byte for byte
against the host's lurk_point_combination and, after normalising, against the oracle.

Every point is P_j = [k_j]G with k_j known, so [sum_j k_j s_j mod r]G is an exact oracle at any size (one Python scalar multiplication);
spec.msm_naive checks the smaller groups a second way.  The kernel's shapes: 4 threads share a window's terms (1 .. 5 terms straddle that),
256 threads build the tables (255 .. 257 wrap the table loop), 64 windows of 4 bits; the group-law branches of XYZZ::add -- an identity
operand, P + P doubling, P + (-P) cancelling -- are reached by the degenerate groups below."""
import ctypes as C
import random
import threading

import numpy as np
import pytest

from oracle import spec

pytestmark = pytest.mark.gpu
CURVES = [0, 1, 2, 3]
FMTS = [0, 1]
LIMIT = 4096                        # LURK_POINT_COMBINATION_MAX_TERMS
CHUNKS, THREADS = 4, 256            # csrc/pointcomb.cu: PC_CHUNKS, PC_THREADS
SIZES = {"1": 1, "2": 2, "3-under-chunks": CHUNKS - 1, "4-chunks": CHUNKS, "5-over-chunks": CHUNKS + 1, "31": 31, "32": 32, "33": 33,
         "48": 48, "130": 130, "255-under-threads": THREADS - 1, "256-threads": THREADS, "257-over-threads": THREADS + 1, "limit": LIMIT}
NAIVE_MAX = 130                     # spec.msm_naive up to this many terms; the discrete-log oracle at every size
POOL = 160                          # distinct points per curve; larger groups reuse them


def moduli(curve):
    c = spec.CURVES[curve]
    return spec.FIELD_MODULUS[c["base"]], spec.FIELD_MODULUS[c["scalar"]]


_pools = {}


def pool(curve):
    """[(k, [k]G)] for POOL random k of `curve`"""
    if curve not in _pools:
        p, r = moduli(curve)
        rng = random.Random(1000 + curve)
        ks = [rng.randrange(1, r) for _ in range(POOL)]
        _pools[curve] = [(k, spec.ec_mul(k, spec.CURVES[curve]["gen"], p)) for k in ks]
    return _pools[curve]


def enc_points(curve, pts, fmt):
    """(x, y) / None -> k x 96 bytes of the header's form in fmt"""
    p, _ = moduli(curve)
    R = (1 << 256) % p if fmt else 1
    vals = []
    for P in pts:
        vals += [0, 0, 0] if P is None else [P[0] * R % p, P[1] * R % p, R % p]
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint8).copy()


def enc_scalars(curve, sc, fmt):
    _, r = moduli(curve)
    R = (1 << 256) % r if fmt else 1
    return np.frombuffer(b"".join(int(s * R % r).to_bytes(32, "little") for s in sc), dtype=np.uint8).copy()


def dec_point(curve, b, fmt):
    p, _ = moduli(curve)
    v = [int.from_bytes(bytes(b[32 * i:32 * i + 32]), "little") for i in range(3)]
    if v == [0, 0, 0]:
        return None
    Ri = pow(1 << 256, -1, p) if fmt else 1
    assert v[2] * Ri % p == 1
    return v[0] * Ri % p, v[1] * Ri % p


def host(L, curve, pb, sb, fmt):
    out = np.zeros(96, dtype=np.uint8)
    n = len(pb) // 96
    L._capi.check(L._capi.lib().lurk_point_combination(curve, L._capi.np_ptr(pb), L._capi.np_ptr(sb), n, fmt, L._capi.np_ptr(out)))
    return out


def batch(L, curve, groups, fmt, stream=0):
    """groups: [(point bytes, scalar bytes)] -> (n_groups, 96)"""
    return L.compress.point_combination_batch(curve, groups, fmt=fmt, stream=stream)


def raw_batch(L, curve, counts, pb, sb, fmt, n_groups=None, stream=None):
    c = np.array(counts, dtype=np.uint32)
    out = np.zeros(96 * max(1, len(counts)), dtype=np.uint8)
    rc = L._capi.lib().lurk_point_combination_batch(curve, len(counts) if n_groups is None else n_groups, L._capi.np_ptr(c), L._capi.np_ptr(pb),
                                                    L._capi.np_ptr(sb), fmt, L._capi.np_ptr(out), stream)
    return rc, out


def dlog_want(curve, ks, sc):
    """[sum k_j s_j]G, ks[j] = None for the identity"""
    p, r = moduli(curve)
    t = sum(k * s for k, s in zip(ks, sc) if k is not None) % r
    return spec.ec_mul(t, spec.CURVES[curve]["gen"], p) if t else None


def random_group(curve, n, seed):
    rng = random.Random(seed)
    _, r = moduli(curve)
    terms = [pool(curve)[rng.randrange(POOL)] for _ in range(n)] if n > POOL else rng.sample(pool(curve), n)
    return [k for k, _ in terms], [P for _, P in terms], [rng.randrange(r) for _ in range(n)]


def check_group(L, curve, fmt, ks, pts, sc, got, naive=None):
    pb, sb = enc_points(curve, pts, fmt), enc_scalars(curve, sc, fmt)
    assert np.array_equal(got, host(L, curve, pb, sb, fmt)), "bytes differ from lurk_point_combination"
    want = dlog_want(curve, ks, sc)
    assert dec_point(curve, got, fmt) == want
    if naive if naive is not None else len(pts) <= NAIVE_MAX:
        assert spec.msm_naive(curve, pts, sc) == want


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("size", list(SIZES.values()), ids=list(SIZES.keys()))
def test_random_group(L, curve, fmt, size):
    ks, pts, sc = random_group(curve, size, 7 * size + curve)
    got = batch(L, curve, [(enc_points(curve, pts, fmt), enc_scalars(curve, sc, fmt))], fmt)
    assert got.shape == (1, 96)
    check_group(L, curve, fmt, ks, pts, sc, got[0])


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("curve", CURVES)
def test_mixed_groups_in_one_call_equal_one_call_each(L, curve, fmt):
    sizes = [3, 130, 1, 33, 2, 257, 48, 4, 31, 5]
    groups = [random_group(curve, n, 50 + i) for i, n in enumerate(sizes)]
    enc = [(enc_points(curve, pts, fmt), enc_scalars(curve, sc, fmt)) for _, pts, sc in groups]
    got = batch(L, curve, enc, fmt)
    assert got.shape == (len(sizes), 96)
    for g, (ks, pts, sc) in enumerate(groups):
        assert np.array_equal(got[g], batch(L, curve, [enc[g]], fmt)[0])
        check_group(L, curve, fmt, ks, pts, sc, got[g], naive=False)


def degenerate_groups(curve):
    """name -> (ks, points, scalars): the group-law branches and the edge scalars"""
    _, r = moduli(curve)
    P = pool(curve)
    (k0, P0), (k1, P1), (k2, P2) = P[0], P[1], P[2]
    p, _ = moduli(curve)
    neg = lambda Q: (Q[0], (-Q[1]) % p)
    rng = random.Random(curve)
    rs = lambda n: [rng.randrange(r) for _ in range(n)]
    return {
        "identity-points": ([None, k0, None, k1, None], [None, P0, None, P1, None], rs(5)),
        "only-identity": ([None] * 3, [None] * 3, rs(3)),
        "zero-scalars": ([k0, k1, k2, k0], [P0, P1, P2, P0], [0, rs(1)[0], 0, rs(1)[0]]),
        "all-zero-scalars": ([k0, k1, k2] * 11, [P0, P1, P2] * 11, [0] * 33),
        "one-and-minus-one": ([k0, k1, k2, k2], [P0, P1, P2, P2], [1, r - 1, 1, r - 1]),
        "repeated-point": ([k0] * 40, [P0] * 40, [rs(1)[0]] * 40),           # every window sum doubles
        "repeated-point-mixed-scalars": ([k1] * 33, [P1] * 33, rs(33)),
        "p-and-minus-p": ([k0, -k0, k1, -k1], [P0, neg(P0), P1, neg(P1)], [5, 5, r - 3, r - 3]),       # every window sum cancels
        "cancelling-total": ([k0, k1, k0], [P0, P1, P0], [k1, (-k0) % r, 0]),      # k0 k1 - k1 k0 = 0: the total is the identity
        "top-digits": ([k0, k1, k2], [P0, P1, P2], [r - 1, r - 2, (1 << (r.bit_length() - 1)) + 15]),
    }


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("curve", CURVES)
def test_group_law_branches(L, curve, fmt):
    cases = degenerate_groups(curve)
    _, r = moduli(curve)
    enc = [(enc_points(curve, pts, fmt), enc_scalars(curve, sc, fmt)) for ks, pts, sc in cases.values()]
    got = batch(L, curve, enc, fmt)
    for g, (name, (ks, pts, sc)) in enumerate(cases.items()):
        ks = [None if k is None else k % r for k in ks]
        check_group(L, curve, fmt, ks, pts, sc, got[g])
        if name in ("only-identity", "all-zero-scalars", "p-and-minus-p", "cancelling-total"):
            assert not got[g].any(), name                      # the identity is all zeros


@pytest.mark.parametrize("curve", CURVES)
def test_refusals_come_before_any_launch_and_leave_the_stream_usable(L, curve):
    import torch
    E = L._capi
    s = torch.cuda.Stream()
    st = C.c_void_p(s.cuda_stream)
    ks, pts, sc = random_group(curve, 6, 3)
    _, r = moduli(curve)
    good_p, good_s = enc_points(curve, pts, 0), enc_scalars(curve, sc, 0)
    counts = [2, 4]

    def bad(pb=good_p, sb=good_s, cnt=counts, cv=curve, fmt=0, n_groups=None):
        rc, _ = raw_batch(L, cv, cnt, pb, sb, fmt, n_groups=n_groups, stream=st)
        return rc, E.lib().lurk_last_error()

    off = good_p.copy()
    off[96 * 3 + 32] ^= 1                                          # y of group 1's term 1
    z2 = good_p.copy()
    z2[96 * 4 + 64:96 * 4 + 96] = np.frombuffer((2).to_bytes(32, "little"), dtype=np.uint8)
    big = good_s.copy()
    big[32 * 5:32 * 6] = np.frombuffer(r.to_bytes(32, "little"), dtype=np.uint8)
    for args, code, msg in [
        (dict(pb=off), E.ERR_RANGE, b"group 1: point 1 is not a point of the header's form"),
        (dict(pb=z2), E.ERR_RANGE, b"group 1: point 2 is not a point of the header's form"),
        (dict(sb=big), E.ERR_RANGE, b"group 1: scalar 3 is not reduced"),
        (dict(cv=9), E.ERR_ARG, b"unknown curve"),
        (dict(fmt=2), E.ERR_ARG, b"bad format"),
        (dict(cnt=[2, 0]), E.ERR_ARG, b"group 1 has 0 terms"),
        (dict(n_groups=0), E.ERR_ARG, b"at least one group"),
    ]:
        rc, m = bad(**args)
        assert rc == code and msg in m, (args, rc, m)
    over = [LIMIT + 1]
    rc, m = bad(pb=np.zeros(96 * (LIMIT + 1), dtype=np.uint8), sb=np.zeros(32 * (LIMIT + 1), dtype=np.uint8), cnt=over)
    assert rc == E.ERR_ARG and b"4097 terms" in m
    # the same stream straight after the refusals
    out = batch(L, curve, [(good_p[:192], good_s[:64]), (good_p[192:], good_s[64:])], 0, stream=s.cuda_stream)
    s.synchronize()
    check_group(L, curve, 0, ks[:2], pts[:2], sc[:2], out[0])
    check_group(L, curve, 0, ks[2:], pts[2:], sc[2:], out[1])


def test_two_host_threads_on_two_streams(L):
    import torch
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    jobs = []
    for t in range(2):
        curve = [0, 2][t]
        groups = [random_group(curve, n, 900 + 10 * t + i) for i, n in enumerate([130, 2, 44, 25, 3])]
        jobs.append((curve, groups, [(enc_points(curve, pts, t), enc_scalars(curve, sc, t)) for _, pts, sc in groups]))
    results, errors = [[None] * 20, [None] * 20], []

    def run(t):
        try:
            curve, _, enc = jobs[t]
            for i in range(20):
                results[t][i] = batch(L, curve, enc, t, stream=streams[t].cuda_stream)
        except Exception as e:           # reported below
            errors.append(e)
    th = [threading.Thread(target=run, args=(t,)) for t in range(2)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors
    for t, (curve, groups, _) in enumerate(jobs):
        for i in range(1, 20):
            assert np.array_equal(results[t][i], results[t][0])
        for g, (ks, pts, sc) in enumerate(groups):
            check_group(L, curve, t, ks, pts, sc, results[t][0][g], naive=False)


def test_list_form_of_the_binding(L):
    """the Python lists of (x, y) / None and ints give what the byte form gives"""
    ks, pts, sc = random_group(1, 9, 11)
    got = L.point_combination_batch(1, [(pts, sc), ([None, pts[0]], [3, 0])])
    assert L.compress.points_of(got) == [dlog_want(1, ks, sc), None]
    with pytest.raises(ValueError):
        L.point_combination_batch(1, [([], [])])
