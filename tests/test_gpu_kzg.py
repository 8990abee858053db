"""GPU parity for the KZG side of the BN256 path (SURVEY.md 8(f) N3 / N4): the powers-of-tau key and the HyperKZG opening prover
through the C ABI -- bit-exact against oracle/kzg.py at small sizes, and at 2^20 coefficients against the MATHS with a key of
known beta: every commitment the GPU returns must be [f(beta)] g for the polynomial f the protocol defines (fold chain, batched
witness quotients), every evaluation must be the oracle's, and the verifier's algebra must accept.
Challenges come from a stand-in function (sha256); Arecibo's Keccak256Transcript is the caller's side of the callback."""
import hashlib
import time

import numpy as np
import pytest

from oracle import kzg, sumcheck as sc
from util import ints, pack, random_elements

pytestmark = pytest.mark.gpu


def to_device(L, field, canon_buf):
    import torch
    import ctypes as C
    t = torch.from_numpy(np.ascontiguousarray(canon_buf, dtype=np.uint8)).cuda()
    L._capi.check(L._capi.lib().lurk_convert_dev(field, C.c_void_p(t.data_ptr()), t.numel() // 32, L.FMT_MONTGOMERY, C.c_void_p(t.data_ptr()), None))
    return t


def key_points(L, spec, curve, ck):
    """the device-resident key of a CommitmentKey made by powers_of_tau, as canonical affine tuples"""
    import ctypes as C
    base = spec.CURVES[curve]["base"]
    c = ck._bases.clone()
    L._capi.check(L._capi.lib().lurk_convert_dev(base, C.c_void_p(c.data_ptr()), c.numel() // 32, L.FMT_CANONICAL, C.c_void_p(c.data_ptr()), None))
    v = ints(c.cpu().numpy())
    return [(x, y) if (x or y) else None for x, y in zip(v[0::2], v[1::2])]


def msg_ints(msg):
    return [int.from_bytes(msg[i:i + 32], "little") for i in range(0, len(msg), 32)]


def chal_fn(p, log):
    def f(rnd, msg):
        log.append((rnd, bytes(msg)))
        return int.from_bytes(hashlib.sha256(bytes([rnd]) + bytes(msg)).digest() + hashlib.sha256(b"x" + bytes(msg)).digest(), "little") % p
    return f


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_powers_of_tau_match_oracle(L, spec, curve):
    Cv = spec.CURVES[curve]
    pb, q = spec.FIELD_MODULUS[Cv["base"]], spec.FIELD_MODULUS[Cv["scalar"]]
    g = spec.ec_mul(987654321, Cv["gen"], pb)
    beta = ints(random_elements(Cv["scalar"], 1, seed=4))[0]
    for n, b in ((70, beta), (1, beta), (5, beta), (9, 0), (6, 1), (7, q - 1)):
        ck = L.CommitmentKey.powers_of_tau(curve, g, b, n)
        assert key_points(L, spec, curve, ck) == kzg.powers_of_tau(curve, g, b, n), (curve, n, b)
    with pytest.raises(L.LurkError) as e:                      # a generator off the curve is refused
        L.CommitmentKey.powers_of_tau(curve, (g[0], (g[1] + 1) % pb), beta, 4)
    assert e.value.code == L._capi.ERR_RANGE


@pytest.mark.parametrize("l", [1, 2, 3, 6, 9])
def test_hyperkzg_prover_matches_oracle(L, oracle, spec, l):
    curve, field = 0, 0
    p = spec.FIELD_MODULUS[field]
    n = 1 << l
    bases = oracle.gen_bases(curve, n, start=3)
    ck = L.CommitmentKey(curve, bases)
    Ph = random_elements(field, n, seed=l, shape="witness" if l == 6 else "uniform")
    x = ints(random_elements(field, l, seed=50 + l))
    log = []
    com, v, w = L.spartan.hyperkzg_prove(curve, ck, to_device(L, field, Ph).data_ptr(), x, chal_fn(p, log))

    def commit(f):
        pt = oracle.msm(curve, bases[:64 * len(f)], pack(f), nthreads=4)
        vv = ints(pt)
        return (vv[0], vv[1]) if vv[2] else None

    def enc(points):
        return b"".join((pack([P[0], P[1], 1]) if P is not None else np.zeros(96, dtype=np.uint8)).tobytes() for P in points)

    def ochal(rnd, msg):
        data = enc(msg) if rnd != 1 else b"".join(pack(row).tobytes() for row in msg)
        return int.from_bytes(hashlib.sha256(bytes([rnd]) + data).digest() + hashlib.sha256(b"x" + data).digest(), "little") % p

    want = kzg.prove(curve, commit, ints(Ph), x, ochal)
    assert com == want["com"] and v == want["v"] and w == want["w"]
    assert [r for r, _ in log] == [0, 1, 2]


def test_hyperkzg_with_known_beta_full_chain(L, spec):
    """2^20 coefficients, key = beta^i g generated on the GPU: commitments equal [f(beta)] g, evaluations equal the oracle's,
    the verifier's algebra accepts"""
    curve, field, l = 0, 0, 20
    Cv = spec.CURVES[curve]
    pb, p = spec.FIELD_MODULUS[Cv["base"]], spec.FIELD_MODULUS[field]
    n = 1 << l
    g = spec.ec_mul(31337, Cv["gen"], pb)
    beta = ints(random_elements(field, 1, seed=77))[0]
    t0 = time.time()
    ck = L.CommitmentKey.powers_of_tau(curve, g, beta, n)
    t_key = time.time() - t0
    Ph = random_elements(field, n, seed=5, shape="witness")
    x = ints(random_elements(field, l, seed=6))
    dP = to_device(L, field, Ph)
    log = []
    import torch
    torch.cuda.synchronize()
    t0 = time.time()
    com, v, w = L.spartan.hyperkzg_prove(curve, ck, dP.data_ptr(), x, chal_fn(p, log))
    t_prove = time.time() - t0
    print(f"\npowers-of-tau key 2^20: {t_key * 1e3:.1f} ms;  HyperKZG prove 2^20 (Python callbacks): {t_prove * 1e3:.1f} ms")
    P = ints(Ph)
    polys = kzg.fold_chain(P, x, p)
    # the key really is beta^i g (spot checks) and the commitments are [P_j(beta)] g
    kp_first = kzg.powers_of_tau(curve, g, beta, 3)
    import ctypes as C
    head = ck._bases[:64 * 3].clone()
    L._capi.check(L._capi.lib().lurk_convert_dev(Cv["base"], C.c_void_p(head.data_ptr()), 6, L.FMT_CANONICAL, C.c_void_p(head.data_ptr()), None))
    hv = ints(head.cpu().numpy())
    assert list(zip(hv[0::2], hv[1::2])) == kp_first
    at_beta = [kzg.poly_eval(f, beta, p) for f in polys]
    assert com == [spec.ec_mul(s, g, pb) for s in at_beta[1:]]
    r = int.from_bytes(hashlib.sha256(bytes([0]) + log[0][1]).digest() + hashlib.sha256(b"x" + log[0][1]).digest(), "little") % p
    u = [r, (-r) % p, r * r % p]
    assert v == [[kzg.poly_eval(f, ut, p) for f in polys] for ut in u]
    q = int.from_bytes(hashlib.sha256(bytes([1]) + log[1][1]).digest() + hashlib.sha256(b"x" + log[1][1]).digest(), "little") % p
    assert msg_ints(log[1][1]) == [e for row in v for e in row]
    # w_t = [h_t(beta)] g with h_t(beta) = (B(beta) - B(u_t)) / (beta - u_t)
    Bbeta = sum(pow(q, j, p) * s for j, s in enumerate(at_beta)) % p
    w_scalars = []
    for t in range(3):
        Bu = sum(pow(q, j, p) * v[t][j] for j in range(l)) % p
        w_scalars.append((Bbeta - Bu) * pow(beta - u[t], -1, p) % p)
    assert w == [spec.ec_mul(s, g, pb) for s in w_scalars]
    assert kzg.verify_known_beta(curve, g, beta, at_beta[0], x, _final_eval(polys, x, p),
                                 at_beta[1:], v, w_scalars, r, q)


def _final_eval(polys, x, p):
    """P(x) = the last fold of the chain: P_l = x_0 (P_{l-1}[1] - P_{l-1}[0]) + P_{l-1}[0]"""
    last = polys[-1]
    return (x[0] * (last[1] - last[0]) + last[0]) % p
