"""The verifiers' CPU checkers: the IPA verifier oracle (tests/ipa_verify_oracle.py) accepts a transcript of a pure-Python
InnerProductArgument::prove built from oracle/sumcheck.py's fold steps and rejects a changed L_j, R_j, a_final, c or comm; the OpenMP port of
matrices_eval (tests/csrc/matrices_eval_cpu.c) equals oracle/spartan.py: matrices_eval on real and adversarial shapes and on points with
coordinates 0, 1, p - 1 and random values, on one thread and on four."""
import hashlib

import numpy as np
import pytest

import ipa_verify_oracle as iv
from oracle import nifs, spec, sumcheck as sc
from util import ints, random_elements


def python_prove(curve, G, gc, a, b, challenge):
    pb, q = spec.FIELD_MODULUS[spec.CURVES[curve]["base"]], spec.FIELD_MODULUS[spec.CURVES[curve]["scalar"]]
    add = lambda P, Q: spec.ec_add(P, Q, pb)
    mul = lambda k, P: spec.ec_mul(k % q, P, pb)
    Ls, Rs = [], []
    while len(a) > 1:
        h = len(a) // 2
        Lj = add(spec.msm_naive(curve, G[h:], a[:h]), mul(sc.inner_product(a[:h], b[h:], q), gc))
        Rj = add(spec.msm_naive(curve, G[:h], a[h:]), mul(sc.inner_product(a[h:], b[:h], q), gc))
        r = challenge(len(Ls), iv.point_bytes(Lj) + iv.point_bytes(Rj)) % q
        ri = pow(r, -1, q)
        Ls.append(Lj)
        Rs.append(Rj)
        a, b = sc.ipa_fold_scalars(a, r, ri, q), sc.ipa_fold_scalars(b, ri, r, q)
        G = sc.ipa_fold_bases(curve, G, ri, r)
    return Ls, Rs, a[0]


def chal(rnd, msg):
    return 1 + int.from_bytes(hashlib.sha256(bytes([rnd]) + msg).digest()[:16], "little")


@pytest.mark.parametrize("curve", [0, 2])
def test_oracle_ipa_verify_accepts_and_rejects(oracle, curve):
    q = spec.FIELD_MODULUS[spec.CURVES[curve]["scalar"]]
    pb = spec.FIELD_MODULUS[spec.CURVES[curve]["base"]]
    n = 8
    bases = ints(oracle.gen_bases(curve, n + 1, start=3))
    pts = list(zip(bases[0::2], bases[1::2]))
    G, gc = pts[:n], pts[n]
    a = ints(random_elements(spec.CURVES[curve]["scalar"], n, seed=curve + 1))
    b = ints(random_elements(spec.CURVES[curve]["scalar"], n, seed=curve + 2, shape="edge"))
    comm, c = spec.msm_naive(curve, G, a), sc.inner_product(a, b, q)
    Ls, Rs, a_hat = python_prove(curve, G, gc, a, b, chal)
    msm = lambda Gs, s: spec.msm_naive(curve, Gs, s)
    ok, ck_hat, b_hat = iv.ipa_verify(curve, G, gc, comm, c, b, Ls, Rs, a_hat, chal, msm)
    assert ok and b_hat == sc.inner_product(b, iv.tensor([chal(j, iv.point_bytes(L) + iv.point_bytes(R)) % q for j, (L, R) in enumerate(zip(Ls, Rs))], q), q)
    other = spec.ec_add(G[0], gc, pb)
    assert not iv.ipa_verify(curve, G, gc, comm, c, b, [other] + Ls[1:], Rs, a_hat, chal, msm)[0]
    assert not iv.ipa_verify(curve, G, gc, comm, c, b, Ls, Rs[:-1] + [other], a_hat, chal, msm)[0]
    assert not iv.ipa_verify(curve, G, gc, comm, c, b, Ls, Rs, (a_hat + 1) % q, chal, msm)[0]
    assert not iv.ipa_verify(curve, G, gc, comm, (c + 1) % q, b, Ls, Rs, a_hat, chal, msm)[0]
    assert not iv.ipa_verify(curve, G, gc, other, c, b, Ls, Rs, a_hat, chal, msm)[0]


# ------------------------------------------------------------------------------------------------ the OpenMP port of matrices_eval
def csr(rows, entries):
    e = np.asarray(entries, dtype=np.int64).reshape(-1, 2)
    e = e[np.argsort(e[:, 0], kind="stable")]
    rp = np.concatenate([[0], np.cumsum(np.bincount(e[:, 0], minlength=rows))]).astype(np.uint64)
    return rp, e[:, 1].astype(np.uint32)


def rows_of(mat):
    rp, col, val = mat
    v = ints(val)
    return [[(int(col[k]), v[k]) for k in range(int(rp[i]), int(rp[i + 1]))] for i in range(len(rp) - 1)]


def shapes():
    """(name, field, mats, n_w, n_x): a real step-circuit shape per field and the adversarial ones"""
    out = []
    for field in range(4):
        mats, n_w, _ = nifs.real_shape_step_circuit(np.random.default_rng(40 + field), spec.FIELD_MODULUS[field], 1, 200, 24, 30)
        out.append((f"real-{field}", field, mats, n_w, 2))
    rng = np.random.default_rng(5)
    n_w, n_x, rows = 3000, 4, 20001
    mats = []
    for m in range(3):
        entries = [(7, int(c)) for c in rng.choice(n_w + 1 + n_x, size=2500, replace=False)] if m == 0 else []
        entries += [(int(r), n_w + m) for r in rng.choice(rows, size=15000, replace=False)]           # u, X0, X1 columns
        entries += [(int(rng.integers(0, rows // 2)), int(c)) for c in rng.integers(0, n_w, size=3000)]
        rp, col = csr(rows, entries)
        mats.append((rp, col, random_elements(0, len(col), seed=10 + m)))
    out.append(("long-row-long-columns-empty-rows", 0, mats, n_w, n_x))
    empty = (np.zeros(3, dtype=np.uint64), np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.uint8))
    out.append(("empty-no-x-two-rows", 1, [empty] * 3, 10, 0))
    rp, col = csr(1, [(0, c) for c in range(12)])
    out.append(("one-row", 3, [(rp, col, random_elements(3, 12, seed=2))] * 3, 11, 0))
    return out


@pytest.mark.parametrize("kind", ["random", "zero", "one", "minus-one", "mixed"])
def test_matrices_eval_port_equals_the_python_oracle(kind):
    import matrices_eval_cpu as mc
    from oracle import spartan as osp
    for name, field, mats, n_w, n_x in shapes():
        p = spec.FIELD_MODULUS[field]
        rows = len(mats[0][0]) - 1
        log_rows = max(1, (rows - 1).bit_length())
        num_vars = 1 << max(1, (max(n_w, n_x + 1) - 1).bit_length())
        rng = np.random.default_rng(len(name))
        rnd = lambda: int.from_bytes(rng.bytes(32), "little") % p
        pick = {"random": rnd, "zero": lambda: 0, "one": lambda: 1, "minus-one": lambda: p - 1,
                "mixed": lambda: [0, 1, p - 1, rnd()][int(rng.integers(0, 4))]}[kind]
        rx, ry = [pick() for _ in range(log_rows)], [pick() for _ in range(num_vars.bit_length())]
        want = tuple(osp.matrices_eval([rows_of(m) for m in mats], n_w, num_vars, rx, ry, p))
        assert mc.matrices_eval(p, mats, n_w, num_vars, rx, ry, nthreads=4) == want, name
        assert mc.matrices_eval(p, mats, n_w, num_vars, rx, ry, nthreads=1) == want, name
