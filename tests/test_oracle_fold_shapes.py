"""The CPU side of the fold-context tests on real row shapes (tests/test_gpu_fold_shapes.py relies on it): the edge-operand
sampler, the real-shape R1CS generator, oracle.c's fold helpers against Python integers on all four fields, and the
oracle's random-oracle absorb patterns."""
import hashlib

import numpy as np
import pytest

from oracle import nifs
from util import edge_values, ints, pack, random_elements

FIELDS = [0, 1, 2, 3]


def test_uniform_shape_unchanged(spec):
    """existing seeds keep their inputs: "uniform" still samples below 2^(bits-1)"""
    digest = {0: "921a9f3fc16b9140", 2: "748bcf07dd29f863"}
    for f in FIELDS:
        out = random_elements(f, 257, seed=11)
        assert hashlib.sha256(out.tobytes()).hexdigest()[:16] == digest[0 if f < 2 else 2]
        assert max(ints(out)) < 1 << (spec.FIELD_MODULUS[f].bit_length() - 1)


@pytest.mark.parametrize("field", FIELDS)
def test_edge_shape_covers_the_field(spec, field):
    p = spec.FIELD_MODULUS[field]
    bits = p.bit_length()
    v = ints(random_elements(field, 3000, seed=4, shape="edge"))
    assert len(v) == 3000 and all(0 <= x < p for x in v)
    assert set(edge_values(field)) <= set(v)
    assert {0, 1, 2, p - 1, p - 2, (p - 1) // 2, (p + 1) // 2, (1 << 256) % p, pow(1 << 256, -1, p)} <= set(edge_values(field))
    top = [x for x in v if x >= 1 << (bits - 1)]
    assert len(top) >= 750                         # a quarter from [2^(bits-1), p), more from the uniform part (BN254)
    mont = [x * (1 << 256) % p for x in v]
    assert sum(1 for m in mont if m >= p - (p >> 4)) >= 750
    assert max(v) > p - (p >> 20)
    assert np.array_equal(random_elements(field, 3000, seed=4, shape="edge"), pack(v))
    assert random_elements(field, 0, seed=1, shape="edge").size == 0


def _real(spec, field, seed, frames=1, free=300, glue=24, lin_rows=24):
    p = spec.FIELD_MODULUS[field]
    rng = np.random.default_rng(seed)
    mats, n_w, glue_fn = nifs.real_shape_step_circuit(rng, p, frames, free, glue, lin_rows)
    return p, mats, n_w, glue_fn


def _rows(mat):
    rp, col, val = mat
    v = ints(val)
    return [[(int(col[k]), v[k]) for k in range(int(rp[i]), int(rp[i + 1]))] for i in range(len(rp) - 1)]


def _witness(field, n_w, glue_fn, seed, zero=False):
    W = [0] * n_w if zero else ints(random_elements(field, n_w, seed=seed, shape="edge"))
    X = ints(random_elements(field, 2, seed=seed + 1, shape="edge"))
    for dst, v in glue_fn(W, X).items():
        W[dst] = v
    return W, X


@pytest.mark.parametrize("field", FIELDS)
def test_real_shape_circuit(spec, field):
    p, mats, n_w, glue_fn = _real(spec, field, seed=field)
    A, B, Cm = (_rows(m) for m in mats)
    assert set(nifs.REAL_ROW_LENGTHS) <= {len(r) for r in A}
    coeffs = {v for r in A + B + Cm for _, v in r}
    assert p - 1 in coeffs and any(v.bit_length() > p.bit_length() - 8 for v in coeffs) and any(v < 37 for v in coeffs)
    assert any(len(r) == 255 and [v for _, v in r] == [pow(2, i, p) for i in range(255)] for r in A)
    cols = {c for r in A + B + Cm for c, _ in r}
    assert n_w in cols and cols & {n_w + 1, n_w + 2}                       # u and X
    assert any(not a and not b and not c for a, b, c in zip(A, B, Cm))
    for zero in (False, True):
        W, X = _witness(field, n_w, glue_fn, seed=10 + field, zero=zero)
        z = W + [1] + X
        dot = lambda r: sum(z[c] * v for c, v in r) % p
        assert all((dot(a) * dot(b) - dot(c)) % p == 0 for a, b, c in zip(A, B, Cm)), "fresh instance satisfies"
    # two fresh instances: the cross term does not vanish on the product rows
    W1, X1 = _witness(field, n_w, glue_fn, seed=30)
    W2, X2 = _witness(field, n_w, glue_fn, seed=40)
    z1, z2 = W1 + [1] + X1, W2 + [1] + X2
    t = [(sum(z1[c] * v for c, v in a) * sum(z2[c] * v for c, v in b) + sum(z2[c] * v for c, v in a) * sum(z1[c] * v for c, v in b)
          - sum(z2[c] * v for c, v in c_) - sum(z1[c] * v for c, v in c_)) % p for a, b, c_ in zip(A, B, Cm)]
    assert sum(1 for x in t if x) > len(t) // 4


@pytest.mark.parametrize("field", FIELDS)
def test_fold_helpers_oracle_matches_python(oracle, spec, field):
    """oracle.c's axpy / spmv / cross_term, which most GPU fold expectations come from, against Python integers"""
    p, mats, n_w, glue_fn = _real(spec, field, seed=100 + field)
    n = n_w + 3
    z = ints(random_elements(field, n, seed=7, shape="edge"))
    for m in mats:
        y = ints(oracle.spmv(field, m[0], m[1], m[2], pack(z), nthreads=2))
        assert y == [sum(z[c] * v for c, v in r) % p for r in _rows(m)]
    a, b = ints(random_elements(field, 600, seed=8, shape="edge")), ints(random_elements(field, 600, seed=9, shape="edge"))
    for r in edge_values(field) + ints(random_elements(field, 3, seed=10, shape="edge")):
        assert ints(oracle.axpy(field, pack(a), pack(b), pack([r]))) == [(x + r * y) % p for x, y in zip(a, b)]
    v = [ints(random_elements(field, 600, seed=20 + k, shape="edge")) for k in range(6)]
    for u1, u2 in ((1, 1), (p - 1, 1), (0, 1), (ints(random_elements(field, 1, 5, "edge"))[0], 1)):
        t = ints(oracle.cross_term(field, *[pack(x) for x in v], pack([u1]), pack([u2])))
        assert t == [(v[0][i] * v[4][i] + v[3][i] * v[1][i] - u1 * v[5][i] - u2 * v[2][i]) % p for i in range(600)]


def test_oracle_ro_patterns(oracle, spec):
    """NovaOracle.prove_step builds the absorb list of a custom pattern as the fold context does; the default pattern is
    Arecibo's NIFS::prove list"""
    curve = 2
    field, pb = spec.CURVES[curve]["scalar"], spec.FIELD_MODULUS[spec.CURVES[curve]["base"]]
    p, mats, n_w, glue_fn = _real(spec, field, seed=5, free=60, glue=12, lin_rows=12)
    bases = oracle.gen_bases(curve, max(n_w, len(mats[0][0]) - 1))
    W, X = _witness(field, n_w, glue_fn, seed=1)
    o1, o2 = (nifs.NovaOracle(curve, bases, mats, n_w, 2, pp_digest=99) for _ in range(2))
    o1.init_running(pack(W), X)
    o2.init_running(pack(W), X)
    W2, X2 = _witness(field, n_w, glue_fn, seed=2)
    a = o1.prove_step(pack(W2), X2)
    b = o2.prove_step(pack(W2), X2, ro_kinds=nifs.DEFAULT_RO_KINDS)
    assert a["absorbed"] == b["absorbed"] and (a["r"], a["hash"]) == (b["r"], b["hash"])
    # the first fold of the instance the chain started from: T = 0, comm_T is the identity, absorbed as (0, 0, 1)
    o = nifs.NovaOracle(curve, bases, mats, n_w, 2, pp_digest=99)
    o.init_running(pack(W), X)
    kinds = [nifs.RO_T_INF, nifs.RO_CONST, nifs.RO_W_INF, nifs.RO_T_X, nifs.RO_W_Y, nifs.RO_T_Y]
    consts = list(range(1000, 1024))
    s = o.prove_step(pack(W), X, challenge_bits=33, ro_kinds=kinds, ro_consts=consts)
    assert not any(ints(s["T"])) and s["comm_T"] is None
    cw = s["comm_W"]
    assert s["absorbed"] == [1, 1001, 0, 0, cw[1], 0]
    r, h = spec.ro_squeeze(spec.CURVES[curve]["base"], s["absorbed"], 33)
    assert (s["r"], s["hash"]) == (r, h) and r < 1 << 33 and h < pb
    assert o.bad_rows() == 0
