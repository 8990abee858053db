"""The oracle's batch_eval_reduce / batch_eval_verify and batched Spartan prover / verifier (tests/batched_oracle.py: prove_batched,
verify_batched) -- SuperNova's `compress` (reference src/proof/supernova.rs:110,293-317) ending in one evaluation claim.
Round trips on all four fields, instances that really went through Nova folds (u != 1, E != 0), and the rejections.  CPU only."""
import numpy as np
import pytest

import batched_oracle as bo
from oracle import sumcheck as sc
from test_gpu_spartan_chain import challenge, folded_instance, rows_of
from util import ints, random_elements


def be_challenge(rnd, values):
    return challenge("batch_eval", (rnd, list(values)))


def random_claims(field, sizes, seed, p):
    polys = [ints(random_elements(field, 1 << n, seed=seed + 10 * i)) for i, n in enumerate(sizes)]
    points = [ints(random_elements(field, max(n, 1), seed=seed + 10 * i + 5))[:n] for i, n in enumerate(sizes)]
    return polys, points, [sc.mle_eval(P, x, p) for P, x in zip(polys, points)]


@pytest.mark.parametrize("field", [0, 1, 2, 3])
@pytest.mark.parametrize("sizes", [[5], [9, 4, 0, 9, 1], [7, 7, 7]])
def test_batch_eval_reduce_round_trip(spec, field, sizes):
    p = spec.FIELD_MODULUS[field]
    polys, points, evals = random_claims(field, sizes, 3 * field + len(sizes), p)
    out = bo.batch_eval_reduce(polys, points, evals, be_challenge, p)
    m = max(sizes)
    assert len(out["rounds"]) == len(out["r"]) == m and len(out["joint"]) == 1 << m
    # L_i is P_i at the tail of r; the joint polynomial is sum_i gamma^i P_i, zero-padded, and its MLE at r is the joint evaluation
    assert out["claims_left"] == [sc.mle_eval(P, out["r"][m - len(x):], p) for P, x in zip(polys, points)]
    assert sc.mle_eval(out["joint"], out["r"], p) == out["joint_eval"]
    got = bo.batch_eval_verify(out["rounds"], points, evals, out["claims_left"], be_challenge, p)
    assert got == (out["r"], out["joint_eval"], out["weights"])
    # a wrong claim, a perturbed L_i or a doctored round are rejected
    bad = list(evals)
    bad[-1] = (bad[-1] + 1) % p
    assert bo.batch_eval_verify(out["rounds"], points, bad, out["claims_left"], be_challenge, p) is None
    left = list(out["claims_left"])
    left[0] = (left[0] + 1) % p
    assert bo.batch_eval_verify(out["rounds"], points, evals, left, be_challenge, p) is None
    if m:
        rounds = [list(r) for r in out["rounds"]]
        rounds[-1][2] = (rounds[-1][2] + 1) % p
        assert bo.batch_eval_verify(rounds, points, evals, out["claims_left"], be_challenge, p) is None


def instance(oracle, spec, seed, frames, slot_elems, glue, lin):
    """a running instance after three Nova folds, as the dict prove_batched / verify_batched take"""
    mats, n_w, o = folded_instance(oracle, spec, np.random.default_rng(seed), frames, slot_elems, glue, lin)
    rows = len(mats[0][0]) - 1
    return dict(R=[rows_of(m) for m in mats], n_w=n_w, nv=1 << max(1, (max(n_w, 3) - 1).bit_length()), s=max(1, (rows - 1).bit_length()),
                rows=rows, W=ints(o.W), E=ints(o.E), u=o.u, X=list(o.X)), mats


SHAPES = [(1, 6, 3, 3), (3, 10, 5, 4), (2, 60, 12, 10)]


@pytest.mark.parametrize("count", [1, 3])
def test_batched_spartan_accepts_folded_instances_and_rejects_tampering(oracle, spec, count):
    p = spec.FIELD_MODULUS[0]
    insts = [instance(oracle, spec, 40 + k, *SHAPES[k if count > 1 else 1])[0] for k in range(count)]
    if count > 1:
        assert len({I["s"] for I in insts}) == count and len({I["nv"] for I in insts}) == count
    proof = bo.prove_batched(insts, challenge, p)
    ok, r, joint_eval, weights = bo.verify_batched(insts, proof, challenge, p)
    assert ok and r == proof["r"] and joint_eval == proof["joint_eval"] and weights == proof["weights"]
    assert sc.mle_eval(proof["joint"], r, p) == joint_eval
    # the claims are the padded vectors' multilinear extensions
    for I, y, x, ew, c in zip(insts, proof["ry"], proof["rx"], proof["eval_W"], proof["claims"]):
        assert ew == sc.mle_eval(I["W"] + [0] * (I["nv"] - I["n_w"]), y[1:], p)
        assert c[3] == sc.mle_eval(I["E"] + [0] * ((1 << I["s"]) - I["rows"]), x, p)
    # one tampered row of E: the instance no longer satisfies the relaxed R1CS
    bad = [dict(I) for I in insts]
    bad[-1]["E"] = list(bad[-1]["E"])
    bad[-1]["E"][1] = (bad[-1]["E"][1] + 1) % p
    assert not bo.verify_batched(insts, bo.prove_batched(bad, challenge, p), challenge, p)[0]
    # the transcript against one instance with another u
    moved = [dict(I) for I in insts]
    moved[0]["u"] = (moved[0]["u"] + 1) % p
    assert not bo.verify_batched(moved, proof, challenge, p)[0]
    # two instances swapped
    if count > 1:
        assert not bo.verify_batched([insts[1], insts[0]] + insts[2:], proof, challenge, p)[0]
    # a perturbed L_i
    for i in (0, len(proof["claims_left"]) - 1):
        left = list(proof["claims_left"])
        left[i] = (left[i] + 1) % p
        assert not bo.verify_batched(insts, dict(proof, claims_left=left), challenge, p)[0]
