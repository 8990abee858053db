"""GPU side of `compress` ending in ONE opening: lurk_batch_eval_reduce_dev (Arecibo's batch_eval_reduce) against the oracle, the Nova
composition RelaxedR1CSSNARK + reduction + one HyperKZG opening, and SuperNova's BatchedRelaxedR1CSSNARK (reference
src/proof/supernova.rs:110,293-317) over running instances of three circuits of different sizes -- folded on the GPU through
SuperNovaFoldContext or by the oracle -- opened with HyperKZG on BN254 and with the inner-product argument on Pallas.
Challenges: the sha256 stand-in of test_gpu_spartan_chain.py for Keccak256Transcript."""
import hashlib

import numpy as np
import pytest

import batched_oracle as bo
from oracle import kzg, nifs, spartan as osp, spec as ospec, sumcheck as sc
from test_gpu_fold_pipeline import _build, _fill, _step_inputs
from test_gpu_spartan_chain import challenge, folded_instance, open_and_check, rows_of, to_device
from test_gpu_sumcheck import from_device
from util import ints, pack, random_elements

pytestmark = pytest.mark.gpu


def be_challenge(rnd, values):
    return challenge("batch_eval", (rnd, list(values)))


def gpu_be_challenge(p):
    return lambda rnd, msg: be_challenge(rnd, [int.from_bytes(msg[i:i + 32], "little") for i in range(0, len(msg), 32)]) % p


def claim_set(field, sizes, seed, p):
    bufs = [random_elements(field, 1 << n, seed=seed + 7 * i) for i, n in enumerate(sizes)]
    points = [ints(random_elements(field, max(n, 1), seed=seed + 7 * i + 3))[:n] for i, n in enumerate(sizes)]
    polys = [ints(b) for b in bufs]
    return bufs, polys, points, [sc.mle_eval(P, x, p) for P, x in zip(polys, points)]


@pytest.mark.parametrize("field", [0, 1, 2, 3])
def test_batch_eval_reduce_matches_oracle(L, field):
    import torch
    p = ospec.FIELD_MODULUS[field]
    rng = np.random.default_rng(field)
    sets = [[5], [9, 4, 0, 9, 1], [7, 7, 7], [int(x) for x in rng.integers(0, 9, size=60)]]
    for k, sizes in enumerate(sets):
        bufs, polys, points, evals = claim_set(field, sizes, 100 * k + field, p)
        want = bo.batch_eval_reduce(polys, points, evals, be_challenge, p)
        dev = [to_device(L, field, b) for b in bufs]
        keep = [d.clone() for d in dev]
        rounds, r, left, w, je, joint = L.spartan.batch_eval_reduce(field, [(d.data_ptr(), n, x, e) for d, n, x, e in zip(dev, sizes, points, evals)],
                                                                    gpu_be_challenge(p))
        assert (rounds, r, left, w, je) == (want["rounds"], want["r"], want["claims_left"], want["weights"], want["joint_eval"]), sizes
        assert from_device(L, field, joint) == want["joint"], sizes
        assert all(torch.equal(a, b) for a, b in zip(dev, keep)), "an input polynomial was modified"
    # 61 claims are refused, a non-reduced evaluation and a non-reduced challenge are out of range, a failing callback aborts
    d = to_device(L, field, random_elements(field, 4, seed=1))
    with pytest.raises(L.LurkError) as e:
        L.spartan.batch_eval_reduce(field, [(d.data_ptr(), 2, [1, 2], 0)] * 61, gpu_be_challenge(p))
    assert e.value.code == L._capi.ERR_ARG
    with pytest.raises(L.LurkError) as e:
        L.spartan.batch_eval_reduce(field, [(d.data_ptr(), 2, [1, 2], p)], gpu_be_challenge(p))
    assert e.value.code == L._capi.ERR_RANGE
    with pytest.raises(L.LurkError) as e:
        L.spartan.batch_eval_reduce(field, [(d.data_ptr(), 2, [1, 2], 0)], lambda rnd, msg: p)
    assert e.value.code == L._capi.ERR_RANGE
    with pytest.raises(ZeroDivisionError):
        L.spartan.batch_eval_reduce(field, [(d.data_ptr(), 2, [1, 2], 0)], lambda rnd, msg: 1 // (2 - rnd))


def test_batch_eval_reduce_at_compress_size(L):
    """W of 2^20 and E of 2^21 elements (fib rc = 100): the oracle verifier accepts the transcript and <joint, eq(r)> is the joint claim"""
    import torch
    field = 0
    p = ospec.FIELD_MODULUS[field]
    sizes = [20, 21]
    dev, points, evals = [], [], []
    for i, n in enumerate(sizes):
        d = to_device(L, field, random_elements(field, 1 << n, seed=50 + i))
        x = ints(random_elements(field, n, seed=60 + i))
        q = torch.empty((1 << n) * 32, dtype=torch.uint8, device="cuda")
        L.spartan.eq_evals(field, x, q.data_ptr())
        dev.append(d)
        points.append(x)
        evals.append(L.spartan.inner_product(field, d.data_ptr(), q.data_ptr(), 1 << n))
    keep = [d.clone() for d in dev]
    rounds, r, left, w, je, joint = L.spartan.batch_eval_reduce(field, [(d.data_ptr(), n, x, e) for d, n, x, e in zip(dev, sizes, points, evals)],
                                                                gpu_be_challenge(p))
    assert bo.batch_eval_verify(rounds, points, evals, left, be_challenge, p) == (r, je, w)
    q = torch.empty((1 << 21) * 32, dtype=torch.uint8, device="cuda")
    L.spartan.eq_evals(field, r, q.data_ptr())
    assert L.spartan.inner_product(field, joint.data_ptr(), q.data_ptr(), 1 << 21) == je
    assert all(torch.equal(a, b) for a, b in zip(dev, keep))


def kzg_setup(L, n):
    g = ospec.ec_mul(4242, ospec.CURVES[0]["gen"], ospec.FIELD_MODULUS[1])
    beta = 0x1234567890abcdef1234567890abcdef % ospec.FIELD_MODULUS[0]
    return g, beta, L.CommitmentKey.powers_of_tau(0, g, beta, n)


def test_nova_compress_with_one_opening(L, oracle):
    """RelaxedR1CSSNARK::prove, then batch_eval_reduce of (W at ry[1:], E at rx), then ONE HyperKZG opening of the joint polynomial"""
    p = ospec.FIELD_MODULUS[0]
    mats, n_w, o = folded_instance(oracle, ospec, np.random.default_rng(31))
    prover = L.spartan.RelaxedR1CSProver(0, mats, n_w, 2)
    z = prover.pad_z(to_device(L, 0, o.W), o.u, o.X)
    proof = prover.prove(z, to_device(L, 0, o.E), o.u, challenge)
    ok, rx, ry = osp.verify([rows_of(m) for m in mats], n_w, prover.num_vars, prover.log_rows, o.u, o.X, proof, challenge, p)
    assert ok
    nvb = prover.num_vars.bit_length() - 1
    claims = [(z.data_ptr(), nvb, ry[1:], proof["eval_W"]), (proof["E_padded"].data_ptr(), prover.log_rows, rx, proof["claims"][3])]
    rounds, r, left, w, je, joint = L.spartan.batch_eval_reduce(0, claims, gpu_be_challenge(p))
    assert bo.batch_eval_verify(rounds, [ry[1:], rx], [proof["eval_W"], proof["claims"][3]], left, be_challenge, p) == (r, je, w)
    Wp = ints(o.W) + [0] * (prover.num_vars - n_w)
    Ep = ints(o.E) + [0] * ((1 << prover.log_rows) - prover.rows)
    ji = from_device(L, 0, joint)
    g, beta, ck = kzg_setup(L, len(ji))
    # the commitment the verifier forms, sum_i w_i C_i, has the discrete log sum_i w_i f_i(beta): that of the joint polynomial
    assert kzg.poly_eval(ji, beta, p) == (w[0] * kzg.poly_eval(Wp, beta, p) + w[1] * kzg.poly_eval(Ep, beta, p)) % p
    assert open_and_check(L, ospec, ck, g, beta, joint, ji, r, je)
    assert not open_and_check(L, ospec, ck, g, beta, joint, ji, r, (je + 1) % p)


# ------------------------------------------------------------------------------------------------ SuperNova
def inst_dict(mats, n_w, W, E, u, X):
    rows = len(mats[0][0]) - 1
    return dict(R=[rows_of(m) for m in mats], n_w=n_w, nv=1 << max(1, (max(n_w, 3) - 1).bit_length()), s=max(1, (rows - 1).bit_length()),
                rows=rows, W=ints(W), E=ints(E), u=u, X=list(X))


def gpu_folded_instances(L, oracle):
    """three circuits -- the Lurk step layout (2^13 variables, 2^10 rows), one arity-8 coprocessor slot (2^9, 2^6) and a host-witness
    circuit (2^5, 2^3) -- folded through one SuperNovaFoldContext on a shared key; returns their running instances"""
    FIELD, p = 0, ospec.FIELD_MODULUS[0]
    rng = np.random.default_rng(8)
    ctx0, lay0, mats0, n_w0, rows0, glue0, bases, ck, bi0 = _build(L, oracle, nifs, ospec, rng, frames=1, glue=150, lin_rows=250)
    blk8 = oracle.witness_block(FIELD, 8)
    glue1 = 10
    mats1, n_w1, glue_fn1 = nifs.synthetic_step_circuit(rng, 1, blk8, glue1, 40)
    ctx1 = L.NovaFoldContext(0, ck, n_w1, 2, mats1, depth=2, fmt=L.FMT_CANONICAL)
    b8 = ctx1.add_slot_batch(8, np.zeros(1, dtype=np.uint64))
    ctx1.set_spans([(blk8, glue1, blk8 + glue1, 1)])
    mats2, n_w2, glue_fn2 = nifs.synthetic_step_circuit(rng, 1, 20, 4, 0)
    ctx2 = L.NovaFoldContext(0, ck, n_w2, 2, mats2, depth=2, fmt=L.FMT_CANONICAL)
    ctx2.set_spans([(0, n_w2, n_w2, 1)])
    nivc = L.SuperNovaFoldContext([ctx0, ctx1, ctx2])

    def ro_bytes(X2):
        ro = np.zeros((24, 32), dtype=np.uint8)
        for pos, v in ((0, 5), (4, X2[0]), (5, X2[1])):
            ro[pos] = np.frombuffer(int(v).to_bytes(32, "little"), dtype=np.uint8)
        return ro.reshape(-1)
    for s, ci in enumerate([0, 1, 2, 2, 0, 1, 1, 2, 0]):
        b = nivc._next[ci]
        if ci == 0:
            _fill(ctx0, b, lay0, _step_inputs(oracle, nifs, ospec, lay0, glue0, 30 + s, rng), 5, bi0)
        elif ci == 1:
            pre = random_elements(FIELD, 8, seed=70 + s, shape="lem")
            W = np.zeros(n_w1 * 32, dtype=np.uint8)
            W[:blk8 * 32] = oracle.poseidon_witness_batch(FIELD, 8, pre, nthreads=4)
            gv = glue_fn1(nifs.ints(W), p)
            X2 = [int(rng.integers(1, 2**61)) for _ in range(2)]
            ctx1.host_buffer(b, b8)[:] = pre
            ctx1.host_buffer(b, -1)[:] = nifs.pack([gv[blk8 + g] for g in range(glue1)])
            ctx1.host_buffer(b, -2)[:] = nifs.pack(X2)
            ctx1.host_buffer(b, -3)[:] = ro_bytes(X2)
        else:
            W = [int(x) % p for x in rng.integers(0, 2**62, size=n_w2)]
            for dst, v in glue_fn2(W, p).items():
                W[dst] = v
            X2 = [int(rng.integers(1, 2**61)) for _ in range(2)]
            ctx2.host_buffer(b, -1)[:] = nifs.pack(W)
            ctx2.host_buffer(b, -2)[:] = nifs.pack(X2)
            ctx2.host_buffer(b, -3)[:] = ro_bytes(X2)
        assert nivc.stage_a(ci) == b
        nivc.fold(ci, b)
        nivc.collect(ci, b)
    out = []
    for c, mats, n_w in ((ctx0, mats0, n_w0), (ctx1, mats1, n_w1), (ctx2, mats2, n_w2)):
        run = c.get_running()
        u = nifs.ints(run["u"])[0]
        assert c.check_running() == (0, True, True) and u != 1 and any(run["E"])
        out.append((mats, n_w, inst_dict(mats, n_w, run["W"], run["E"], u, nifs.ints(run["X"]))))
    return out


def oracle_folded_instances(oracle):
    """three circuits (2^11 / 2^7 / 2^3 variables, 2^9 / 2^6 / 2^2 rows) folded by the oracle"""
    out = []
    for k, shape in enumerate([(1, 1000, 100, 200), (1, 100, 20, 10), (1, 6, 2, 0)]):
        mats, n_w, o = folded_instance(oracle, ospec, np.random.default_rng(90 + k), *shape)
        out.append((mats, n_w, inst_dict(mats, n_w, o.W, o.E, o.u, o.X)))
    return out


def prove_on_gpu(L, field, circuits, insts, E_override=None):
    prover = L.spartan.BatchedRelaxedR1CSProver(field, [(mats, n_w, 2) for mats, n_w, _ in circuits])
    dev = []
    for i, I in enumerate(insts):
        E = I["E"] if E_override is None or i not in E_override else E_override[i]
        dev.append((prover.pad_z(i, to_device(L, field, pack(I["W"])), I["u"], I["X"]), to_device(L, field, pack(E)), I["u"]))
    return prover, prover.prove(dev, challenge)


KEYS = ("outer_rounds", "inner_rounds", "claims", "eval_W", "reduce_rounds", "claims_left", "rx", "ry", "r", "weights", "joint_eval")


def check_batched(L, field, circuits, compare_oracle=True):
    p = ospec.FIELD_MODULUS[field]
    insts = [c[2] for c in circuits]
    prover, proof = prove_on_gpu(L, field, circuits, insts)
    joint = from_device(L, field, proof["joint"])
    if compare_oracle:
        want = bo.prove_batched(insts, challenge, p)
        for k in KEYS:
            assert [tuple(c) for c in proof[k]] == [tuple(c) for c in want[k]] if k == "claims" else proof[k] == want[k], k
        assert joint == want["joint"]
    ok, r, je, w = bo.verify_batched(insts, proof, challenge, p)
    assert ok and (r, je, w) == (proof["r"], proof["joint_eval"], proof["weights"])
    assert sc.mle_eval(joint, r, p) == je
    # rejections: a tampered E row, another u, swapped instances, a perturbed L_i
    bad = list(insts[-1]["E"])
    bad[0] = (bad[0] + 1) % p
    assert not bo.verify_batched(insts, prove_on_gpu(L, field, circuits, insts, {len(insts) - 1: bad})[1], challenge, p)[0]
    assert not bo.verify_batched([dict(insts[0], u=(insts[0]["u"] + 1) % p)] + insts[1:], proof, challenge, p)[0]
    if len(insts) > 1:
        assert not bo.verify_batched([insts[1], insts[0]] + insts[2:], proof, challenge, p)[0]
    left = list(proof["claims_left"])
    left[1] = (left[1] + 1) % p
    assert not bo.verify_batched(insts, dict(proof, claims_left=left), challenge, p)[0]
    polys = [I["W"] + [0] * (I["nv"] - I["n_w"]) for I in insts] + [I["E"] + [0] * ((1 << I["s"]) - I["rows"]) for I in insts]
    return proof, joint, polys


def joint_commitment(ck, curve, polys, weights):
    """sum_i w_i C_i from the per-polynomial commitments"""
    pb = ospec.FIELD_MODULUS[ospec.CURVES[curve]["base"]]
    acc = None
    for P, w in zip(polys, weights):
        acc = ospec.ec_add(acc, ospec.ec_mul(w, nifs.point_of(ck.commit(pack(P))), pb), pb)
    return acc


@pytest.mark.parametrize("source", ["gpu_folds", "oracle_folds", "one_instance"])
def test_supernova_compress_hyperkzg(L, oracle, source):
    p = ospec.FIELD_MODULUS[0]
    if source == "gpu_folds":
        circuits = gpu_folded_instances(L, oracle)
    else:
        circuits = oracle_folded_instances(oracle)
        if source == "one_instance":
            circuits = circuits[1:2]
    if len(circuits) == 3:
        nv = [c[2]["nv"] for c in circuits]
        s = [c[2]["s"] for c in circuits]
        assert min(a // b for a, b in zip(nv, nv[1:])) >= 8 and min(s[k] - s[k + 1] for k in range(2)) >= 3
    proof, joint, polys = check_batched(L, 0, circuits)
    g, beta, ck = kzg_setup(L, len(joint))
    assert joint_commitment(ck, 0, polys, proof["weights"]) == nifs.point_of(ck.commit(pack(joint)))
    assert open_and_check(L, ospec, ck, g, beta, proof["joint"], joint, proof["r"], proof["joint_eval"])
    assert not open_and_check(L, ospec, ck, g, beta, proof["joint"], joint, proof["r"], (proof["joint_eval"] + 1) % p)


def test_supernova_compress_pallas_ipa(L, oracle):
    """the Pasta cycle's EE1: the joint polynomial opened with the inner-product argument, b = eq(r); the closing relation
    a' G' + a' b' ck_c = commit(joint) + joint_eval ck_c + sum_j (r_j^2 L_j + r_j^-2 R_j) holds"""
    import torch
    curve = 2
    field, pb = ospec.CURVES[curve]["scalar"], ospec.FIELD_MODULUS[ospec.CURVES[curve]["base"]]
    p = ospec.FIELD_MODULUS[field]
    circuits = []
    for k, (frames, slot, glue, lin) in enumerate([(1, 300, 30, 40), (1, 30, 6, 2), (1, 6, 2, 0)]):
        rng = np.random.default_rng(120 + k)
        mats, n_w, glue_fn = nifs.synthetic_step_circuit(rng, frames, slot, glue, lin)
        bases = oracle.gen_bases(curve, max(n_w, len(mats[0][0]) - 1))
        o = nifs.NovaOracle(curve, bases, mats, n_w, 2, pp_digest=3)
        for step in range(3):
            W = [int(x) % p for x in rng.integers(0, 2**62, size=n_w)]
            for dst, v in glue_fn(W, p).items():
                W[dst] = v
            X2 = [int(rng.integers(1, 2**60)) for _ in range(2)]
            (o.init_running if step == 0 else o.prove_step)(nifs.pack(W), X2)
        assert o.bad_rows() == 0 and o.u != 1 and any(ints(o.E))
        circuits.append((mats, n_w, inst_dict(mats, n_w, o.W, o.E, o.u, o.X)))
    proof, joint, polys = check_batched(L, field, circuits)
    m, r, je = len(proof["r"]), proof["r"], proof["joint_eval"]
    n = 1 << m
    bases = oracle.gen_bases(curve, n + 1, start=5)
    gc = tuple(ints(bases[64 * n:]))
    ck = L.CommitmentKey(curve, bases[:64 * n])
    assert joint_commitment(ck, curve, polys, proof["weights"]) == nifs.point_of(ck.commit(pack(joint)))
    b = torch.empty(n * 32, dtype=torch.uint8, device="cuda")
    L.spartan.eq_evals(field, r, b.data_ptr())
    eq_r = sc.eq_evals(r, p)
    chals = []

    def chal(rnd, msg):
        chals.append(1 + int.from_bytes(hashlib.sha256(bytes([rnd]) + msg).digest()[:16], "little"))
        return chals[-1]
    Ls, Rs, a_fin, b_fin = L.spartan.ipa_prove(curve, ck, gc, proof["joint"].clone().data_ptr(), b.data_ptr(), m, chal)
    add = lambda P, Q: ospec.ec_add(P, Q, pb)
    mul = lambda k, P: ospec.ec_mul(k % p, P, pb)
    acc = add(nifs.point_of(ck.commit(pack(joint))), mul(je, gc))
    for rj, Lj, Rj in zip(chals, Ls, Rs):
        ri = pow(rj, -1, p)
        acc = add(acc, add(mul(rj * rj, Lj), mul(ri * ri, Rj)))
    # the folded key's single base is sum_k s_k G_k with s_k = prod_j (bit j of k from the top ? r_j : r_j^-1); b folds the same way
    s = []
    for k in range(n):
        v = 1
        for j, rj in enumerate(chals):
            v = v * (rj if (k >> (m - 1 - j)) & 1 else pow(rj, -1, p)) % p
        s.append(v)
    assert b_fin == sum(x * y for x, y in zip(s, eq_r)) % p
    G0 = nifs.point_of(oracle.msm(curve, bases[:64 * n], pack(s), nthreads=4))
    assert add(mul(a_fin, G0), mul(a_fin * b_fin, gc)) == acc
