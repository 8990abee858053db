"""The verifier side on the GPU (lurk_spartan_matrix_evals_dev, lurk_spartan_verify, lurk_spartan_verify_batch, lurk_ipa_verify_dev;
csrc/spartan.cu, csrc/ipa.cu): the matrix evaluations bit-exact with oracle/spartan.py: matrices_eval on real and adversarial shapes (and
with the prover's composition eq table -> evaluation table -> inner product at full size); the verifiers accept what the
provers make, write the prover's derived bytes, decide as the oracle verifiers decide in both round encodings and reject every tampered
field, in shapes with 0 to 11 public inputs and with 2^24 + 3 rows; a failing transcript callback is LURK_ERR_ARG from the C entry points;
the IPA verifier accepts lurk_ipa_prove_dev transcripts on all four curves with ck_hat and b_hat equal to the oracle's; a fold chain proved,
opened and verified end to end.  At full size (fib rc = 100, trie_nivc's rc = 400) A, B and C are each compared with the OpenMP port of
matrices_eval (tests/csrc/matrices_eval_cpu.c).  Challenges: the sha256 stand-in of test_gpu_spartan_chain.py."""
import hashlib
import os
import threading

import numpy as np
import pytest

import batched_oracle as bo
import ipa_verify_oracle as iv
from oracle import nifs, spartan as osp, spec as ospec, sumcheck as sc
from test_gpu_spartan_batched import oracle_folded_instances
from test_gpu_spartan_chain import challenge, rows_of, to_device
from test_gpu_spartan_ctx import csr_from_entries, folded, pallas_circuits, z_of
from util import ints, pack, random_elements

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DERIVED = ("rx", "ry", "r", "weights", "joint_eval")


def points(p, k, seed, kind):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return [int.from_bytes(rng.bytes(32), "little") % p for _ in range(k)]
    if kind == "mixed":
        return [[0, 1, p - 1, int.from_bytes(rng.bytes(32), "little") % p][int(rng.integers(0, 4))] for _ in range(k)]
    return [{"zero": 0, "one": 1, "minus-one": p - 1}[kind]] * k


def check_evals(L, field, mats, n_w, n_x, kinds=("random", "zero", "one", "minus-one", "mixed")):
    p = ospec.FIELD_MODULUS[field]
    ctx = L.spartan.SpartanContext(field, mats, n_w, n_x)
    rows_lists = [rows_of(m) for m in mats]
    for t, kind in enumerate(kinds):
        rx, ry = points(p, ctx.log_rows, 10 + t, kind), points(p, ctx.log_vars + 1, 20 + t, kind)
        assert ctx.matrix_evals(rx, ry) == tuple(osp.matrices_eval(rows_lists, n_w, ctx.num_vars, rx, ry, p)), kind
    return ctx


# ------------------------------------------------------------------------------------------------ matrix evaluations
@pytest.mark.parametrize("field", [0, 1, 2, 3])
def test_matrix_evals_real_shape(L, field):
    p = ospec.FIELD_MODULUS[field]
    mats, n_w, _ = nifs.real_shape_step_circuit(np.random.default_rng(40 + field), p, 1, 200, 24, 30)
    check_evals(L, field, mats, n_w, 2)


def test_matrix_evals_adversarial_shapes(L):
    """a row of 2500 non-zeros among empty rows, u / X columns of 70 000 entries, a row count that is not a power of two"""
    field, rng = 0, np.random.default_rng(5)
    n_w, n_x, rows = 3000, 2, 80001
    mats = []
    for m in range(3):
        entries = [(7, int(c)) for c in rng.choice(n_w + 1 + n_x, size=2500, replace=False)] if m == 0 else []
        entries += [(int(r), n_w + (m % 3)) for r in rng.choice(rows, size=70000, replace=False)]     # the u column, then X0, X1
        entries += [(int(rng.integers(0, rows // 2)), int(c)) for c in rng.integers(0, n_w, size=3000)]
        rp, col = csr_from_entries(rows, entries)
        mats.append((rp, col, random_elements(field, len(col), seed=10 + m)))
    check_evals(L, field, mats, n_w, n_x, kinds=("random", "mixed"))


def test_matrix_evals_empty_matrices_no_x_and_two_rows(L):
    rows = 2
    empty = (np.zeros(rows + 1, dtype=np.uint64), np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.uint8))
    ctx = check_evals(L, 1, [empty] * 3, 10, 0)
    assert ctx.log_rows == 1 and ctx.matrix_evals([5], [1, 2, 3, 4, 5]) == (0, 0, 0)
    one = (np.array([0, 1, 1], dtype=np.uint64), np.array([10], dtype=np.uint32), random_elements(3, 1, seed=1))
    check_evals(L, 3, [empty, one, empty], 10, 0)
    rp, col = csr_from_entries(1, [(0, c) for c in range(12)])
    check_evals(L, 2, [(rp, col, random_elements(2, 12, seed=2))] * 3, 11, 0)     # one row, log_rows = 1


def test_matrix_evals_with_four_column_tables(L):
    """n_w = 2^23 + 5: the padded z has 2^25 entries, four 8-bit group tables for the columns (the largest table set of a real shape)"""
    field = 2
    p = ospec.FIELD_MODULUS[field]
    n_w, n_x, rows = (1 << 23) + 5, 3, 300
    rng = np.random.default_rng(9)
    cols = [0, 1, 255, 256, 65535, 65536, (1 << 23) - 1, 1 << 23, n_w - 1, n_w, n_w + 1, n_w + 3] + [int(c) for c in rng.integers(0, n_w + 4, size=200)]
    rp, col = csr_from_entries(rows, [(int(rng.integers(0, rows)), c) for c in cols])
    mats = [(rp, col, random_elements(field, len(col), seed=30 + m)) for m in range(3)]
    ctx = L.spartan.SpartanContext(field, mats, n_w, n_x)
    assert ctx.log_vars + 1 == 25
    rx, ry = points(p, ctx.log_rows, 1, "mixed"), points(p, ctx.log_vars + 1, 2, "random")

    def eq_bits(idx, r):
        l = len(r)
        return bo.eq_at([(idx >> (l - 1 - j)) & 1 for j in range(l)], r, p)
    want = []
    for _, c_, v in mats:
        vals = ints(v)
        total = 0
        for i in range(rows):
            for k in range(int(rp[i]), int(rp[i + 1])):
                total += eq_bits(i, rx) * vals[k] * eq_bits(osp.col_map(int(col[k]), n_w, ctx.num_vars), ry)
        want.append(total % p)
    assert ctx.matrix_evals(rx, ry) == tuple(want)


@pytest.mark.parametrize("rc", [100, 400], ids=["fib-rc100", "trie_nivc-rc400"])
def test_matrix_evals_at_full_size(L, rc):
    """bench.step_circuit at rc = 100 (5.1 M non-zeros, 2^21 rows) and rc = 400 (the trie_nivc Lurk circuit, 20.4 M non-zeros, 2^23 rows):
    A, B and C each bit-exact with the OpenMP port of matrices_eval, and A + r B + r^2 C with the prover's composition
    <eval_table(eq(rx), r), eq(ry)>"""
    import sys
    import torch
    import matrices_eval_cpu as mc
    sys.path.insert(0, ROOT)
    import bench
    field = 0
    p = ospec.FIELD_MODULUS[field]
    mats, n_w, rows, _ = bench.step_circuit(1, rc)
    ctx = L.spartan.SpartanContext(field, mats, n_w, 2)
    rx, ry = points(p, ctx.log_rows, 3, "random"), points(p, ctx.log_vars + 1, 4, "random")
    A, B, Cc = ctx.matrix_evals(rx, ry)
    assert (A, B, Cc) == mc.matrices_eval(p, mats, n_w, ctx.num_vars, rx, ry)
    r = 0x1234567 * 0xfedcba98765 % p
    eq_x = torch.empty((1 << ctx.log_rows) * 32, dtype=torch.uint8, device="cuda")
    eq_y = torch.empty(2 * ctx.num_vars * 32, dtype=torch.uint8, device="cuda")
    tab = torch.empty_like(eq_y)
    L.spartan.eq_evals(field, rx, eq_x.data_ptr())
    L.spartan.eq_evals(field, ry, eq_y.data_ptr())
    ctx.eval_table(eq_x.data_ptr(), r, tab.data_ptr())
    assert (A + r * B + r * r * Cc) % p == L.spartan.inner_product(field, tab.data_ptr(), eq_y.data_ptr(), 2 * ctx.num_vars)


# ------------------------------------------------------------------------------------------------ plain verifier
def compress(rounds, p):
    """evaluations s(0) .. s(d) -> CompressedUniPoly (coefficients without the linear one, constant first), by Lagrange on 0 .. d"""
    out = []
    for ev in rounds:
        d = len(ev) - 1
        coeffs = [0] * (d + 1)
        for i in range(d + 1):
            basis, den = [1], 1                                  # prod_{j != i} (x - j) as a coefficient list
            for j in range(d + 1):
                if j != i:
                    basis = [((basis[k - 1] if k else 0) - j * (basis[k] if k < len(basis) else 0)) % p for k in range(len(basis) + 1)]
                    den = den * (i - j) % p
            f = ev[i] * pow(den, -1, p) % p
            coeffs = [(a + f * b) % p for a, b in zip(coeffs, basis)]
        out.append([coeffs[0]] + coeffs[2:])
    return out


def compressed(proof, p):
    return dict(proof, **{k: compress(proof[k], p) for k in ("outer_rounds", "inner_rounds", "reduce_rounds")})


def oracle_plain(ctx, mats, n_w, u, X, proof, chal, p):
    ok, rx, ry = osp.verify([rows_of(m) for m in mats], n_w, ctx.num_vars, ctx.log_rows, u, X, proof, chal, p)
    if not ok:
        return False
    return bo.batch_eval_verify(proof["reduce_rounds"], [ry[1:], rx], [proof["eval_W"], proof["claims"][3]], proof["claims_left"],
                                lambda rnd, v: chal("batch_eval", (rnd, list(v))), p) is not None


def bumped(proof, key, path, p):
    """the proof with one element (path into the nested lists) changed by + 1"""
    def bump(v, path):
        if not path:
            return (v + 1) % p
        v = list(v)
        v[path[0]] = bump(v[path[0]], path[1:])
        return v
    return dict(proof, **{key: bump(proof[key], path)})


def tampers(proof):
    out = []
    for key in ("outer_rounds", "inner_rounds", "reduce_rounds"):
        for t in range(len(proof[key][0])):
            out.append((key, (len(proof[key]) // 2, t)))
    for k in range(4):
        out.append(("claims", (k,) if not isinstance(proof["claims"][0], (list, tuple)) else (0, k)))
    out.append(("eval_W", () if not isinstance(proof["eval_W"], list) else (0,)))
    for k in range(len(proof["claims_left"])):
        out.append(("claims_left", (k,)))
    return out


def other_challenge(label_to_change):
    def chal(label, data):
        x = challenge(label, data)
        return x + 1 if label == label_to_change else x
    return chal


def failing_at(label_to_fail):
    def chal(label, data):
        if label == label_to_fail:
            raise RuntimeError("transcript failure")
        return challenge(label, data)
    return chal


def raw_verify(L, ctx, proof, u, X, chal):
    """lurk_spartan_verify called directly (the Python wrapper re-raises a callback's exception before it looks at the return code): returns the
    status and checks that a failed call did not report an acceptance"""
    import ctypes as C
    E = L._capi
    fes = L.spartan._fes
    bufs = {k: fes(x for rnd in proof[k] for x in rnd) for k in ("outer_rounds", "inner_rounds", "reduce_rounds")}
    bufs.update(claims=fes(proof["claims"]), eval_W=fes([proof["eval_W"]]), claims_left=fes(proof["claims_left"]))
    rec = E.SpartanProof(**{k: b.ctypes.data for k, b in bufs.items()})
    acc = C.c_int(7)
    cb = L.spartan._spartan_callback(chal, ctx.p, 1, False, [])
    rc = E.lib().lurk_spartan_verify(ctx._ctx, E.np_ptr(fes([u])), E.np_ptr(fes(X)), C.byref(rec), E.SPARTAN_ROUNDS_EVALS, cb, None, C.byref(acc),
                                     E.FMT_CANONICAL, None)
    assert acc.value == (1 if rc == E.OK else 0)
    return rc


@pytest.mark.parametrize("field", [0, 1, 2, 3])
def test_plain_verifier_accepts_decides_as_the_oracle_and_rejects_tampering(L, oracle, field):
    p = ospec.FIELD_MODULUS[field]
    mats, n_w, o = folded(oracle, field, 300 + field)
    ctx = L.spartan.SpartanContext(field, mats, n_w, 2)
    dz, dE = z_of(L, field, o.W, o.u, o.X), to_device(L, field, o.E)
    got = ctx.prove(dz.data_ptr(), dE.data_ptr(), challenge)
    ok, d = ctx.verify(got, o.u, o.X, challenge)
    assert ok and all(d[k] == got[k] for k in DERIVED)
    assert ctx.verify(compressed(got, p), o.u, o.X, challenge, compressed=True) == (True, d)
    assert oracle_plain(ctx, mats, n_w, o.u, o.X, got, challenge, p)
    for key, path in tampers(got):
        bad = bumped(got, key, path, p)
        assert not ctx.verify(bad, o.u, o.X, challenge)[0], (key, path)
        assert not oracle_plain(ctx, mats, n_w, o.u, o.X, bad, challenge, p), (key, path)
        if key.endswith("_rounds"):
            assert not ctx.verify(bumped(compressed(got, p), key, (path[0], min(path[1], len(compressed(got, p)[key][0]) - 1)), p), o.u, o.X,
                                  challenge, compressed=True)[0], (key, path)
    X2 = [o.X[0], (o.X[1] + 1) % p]
    for u, X in (((o.u + 1) % p, o.X), (o.u, X2)):
        assert not ctx.verify(got, u, X, challenge)[0] and not oracle_plain(ctx, mats, n_w, u, X, got, challenge, p)
    for label in ("tau", "outer", "inner_r", "inner", "batch_eval"):
        assert not ctx.verify(got, o.u, o.X, other_challenge(label))[0], label
        assert not oracle_plain(ctx, mats, n_w, o.u, o.X, got, other_challenge(label), p), label
    # a callback that fails is an error (LURK_ERR_ARG from the C entry point, not a rejection), a value >= p is out of range
    for label in ("tau", "inner", "batch_eval"):
        assert raw_verify(L, ctx, got, o.u, o.X, failing_at(label)) == L._capi.ERR_ARG, label
    assert raw_verify(L, ctx, got, o.u, o.X, challenge) == L._capi.OK
    with pytest.raises(L.LurkError) as e:
        ctx.verify(got, o.u + p, o.X, challenge)
    assert e.value.code == L._capi.ERR_RANGE


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_verifier_on_fold_context_proofs(L, oracle, curve):
    """a NovaFoldContext chain proved from LURK_FOLD_BUF_Z1 / _E1 and verified; the joint opening checked with lurk_ipa_verify_dev (Grumpkin,
    Pallas, Vesta) or oracle/kzg.py's verify_known_beta (BN254); the same chain with a tampered E is rejected"""
    import torch
    from test_gpu_spartan_batched import kzg_setup
    from test_gpu_spartan_chain import open_and_check
    field = ospec.CURVES[curve]["scalar"]
    p, pb = ospec.FIELD_MODULUS[field], ospec.FIELD_MODULUS[ospec.CURVES[curve]["base"]]
    rng = np.random.default_rng(700 + curve)
    mats, n_w, glue_fn = nifs.real_shape_step_circuit(rng, p, 1, 150, 20, 30)
    rows = len(mats[0][0]) - 1
    bases = oracle.gen_bases(curve, max(n_w, rows))
    key = L.CommitmentKey(curve, bases)
    fctx = L.NovaFoldContext(curve, key, n_w, 2, mats, depth=1, fmt=L.FMT_CANONICAL)
    fctx.set_spans([(0, n_w, n_w, 1)])
    o = nifs.NovaOracle(curve, bases, mats, n_w, 2, nthreads=4, pp_digest=5)
    for step in range(3):
        W = ints(random_elements(field, n_w, seed=40 * curve + step, shape="edge"))
        X = ints(random_elements(field, 2, seed=40 * curve + step + 20, shape="edge"))
        for dst, v in glue_fn(W, X).items():
            W[dst] = v
        fctx.host_buffer(0, -1)[:] = pack(W)
        fctx.host_buffer(0, -2)[:] = pack(X)
        fctx.host_buffer(0, -3)[:] = pack([int(c) % pb for c in o.ro_consts(X)] + [0] * (24 - len(o.ro_consts(X))))
        fctx.stage_a(0)
        (fctx.init_running if step == 0 else fctx.stage_b_launch)(0)
        fctx.collect(0)
        o.init_running(pack(W), X) if step == 0 else o.prove_step(pack(W), X)
    dz, _ = fctx.device_buffer(0, L._capi.FOLD_BUF_Z1)
    de, _ = fctx.device_buffer(0, L._capi.FOLD_BUF_E1)
    run = fctx.get_running()
    u, X = ints(run["u"])[0], ints(run["X"])
    ctx = L.spartan.SpartanContext(field, mats, n_w, 2)
    got = ctx.prove(dz, de, challenge)
    ok, d = ctx.verify(got, u, X, challenge)
    assert ok and all(d[k] == got[k] for k in DERIVED)
    m = len(got["r"])
    n = 1 << m
    if curve == 0:
        from test_gpu_sumcheck import from_device
        g, beta, ck = kzg_setup(L, n)
        joint = from_device(L, field, got["joint"])
        assert open_and_check(L, ospec, ck, g, beta, got["joint"], joint, got["r"], got["joint_eval"])
    else:
        # the joint commitment from the running instance's commitments, the opening under a key of 2^m bases
        kb = oracle.gen_bases(curve, n + 1, start=5)
        ck, gc = L.CommitmentKey(curve, kb[:64 * n]), tuple(ints(kb[64 * n:]))
        padW = pack(ints(run["W"]) + [0] * (n - n_w))
        padE = pack(ints(run["E"]) + [0] * (n - rows))
        cW, cE = nifs.point_of(ck.commit(padW)), nifs.point_of(ck.commit(padE))
        add = lambda P, Q: ospec.ec_add(P, Q, pb)
        comm = add(ospec.ec_mul(got["weights"][0], cW, pb), ospec.ec_mul(got["weights"][1], cE, pb))
        b = torch.empty(n * 32, dtype=torch.uint8, device="cuda")
        L.spartan.eq_evals(field, got["r"], b.data_ptr())
        chal = lambda rnd, msg: 1 + int.from_bytes(hashlib.sha256(bytes([rnd]) + msg).digest()[:16], "little")
        work, bw = got["joint"].clone(), b.clone()           # consumed by the prover
        Ls, Rs, a_fin, _ = L.spartan.ipa_prove(curve, ck, gc, work.data_ptr(), bw.data_ptr(), m, chal)
        assert L.spartan.ipa_verify(curve, ck, gc, comm, got["joint_eval"], b.data_ptr(), m, Ls, Rs, a_fin, chal)[0]
        assert not L.spartan.ipa_verify(curve, ck, gc, comm, (got["joint_eval"] + 1) % p, b.data_ptr(), m, Ls, Rs, a_fin, chal)[0]
    bad = run["E"].copy()
    bad[0] ^= 1
    dbad = to_device(L, field, bad)
    tampered = ctx.prove(dz, dbad.data_ptr(), challenge)
    assert not ctx.verify(tampered, u, X, challenge)[0]


# ------------------------------------------------------------------------------------------------ batched verifier
@pytest.mark.parametrize("field", [0, 2])
def test_batched_verifier(L, oracle, field):
    p = ospec.FIELD_MODULUS[field]
    circuits = oracle_folded_instances(oracle) if field == 0 else pallas_circuits(oracle)
    insts = [c[2] for c in circuits]
    ctxs = [L.spartan.SpartanContext(field, mats, n_w, 2) for mats, n_w, _ in circuits]
    dev = [(z_of(L, field, pack(I["W"]), I["u"], I["X"]), to_device(L, field, pack(I["E"]))) for I in insts]
    got = L.spartan.spartan_prove_batch(ctxs, [(a.data_ptr(), b.data_ptr()) for a, b in dev], challenge)
    pub = [(I["u"], I["X"]) for I in insts]
    ok, d = L.spartan.spartan_verify_batch(ctxs, pub, got, challenge)
    assert ok and all(d[k] == got[k] for k in DERIVED)
    assert L.spartan.spartan_verify_batch(ctxs, pub, compressed(got, p), challenge, compressed=True) == (True, d)
    assert bo.verify_batched(insts, got, challenge, p)[0]
    for key, path in tampers(got):
        bad = bumped(got, key, path, p)
        assert not L.spartan.spartan_verify_batch(ctxs, pub, bad, challenge)[0], (key, path)
        assert not bo.verify_batched(insts, bad, challenge, p)[0], (key, path)
    order = [1, 0] + list(range(2, len(ctxs)))
    assert not L.spartan.spartan_verify_batch([ctxs[i] for i in order], [pub[i] for i in order], got, challenge)[0]
    assert not bo.verify_batched([insts[i] for i in order], got, challenge, p)[0]
    wrong_u = [((pub[0][0] + 1) % p, pub[0][1])] + pub[1:]
    assert not L.spartan.spartan_verify_batch(ctxs, wrong_u, got, challenge)[0]
    wrong_x = pub[:-1] + [(pub[-1][0], [(pub[-1][1][0] + 1) % p] + list(pub[-1][1][1:]))]
    assert not L.spartan.spartan_verify_batch(ctxs, wrong_x, got, challenge)[0]
    assert not L.spartan.spartan_verify_batch(ctxs, pub, got, other_challenge("outer_r"))[0]


# ------------------------------------------------------------------------------------------------ IPA verifier
def ipa_chal(rnd, msg):
    return 1 + int.from_bytes(hashlib.sha256(bytes([rnd]) + msg).digest()[:16], "little")


@pytest.mark.parametrize("log_n", [1, 2, 5, 10, 16])
@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_ipa_verifier(L, oracle, curve, log_n):
    import torch
    Cv = ospec.CURVES[curve]
    field, pb, q = Cv["scalar"], ospec.FIELD_MODULUS[Cv["base"]], ospec.FIELD_MODULUS[Cv["scalar"]]
    n = 1 << log_n
    a_h, b_h = random_elements(field, n, seed=3 + log_n), random_elements(field, n, seed=4 + log_n, shape="edge")
    a, b = ints(a_h), ints(b_h)
    bases = oracle.gen_bases(curve, n + 1, start=5)
    gc = tuple(ints(bases[64 * n:]))
    ck = L.CommitmentKey(curve, bases[:64 * n])
    comm, c = nifs.point_of(ck.commit(a_h)), sc.inner_product(a, b, q)
    db = to_device(L, field, b_h)
    keep = db.clone()
    def prove():
        da, dbw = to_device(L, field, a_h), to_device(L, field, b_h)       # consumed by the prover; kept alive until it returns
        return L.spartan.ipa_prove(curve, ck, gc, da.data_ptr(), dbw.data_ptr(), log_n, ipa_chal)
    Ls, Rs, a_fin, b_fin = prove()
    ok, ck_hat, b_hat = L.spartan.ipa_verify(curve, ck, gc, comm, c, db.data_ptr(), log_n, Ls, Rs, a_fin, ipa_chal)
    torch.cuda.synchronize()
    assert torch.equal(db, keep), "b was modified"
    msm = lambda G, s: nifs.point_of(oracle.msm(curve, bases[:64 * n], pack(s), nthreads=4))
    want = iv.ipa_verify(curve, None, gc, comm, c, b, Ls, Rs, a_fin, ipa_chal, msm)
    assert ok and want[0] and (ck_hat, b_hat) == (want[1], want[2])
    # the key context is not consumed: a proof after a verify is unchanged
    assert b_hat == b_fin
    assert prove() == (Ls, Rs, a_fin, b_fin)
    if log_n == 5:
        other = ospec.ec_add(gc, gc, pb)
        cases = [([other] + Ls[1:], Rs, a_fin, c, comm), (Ls, Rs[:-1] + [other], a_fin, c, comm), (Ls, Rs, (a_fin + 1) % q, c, comm),
                 (Ls, Rs, a_fin, (c + 1) % q, comm), (Ls, Rs, a_fin, c, other)]
        for Lx, Rx, ax, cx, comx in cases:
            assert not L.spartan.ipa_verify(curve, ck, gc, comx, cx, db.data_ptr(), log_n, Lx, Rx, ax, ipa_chal)[0]
            assert not iv.ipa_verify(curve, None, gc, comx, cx, b, Lx, Rx, ax, ipa_chal, msm)[0]
        with pytest.raises(L.LurkError) as e:                   # a point off the curve
            L.spartan.ipa_verify(curve, ck, gc, (comm[0], (comm[1] + 1) % pb), c, db.data_ptr(), log_n, Ls, Rs, a_fin, ipa_chal)
        assert e.value.code == L._capi.ERR_RANGE


# ------------------------------------------------------------------------------------------------ concurrency
def test_primary_and_secondary_verifies_at_once(L, oracle):
    """a BN254 and a Grumpkin verify from two host threads on two streams decide and derive what they do one after the other"""
    import torch
    jobs = []
    for field, seed in ((0, 11), (1, 12)):
        mats, n_w, o = folded(oracle, field, seed, free=400, glue=40, lin_rows=60)
        ctx = L.spartan.SpartanContext(field, mats, n_w, 2)
        dz, dE = z_of(L, field, o.W, o.u, o.X), to_device(L, field, o.E)
        proof = ctx.prove(dz.data_ptr(), dE.data_ptr(), challenge)
        jobs.append((ctx, proof, o.u, o.X))
    seq = [ctx.verify(pr, u, X, challenge) for ctx, pr, u, X in jobs]
    assert all(ok for ok, _ in seq)
    results, errors = [None, None], []

    def run(i):
        try:
            ctx, pr, u, X = jobs[i]
            s = torch.cuda.Stream()
            for _ in range(3):
                results[i] = ctx.verify(pr, u, X, challenge, stream=s.cuda_stream)
            s.synchronize()
        except Exception as ex:        # reported below
            errors.append(ex)
    threads = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    assert results == seq


# ------------------------------------------------------------------------------------------------ public inputs of every length, four row tables
def relaxed_instance(field, rows, n_w, n_x, per_matrix, seed):
    """a satisfied relaxed R1CS instance of random shape: random (W, u, X), E = Az o Bz - u Cz (computed over the rows that have entries);
    the matrices touch the u column and every X column"""
    p = ospec.FIELD_MODULUS[field]
    rng = np.random.default_rng(seed)
    nz = n_w + 1 + n_x
    mats, sparse = [], []
    for m in range(3):
        cols = [int(c) for c in rng.integers(0, nz, size=per_matrix)] + list(range(n_w, nz))
        entries = [(int(rng.integers(0, rows)), c) for c in cols] + ([(rows - 1, 0)] if m == 0 else [])
        rp, col = csr_from_entries(rows, entries)
        val = random_elements(field, len(col), seed=seed + m)
        mats.append((rp, col, val))
        vals, row_of = ints(val), np.repeat(np.arange(rows), np.diff(rp.astype(np.int64)))
        M = {}
        for k in range(len(col)):
            M.setdefault(int(row_of[k]), []).append((int(col[k]), vals[k]))
        sparse.append(M)
    W = ints(random_elements(field, n_w, seed=seed + 5))
    u = int.from_bytes(np.random.default_rng(seed + 6).bytes(32), "little") % p
    X = ints(random_elements(field, n_x, seed=seed + 7)) if n_x else []
    z = W + [u] + X
    E = np.zeros((rows, 32), dtype=np.uint8)
    for i in sorted(set().union(*sparse)):
        az, bz, cz = (sum(v * z[c] for c, v in M.get(i, [])) % p for M in sparse)
        E[i] = np.frombuffer(((az * bz - u * cz) % p).to_bytes(32, "little"), dtype=np.uint8)
    return mats, pack(W), E.reshape(-1), u, X


@pytest.mark.parametrize("n_x", [0, 1, 4, 11])
def test_plain_verifier_with_public_inputs_of_every_length(L, n_x):
    """eval_X over (u, X) of 1, 2, 5 and 12 entries: accepted, the oracle agrees, and a changed X (or u) is rejected by both"""
    field = 1
    p = ospec.FIELD_MODULUS[field]
    n_w = 37
    mats, Wb, Eb, u, X = relaxed_instance(field, 53, n_w, n_x, 120, 500 + n_x)
    ctx = L.spartan.SpartanContext(field, mats, n_w, n_x)
    dz, dE = z_of(L, field, Wb, u, X), to_device(L, field, Eb)
    got = ctx.prove(dz.data_ptr(), dE.data_ptr(), challenge)
    ok, d = ctx.verify(got, u, X, challenge)
    assert ok and all(d[k] == got[k] for k in DERIVED)
    assert oracle_plain(ctx, mats, n_w, u, X, got, challenge, p)
    for k in range(n_x):
        X2 = list(X)
        X2[k] = (X2[k] + 1) % p
        assert not ctx.verify(got, u, X2, challenge)[0] and not oracle_plain(ctx, mats, n_w, u, X2, got, challenge, p), k
    assert not ctx.verify(got, (u + 1) % p, X, challenge)[0]


def test_plain_verifier_with_four_row_tables(L):
    """2^24 + 3 constraints: log_rows = 25, four 8-bit group tables for eq(r_x); an honest proof is accepted, a changed E row rejected"""
    field = 0
    rows, n_w, n_x = (1 << 24) + 3, 300, 2
    mats, Wb, Eb, u, X = relaxed_instance(field, rows, n_w, n_x, 400, 77)
    ctx = L.spartan.SpartanContext(field, mats, n_w, n_x)
    assert ctx.log_rows == 25
    dz, dE = z_of(L, field, Wb, u, X), to_device(L, field, Eb)
    got = ctx.prove(dz.data_ptr(), dE.data_ptr(), challenge)
    ok, d = ctx.verify(got, u, X, challenge)
    assert ok and all(d[k] == got[k] for k in DERIVED)
    bad = Eb.copy()
    bad[32 * (rows - 1)] ^= 1                      # the last row (it has an entry of A): its index sets bits of the top table
    dbad = to_device(L, field, bad)
    assert not ctx.verify(ctx.prove(dz.data_ptr(), dbad.data_ptr(), challenge), u, X, challenge)[0]


def test_ipa_verifier_callback_failure_is_an_error(L, oracle):
    """lurk_ipa_verify_dev called directly: a transcript callback that fails in any round gives LURK_ERR_ARG, not a rejection"""
    import ctypes as C
    curve, log_n = 2, 4
    field = ospec.CURVES[curve]["scalar"]
    n = 1 << log_n
    a_h, b_h = random_elements(field, n, seed=1), random_elements(field, n, seed=2)
    bases = oracle.gen_bases(curve, n + 1, start=5)
    gc = tuple(ints(bases[64 * n:]))
    ck = L.CommitmentKey(curve, bases[:64 * n])
    comm, c = nifs.point_of(ck.commit(a_h)), sc.inner_product(ints(a_h), ints(b_h), ospec.FIELD_MODULUS[field])
    da, dbw, db = to_device(L, field, a_h), to_device(L, field, b_h), to_device(L, field, b_h)
    Ls, Rs, a_fin, _ = L.spartan.ipa_prove(curve, ck, gc, da.data_ptr(), dbw.data_ptr(), log_n, ipa_chal)
    E, fes, pb = L._capi, L.spartan._fes, L.spartan._point_bytes
    Lb, Rb = np.concatenate([pb(P) for P in Ls]), np.concatenate([pb(P) for P in Rs])

    def run(chal):
        acc = C.c_int(7)
        rc = E.lib().lurk_ipa_verify_dev(curve, ck._ctx, E.np_ptr(fes(gc)), E.np_ptr(pb(comm)), E.np_ptr(fes([c])), C.c_void_p(db.data_ptr()), log_n,
                                         E.np_ptr(Lb), E.np_ptr(Rb), E.np_ptr(fes([a_fin])), L.spartan._callback(chal, []), None, C.byref(acc), None,
                                         None, E.FMT_CANONICAL, None)
        assert acc.value == (1 if rc == E.OK else 0)
        return rc
    assert run(ipa_chal) == E.OK
    for bad_round in (0, log_n - 1):
        def chal(rnd, msg, bad_round=bad_round):
            if rnd == bad_round:
                raise RuntimeError("transcript failure")
            return ipa_chal(rnd, msg)
        assert run(chal) == E.ERR_ARG, bad_round
