"""The compress context (lurk_compress_ctx_*, lurk_compress_prove_dev; csrc/compress.cu) on the GPU: CompressedSNARK::prove in one call,
bit-exact with the composition it replaces -- SpartanContext.prove (or spartan_prove_batch), the joint commitment sum_i w_i C_i, then
hyperkzg_prove or ipa_prove under the same transcript -- from the running instances of two fold contexts (the secondary's last fold
included), accepted by the oracle verifiers, with HyperKZG's algebra checked under a key of known beta and the inner-product argument's
closing relation checked on the returned L, R, a_final, b_final.  Also: concurrent and sequential calls agree, a context carries nothing
from one proof to the next, a fold step on a shared key between two proofs changes nothing, and the errors and refusals.
Challenges: the sha256 stand-in of test_gpu_spartan_chain.py for Keccak256Transcript, one transcript per circuit."""
import os
import subprocess

import numpy as np
import pytest

import batched_oracle as bo
from oracle import nifs, spartan as osp, spec as ospec, sumcheck as sc
from test_gpu_spartan_batched import inst_dict, kzg_setup
from test_gpu_spartan_chain import challenge, folded_instance, open_and_check, rows_of, to_device
from test_gpu_spartan_ctx import z_of
from test_gpu_sumcheck import from_device
from util import ints, pack, random_elements

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def chal_of(k):
    """the transcript of circuit k (0 primary, 1 secondary)"""
    return challenge if k == 0 else (lambda label, data: challenge(("secondary", label), data))


def cchal(k, label, data):
    return chal_of(k)(label, data)


def point96(P):
    return pack([0, 0, 0]) if P is None else pack([P[0], P[1], 1])


def fold_chain(L, oracle, curve, steps, seed, free=150, glue=20, lin_rows=30):
    """a NovaFoldContext on nifs.real_shape_step_circuit after `steps` GPU folds, checked step by step against nifs.NovaOracle; the key
    (also the IPA key of the opening) has joint_len bases"""
    field = ospec.CURVES[curve]["scalar"]
    p, pb = ospec.FIELD_MODULUS[field], ospec.FIELD_MODULUS[ospec.CURVES[curve]["base"]]
    rng = np.random.default_rng(seed)
    mats, n_w, glue_fn = nifs.real_shape_step_circuit(rng, p, 1, free, glue, lin_rows)
    rows = len(mats[0][0]) - 1
    n_key = 1 << max((rows - 1).bit_length(), (max(n_w, 3) - 1).bit_length())
    bases = oracle.gen_bases(curve, n_key)
    ck = L.CommitmentKey(curve, bases)
    fctx = L.NovaFoldContext(curve, ck, n_w, 2, mats, depth=1, fmt=L.FMT_CANONICAL)
    fctx.set_spans([(0, n_w, n_w, 1)])
    o = nifs.NovaOracle(curve, bases, mats, n_w, 2, nthreads=4, pp_digest=5)
    c = dict(curve=curve, field=field, p=p, mats=mats, n_w=n_w, rows=rows, bases=bases, ck=ck, fctx=fctx, o=o, glue_fn=glue_fn, pb=pb, step=0, seed=seed)
    for _ in range(steps):
        fold_step(L, c)
    return c


def fold_step(L, c):
    """one step through the fold context, its record checked against the oracle's NIFS::prove"""
    fctx, o, field, step = c["fctx"], c["o"], c["field"], c["step"]
    W = ints(random_elements(field, c["n_w"], seed=40 * c["seed"] + step, shape="edge"))
    X = ints(random_elements(field, 2, seed=40 * c["seed"] + step + 20, shape="edge"))
    for dst, v in c["glue_fn"](W, X).items():
        W[dst] = v
    fctx.host_buffer(0, -1)[:] = pack(W)
    fctx.host_buffer(0, -2)[:] = pack(X)
    fctx.host_buffer(0, -3)[:] = pack([int(v) % c["pb"] for v in o.ro_consts(X)] + [0] * (24 - len(o.ro_consts(X))))
    fctx.stage_a(0)
    (fctx.init_running if step == 0 else fctx.stage_b_launch)(0)
    rec = fctx.collect(0)
    want = o.init_running(pack(W), X) if step == 0 else o.prove_step(pack(W), X)
    if step:
        assert nifs.point_of(rec.comm_T) == want["comm_T"]
    assert nifs.point_of(rec.running_comm_W) == o.comm_W and nifs.point_of(rec.running_comm_E) == o.comm_E
    c["rec"], c["step"] = rec, step + 1
    return rec


def running(L, c):
    """(d_z, d_E, comm_W, comm_E) of the fold context's running instance, straight from LURK_FOLD_BUF_Z1 / E1"""
    dz, _ = c["fctx"].device_buffer(0, L._capi.FOLD_BUF_Z1)
    de, _ = c["fctx"].device_buffer(0, L._capi.FOLD_BUF_E1)
    return dz, de, nifs.point_of(c["rec"].running_comm_W), nifs.point_of(c["rec"].running_comm_E)


def snapshot(L, c):
    import torch
    c["fctx"].sync()
    out = []
    for which in (L._capi.FOLD_BUF_Z1, L._capi.FOLD_BUF_E1):
        ptr, n = c["fctx"].device_buffer(0, which)
        out.append(L.fold.device_tensor(ptr, n).clone())
    torch.cuda.synchronize()
    return out


def joint_comm(curve, comms, weights):
    pb = ospec.FIELD_MODULUS[ospec.CURVES[curve]["base"]]
    acc = None
    for C_, w in zip(comms, weights):
        acc = ospec.ec_add(acc, ospec.ec_mul(w, C_, pb), pb)
    return acc


def composition(L, k, curve, ctxs, insts, pcs, batched):
    """today's composition for circuit k: SpartanContext.prove / spartan_prove_batch, sum_i w_i C_i on the host, then the opening under the
    same transcript.  insts: [(d_z, d_E, comm_W, comm_E)]."""
    import torch
    chal = chal_of(k)
    field = ospec.CURVES[curve]["scalar"]
    p, pb = ospec.FIELD_MODULUS[field], ospec.FIELD_MODULUS[ospec.CURVES[curve]["base"]]
    if batched:
        got = L.spartan.spartan_prove_batch(ctxs, [(z, e) for z, e, _, _ in insts], chal)
    else:
        got = ctxs[0].prove(insts[0][0], insts[0][1], chal)
    got["comm"] = joint_comm(curve, [x[2] for x in insts] + [x[3] for x in insts], got["weights"])
    r, m = got["r"], len(got["r"])
    if pcs[0] == "hyperkzg":
        got["com"], got["v"], got["w"] = L.spartan.hyperkzg_prove(curve, pcs[1], got["joint"].data_ptr(), r, lambda rnd, msg: chal("pcs", (rnd, bytes(msg))) % p)
    else:
        scale = chal("pcs", (0, point96(got["comm"]).tobytes() + int(got["joint_eval"]).to_bytes(32, "little"))) % p
        gc = ospec.ec_mul(scale, pcs[2], pb)
        b = torch.empty((1 << m) * 32, dtype=torch.uint8, device="cuda")
        L.spartan.eq_evals(field, r, b.data_ptr())
        got["L"], got["R"], got["a_final"], got["b_final"] = L.spartan.ipa_prove(curve, pcs[1], gc, got["joint"].clone().data_ptr(), b.data_ptr(), m,
                                                                                 lambda rnd, msg: chal("pcs", (rnd + 1, bytes(msg))) % p)
        got["gc"] = gc
    return got


PROOF_KEYS = ("outer_rounds", "inner_rounds", "claims", "eval_W", "rx", "ry", "reduce_rounds", "r", "claims_left", "weights", "joint_eval", "comm")
OPEN_KEYS = {"hyperkzg": ("com", "v", "w"), "ipa": ("L", "R", "a_final", "b_final")}


def same(a, b, kind):
    return all(a[k] == b[k] for k in PROOF_KEYS + OPEN_KEYS[kind])


def ipa_relation(oracle, k, curve, bases, ck_c, proof):
    """the inner-product argument's closing relation on the returned L, R, a_final, b_final: a' G' + a' b' ck_c' = comm + joint_eval ck_c' +
    sum_j (r_j^2 L_j + r_j^-2 R_j), with ck_c' = (the round-0 challenge) ck_c, G' = sum_i s_i G_i and b' = <s, eq(r)>"""
    field = ospec.CURVES[curve]["scalar"]
    p, pb = ospec.FIELD_MODULUS[field], ospec.FIELD_MODULUS[ospec.CURVES[curve]["base"]]
    chal = chal_of(k)
    scale = chal("pcs", (0, point96(proof["comm"]).tobytes() + int(proof["joint_eval"]).to_bytes(32, "little"))) % p
    gc = ospec.ec_mul(scale, ck_c, pb)
    r, m = proof["r"], len(proof["r"])
    add = lambda P, Q: ospec.ec_add(P, Q, pb)
    mul = lambda s, P: ospec.ec_mul(s % p, P, pb)
    acc = add(proof["comm"], mul(proof["joint_eval"], gc))
    chals = []
    for j, (Lj, Rj) in enumerate(zip(proof["L"], proof["R"])):
        rj = chal("pcs", (j + 1, point96(Lj).tobytes() + point96(Rj).tobytes())) % p
        chals.append(rj)
        acc = add(acc, add(mul(rj * rj, Lj), mul(pow(rj, -2, p), Rj)))
    s = []
    for i in range(1 << m):
        v = 1
        for j, rj in enumerate(chals):
            v = v * (rj if (i >> (m - 1 - j)) & 1 else pow(rj, -1, p)) % p
        s.append(v)
    if proof["b_final"] != sum(x * y for x, y in zip(s, sc.eq_evals(r, p))) % p:
        return False
    G0 = nifs.point_of(oracle.msm(curve, bases[:64 << m], pack(s), nthreads=4))
    a = proof["a_final"]
    return add(mul(a, G0), mul(a * proof["b_final"], gc)) == acc


def pcs_of(L, oracle, c, kind):
    if kind == "hyperkzg":
        g, beta, ck = kzg_setup(L, c["ctx"].joint_len)
        return ("hyperkzg", ck), (g, beta)
    gc = tuple(ints(oracle.gen_bases(c["curve"], 1, start=len(c["bases"]) // 64 + 7)))
    return ("ipa", c["ck"], gc), None


def check_circuit(L, oracle, k, c, got, want, kind, extra, tampered=False):
    """the compress proof of circuit k equals the composition's, the oracle verifiers accept it, the opening checks out"""
    assert same(got, want, kind), [key for key in PROOF_KEYS + OPEN_KEYS[kind] if got[key] != want[key]]
    p = c["p"]
    run = c["fctx"].get_running()
    u, X = ints(run["u"])[0], ints(run["X"])
    ok, rx, ry = osp.verify([rows_of(m) for m in c["mats"]], c["n_w"], c["ctx"].num_vars, c["ctx"].log_rows, u, X, got, chal_of(k), p)
    assert ok
    assert bo.batch_eval_verify(got["reduce_rounds"], [ry[1:], rx], [got["eval_W"], got["claims"][3]], got["claims_left"],
                                lambda rnd, v: chal_of(k)("batch_eval", (rnd, list(v))), p) == (got["r"], got["joint_eval"], got["weights"])
    joint = from_device(L, c["field"], want["joint"])
    assert got["comm"] == nifs.point_of(c["ck"].commit(pack(joint)))          # sum_i w_i C_i = commit(joint) under the fold key
    if kind == "hyperkzg":
        g, beta = extra
        ck = kzg_setup(L, len(joint))[2]
        assert open_and_check(L, ospec, ck, g, beta, want["joint"], joint, got["r"], got["joint_eval"])
    else:
        assert ipa_relation(oracle, k, c["curve"], c["bases"], c["pcs"][2], got)


_CACHE = {}


def nova_setup(L, oracle, curves, kinds):
    """primary and secondary fold chains of 3 steps each, then the secondary's final fold (l_u_secondary into r_U_secondary)"""
    key = (curves, kinds)
    if key not in _CACHE:
        cs = []
        for k, (curve, kind) in enumerate(zip(curves, kinds)):
            c = fold_chain(L, oracle, curve, 3, seed=11 + 7 * curve)
            if k == 1:
                fold_step(L, c)             # the secondary's last fold: its record carries comm_T, checked against NovaOracle
            assert c["fctx"].check_running() == (0, True, True)
            run = c["fctx"].get_running()
            assert np.array_equal(run["W"], c["o"].W) and np.array_equal(run["E"], c["o"].E) and ints(run["u"])[0] == c["o"].u
            c["ctx"] = L.spartan.SpartanContext(c["field"], c["mats"], c["n_w"], 2)
            c["pcs"], c["extra"] = pcs_of(L, oracle, c, kind)
            cs.append(c)
        _CACHE[key] = cs
    return _CACHE[key]


@pytest.mark.parametrize("curves,kinds", [((0, 1), ("hyperkzg", "ipa")), ((2, 3), ("ipa", "ipa"))], ids=["bn254-grumpkin", "pallas-vesta"])
def test_nova_compress_from_the_fold_contexts(L, oracle, curves, kinds):
    cs = nova_setup(L, oracle, curves, kinds)
    cctx = L.CompressContext(cs[0]["ctx"], cs[1]["ctx"], cs[0]["pcs"], cs[1]["pcs"])
    assert cctx.info()["device_bytes"] == 0
    insts = [running(L, c) for c in cs]
    keep = [snapshot(L, c) for c in cs]
    got = cctx.prove([insts[0]], insts[1], cchal)
    for c, before in zip(cs, keep):
        assert all(a.equal(b) for a, b in zip(snapshot(L, c), before)), "a fold context's buffers were modified"
    assert cctx.info()["device_bytes"] > 0
    for k, c in enumerate(cs):
        want = composition(L, k, c["curve"], [c["ctx"]], [insts[k]], c["pcs"], batched=False)
        check_circuit(L, oracle, k, c, got[k], want, kinds[k], c["extra"])
    # the sequential call gives the same bytes
    seq = cctx.prove([insts[0]], insts[1], cchal, sequential=True)
    assert all(same(a, b, kind) for a, b, kind in zip(got, seq, kinds))


def test_nova_compress_rejects_a_tampered_E_and_survives_a_failing_callback(L, oracle):
    import torch
    kinds = ("hyperkzg", "ipa")
    cs = nova_setup(L, oracle, (0, 1), kinds)
    cctx = L.CompressContext(cs[0]["ctx"], cs[1]["ctx"], cs[0]["pcs"], cs[1]["pcs"])
    insts = [running(L, c) for c in cs]
    good = cctx.prove([insts[0]], insts[1], cchal)
    # one tampered row of the primary's E: the proof is made, and the oracle verifier rejects it
    c = cs[0]
    E = c["fctx"].get_running()["E"].copy()
    E[0] ^= 1
    dE = to_device(L, c["field"], E)
    bad = cctx.prove([(insts[0][0], dE.data_ptr(), insts[0][2], insts[0][3])], insts[1], cchal)
    run = c["fctx"].get_running()
    assert not osp.verify([rows_of(m) for m in c["mats"]], c["n_w"], c["ctx"].num_vars, c["ctx"].log_rows, ints(run["u"])[0], ints(run["X"]), bad[0],
                          chal_of(0), c["p"])[0]
    # a callback that fails on the secondary circuit: LURK_ERR_ARG naming the secondary; the next call on the context succeeds
    def failing(k, label, data):
        if k == 1 and label == "pcs":
            raise KeyError("secondary transcript")
        return cchal(k, label, data)
    with pytest.raises(KeyError):
        cctx.prove([insts[0]], insts[1], failing)
    with pytest.raises(L.LurkError) as e:
        _raw_failing_call(L, cctx, insts)
    assert e.value.code == L._capi.ERR_ARG and "secondary" in str(e.value)
    again = cctx.prove([insts[0]], insts[1], cchal)
    assert all(same(a, b, kind) for a, b, kind in zip(good, again, kinds))
    torch.cuda.synchronize()


def _raw_failing_call(L, cctx, insts):
    """a C-level callback that returns non-zero in the secondary's opening (the Python wrapper re-raises the Python exception instead)"""
    calls = []

    def fn(user, circuit, phase, rnd, msg, n, out):
        calls.append((circuit, phase))
        if circuit == 1 and phase == L._capi.SPARTAN_PCS:
            return 5
        for i in range(32):
            out[i] = 0
        out[0] = 3 + len(calls) % 200
        return 0
    return cctx.prove([insts[0]], insts[1], None, native=(L._capi.COMPRESS_CHALLENGE_FN(fn), None))


def test_compress_context_carries_nothing_between_proofs(L, oracle):
    """three calls on one context, another instance in the middle, give the bytes fresh contexts give; a fold step on the key a compress
    context shares with the fold context, between two proofs, changes neither the fold record (checked against the oracle) nor the proof"""
    kinds = ("hyperkzg", "ipa")
    cs = [fold_chain(L, oracle, 0, 3, seed=61), fold_chain(L, oracle, 1, 4, seed=62)]
    for c, kind in zip(cs, kinds):
        c["ctx"] = L.spartan.SpartanContext(c["field"], c["mats"], c["n_w"], 2)
        c["pcs"], c["extra"] = pcs_of(L, oracle, c, kind)
    # the secondary's key context is the one its fold context commits with
    assert cs[1]["pcs"][1] is cs[1]["ck"]
    fresh = lambda: L.CompressContext(cs[0]["ctx"], cs[1]["ctx"], cs[0]["pcs"], cs[1]["pcs"])
    cctx = fresh()
    a = [running(L, c) for c in cs]
    E = cs[0]["fctx"].get_running()["E"].copy()
    E[3] ^= 2
    dE = to_device(L, 0, E)
    b0 = (a[0][0], dE.data_ptr(), a[0][2], a[0][3])                             # another primary instance of the same shape
    p1 = cctx.prove([a[0]], a[1], cchal)
    p2 = cctx.prove([b0], a[1], cchal)
    p3 = cctx.prove([a[0]], a[1], cchal)
    f1 = fresh().prove([a[0]], a[1], cchal)
    f2 = fresh().prove([b0], a[1], cchal)
    for x, y in ((p1, f1), (p3, f1), (p2, f2)):
        assert all(same(u, v, kind) for u, v, kind in zip(x, y, kinds))
    assert not same(p1[0], p2[0], kinds[0])
    # a fold step of the secondary's fold context between two proofs, on the key the compress context cloned
    fold_step(L, cs[1])
    assert cs[1]["fctx"].check_running() == (0, True, True)
    a = [running(L, c) for c in cs]
    after = cctx.prove([a[0]], a[1], cchal)
    assert all(same(u, v, kind) for u, v, kind in zip(after, fresh().prove([a[0]], a[1], cchal), kinds))
    check_circuit(L, oracle, 1, cs[1], after[1], composition(L, 1, 1, [cs[1]["ctx"]], [a[1]], cs[1]["pcs"], batched=False), "ipa", None)


def test_supernova_compress(L, oracle):
    """a batched primary of three BN254 circuits of different shapes (oracle-folded) and a Grumpkin secondary from its fold context:
    bit-exact with spartan_prove_batch + the opening, accepted by the batched verifier"""
    p = ospec.FIELD_MODULUS[0]
    circuits, insts, prim = [], [], []
    for k, shape in enumerate([(1, 1000, 100, 200), (1, 100, 20, 10), (1, 6, 2, 0)]):
        mats, n_w, o = folded_instance(oracle, ospec, np.random.default_rng(90 + k), *shape)
        circuits.append((mats, n_w))
        insts.append(inst_dict(mats, n_w, o.W, o.E, o.u, o.X))
        prim.append((z_of(L, 0, o.W, o.u, o.X), to_device(L, 0, o.E), o.comm_W, o.comm_E))
    ctxs = [L.spartan.SpartanContext(0, mats, n_w, 2) for mats, n_w in circuits]
    sec = nova_setup(L, oracle, (0, 1), ("hyperkzg", "ipa"))[1]
    m = max(max(c.log_rows, c.log_vars) for c in ctxs)
    g, beta, kck = kzg_setup(L, 1 << m)
    cctx = L.CompressContext(ctxs, sec["ctx"], ("hyperkzg", kck), sec["pcs"])
    assert cctx.info()["joint_len_primary"] == 1 << m
    pi = [(z.data_ptr(), e.data_ptr(), cw, ce) for z, e, cw, ce in prim]
    s_inst = running(L, sec)
    got = cctx.prove(pi, s_inst, cchal)
    want = composition(L, 0, 0, ctxs, pi, ("hyperkzg", kck), batched=True)
    assert same(got[0], want, "hyperkzg")
    ok, r, je, w = bo.verify_batched(insts, got[0], challenge, p)
    assert ok and (r, je, w) == (got[0]["r"], got[0]["joint_eval"], got[0]["weights"])
    joint = from_device(L, 0, want["joint"])
    assert open_and_check(L, ospec, kck, g, beta, want["joint"], joint, got[0]["r"], got[0]["joint_eval"])
    check_circuit(L, oracle, 1, sec, got[1], composition(L, 1, 1, [sec["ctx"]], [s_inst], sec["pcs"], batched=False), "ipa", None)
    seq = cctx.prove(pi, s_inst, cchal, sequential=True)
    assert same(seq[0], got[0], "hyperkzg") and same(seq[1], got[1], "ipa")


def test_create_refuses_short_keys_mixed_fields_and_duplicates(L, oracle):
    cs = nova_setup(L, oracle, (0, 1), ("hyperkzg", "ipa"))
    p0, p1 = cs[0]["pcs"], cs[1]["pcs"]
    short = L.CommitmentKey(0, oracle.gen_bases(0, cs[0]["ctx"].joint_len // 2))
    pasta = nova_setup(L, oracle, (2, 3), ("ipa", "ipa"))
    cases = [
        (lambda: L.CompressContext(cs[0]["ctx"], cs[1]["ctx"], ("hyperkzg", short), p1), "bases"),
        (lambda: L.CompressContext(cs[0]["ctx"], pasta[1]["ctx"], p0, p1), "field"),                      # a Vesta secondary for a BN254 primary
        (lambda: L.CompressContext([cs[0]["ctx"], pasta[0]["ctx"]], cs[1]["ctx"], p0, p1), "field"),       # mixed primary fields
        (lambda: L.CompressContext(cs[0]["ctx"], cs[1]["ctx"], p0, ("ipa", pasta[1]["ck"], p1[2])), "curve"),
        (lambda: L.CompressContext([cs[0]["ctx"], cs[0]["ctx"]], cs[1]["ctx"], p0, p1), "same context"),
    ]
    for make, message in cases:
        with pytest.raises(L.LurkError) as e:
            make()
        assert e.value.code == L._capi.ERR_ARG and message in str(e.value), str(e.value)


def test_plain_c_client_proves_on_the_gpu(tmp_path):
    exe, libdir = str(tmp_path / "compress_client"), os.path.join(ROOT, "lurk-beta_b200")
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "csrc", "compress_client.c"), "-o", exe, "-L", libdir, "-llurk_b200", "-Wl,-rpath," + libdir])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    assert out.stdout.strip() == "compress_client ok"
