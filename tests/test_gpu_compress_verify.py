"""The compressed verifier (lurk_compress_verify; csrc/compress_verify.cu) on the GPU: CompressedSNARK::verify in one call on the proofs
lurk_compress_prove_dev makes from fold contexts (the secondary's last fold included).  The primary's fold key is a KZG key of known beta,
so the pairing callback checks P == beta Q in G1, and P, Q are pinned to kzg_verifier_oracle.verifier_points.  Every verdict is compared with
the composed path -- SpartanContext.verify / spartan_verify_batch, the joint commitment, ipa_verify on eq(r), or HyperKZG's fold check and
kzg.verify_known_beta -- on the good proofs and on one tamper at a time; the transcripts are the prover's, byte for byte.  Also: the
errors come before any callback, failing callbacks name their circuit, concurrent and sequential calls, verifier-only contexts and two host
threads agree, and the key contexts are left as they were."""
import os
import subprocess
import threading

import numpy as np
import pytest

from kzg_verifier_oracle import verifier_points
from oracle import kzg, spec as ospec
from test_gpu_compress import chal_of, composition, fold_chain, fold_step, point96, running
from test_gpu_spartan_batched import kzg_setup
from test_gpu_spartan_chain import folded_instance, to_device
from test_gpu_spartan_ctx import z_of
from test_gpu_spartan_verify import compressed
from test_gpu_sumcheck import from_device
from util import ints, pack

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class KzgKeyOracle:
    """the oracle with gen_bases on BN254 replaced by the powers of tau of kzg_setup's (g, beta): fold contexts and NovaOracle then commit
    under the KZG key, so that the primary's commitments open with HyperKZG"""

    def __init__(self, oracle, g, beta):
        self.oracle, self.g, self.beta = oracle, g, beta

    def gen_bases(self, curve, n, start=0):
        if curve != 0:
            return self.oracle.gen_bases(curve, n, start=start)
        return pack([c for P in kzg.powers_of_tau(0, self.g, self.beta, n) for c in P])

    def __getattr__(self, name):
        return getattr(self.oracle, name)


def logged(logs):
    """the transcript of test_gpu_compress (one per circuit), every call appended to logs[circuit]"""
    def chal(k, label, data):
        logs[k].append((label, repr(data)))
        return chal_of(k)(label, data)
    return chal


def kzg_pairing(beta, calls=None, answer=None):
    pb = ospec.FIELD_MODULUS[1]

    def pairing(k, P, Q):
        if calls is not None:
            calls.append((k, P, Q))
        return ospec.ec_mul(beta, Q, pb) == P if answer is None else answer
    return pairing


_CACHE = {}


def setup(L, oracle, curves):
    """Nova: the primary and secondary fold chains (3 steps, the secondary's last fold on top), their compress proof and everything the
    verifier takes"""
    if curves in _CACHE:
        return _CACHE[curves]
    g, beta, _ = kzg_setup(L, 1)
    kinds = ("hyperkzg", "ipa") if curves == (0, 1) else ("ipa", "ipa")
    cs = []
    for k, curve in enumerate(curves):
        c = fold_chain(L, KzgKeyOracle(oracle, g, beta) if kinds[k] == "hyperkzg" else oracle, curve, 3, seed=13 + 5 * curve)
        if k == 1:
            fold_step(L, c)
        c["ctx"] = L.spartan.SpartanContext(c["field"], c["mats"], c["n_w"], 2)
        if kinds[k] == "hyperkzg":
            c["pcs"], c["vk"] = ("hyperkzg", c["ck"]), ("hyperkzg", g)
        else:
            gc = tuple(ints(oracle.gen_bases(curve, 1, start=len(c["bases"]) // 64 + 7)))
            c["pcs"], c["vk"] = ("ipa", c["ck"], gc), ("ipa", c["ck"], gc)
        run = c["fctx"].get_running()
        c["inst"] = (ints(run["u"])[0], ints(run["X"]), *running(L, c)[2:])
        c["W"], c["E"] = ints(run["W"]), ints(run["E"])
        cs.append(c)
    cctx = L.CompressContext(cs[0]["ctx"], cs[1]["ctx"], cs[0]["pcs"], cs[1]["pcs"])
    logs = [[], []]
    proof = cctx.prove([running(L, cs[0])], running(L, cs[1]), logged(logs))
    s = dict(cs=cs, kinds=kinds, g=g, beta=beta, proof=proof, logs=logs, cctx=cctx)
    _CACHE[curves] = s
    return s


def verify(L, s, proof=None, insts=None, chal=None, pairing=None, ctxs=None, **kw):
    cs = s["cs"]
    ctxs = ctxs or [c["ctx"] for c in cs]
    insts = insts or [c["inst"] for c in cs]
    return L.compress_verify(ctxs[0], ctxs[1], cs[0]["vk"], cs[1]["vk"], [insts[0]], insts[1], proof or s["proof"], chal or logged([[], []]),
                             pairing or kzg_pairing(s["beta"]), **kw)


def kzg_scalars(L, s):
    """the discrete logs (w.r.t. g) of the primary's commitments and of the honest opening: C_i, com_j, w_t"""
    if "scal" in s:
        return s["scal"]
    c, pr, p = s["cs"][0], s["proof"][0], ospec.FIELD_MODULUS[0]
    beta = s["beta"]
    want = composition(L, 0, 0, [c["ctx"]], [running(L, c)], c["pcs"], batched=False)
    joint = from_device(L, 0, want["joint"])
    polys = kzg.fold_chain(joint, pr["r"], p)
    at_beta = [kzg.poly_eval(f, beta, p) for f in polys]
    r = chal_of(0)("pcs", (0, b"".join(point96(P).tobytes() for P in pr["com"]))) % p
    q = chal_of(0)("pcs", (1, pack([x for t in pr["v"] for x in t]).tobytes())) % p
    u = [r, (-r) % p, r * r % p]
    Bb = sum(pow(q, j, p) * x for j, x in enumerate(at_beta)) % p
    w = [(Bb - sum(pow(q, j, p) * pr["v"][t][j] for j in range(len(pr["r"])))) * pow(beta - u[t], -1, p) % p for t in range(3)]
    s["scal"] = dict(C=[kzg.poly_eval(c["W"], beta, p), kzg.poly_eval(c["E"], beta, p)], com=at_beta[1:], w=w)
    return s["scal"]


def composed(L, s, k, proof, inst, chal, scal=None, compressed_rounds=False):
    """the verdict of the composed path for circuit k: (snark_ok, eval_ok, opening_ok)"""
    import torch
    c = s["cs"][k]
    curve, p, pb = c["curve"], c["p"], c["pb"]
    ok, d = c["ctx"].verify(proof, inst[0], inst[1], lambda label, data: chal(k, label, data), compressed=compressed_rounds)
    if not ok:
        return (0, -1, -1)
    m = len(d["r"])
    comm = ospec.ec_add(ospec.ec_mul(d["weights"][0], inst[2], pb), ospec.ec_mul(d["weights"][1], inst[3], pb), pb)
    if c["vk"][0] == "ipa":
        scale = chal(k, "pcs", (0, point96(comm).tobytes() + int(d["joint_eval"]).to_bytes(32, "little"))) % p
        gc = ospec.ec_mul(scale, c["vk"][2], pb)
        b = torch.empty((1 << m) * 32, dtype=torch.uint8, device="cuda")
        L.spartan.eq_evals(c["field"], d["r"], b.data_ptr())
        acc = L.spartan.ipa_verify(curve, c["ck"], gc, comm, d["joint_eval"], b.data_ptr(), m, proof["L"], proof["R"], proof["a_final"],
                                   lambda rnd, msg: chal(k, "pcs", (rnd + 1, bytes(msg))) % p)[0]
        return (1, 1, int(acc))
    # HyperKZG with every commitment as its discrete log
    r = chal(k, "pcs", (0, b"".join(point96(P).tobytes() for P in proof["com"]))) % p
    v, x = proof["v"], d["r"]
    Y = list(v[2]) + [d["joint_eval"]]
    if any(2 * r * Y[i + 1] % p != (r * (1 - x[m - 1 - i]) * (v[0][i] + v[1][i]) + x[m - 1 - i] * (v[0][i] - v[1][i])) % p for i in range(m)):
        return (1, 0, -1)
    q = chal(k, "pcs", (1, pack([e for t in v for e in t]).tobytes())) % p
    chal(k, "pcs", (2, b"".join(point96(P).tobytes() for P in proof["w"])))
    C0 = (d["weights"][0] * scal["C"][0] + d["weights"][1] * scal["C"][1]) % p
    return (1, 1, int(kzg.verify_known_beta(0, s["g"], s["beta"], C0, x, d["joint_eval"], scal["com"], v, scal["w"], r, q)))


@pytest.mark.parametrize("compressed_rounds", [False, True], ids=["evals", "compressed"])
@pytest.mark.parametrize("curves", [(0, 1), (2, 3)], ids=["bn254-grumpkin", "pallas-vesta"])
def test_round_trip_is_accepted_with_the_provers_transcript(L, oracle, curves, compressed_rounds):
    s = setup(L, oracle, curves)
    proof = [compressed(pr, c["p"]) for pr, c in zip(s["proof"], s["cs"])] if compressed_rounds else s["proof"]
    logs, calls = [[], []], []
    acc, verdicts = verify(L, s, proof=proof, chal=logged(logs), pairing=kzg_pairing(s["beta"], calls), compressed=compressed_rounds)
    assert acc and verdicts == [(1, 1, 1), (1, 1, 1)]
    assert logs == s["logs"]                        # per circuit, the prover's transcript byte for byte
    scal = kzg_scalars(L, s) if curves == (0, 1) else None
    for k in range(2):
        assert composed(L, s, k, proof[k], s["cs"][k]["inst"], logged([[], []]), scal, compressed_rounds) == (1, 1, 1)
    if curves == (0, 1):
        assert len(calls) == 1 and calls[0][0] == 0
        pr, p, pb = s["proof"][0], ospec.FIELD_MODULUS[0], ospec.FIELD_MODULUS[1]
        r = chal_of(0)("pcs", (0, b"".join(point96(P).tobytes() for P in pr["com"]))) % p
        q = chal_of(0)("pcs", (1, pack([x for t in pr["v"] for x in t]).tobytes())) % p
        d = chal_of(0)("pcs", (2, b"".join(point96(P).tobytes() for P in pr["w"]))) % p
        C0 = (pr["weights"][0] * scal["C"][0] + pr["weights"][1] * scal["C"][1]) % p
        Ps, Qs = verifier_points(0, C0, scal["com"], pr["v"], scal["w"], r, q, d)
        assert calls[0][1] == ospec.ec_mul(Ps, s["g"], pb) and calls[0][2] == ospec.ec_mul(Qs, s["g"], pb)
        assert Ps == s["beta"] * Qs % p
    else:
        assert calls == []


def _bump(x, p):
    return (x + 1) % p


def _tampers(s):
    """(name, circuit, check index, function (proof, insts, scal) -> (proof, insts, scal, chal, pairing)) -- one field at a time"""
    out = []
    for k, c in enumerate(s["cs"]):
        p, pb, curve = c["p"], c["pb"], c["curve"]
        gen = s["g"] if c["vk"][0] == "hyperkzg" else ospec.CURVES[curve]["gen"]

        def field(key, path, k=k, p=p):
            def f(proof, insts, scal):
                pr = dict(proof[k])
                v = pr[key]
                if path is None:
                    pr[key] = _bump(v, p)
                else:
                    v = [list(x) if isinstance(x, (list, tuple)) else x for x in v]
                    i, j = path
                    if j is None:
                        v[i] = _bump(v[i], p)
                    else:
                        v[i][j] = _bump(v[i][j], p)
                    pr[key] = v
                proof = list(proof)
                proof[k] = pr
                return proof, insts, scal, None, None
            return f

        def point(key, i, k=k, pb=pb, gen=gen, shift=None):
            def f(proof, insts, scal):
                pr = dict(proof[k])
                pts = list(pr[key])
                pts[i] = ospec.ec_add(pts[i], gen, pb)
                pr[key] = pts
                proof = list(proof)
                proof[k] = pr
                if shift:
                    scal = dict(scal, **{shift: [x + (1 if j == i else 0) for j, x in enumerate(scal[shift])]})
                return proof, insts, scal, None, None
            return f

        def inst(pos, k=k, p=p, pb=pb, gen=gen):
            def f(proof, insts, scal):
                x = list(insts[k])
                if pos == 0:
                    x[0] = _bump(x[0], p)
                elif pos == 1:
                    x[1] = [_bump(x[1][0], p)] + list(x[1][1:])
                else:
                    x[pos] = ospec.ec_add(x[pos], gen, pb)
                    if scal and k == 0:
                        scal = dict(scal, C=[v + (1 if j == pos - 2 else 0) for j, v in enumerate(scal["C"])])
                insts = list(insts)
                insts[k] = tuple(x)
                return proof, insts, scal, None, None
            return f
        out += [(f"{k}-outer", k, 0, field("outer_rounds", (0, 1))), (f"{k}-inner", k, 0, field("inner_rounds", (1, 0))),
                (f"{k}-reduce", k, 0, field("reduce_rounds", (0, 2))), (f"{k}-claims", k, 0, field("claims", (1, None))),
                (f"{k}-eval_W", k, 0, field("eval_W", None)), (f"{k}-claims_left", k, 0, field("claims_left", (1, None))),
                (f"{k}-u", k, 0, inst(0)), (f"{k}-X", k, 0, inst(1)), (f"{k}-comm_W", k, 2, inst(2)), (f"{k}-comm_E", k, 2, inst(3))]
        if c["vk"][0] == "hyperkzg":
            out += [(f"{k}-com", k, 1, point("com", 1, shift="com")), (f"{k}-v", k, 1, field("v", (2, 1))), (f"{k}-w", k, 2, point("w", 1, shift="w"))]
        else:
            out += [(f"{k}-L", k, 2, point("L", 2)), (f"{k}-R", k, 2, point("R", 0)), (f"{k}-a_final", k, 2, field("a_final", None))]

        def other_chal(proof, insts, scal, k=k):
            def chal(kk, label, data):
                x = chal_of(kk)(label, data)
                return x + 1 if kk == k and label == "pcs" and data[0] == 1 else x
            return proof, insts, scal, chal, None
        out.append((f"{k}-transcript", k, 2, other_chal))
    out.append(("0-pairing-no", 0, 2, lambda proof, insts, scal: (proof, insts, scal, None, kzg_pairing(s["beta"], answer=False))))
    return out


def test_every_tamper_is_rejected_by_its_circuit_alone_as_the_composed_path_rejects_it(L, oracle):
    s = setup(L, oracle, (0, 1))
    scal0 = kzg_scalars(L, s)
    insts0 = [c["inst"] for c in s["cs"]]
    names = []
    for name, k, check, tamper in _tampers(s):
        proof, insts, scal, chal, pairing = tamper(s["proof"], insts0, scal0)
        chal = chal or (lambda kk, label, data: chal_of(kk)(label, data))
        for sequential in (False, True):
            logs = [[], []]
            acc, verdicts = verify(L, s, proof=proof, insts=insts, chal=lambda kk, label, data: (logs[kk].append((label, repr(data))), chal(kk, label, data))[1],
                                   pairing=pairing, sequential=sequential)
            want = tuple([1] * check + [0] + [-1] * (2 - check))
            assert not acc and verdicts[k] == want and verdicts[1 - k] == (1, 1, 1), (name, verdicts)
            assert logs[1 - k] == s["logs"][1 - k], name
            if sequential:
                assert (verdicts, logs) == seen, name
            seen = (verdicts, logs)
        if name != "0-pairing-no":
            assert composed(L, s, k, proof[k], insts[k], chal, scal) == want, name
        names.append(name)
    assert len(names) == 29


def test_supernova_batched_primary_round_trip_and_swapped_instances(L, oracle):
    g, beta, _ = kzg_setup(L, 1)
    ko = KzgKeyOracle(oracle, g, beta)
    circuits, prim, insts = [], [], []
    for k, shape in enumerate([(1, 1000, 100, 200), (1, 100, 20, 10), (1, 6, 2, 0)]):
        mats, n_w, o = folded_instance(ko, ospec, np.random.default_rng(90 + k), *shape)
        circuits.append((mats, n_w))
        prim.append((z_of(L, 0, o.W, o.u, o.X), to_device(L, 0, o.E), o.comm_W, o.comm_E))
        insts.append((o.u, [int(x) for x in o.X], o.comm_W, o.comm_E))
    ctxs = [L.spartan.SpartanContext(0, mats, n_w, 2) for mats, n_w in circuits]
    m = max(max(c.log_rows, c.log_vars) for c in ctxs)
    _, _, kck = kzg_setup(L, 1 << m)
    sec = setup(L, oracle, (0, 1))["cs"][1]
    cctx = L.CompressContext(ctxs, sec["ctx"], ("hyperkzg", kck), sec["pcs"])
    logs = [[], []]
    proof = cctx.prove([(z.data_ptr(), e.data_ptr(), cw, ce) for z, e, cw, ce in prim], running(L, sec), logged(logs))
    for compressed_rounds in (False, True):
        pr = [compressed(proof[0], ospec.FIELD_MODULUS[0]), compressed(proof[1], sec["p"])] if compressed_rounds else proof
        vlogs = [[], []]
        acc, verdicts = L.compress_verify(ctxs, sec["ctx"], ("hyperkzg", g), sec["vk"], insts, sec["inst"], pr, logged(vlogs), kzg_pairing(beta),
                                          compressed=compressed_rounds)
        assert acc and verdicts == [(1, 1, 1), (1, 1, 1)] and vlogs == logs
        ok, _ = L.spartan.spartan_verify_batch(ctxs, [x[:2] for x in insts], pr[0], chal_of(0), compressed=compressed_rounds)
        assert ok
    swapped = [insts[1], insts[0], insts[2]]
    acc, verdicts = L.compress_verify(ctxs, sec["ctx"], ("hyperkzg", g), sec["vk"], swapped, sec["inst"], proof, logged([[], []]), kzg_pairing(beta))
    assert not acc and verdicts == [(0, -1, -1), (1, 1, 1)]
    assert not L.spartan.spartan_verify_batch(ctxs, [x[:2] for x in swapped], proof[0], chal_of(0))[0]


def _counting(calls):
    def chal(k, label, data):
        calls.append(k)
        return chal_of(k)(label, data)
    return chal


def test_errors_come_before_any_callback_and_leave_the_contexts_usable(L, oracle):
    s = setup(L, oracle, (0, 1))
    cs, p0 = s["cs"], s["cs"][0]["p"]
    pasta = setup(L, oracle, (2, 3))["cs"]
    short = L.CommitmentKey(1, oracle.gen_bases(1, cs[1]["ctx"].joint_len // 2))
    insts = [c["inst"] for c in cs]
    bad_claims = dict(s["proof"][0], claims=(p0,) + tuple(s["proof"][0]["claims"][1:]))
    twice = dict(s["proof"][0], claims=[s["proof"][0]["claims"]] * 2, eval_W=[s["proof"][0]["eval_W"]] * 2, claims_left=s["proof"][0]["claims_left"] * 2)
    off = list(s["proof"][1]["L"])
    off[0] = (1, 1)
    cases = [
        (dict(proof=[bad_claims, s["proof"][1]]), L._capi.ERR_RANGE, "claims"),
        (dict(proof=[s["proof"][0], dict(s["proof"][1], L=off)]), L._capi.ERR_RANGE, "secondary"),
        (dict(proof=[dict(s["proof"][0], v=[[p0] + list(s["proof"][0]["v"][0][1:])] + list(s["proof"][0]["v"][1:])), s["proof"][1]]), L._capi.ERR_RANGE, "v"),
        (dict(insts=[(p0,) + tuple(insts[0][1:]), insts[1]]), L._capi.ERR_RANGE, "u"),
        (dict(insts=[insts[0][:2] + ((1, 1),) + insts[0][3:], insts[1]]), L._capi.ERR_RANGE, "commitment"),
        (dict(ctxs=[cs[0]["ctx"], pasta[1]["ctx"]]), L._capi.ERR_ARG, "field"),
        (dict(ctxs=[cs[0]["ctx"], cs[0]["ctx"]]), L._capi.ERR_ARG, "secondary context"),
    ]
    for kw, code, message in cases:
        calls = []
        with pytest.raises(L.LurkError) as e:
            verify(L, s, chal=_counting(calls), **kw)
        assert e.value.code == code and message in str(e.value), str(e.value)
        assert calls == [], message
        assert verify(L, s)[0]
    for make, message in [
        (lambda chal: L.compress_verify(cs[0]["ctx"], cs[1]["ctx"], cs[0]["vk"], ("ipa", short, cs[1]["vk"][2]), [insts[0]], insts[1], s["proof"], chal,
                                        kzg_pairing(s["beta"])), "bases"),
        (lambda chal: L.compress_verify(cs[0]["ctx"], cs[1]["ctx"], cs[0]["vk"], ("ipa", pasta[1]["ck"], cs[1]["vk"][2]), [insts[0]], insts[1], s["proof"],
                                        chal, kzg_pairing(s["beta"])), "curve"),
        (lambda chal: L.compress_verify(cs[0]["ctx"], cs[1]["ctx"], cs[0]["vk"], cs[1]["vk"], [insts[0]], insts[1], s["proof"], chal), "pairing"),
        (lambda chal: L.compress_verify([cs[0]["ctx"], cs[0]["ctx"]], cs[1]["ctx"], cs[0]["vk"], cs[1]["vk"], [insts[0]] * 2, insts[1], [twice, s["proof"][1]],
                                        chal, kzg_pairing(s["beta"])), "same context"),
    ]:
        calls = []
        with pytest.raises(L.LurkError) as e:
            make(_counting(calls))
        assert e.value.code == L._capi.ERR_ARG and message in str(e.value), str(e.value)
        assert calls == []
        assert verify(L, s)[0]
    # failing C callbacks: LURK_ERR_ARG naming the circuit, never a rejection
    def failing_transcript(user, circuit, phase, rnd, msg, n, out):
        if circuit == 1:
            return 5
        for i in range(32):
            out[i] = 0
        out[0] = 3 + rnd
        return 0
    with pytest.raises(L.LurkError) as e:
        verify(L, s, native=(L._capi.COMPRESS_CHALLENGE_FN(failing_transcript), None), native_pairing=L._capi.PAIRING_CHECK_FN(lambda *a: 0))
    assert e.value.code == L._capi.ERR_ARG and "secondary" in str(e.value)
    with pytest.raises(L.LurkError) as e:
        verify(L, s, native_pairing=L._capi.PAIRING_CHECK_FN(lambda *a: 7))
    assert e.value.code == L._capi.ERR_ARG and "primary" in str(e.value) and "pairing" in str(e.value)
    assert verify(L, s) == (True, [(1, 1, 1), (1, 1, 1)])


def test_verifier_only_contexts_threads_and_the_key_contexts(L, oracle):
    s = setup(L, oracle, (0, 1))
    cs = s["cs"]
    vctx = [L.spartan.SpartanContext.verifier(c["field"], c["mats"], c["n_w"], 2) for c in cs]
    want = verify(L, s)
    assert verify(L, s, ctxs=vctx) == want and verify(L, s, ctxs=vctx, sequential=True) == want
    # a commitment on the borrowed key gives the same bytes before and after a call, and nothing is left pending on it
    probe = pack(list(range(1, 65)))
    before = cs[1]["ck"].commit(probe)
    assert verify(L, s)[0]
    assert np.array_equal(cs[1]["ck"].commit(probe), before)
    # two host threads, two proofs at once, on separate key contexts
    other = L.CommitmentKey(1, cs[1]["bases"])
    vk2 = ("ipa", other, cs[1]["vk"][2])
    results = [None, None]

    def work(i):
        if i == 0:
            results[i] = verify(L, s)
        else:
            results[i] = L.compress_verify(vctx[0], vctx[1], cs[0]["vk"], vk2, [cs[0]["inst"]], cs[1]["inst"], s["proof"], logged([[], []]),
                                           kzg_pairing(s["beta"]))
    th = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert results == [want, want]


def test_plain_c_client_verifies_on_the_gpu(tmp_path):
    exe, libdir = str(tmp_path / "compress_verify_client"), os.path.join(ROOT, "lurk-beta_b200")
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "csrc", "compress_verify_client.c"), "-o", exe, "-L", libdir, "-llurk_b200", "-Wl,-rpath," + libdir])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    assert out.stdout.strip() == "compress_verify_client ok"
