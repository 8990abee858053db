"""The recursive verifier (lurk_recursive_verify, _dev; csrc/recursive.cu) on the GPU: RecursiveSNARK::verify's satisfiability checks --
is_sat_relaxed on the running instances, is_sat on the secondary's last fresh one -- in one call, every verdict equal to the oracle's
(nifs.NovaOracle: its sparse products for the rows, its MSM for the commitments), for instances straight from fold contexts, host and
device forms, full and verifier-only shapes, tampered proofs and the fib rc = 100 shapes after real folds.  lurk_fold_ctx_check_running,
which runs the same kernel with the fold's kept products, must agree."""
import ctypes as C
import os
import subprocess
import threading

import numpy as np
import pytest

from oracle import nifs, spec as ospec
from test_gpu_compress import fold_chain, snapshot
from test_gpu_spartan_chain import challenge, folded_instance, to_device
from test_gpu_spartan_ctx import z_of
from test_gpu_spartan_verify import relaxed_instance
from util import ints, pack, random_elements

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def oracle_verdict(o, W, E, u, X, comm_W, comm_E):
    """the verdict of R1CSShape::is_sat_relaxed (E given) or is_sat (E None: E = 0, u must be 1) from the oracle"""
    p = o.p
    strict = E is None
    az, bz, cz = (ints(v) for v in o.mv(o.z(W, u, X)))
    e = [0] * o.rows if strict else ints(E)
    bad = [i for i, (a, b, c, d) in enumerate(zip(az, bz, cz, e)) if (a * b - u * c - d) % p]
    if not strict:
        assert len(bad) == o.bad_rows(W, E, u, X)
    return dict(bad_rows=len(bad), first_bad_row=bad[0] if bad else None, u_ok=u == 1 if strict else True, comm_W_ok=o.commit_w(W) == comm_W,
                comm_E_ok=True if strict else o.commit_t(E) == comm_E)


def stage_fresh(L, c):
    """stage the next fresh instance (u = 1) of the chain's fold context without folding it: (W bytes, X), its z in LURK_FOLD_BUF_W2"""
    fctx, o, field, step = c["fctx"], c["o"], c["field"], c["step"]
    W = ints(random_elements(field, c["n_w"], seed=40 * c["seed"] + step, shape="edge"))
    X = ints(random_elements(field, 2, seed=40 * c["seed"] + step + 20, shape="edge"))
    for dst, v in c["glue_fn"](W, X).items():
        W[dst] = v
    fctx.host_buffer(0, -1)[:] = pack(W)
    fctx.host_buffer(0, -2)[:] = pack(X)
    fctx.host_buffer(0, -3)[:] = pack([int(v) % c["pb"] for v in o.ro_consts(X)] + [0] * (24 - len(o.ro_consts(X))))
    fctx.stage_a(0)
    fctx.sync()
    return pack(W), X


_CACHE = {}


def nova(L, oracle, curves):
    """a primary and a secondary fold chain on nifs.real_shape_step_circuit (rows of 0 to 2000 non-zeros), the secondary's next fresh
    instance staged; one Spartan shape per circuit"""
    if curves not in _CACHE:
        cs = []
        for k, curve in enumerate(curves):
            c = fold_chain(L, oracle, curve, 3, seed=31 + 5 * curve)
            c["shape"] = L.spartan.SpartanContext(c["field"], c["mats"], c["n_w"], 2)
            if k == 1:
                c["fresh"] = stage_fresh(L, c)
            cs.append(c)
        _CACHE[curves] = cs
    return _CACHE[curves]


def dev_instances(L, cs):
    """[primary running, secondary running, secondary fresh] as the fold contexts hold them"""
    out = []
    for c in cs:
        dz, _ = c["fctx"].device_buffer(0, L._capi.FOLD_BUF_Z1)
        de, _ = c["fctx"].device_buffer(0, L._capi.FOLD_BUF_E1)
        out.append(dict(shape=c["shape"], ck=c["ck"], z=dz, E=de, comm_W=nifs.point_of(c["rec"].running_comm_W), comm_E=nifs.point_of(c["rec"].running_comm_E)))
    s = cs[1]
    dz2, _ = s["fctx"].device_buffer(0, L._capi.FOLD_BUF_W2)
    out.append(dict(shape=s["shape"], ck=s["ck"], z=dz2, E=None, comm_W=s["o"].commit_w(s["fresh"][0]), comm_E=None))
    return out


def host_parts(cs):
    """(o, W, E, u, X, comm_W, comm_E) of the same three instances, canonical, from the oracles"""
    out = [(c["o"], c["o"].W, c["o"].E, c["o"].u, c["o"].X, c["o"].comm_W, c["o"].comm_E) for c in cs]
    s = cs[1]
    W, X = s["fresh"]
    out.append((s["o"], W, None, 1, X, s["o"].commit_w(W), None))
    return out


def host_instances(cs, parts):
    insts = []
    for c, (o, W, E, u, X, cw, ce) in zip([cs[0], cs[1], cs[1]], parts):
        insts.append(dict(shape=c["shape"], ck=c["ck"], z=o.z(W, u, X), E=E, comm_W=cw, comm_E=ce))
    return insts


@pytest.mark.parametrize("curves", [(0, 1), (2, 3)], ids=["bn254-grumpkin", "pallas-vesta"])
def test_nova_from_the_fold_contexts(L, oracle, curves):
    cs = nova(L, oracle, curves)
    keep = [snapshot(L, c) for c in cs]
    w2_ptr, w2_len = cs[1]["fctx"].device_buffer(0, L._capi.FOLD_BUF_W2)
    w2 = L.fold.device_tensor(w2_ptr, w2_len).clone()
    ok, got = L.recursive_verify(dev_instances(L, cs))
    assert ok
    for v, part in zip(got, host_parts(cs)):
        assert v == oracle_verdict(*part)
    for c, before in zip(cs, keep):
        assert all(a.equal(b) for a, b in zip(snapshot(L, c), before)), "a fold context's buffers were modified"
    assert L.fold.device_tensor(w2_ptr, w2_len).equal(w2)
    for c in cs:
        assert c["fctx"].check_running() == (0, True, True)


def tamper(p, parts, which, what):
    """a copy of the instance parts with one thing changed: instance `which`, field `what`"""
    parts = [list(x) for x in parts]
    o, W, E, u, X, cw, ce = parts[which]
    pb = ospec.FIELD_MODULUS[ospec.CURVES[o.curve_id]["base"]]
    if what == "W":
        v = ints(W)
        v[3] = (v[3] + 1) % p
        parts[which][1] = pack(v)
    elif what == "E":
        v = ints(E)
        v[5] = (v[5] + 1) % p
        parts[which][2] = pack(v)
    elif what == "u":
        parts[which][3] = (u + 1) % p
    elif what == "X":
        parts[which][4] = [(X[0] + 1) % p] + list(X[1:])
    elif what == "comm_W":
        parts[which][5] = ospec.ec_add(cw, cw, pb)
    elif what == "comm_E":
        parts[which][6] = ospec.ec_add(ce, cw, pb)
    return [tuple(x) for x in parts]


@pytest.mark.parametrize("which,what", [(0, "W"), (0, "E"), (0, "u"), (0, "X"), (0, "comm_W"), (0, "comm_E"), (1, "W"), (1, "E"), (1, "comm_E"),
                                        (2, "W"), (2, "u"), (2, "X"), (2, "comm_W")])
def test_nova_rejections(L, oracle, which, what):
    cs = nova(L, oracle, (0, 1))
    parts = tamper(cs[which if which < 2 else 1]["p"], host_parts(cs), which, what)
    ok, got = L.recursive_verify(host_instances(cs, parts), device=False)
    assert not ok
    want = [oracle_verdict(*x) for x in parts]
    assert got == want
    assert [i for i in range(3) if got[i] != want[i] or not all((got[i]["bad_rows"] == 0, got[i]["u_ok"], got[i]["comm_W_ok"], got[i]["comm_E_ok"]))] == [which]


def test_nova_swapped_secondary_instances(L, oracle):
    """the secondary's running and fresh instances swapped (one shape, one key): each position checked as what it claims to be"""
    cs = nova(L, oracle, (0, 1))
    parts = host_parts(cs)
    (o, W1, E1, u1, X1, cw1, ce1), (_, W2, _, u2, X2, cw2, _) = parts[1], parts[2]
    swapped = [parts[0], (o, W2, E1, u2, X2, cw2, ce1), (o, W1, None, u1, X1, cw1, None)]
    ok, got = L.recursive_verify(host_instances(cs, swapped), device=False)
    assert not ok
    assert got == [oracle_verdict(*x) for x in swapped]
    assert not got[2]["u_ok"] and got[1]["bad_rows"] > 0


@pytest.mark.parametrize("fmt", [0, 1], ids=["canonical", "montgomery"])
def test_host_form_equals_device_form(L, oracle, fmt):
    cs = nova(L, oracle, (0, 1))
    parts = tamper(cs[0]["p"], host_parts(cs), 0, "E")          # a rejection, so that the verdicts carry a row
    insts = host_instances(cs, parts)
    want = L.recursive_verify(insts, device=False)
    dev = []
    for x in insts:
        y = dict(x)
        y["z"] = to_device(L, x["shape"].field, x["z"])
        y["E"] = None if x["E"] is None else to_device(L, x["shape"].field, x["E"])
        dev.append(y)
    got = L.recursive_verify([dict(x, z=x["z"].data_ptr(), E=None if x["E"] is None else x["E"].data_ptr()) for x in dev], fmt=fmt)
    assert got == want
    if fmt == 1:
        mont = [dict(x, z=x["z"], E=x["E"]) for x in insts]
        for x, y in zip(mont, dev):
            x["z"] = y["z"].cpu().numpy()
            x["E"] = None if y["E"] is None else y["E"].cpu().numpy()
        assert L.recursive_verify(mont, fmt=1, device=False) == want


def test_supernova_three_circuits_one_key(L, oracle):
    """three BN254 running instances of different shapes on one key, then a Grumpkin secondary; a tamper in the middle circuit fails
    only that circuit's verdict"""
    prim = []
    for k, shape in enumerate([(1, 100, 20, 10), (1, 30, 5, 4), (1, 6, 2, 0)]):
        mats, n_w, o = folded_instance(oracle, ospec, np.random.default_rng(70 + k), *shape)
        prim.append((L.spartan.SpartanContext(0, mats, n_w, 2), o))
    need = max(max(o.n_w, o.rows) for _, o in prim)
    ck = L.CommitmentKey(0, oracle.gen_bases(0, need))
    cs = nova(L, oracle, (0, 1))
    insts = [dict(shape=s, ck=ck, z=o.z(o.W, o.u, o.X), E=o.E, comm_W=o.comm_W, comm_E=o.comm_E) for s, o in prim]
    insts += host_instances(cs, host_parts(cs))[1:]
    ok, got = L.recursive_verify(insts, device=False)
    assert ok and all(v == dict(bad_rows=0, first_bad_row=None, u_ok=True, comm_W_ok=True, comm_E_ok=True) for v in got)
    s, o = prim[1]
    E = ints(o.E)
    E[2] = (E[2] + 1) % o.p
    insts[1] = dict(insts[1], E=pack(E))
    ok, got = L.recursive_verify(insts, device=False)
    assert not ok
    assert got[1] == oracle_verdict(o, o.W, pack(E), o.u, o.X, o.comm_W, o.comm_E) and got[1]["first_bad_row"] == 2
    assert all(v["bad_rows"] == 0 and v["comm_W_ok"] and v["comm_E_ok"] and v["u_ok"] for i, v in enumerate(got) if i != 1)


@pytest.mark.parametrize("n_x,rows", [(0, 53), (1, 256), (4, 257), (11, 600)])
def test_public_inputs_empty_rows_and_row_counts(L, oracle, n_x, rows):
    """relaxed instances with 0 to 11 public inputs, rows without entries and row counts on both sides of a CTA; full and
    verifier-only shapes agree"""
    field, curve = 1, 1
    n_w = 37
    mats, Wb, Eb, u, X = relaxed_instance(field, rows, n_w, n_x, 120, 700 + n_x)
    assert any(mats[0][0][i] == mats[0][0][i + 1] for i in range(rows))
    bases = oracle.gen_bases(curve, max(n_w, rows))
    ck = L.CommitmentKey(curve, bases)
    o = nifs.NovaOracle(curve, bases, mats, n_w, n_x)
    cw, ce = o.commit_w(Wb), o.commit_t(Eb)
    for verifier_only in (False, True):
        shape = L.spartan.SpartanContext(field, mats, n_w, n_x, verifier_only=verifier_only)
        z = o.z(Wb, u, X)
        ok, got = L.recursive_verify([dict(shape=shape, ck=ck, z=z, E=Eb, comm_W=cw, comm_E=ce)], device=False)
        assert ok and got[0] == oracle_verdict(o, Wb, Eb, u, X, cw, ce)
        E2 = ints(Eb)
        E2[rows - 1] = (E2[rows - 1] + 3) % o.p
        ok, got = L.recursive_verify([dict(shape=shape, ck=ck, z=z, E=pack(E2), comm_W=cw, comm_E=ce)], device=False)
        assert not ok and got[0]["bad_rows"] == 1 and got[0]["first_bad_row"] == rows - 1 and not got[0]["comm_E_ok"]


def test_rows_past_two_to_the_24(L, oracle):
    """a 2^24 + 3-row shape (one entry per row but the last, which is empty): accepted, and a bad last-but-one row is found"""
    import torch
    field, curve = 0, 0
    rows, n_w = (1 << 24) + 3, 8
    rp = np.concatenate([np.arange(rows, dtype=np.uint64), np.array([rows - 1], dtype=np.uint64)])
    col = (np.arange(rows - 1) % n_w).astype(np.uint32)
    one = pack([1])
    val = np.tile(one, rows - 1)
    mats = [(rp, col, val), (rp, np.full(rows - 1, n_w, dtype=np.uint32), val), (rp, col, val)]     # (W_j)(u) = u W_j + E, E = 0
    shape = L.spartan.SpartanContext.verifier(field, mats, n_w, 0)
    ck = L.CommitmentKey(curve, oracle.gen_bases(curve, rows))
    W = ints(random_elements(field, n_w, seed=3))
    z = pack(W + [1])
    E = torch.zeros(rows * 32, dtype=torch.uint8, device="cuda")
    dz = to_device(L, field, z)
    ident = None
    o = nifs.NovaOracle(curve, oracle.gen_bases(curve, n_w), [(np.array([0, 0], dtype=np.uint64), np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.uint8))] * 3, n_w, 0)
    cw = o.commit_w(pack(W))
    ok, got = L.recursive_verify([dict(shape=shape, ck=ck, z=dz.data_ptr(), E=E.data_ptr(), comm_W=cw, comm_E=ident)])
    assert ok and got[0]["bad_rows"] == 0
    E[(rows - 2) * 32] = 1
    ok, got = L.recursive_verify([dict(shape=shape, ck=ck, z=dz.data_ptr(), E=E.data_ptr(), comm_W=cw, comm_E=ident)])
    assert not ok and got[0]["bad_rows"] == 1 and got[0]["first_bad_row"] == rows - 2 and not got[0]["comm_E_ok"]


def test_verifier_only_context_matches_a_full_one_and_refuses_to_prove(L, oracle):
    import torch
    field = 0
    mats, n_w, o = folded_instance(oracle, ospec, np.random.default_rng(5), 1, 30, 5, 4)
    full = L.spartan.SpartanContext(field, mats, n_w, 2)
    ver = L.spartan.SpartanContext.verifier(field, mats, n_w, 2)
    assert (full.log_rows, full.log_vars, full.joint_len) == (ver.log_rows, ver.log_vars, ver.joint_len)
    p = ospec.FIELD_MODULUS[field]
    rng = np.random.default_rng(9)
    rx = [int(rng.integers(0, 2**62)) * 7919 % p for _ in range(full.log_rows)]
    ry = [int(rng.integers(0, 2**62)) * 104729 % p for _ in range(full.log_vars + 1)]
    assert full.matrix_evals(rx, ry) == ver.matrix_evals(rx, ry)
    dz, dE = z_of(L, field, o.W, o.u, o.X), to_device(L, field, o.E)
    proof = full.prove(dz.data_ptr(), dE.data_ptr(), challenge)
    assert full.verify(proof, o.u, o.X, challenge) == ver.verify(proof, o.u, o.X, challenge)
    assert ver.verify(proof, o.u, o.X, challenge)[0]
    lib = L._capi.lib()
    joint = torch.empty(full.joint_len * 32, dtype=torch.uint8, device="cuda")
    rec = L._capi.SpartanProof()
    fn = L._capi.SPARTAN_CHALLENGE_FN(lambda *a: 0)
    arr = (C.c_void_p * 1)(ver._ctx.value)
    zs = (C.c_void_p * 1)(dz.data_ptr())
    es = (C.c_void_p * 1)(dE.data_ptr())
    calls = [lambda: lib.lurk_spartan_prove_dev(ver._ctx, C.c_void_p(dz.data_ptr()), C.c_void_p(dE.data_ptr()), fn, None, C.byref(rec),
                                                C.c_void_p(joint.data_ptr()), 0, None),
             lambda: lib.lurk_spartan_prove_batch_dev(1, arr, zs, es, fn, None, C.byref(rec), C.c_void_p(joint.data_ptr()), 0, None),
             lambda: lib.lurk_spartan_eval_table_dev(ver._ctx, C.c_void_p(joint.data_ptr()), L._capi.np_ptr(pack([3])), C.c_void_p(joint.data_ptr()), 0, None)]
    for call in calls:
        assert call() == L._capi.ERR_ARG
        assert b"verifier" in lib.lurk_last_error() or b"transpose" in lib.lurk_last_error()
    prim, sec = nova(L, oracle, (0, 1))
    for primary, secondary in ((ver, sec["shape"]), (prim["shape"], L.spartan.SpartanContext.verifier(1, sec["mats"], sec["n_w"], 2))):
        with pytest.raises(L.LurkError, match="transpose") as e:
            L.CompressContext(primary, secondary, ("ipa", prim["ck"], (1, 2)), ("ipa", sec["ck"], (1, 2)))
        assert e.value.code == L._capi.ERR_ARG


def test_verify_batch_on_a_verifier_only_context(L, oracle):
    field = 0
    shapes = [(1, 30, 5, 4), (1, 6, 2, 0)]
    full, ver, insts = [], [], []
    for k, sh in enumerate(shapes):
        mats, n_w, o = folded_instance(oracle, ospec, np.random.default_rng(50 + k), *sh)
        full.append(L.spartan.SpartanContext(field, mats, n_w, 2))
        ver.append(L.spartan.SpartanContext.verifier(field, mats, n_w, 2))
        insts.append((z_of(L, field, o.W, o.u, o.X), to_device(L, field, o.E), o))
    proof = L.spartan.spartan_prove_batch(full, [(z.data_ptr(), e.data_ptr()) for z, e, _ in insts], challenge)
    pub = [(o.u, o.X) for _, _, o in insts]
    a = L.spartan.spartan_verify_batch(full, pub, proof, challenge)
    b = L.spartan.spartan_verify_batch(ver, pub, proof, challenge)
    assert a == b and a[0]


def test_errors_leave_nothing_behind(L, oracle):
    cs = nova(L, oracle, (0, 1))
    parts = host_parts(cs)
    insts = host_instances(cs, parts)
    p = cs[0]["p"]
    bad_z = [dict(x) for x in insts]
    z = bad_z[0]["z"].copy()
    z[32 * 2:32 * 3] = np.frombuffer(p.to_bytes(32, "little"), dtype=np.uint8)
    bad_z[0]["z"] = z
    bad_e = [dict(x) for x in insts]
    E = bad_e[1]["E"].copy()
    E[-32:] = 0xff
    bad_e[1]["E"] = E
    off = [dict(x) for x in insts]
    cw = off[2]["comm_W"]
    off[2]["comm_W"] = (cw[0], (cw[1] + 1) % cs[1]["pb"])
    for case in (bad_z, bad_e, off):
        with pytest.raises(L.LurkError) as e:
            L.recursive_verify(case, device=False)
        assert e.value.code == L._capi.ERR_RANGE
    ok, got = L.recursive_verify(insts, device=False)
    assert ok and got == [oracle_verdict(*x) for x in parts]
    assert L.recursive_verify(dev_instances(L, cs))[0]


def test_refusals_on_the_device(L, oracle):
    cs = nova(L, oracle, (0, 1))
    insts = host_instances(cs, host_parts(cs))
    short = L.CommitmentKey(0, oracle.gen_bases(0, 8))
    pasta = nova(L, oracle, (2, 3))
    for case, msg in ((dict(insts[0], ck=short), "bases"), (dict(insts[0], ck=cs[1]["ck"]), "curve"), (dict(insts[0], ck=pasta[0]["ck"]), "curve")):
        with pytest.raises(L.LurkError, match=msg) as e:
            L.recursive_verify([case] + insts[1:], device=False)
        assert e.value.code == L._capi.ERR_ARG


def test_two_threads_on_different_keys(L, oracle):
    jobs = []
    for curves in ((0, 1), (2, 3)):
        cs = nova(L, oracle, curves)
        parts = host_parts(cs)
        jobs.append((host_instances(cs, parts), host_instances(cs, tamper(cs[0]["p"], parts, 0, "W"))))
    want = [[L.recursive_verify(x, device=False) for x in j] for j in jobs]
    got = [None, None]

    def run(k):
        got[k] = [L.recursive_verify(x, device=False) for x in jobs[k] * 3]

    th = [threading.Thread(target=run, args=(k,)) for k in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for k in range(2):
        assert got[k] == want[k] * 3


def test_plain_c_client_verifies_on_the_gpu(tmp_path):
    exe, libdir = str(tmp_path / "recursive_client"), os.path.join(ROOT, "lurk-beta_b200")
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "csrc", "recursive_client.c"), "-o", exe, "-L", libdir, "-llurk_b200", "-Wl,-rpath," + libdir])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    assert out.stdout.strip() == "recursive_client ok"


def test_full_size_fib_rc100(L, oracle):
    """the fib rc = 100 primary circuit and bench.SECONDARY after real folds through their fold contexts (bench's workload): the call
    accepts [primary running, secondary running, the secondary's prefetched and unfolded fresh instance], the primary's commitments are the
    CPU oracle's, and one changed E row is found"""
    import bench
    import torch
    wl = bench.FoldStepGPU(0, 1)
    wl.start(staged=True)
    for _ in range(3):
        wl.step(staged=True)
    wl.drain()
    prim, sec = wl.inst[0], wl.inst[-1]
    shapes = [L.spartan.SpartanContext.verifier(i.field, i.mats, i.nW, 2) for i in (prim, sec)]
    insts = []
    for i, shape, ck, rec in ((prim, shapes[0], wl.ck_w, wl.last[0]), (sec, shapes[1], wl.ck2, wl.last[-1])):
        dz, _ = i.ctx.device_buffer(0, L._capi.FOLD_BUF_Z1)
        de, _ = i.ctx.device_buffer(0, L._capi.FOLD_BUF_E1)
        insts.append(dict(shape=shape, ck=ck, z=dz, E=de, comm_W=nifs.point_of(rec.running_comm_W), comm_E=nifs.point_of(rec.running_comm_E)))
    staged = wl.step_index & 1                   # stage A of the next step, never folded: a fresh instance with u = 1
    dw2, _ = sec.ctx.device_buffer(staged, L._capi.FOLD_BUF_W2)
    w2 = L.fold.device_tensor(dw2, sec.nW * 32).clone()
    L._capi.check(L._capi.lib().lurk_convert_dev(sec.field, C.c_void_p(w2.data_ptr()), sec.nW, L.FMT_CANONICAL, C.c_void_p(w2.data_ptr()), None))
    torch.cuda.synchronize()
    cw2 = nifs.point_of(oracle.msm(1, L.synthetic_bases(1, sec.nW), w2.cpu().numpy(), nthreads=bench.host_threads()))
    insts.append(dict(shape=shapes[1], ck=wl.ck2, z=dw2, E=None, comm_W=cw2, comm_E=None))
    ok, got = L.recursive_verify(insts)
    assert ok, got
    assert all(v == dict(bad_rows=0, first_bad_row=None, u_ok=True, comm_W_ok=True, comm_E_ok=True) for v in got)
    # the primary's commitments against the CPU oracle on all host threads
    z = prim.ctx.read_device(0, L._capi.FOLD_BUF_Z1)
    E = prim.ctx.read_device(0, L._capi.FOLD_BUF_E1)
    both = torch.from_numpy(np.concatenate([z[:prim.nW * 32], E])).cuda()
    L._capi.check(L._capi.lib().lurk_convert_dev(0, C.c_void_p(both.data_ptr()), both.numel() // 32, L.FMT_CANONICAL, C.c_void_p(both.data_ptr()), None))
    torch.cuda.synchronize()
    both = both.cpu().numpy()
    bases = L.synthetic_bases(0, max(prim.nW, prim.nT))
    th = bench.host_threads()
    assert nifs.point_of(oracle.msm(0, bases, both[:prim.nW * 32], nthreads=th)) == insts[0]["comm_W"]
    assert nifs.point_of(oracle.msm(0, bases, both[prim.nW * 32:], nthreads=th)) == insts[0]["comm_E"]
    # one E row changed (in a copy): exactly that row fails
    row = prim.nT // 2 + 17
    e2 = torch.from_numpy(E.copy()).cuda()
    e2[row * 32] ^= 1
    ok, got = L.recursive_verify([dict(insts[0], E=e2.data_ptr())] + insts[1:])
    assert not ok and got[0]["bad_rows"] == 1 and got[0]["first_bad_row"] == row and not got[0]["comm_E_ok"] and got[0]["comm_W_ok"]
    assert got[1:] == [dict(bad_rows=0, first_bad_row=None, u_ok=True, comm_W_ok=True, comm_E_ok=True)] * 2


def test_check_running_finds_bad_rows_and_stale_kept_products(L, oracle):
    """lurk_fold_ctx_check_running on a folded chain: an E row changed in place fails that row alone; a W element changed in place fails
    every row whose products use it (the fresh products no longer equal the ones the folds kept) and every row whose relation breaks;
    after set_running (no kept products) a tampered W fails exactly the oracle's rows"""
    import torch
    c = fold_chain(L, oracle, 0, 3, seed=77)
    fctx, o, p = c["fctx"], c["o"], c["p"]
    assert fctx.check_running() == (0, True, True)
    fctx.sync()
    dz, nz = fctx.device_buffer(0, L._capi.FOLD_BUF_Z1)
    de, ne = fctx.device_buffer(0, L._capi.FOLD_BUF_E1)
    z_dev, e_dev = L.fold.device_tensor(dz, nz), L.fold.device_tensor(de, ne)
    # one E row (non-zero) set to zero
    E = ints(o.E)
    k = next(i for i in range(len(E)) if E[i])
    saved = e_dev[32 * k:32 * k + 32].clone()
    e_dev[32 * k:32 * k + 32] = 0
    torch.cuda.synchronize()
    assert fctx.check_running() == (1, True, False)
    e_dev[32 * k:32 * k + 32] = saved
    torch.cuda.synchronize()
    assert fctx.check_running() == (0, True, True)
    # one W element (non-zero, used by the matrices) set to zero
    W = ints(o.W)
    uses = {}
    for rp, col, val in c["mats"]:
        row_of = np.repeat(np.arange(len(rp) - 1), np.diff(np.asarray(rp, dtype=np.int64)))
        for r, cc, v in zip(row_of, np.asarray(col), ints(val)):
            if v % p:
                uses.setdefault(int(cc), set()).add(int(r))
    j = next(j for j in sorted(uses) if j < c["n_w"] and W[j] and len(uses[j]) > 1)
    W2 = list(W)
    W2[j] = 0
    relation = oracle_verdict(o, pack(W2), o.E, o.u, o.X, o.comm_W, o.comm_E)
    az, bz, cz = (ints(v) for v in o.mv(o.z(pack(W2), o.u, o.X)))
    fails = {i for i, (a, b, cc, d) in enumerate(zip(az, bz, cz, E)) if (a * b - o.u * cc - d) % p}
    want = len(uses[j] | fails)
    saved = z_dev[32 * j:32 * j + 32].clone()
    z_dev[32 * j:32 * j + 32] = 0
    torch.cuda.synchronize()
    assert fctx.check_running() == (want, False, True)
    z_dev[32 * j:32 * j + 32] = saved
    torch.cuda.synchronize()
    assert fctx.check_running() == (0, True, True)
    # the same W through set_running: no kept products, the relation alone
    fctx.set_running(pack(W2), o.E, pack([o.u]), pack(o.X), nifs.point_bytes(o.comm_W), nifs.point_bytes(o.comm_E))
    assert fctx.check_running() == (relation["bad_rows"], False, True)
    assert relation["bad_rows"] > 0
