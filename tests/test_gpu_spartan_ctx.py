"""The Spartan prover context (lurk_spartan_ctx_*, lurk_spartan_prove_dev / lurk_spartan_prove_batch_dev; csrc/spartan.cu) on the GPU:
bit-exact with the Python compositions it replaces (spartan.RelaxedR1CSProver + batch_eval_reduce, spartan.BatchedRelaxedR1CSProver) on all
four fields, accepted by the verifiers (oracle/spartan.py, tests/batched_oracle.py), proved straight from the fold context's running
instance and opened with HyperKZG (BN254) or the inner-product argument (Grumpkin, Pallas, Vesta); the fused evaluation table against three
transposed SpMVs and two AXPYs on adversarial column lengths; a primary and a secondary proof from two host threads at once.
Challenges: the sha256 stand-in of test_gpu_spartan_chain.py for Keccak256Transcript."""
import ctypes as C
import hashlib
import os
import subprocess
import threading

import numpy as np
import pytest

import batched_oracle as bo
from oracle import nifs, spartan as osp, spec as ospec, sumcheck as sc
from test_gpu_spartan_batched import KEYS, gpu_be_challenge, inst_dict, joint_commitment, kzg_setup, oracle_folded_instances, prove_on_gpu
from test_gpu_spartan_chain import challenge, open_and_check, rows_of, to_device
from test_gpu_sumcheck import from_device
from util import ints, pack, random_elements

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CURVE_OF_FIELD = {0: 0, 1: 1, 2: 2, 3: 3}          # the curve whose scalar field is the witness field


def folded(oracle, field, seed, free=200, glue=24, lin_rows=30):
    """a running instance of nifs.real_shape_step_circuit after init + 2 folds by nifs.NovaOracle (u != 1, E != 0)"""
    curve, p = CURVE_OF_FIELD[field], ospec.FIELD_MODULUS[field]
    rng = np.random.default_rng(seed)
    mats, n_w, glue_fn = nifs.real_shape_step_circuit(rng, p, 1, free, glue, lin_rows)
    o = nifs.NovaOracle(curve, oracle.gen_bases(curve, max(n_w, len(mats[0][0]) - 1)), mats, n_w, 2, nthreads=4, pp_digest=9)
    for step in range(3):
        W = ints(random_elements(field, n_w, seed=seed + 10 * step, shape="edge"))
        X = ints(random_elements(field, 2, seed=seed + 10 * step + 1, shape="edge"))
        for dst, v in glue_fn(W, X).items():
            W[dst] = v
        (o.init_running if step == 0 else o.prove_step)(pack(W), X)
    assert o.bad_rows() == 0 and o.u != 1 and any(ints(o.E))
    return mats, n_w, o


def z_of(L, field, W_bytes, u, X):
    return to_device(L, field, np.concatenate([np.ascontiguousarray(W_bytes, dtype=np.uint8).reshape(-1), pack([u] + list(X))]))


def python_composition(L, field, mats, n_w, W_bytes, E_bytes, u, X):
    """RelaxedR1CSProver.prove followed by batch_eval_reduce([W, E]): the reference the context is compared with"""
    p = ospec.FIELD_MODULUS[field]
    prover = L.spartan.RelaxedR1CSProver(field, mats, n_w, 2)
    zp = prover.pad_z(to_device(L, field, W_bytes), u, X)
    proof = prover.prove(zp, to_device(L, field, E_bytes), u, challenge)
    nvb = prover.num_vars.bit_length() - 1
    claims = [(zp.data_ptr(), nvb, proof["ry"][1:], proof["eval_W"]), (proof["E_padded"].data_ptr(), prover.log_rows, proof["rx"], proof["claims"][3])]
    rounds, r, left, w, je, joint = L.spartan.batch_eval_reduce(field, claims, gpu_be_challenge(p))
    proof.update(reduce_rounds=rounds, r=r, claims_left=left, weights=w, joint_eval=je, joint=joint)
    return prover, proof


PLAIN_KEYS = ("outer_rounds", "inner_rounds", "claims", "eval_W", "rx", "ry", "reduce_rounds", "r", "claims_left", "weights", "joint_eval")


def check_plain(L, field, ctx, mats, n_w, W, E, u, X, d_z, d_E):
    """the context's proof from (d_z, d_E) is bit-exact with the Python composition; the verifiers accept it and reject a changed u"""
    import torch
    p = ospec.FIELD_MODULUS[field]
    keep = (d_z.clone(), d_E.clone())
    got = ctx.prove(d_z.data_ptr(), d_E.data_ptr(), challenge)
    torch.cuda.synchronize()
    assert torch.equal(d_z, keep[0]) and torch.equal(d_E, keep[1]), "an input was modified"
    prover, want = python_composition(L, field, mats, n_w, W, E, u, X)
    for k in PLAIN_KEYS:
        assert got[k] == want[k], k
    assert torch.equal(got["joint"], want["joint"]), "joint polynomial bytes"
    rows_lists = [rows_of(m) for m in mats]
    ok, rx, ry = osp.verify(rows_lists, n_w, ctx.num_vars, ctx.log_rows, u, X, got, challenge, p)
    assert ok and rx == got["rx"] and ry == got["ry"]
    assert bo.batch_eval_verify(got["reduce_rounds"], [ry[1:], rx], [got["eval_W"], got["claims"][3]], got["claims_left"],
                                lambda rnd, v: challenge("batch_eval", (rnd, list(v))), p) == (got["r"], got["joint_eval"], got["weights"])
    assert not osp.verify(rows_lists, n_w, ctx.num_vars, ctx.log_rows, (u + 1) % p, X, got, challenge, p)[0]
    return got


@pytest.mark.parametrize("field", [0, 1, 2, 3])
def test_plain_prover_matches_the_python_composition(L, oracle, field):
    p = ospec.FIELD_MODULUS[field]
    mats, n_w, o = folded(oracle, field, 300 + field)
    ctx = L.spartan.SpartanContext(field, mats, n_w, 2)
    check_plain(L, field, ctx, mats, n_w, o.W, o.E, o.u, o.X, z_of(L, field, o.W, o.u, o.X), to_device(L, field, o.E))
    # one tampered row of E: the instance is no longer satisfied and the verifier rejects the context's proof
    bad = o.E.copy()
    bad[0] ^= 1
    dz, dE = z_of(L, field, o.W, o.u, o.X), to_device(L, field, bad)
    proof = ctx.prove(dz.data_ptr(), dE.data_ptr(), challenge)
    assert not osp.verify([rows_of(m) for m in mats], n_w, ctx.num_vars, ctx.log_rows, o.u, o.X, proof, challenge, p)[0]


def ipa_closes(L, oracle, curve, joint_t, joint, r, je, commitment=None):
    """test_supernova_compress_pallas_ipa's closing relation: a' G' + a' b' ck_c = commit(joint) + joint_eval ck_c + sum_j (r_j^2 L_j + r_j^-2 R_j)"""
    import torch
    field, pb = ospec.CURVES[curve]["scalar"], ospec.FIELD_MODULUS[ospec.CURVES[curve]["base"]]
    p = ospec.FIELD_MODULUS[field]
    m = len(r)
    n = 1 << m
    bases = oracle.gen_bases(curve, n + 1, start=5)
    gc = tuple(ints(bases[64 * n:]))
    ck = L.CommitmentKey(curve, bases[:64 * n])
    b = torch.empty(n * 32, dtype=torch.uint8, device="cuda")
    L.spartan.eq_evals(field, r, b.data_ptr())
    chals = []

    def chal(rnd, msg):
        chals.append(1 + int.from_bytes(hashlib.sha256(bytes([rnd]) + msg).digest()[:16], "little"))
        return chals[-1]
    Ls, Rs, a_fin, b_fin = L.spartan.ipa_prove(curve, ck, gc, joint_t.clone().data_ptr(), b.data_ptr(), m, chal)
    add = lambda P, Q: ospec.ec_add(P, Q, pb)
    mul = lambda k, P: ospec.ec_mul(k % p, P, pb)
    acc = add(nifs.point_of(ck.commit(pack(joint))), mul(je, gc))
    for rj, Lj, Rj in zip(chals, Ls, Rs):
        ri = pow(rj, -1, p)
        acc = add(acc, add(mul(rj * rj, Lj), mul(ri * ri, Rj)))
    s = []
    for k in range(n):
        v = 1
        for j, rj in enumerate(chals):
            v = v * (rj if (k >> (m - 1 - j)) & 1 else pow(rj, -1, p)) % p
        s.append(v)
    eq_r = sc.eq_evals(r, p)
    assert b_fin == sum(x * y for x, y in zip(s, eq_r)) % p
    G0 = nifs.point_of(oracle.msm(curve, bases[:64 * n], pack(s), nthreads=4))
    return ck, add(mul(a_fin, G0), mul(a_fin * b_fin, gc)) == acc


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_proof_straight_from_the_fold_context(L, oracle, curve):
    """a NovaFoldContext chain of 4 GPU steps, proved from the pointers LURK_FOLD_BUF_Z1 / LURK_FOLD_BUF_E1 return (no host copy of W or
    E on the way in); the joint polynomial opens (HyperKZG on BN254, IPA elsewhere) and sum_i w_i C_i = commit(joint)"""
    import torch
    field = ospec.CURVES[curve]["scalar"]
    p = ospec.FIELD_MODULUS[field]
    rng = np.random.default_rng(700 + curve)
    mats, n_w, glue_fn = nifs.real_shape_step_circuit(rng, p, 1, 150, 20, 30)
    rows = len(mats[0][0]) - 1
    bases = oracle.gen_bases(curve, max(n_w, rows))
    fctx = L.NovaFoldContext(curve, L.CommitmentKey(curve, bases), n_w, 2, mats, depth=1, fmt=L.FMT_CANONICAL)
    fctx.set_spans([(0, n_w, n_w, 1)])
    o = nifs.NovaOracle(curve, bases, mats, n_w, 2, nthreads=4, pp_digest=5)
    pb = ospec.FIELD_MODULUS[ospec.CURVES[curve]["base"]]
    for step in range(4):
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
        (o.init_running if step == 0 else o.prove_step)(pack(W), X)
    assert fctx.check_running() == (0, True, True)
    dz, zbytes = fctx.device_buffer(0, L._capi.FOLD_BUF_Z1)
    de, ebytes = fctx.device_buffer(0, L._capi.FOLD_BUF_E1)
    assert (zbytes, ebytes) == (32 * (n_w + 3), 32 * rows)
    run = fctx.get_running()
    u, X = ints(run["u"])[0], ints(run["X"])
    assert np.array_equal(run["W"], o.W) and np.array_equal(run["E"], o.E) and u == o.u
    ctx = L.spartan.SpartanContext(field, mats, n_w, 2)
    # byte copies of the fold context's buffers before and after the proof (out = a + 0 b)
    zero = L._capi.np_ptr(np.zeros(32, dtype=np.uint8))

    def snapshot(ptr, nbytes):
        t = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        L._capi.check(L._capi.lib().lurk_axpy_dev(field, C.c_void_p(ptr), C.c_void_p(ptr), zero, nbytes // 32, C.c_void_p(t.data_ptr()), None))
        return t
    keep_z, keep_e = snapshot(dz, zbytes), snapshot(de, ebytes)
    got = ctx.prove(dz, de, challenge)
    assert torch.equal(snapshot(dz, zbytes), keep_z) and torch.equal(snapshot(de, ebytes), keep_e), "the fold context's running instance was modified"
    _, want = python_composition(L, field, mats, n_w, run["W"], run["E"], u, X)
    for k in PLAIN_KEYS:
        assert got[k] == want[k], k
    assert torch.equal(got["joint"], want["joint"])
    ok, rx, ry = osp.verify([rows_of(m) for m in mats], n_w, ctx.num_vars, ctx.log_rows, u, X, got, challenge, p)
    assert ok
    joint = from_device(L, field, got["joint"])
    polys = [ints(run["W"]) + [0] * (ctx.num_vars - n_w), ints(run["E"]) + [0] * ((1 << ctx.log_rows) - rows)]
    if curve == 0:
        g, beta, ck = kzg_setup(L, len(joint))
        assert open_and_check(L, ospec, ck, g, beta, got["joint"], joint, got["r"], got["joint_eval"])
        assert not open_and_check(L, ospec, ck, g, beta, got["joint"], joint, got["r"], (got["joint_eval"] + 1) % p)
    else:
        ck, closes = ipa_closes(L, oracle, curve, got["joint"], joint, got["r"], got["joint_eval"])
        assert closes
    assert joint_commitment(ck, curve, polys, got["weights"]) == nifs.point_of(ck.commit(pack(joint)))


# ------------------------------------------------------------------------------------------------ the fused evaluation table
def csr_from_entries(rows, entries):
    """entries: (row, col) pairs -> row_ptr, col (sorted by row)"""
    e = np.asarray(entries, dtype=np.int64).reshape(-1, 2)
    order = np.argsort(e[:, 0], kind="stable")
    e = e[order]
    rp = np.concatenate([[0], np.cumsum(np.bincount(e[:, 0], minlength=rows))]).astype(np.uint64)
    return rp, e[:, 1].astype(np.uint32)


def check_table(L, field, mats, n_w, n_x, seed):
    """sp_eval_table_kernel against the composition it replaces: three transposed lurk_spmv_csr_dev calls and two lurk_axpy_dev calls"""
    import torch
    p = ospec.FIELD_MODULUS[field]
    ctx = L.spartan.SpartanContext(field, mats, n_w, n_x)
    prover = L.spartan.RelaxedR1CSProver(field, mats, n_w, n_x)
    eq = to_device(L, field, random_elements(field, 1 << ctx.log_rows, seed=seed))
    r = ints(random_elements(field, 1, seed=seed + 1))[0]
    nz = 2 * ctx.num_vars
    got = torch.full((nz * 32,), 0xAB, dtype=torch.uint8, device="cuda")      # every output must be written, empty columns included
    ctx.eval_table(eq.data_ptr(), r, got.data_ptr())
    ys = [torch.empty(nz * 32, dtype=torch.uint8, device="cuda") for _ in range(3)]
    for M, y in zip(prover.MT, ys):
        M.mv(field, eq.data_ptr(), y.data_ptr())
    want = torch.empty_like(ys[0])
    prover._axpy(ys[0], ys[1], r, want)
    prover._axpy(want, ys[2], r * r % p, want)
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    # and twice in a row: the per-row tickets of the split columns are reset by the kernel itself
    ctx.eval_table(eq.data_ptr(), r, got.data_ptr())
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_eval_table_on_adversarial_column_lengths(L):
    """columns of the padded z with 0, 1, 1024, 1025 and 70 000 entries (split over 4 375 chunks), across the three matrices"""
    field, rng = 0, np.random.default_rng(5)
    n_w, n_x, rows = 3000, 2, 80000
    lens = {0: 0, 1: 1, 2: 1024, 3: 1025, n_w: 70000, n_w + 1: 1025, n_w + 2: 3}       # n_w = the u column, then X
    mats = []
    for m in range(3):
        entries = []
        for c, k in lens.items():
            if k:
                share = k // 3 + (1 if m < k % 3 else 0)
                entries += [(int(rw), c) for rw in rng.choice(rows, size=share, replace=False)]
        entries += [(int(rng.integers(0, rows)), int(c)) for c in rng.integers(4, n_w, size=5000)]
        rp, col = csr_from_entries(rows, entries)
        mats.append((rp, col, random_elements(field, len(col), seed=10 + m)))
    check_table(L, field, mats, n_w, n_x, seed=1)


def test_eval_table_many_long_columns_no_x_and_empty_matrix(L):
    """more than 4096 columns of over 1024 entries each (what a long-row list of fixed capacity could not hold), with n_x = 0 and an
    empty C"""
    field, rng = 2, np.random.default_rng(6)
    n_w, rows, ncols, per = 4200, 2048, 4100, 1030
    mats = []
    for m in range(2):
        r_idx = rng.integers(0, rows, size=ncols * per)
        c_idx = np.repeat(np.arange(ncols), per)
        rp, col = csr_from_entries(rows, np.stack([r_idx, c_idx], axis=1))
        mats.append((rp, col, random_elements(field, len(col), seed=20 + m)))
    mats.append((np.zeros(rows + 1, dtype=np.uint64), np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.uint8)))
    check_table(L, field, mats, n_w, 0, seed=2)


def test_eval_table_all_matrices_empty(L):
    rows = 8
    empty = (np.zeros(rows + 1, dtype=np.uint64), np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.uint8))
    check_table(L, 1, [empty] * 3, 10, 2, seed=3)


def test_eval_table_at_fib_rc100_shape(L):
    import sys
    sys.path.insert(0, ROOT)
    import bench
    mats, n_w, rows, _ = bench.step_circuit(1, 100)
    check_table(L, 0, mats, n_w, 2, seed=4)


# ------------------------------------------------------------------------------------------------ batched
def pallas_circuits(oracle):
    curve, field = 2, 2
    p = ospec.FIELD_MODULUS[field]
    out = []
    for k, (slot, glue, lin) in enumerate([(300, 30, 40), (30, 6, 2), (6, 2, 0)]):
        rng = np.random.default_rng(120 + k)
        mats, n_w, glue_fn = nifs.synthetic_step_circuit(rng, 1, slot, glue, lin)
        o = nifs.NovaOracle(curve, oracle.gen_bases(curve, max(n_w, len(mats[0][0]) - 1)), mats, n_w, 2, pp_digest=3)
        for step in range(3):
            W = [int(x) % p for x in rng.integers(0, 2**62, size=n_w)]
            for dst, v in glue_fn(W, p).items():
                W[dst] = v
            (o.init_running if step == 0 else o.prove_step)(nifs.pack(W), [int(rng.integers(1, 2**60)) for _ in range(2)])
        out.append((mats, n_w, inst_dict(mats, n_w, o.W, o.E, o.u, o.X)))
    return out


@pytest.mark.parametrize("field", [0, 2])
def test_batched_prover_matches_the_python_composition(L, oracle, field):
    import torch
    p = ospec.FIELD_MODULUS[field]
    circuits = oracle_folded_instances(oracle) if field == 0 else pallas_circuits(oracle)
    insts = [c[2] for c in circuits]
    ctxs = [L.spartan.SpartanContext(field, mats, n_w, 2) for mats, n_w, _ in circuits]
    dev = [(z_of(L, field, pack(I["W"]), I["u"], I["X"]), to_device(L, field, pack(I["E"]))) for I in insts]
    keep = [(a.clone(), b.clone()) for a, b in dev]
    got = L.spartan.spartan_prove_batch(ctxs, [(a.data_ptr(), b.data_ptr()) for a, b in dev], challenge)
    torch.cuda.synchronize()
    assert all(torch.equal(a, c) and torch.equal(b, d) for (a, b), (c, d) in zip(dev, keep))
    _, want = prove_on_gpu(L, field, circuits, insts)
    for k in KEYS:
        assert got[k] == want[k], k
    assert torch.equal(got["joint"], want["joint"])
    ok, r, je, w = bo.verify_batched(insts, got, challenge, p)
    assert ok and (r, je, w) == (got["r"], got["joint_eval"], got["weights"])
    # a context of another field is refused before any device work
    other = L.spartan.SpartanContext(1 if field == 0 else 3, circuits[-1][0], circuits[-1][1], 2)
    with pytest.raises(L.LurkError) as e:
        L.spartan.spartan_prove_batch(ctxs[:-1] + [other], [(a.data_ptr(), b.data_ptr()) for a, b in dev], challenge)
    assert e.value.code == L._capi.ERR_ARG and "field" in str(e.value)
    # a joint buffer over an input is refused
    with pytest.raises(L.LurkError) as e:
        L.spartan.spartan_prove_batch(ctxs, [(a.data_ptr(), b.data_ptr()) for a, b in dev], challenge, d_joint_ptr=dev[0][1].data_ptr())
    assert e.value.code == L._capi.ERR_ARG and "overlaps" in str(e.value)


# ------------------------------------------------------------------------------------------------ both halves of CompressedSNARK::prove
def test_primary_and_secondary_proofs_at_once(L, oracle):
    """a BN254 primary proof and a Grumpkin (BN254 Fq) secondary proof from two host threads on two streams give the bytes they give
    one after the other"""
    import torch
    jobs = []
    for field, seed in ((0, 11), (1, 12)):
        mats, n_w, o = folded(oracle, field, seed, free=400, glue=40, lin_rows=60)
        ctx = L.spartan.SpartanContext(field, mats, n_w, 2)
        jobs.append((ctx, z_of(L, field, o.W, o.u, o.X), to_device(L, field, o.E)))
    torch.cuda.synchronize()
    seq = [ctx.prove(z.data_ptr(), e.data_ptr(), challenge) for ctx, z, e in jobs]
    results, errors = [None, None], []

    def run(i):
        try:
            ctx, z, e = jobs[i]
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                results[i] = ctx.prove(z.data_ptr(), e.data_ptr(), challenge, stream=s.cuda_stream)
            s.synchronize()
        except Exception as ex:        # reported below
            errors.append(ex)
    threads = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for a, b in zip(seq, results):
        for k in PLAIN_KEYS:
            assert a[k] == b[k], k
        assert torch.equal(a["joint"], b["joint"])


def test_plain_c_client_proves_on_the_gpu(tmp_path):
    exe, libdir = str(tmp_path / "spartan_client"), os.path.join(ROOT, "lurk-beta_b200")
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "csrc", "spartan_client.c"), "-o", exe, "-L", libdir, "-llurk_b200", "-Wl,-rpath," + libdir])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    assert out.stdout.strip() == "spartan_client ok"
