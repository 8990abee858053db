"""The fold context (lurk_fold_ctx_*, csrc/foldctx_impl.cuh) on every curve of both cycles -- BN254 / Grumpkin and Pallas /
Vesta, the reference's default (src/proof/nova.rs:58) -- with R1CS rows of real shape (nifs.real_shape_step_circuit: empty
rows, the lazy-reduction group boundaries, 255-term bit packings, p - 1 and full-width coefficients, a 2000-term row, u and
X columns) and operands over the whole field (util.random_elements shape "edge"): the IVC chain against the oracle, one
step against plain Python integers, the identity commitments of the sponge (W_INF / T_INF), custom absorb patterns and
challenge widths (lurk_fold_ctx_set_ro), and the stand-alone fold helpers."""
import numpy as np
import pytest

from oracle import nifs
from util import edge_values, ints, montgomery_top, pack, random_elements

pytestmark = pytest.mark.gpu
CURVES = [0, 1, 2, 3]          # BN254 G1, Grumpkin, Pallas, Vesta
R = 1 << 256
PP = 0x1234567890abcdef1122334455667788


def _fields(spec, curve):
    C = spec.CURVES[curve]
    return C["scalar"], C["base"], spec.FIELD_MODULUS[C["scalar"]], spec.FIELD_MODULUS[C["base"]]


def _mont(spec, field, buf):
    p = spec.FIELD_MODULUS[field]
    return pack([x * R % p for x in ints(buf)])


def _unmont(spec, field, buf):
    p = spec.FIELD_MODULUS[field]
    rinv = pow(R, -1, p)
    return [x * rinv % p for x in ints(buf)]


def _ro_buffer(pb, consts):
    """the step's CONST elements by absorb position, as the host writes them (reduced into the commitment field)"""
    return pack([int(c) % pb for c in consts] + [0] * (24 - len(consts)))


def _same_point(buf96, P):
    return np.array_equal(buf96, nifs.point_bytes(P))


def _check_record(rec, want, o, s):
    assert _same_point(rec.comm_W, want["comm_W"]), f"step {s}: comm_W"
    assert _same_point(rec.comm_T, want["comm_T"]), f"step {s}: comm_T"
    assert int.from_bytes(rec.ro_hash.tobytes(), "little") == want["hash"], f"step {s}: sponge output"
    assert int.from_bytes(rec.r.tobytes(), "little") == want["r"], f"step {s}: challenge"
    assert _same_point(rec.running_comm_W, o.comm_W) and _same_point(rec.running_comm_E, o.comm_E), f"step {s}: folded commitments"


def _check_final(ctx, o):
    run = ctx.get_running()
    assert np.array_equal(run["W"], o.W) and np.array_equal(run["E"], o.E)
    assert ints(run["u"]) == [o.u] and ints(run["X"]) == o.X
    assert _same_point(run["comm_W"], o.comm_W) and _same_point(run["comm_E"], o.comm_E)
    assert o.bad_rows(run["W"], run["E"], ints(run["u"])[0], ints(run["X"])) == 0
    assert ctx.check_running() == (0, True, True)


def _key(L, oracle, curve, mats, n_w):
    bases = oracle.gen_bases(curve, max(n_w, len(mats[0][0]) - 1))
    return bases, L.CommitmentKey(curve, bases)


# ----------------------------------------------------------------------------------------------------------- slot context
def _layout(oracle, field, frames, glue, slots_per_frame=((4, 6), (8, 3), (3, 1)), bd_per_frame=2):
    """per frame [slot blocks in slot order | bit decompositions | glue] (src/lem/multiframe.rs:635-712)"""
    blocks = {a: oracle.witness_block(field, a) for a, _ in slots_per_frame}
    bd_block = oracle.bitdecomp_size(field)
    slot_elems = sum(n * blocks[a] for a, n in slots_per_frame) + bd_per_frame * bd_block
    per = slot_elems + glue
    offs, cur = {}, 0
    for a, n in slots_per_frame:
        offs[a] = np.array([f * per + cur + k * blocks[a] for f in range(frames) for k in range(n)], dtype=np.uint64)
        cur += n * blocks[a]
    offs[0] = np.array([f * per + cur + k * bd_block for f in range(frames) for k in range(bd_per_frame)], dtype=np.uint64)
    return dict(blocks=blocks, bd_block=bd_block, slot_elems=slot_elems, per=per, offs=offs, frames=frames, glue=glue,
                slots=[(a, n * frames) for a, n in slots_per_frame], nbd=bd_per_frame * frames)


def _slot_step(oracle, field, lay, glue_fn, seed, rng, dummy=False):
    """slot preimages of one step (edge operands; most slots dummies, or all of them) and the fresh witness the reference
    assembles from them"""
    pre = {}
    for a, n in lay["slots"]:
        x = random_elements(field, n * a, seed=100 * seed + a, shape="edge").reshape(n, a * 32)
        x[rng.random(n) < 0.6] = 0                       # dummy slots (multiframe.rs:553-577)
        pre[a] = np.zeros_like(x).reshape(-1) if dummy else x.reshape(-1)
    bd = random_elements(field, lay["nbd"], seed=50 + seed, shape="edge")
    if dummy:
        bd = np.zeros_like(bd)
    n_w = lay["frames"] * lay["per"]
    Wv = np.zeros((n_w, 32), dtype=np.uint8)
    for a, n in lay["slots"]:
        blk = lay["blocks"][a]
        wit = oracle.poseidon_witness_batch(field, a, pre[a], nthreads=8).reshape(n, blk, 32)
        for k, off in enumerate(lay["offs"][a]):
            Wv[int(off):int(off) + blk] = wit[k]
    wit = oracle.bitdecomp_witness_batch(field, bd).reshape(lay["nbd"], lay["bd_block"], 32)
    for k, off in enumerate(lay["offs"][0]):
        Wv[int(off):int(off) + lay["bd_block"]] = wit[k]
    X2 = ints(random_elements(field, 2, seed=70 + seed, shape="edge"))
    Wi = ints(Wv)
    gv = glue_fn(Wi, X2)
    for dst, v in gv.items():
        Wi[dst] = v
    glue = pack([gv[f * lay["per"] + lay["slot_elems"] + g] for f in range(lay["frames"]) for g in range(lay["glue"])])
    return dict(pre=pre, bd=bd, W2=pack(Wi), glue=glue, X2=X2)


def _slot_fill(ctx, b, lay, st, bi, pb, conv_s, conv_b):
    for a, _ in lay["slots"]:
        ctx.host_buffer(b, bi[a])[:] = conv_s(st["pre"][a])
    ctx.host_buffer(b, bi[0])[:] = conv_s(st["bd"])
    ctx.host_buffer(b, -1)[:] = conv_s(st["glue"])
    ctx.host_buffer(b, -2)[:] = conv_s(pack(st["X2"]))
    ctx.host_buffer(b, -3)[:] = conv_b(_ro_buffer(pb, [PP, 0, 0, 0] + st["X2"]))


@pytest.mark.parametrize("curve", CURVES)
def test_ivc_chain_real_shapes(L, oracle, spec, curve):
    """init_running and four folds at depth 2 with slot batches: every record and the running instance equal the oracle;
    the last step's slots are all dummies (W2 = D on the slot spans, so commit(W2 - D) sees zero scalars there).  The
    Pallas chain takes Montgomery inputs."""
    field, base, p, pb = _fields(spec, curve)
    rng = np.random.default_rng(1000 + curve)
    lay = _layout(oracle, field, frames=2, glue=33)
    mats, n_w, glue_fn = nifs.real_shape_step_circuit(rng, p, 2, lay["slot_elems"], lay["glue"], lin_rows=33)
    bases, ck = _key(L, oracle, curve, mats, n_w)
    ctx = L.NovaFoldContext(curve, ck, n_w, 2, mats, depth=2, fmt=L.FMT_CANONICAL)
    bi = {a: ctx.add_slot_batch(a, lay["offs"][a]) for a, _ in lay["slots"]}
    bi[0] = ctx.add_slot_batch(0, lay["offs"][0])
    ctx.set_spans([(lay["slot_elems"], lay["glue"], lay["per"], lay["frames"])])
    o = nifs.NovaOracle(curve, bases, mats, n_w, 2, nthreads=8, pp_digest=PP)
    fmt = L.FMT_MONTGOMERY if curve == 2 else L.FMT_CANONICAL
    if fmt == L.FMT_MONTGOMERY:
        conv_s, conv_b = (lambda x: _mont(spec, field, x)), (lambda x: _mont(spec, base, x))
    else:
        conv_s = conv_b = lambda x: x
    n_steps = 5
    steps = [_slot_step(oracle, field, lay, glue_fn, s, rng, dummy=s == n_steps - 1) for s in range(n_steps)]
    _slot_fill(ctx, 0, lay, steps[0], bi, pb, conv_s, conv_b)
    ctx.stage_a(0, fmt=fmt)
    ctx.init_running(0)
    _slot_fill(ctx, 1, lay, steps[1], bi, pb, conv_s, conv_b)
    ctx.stage_a(1, fmt=fmt)
    rec = ctx.collect(0)
    want = o.init_running(steps[0]["W2"], steps[0]["X2"])
    assert _same_point(rec.comm_W, want["comm_W"]) and _same_point(rec.running_comm_W, want["comm_W"])
    assert not rec.running_comm_E.any() and not rec.comm_T.any()
    for s in range(1, n_steps):
        b = s & 1
        ctx.stage_b_launch(b)
        rec = ctx.collect(b)
        if s + 1 < n_steps:
            _slot_fill(ctx, b ^ 1, lay, steps[s + 1], bi, pb, conv_s, conv_b)
            ctx.stage_a(b ^ 1, fmt=fmt)
        _check_record(rec, o.prove_step(steps[s]["W2"], steps[s]["X2"]), o, s)
    _check_final(ctx, o)


# -------------------------------------------------------------------------------------------------------- no-slot context
def _host_ctx(L, oracle, spec, curve, seed, free, glue, lin_rows, pp=PP):
    field, base, p, pb = _fields(spec, curve)
    rng = np.random.default_rng(seed)
    mats, n_w, glue_fn = nifs.real_shape_step_circuit(rng, p, 1, free, glue, lin_rows)
    bases, ck = _key(L, oracle, curve, mats, n_w)
    ctx = L.NovaFoldContext(curve, ck, n_w, 2, mats, depth=1, fmt=L.FMT_CANONICAL)
    ctx.set_spans([(0, n_w, n_w, 1)])                      # the host supplies every witness value
    o = nifs.NovaOracle(curve, bases, mats, n_w, 2, nthreads=8, pp_digest=pp)
    return ctx, o, mats, n_w, glue_fn, bases


def _witness(spec, curve, n_w, glue_fn, seed, zero=False, X=None, mont_top=False):
    field = spec.CURVES[curve]["scalar"]
    p = spec.FIELD_MODULUS[field]
    if mont_top:            # every value's Montgomery form near p: the lazy reductions of A z, B z, C z at their bound
        W = [montgomery_top(p, int(k)) for k in np.random.default_rng(seed).integers(0, 2**32, size=n_w)]
    else:
        W = [0] * n_w if zero else ints(random_elements(field, n_w, seed=seed, shape="edge"))
    X = ints(random_elements(field, 2, seed=seed + 1, shape="edge")) if X is None else X
    for dst, v in glue_fn(W, X).items():
        W[dst] = v
    return pack(W), X


def _host_step(ctx, o, pb, W, X, first, consts=None):
    ctx.host_buffer(0, -1)[:] = W
    ctx.host_buffer(0, -2)[:] = pack(X)
    ctx.host_buffer(0, -3)[:] = _ro_buffer(pb, o.ro_consts(X) if consts is None else consts)
    ctx.stage_a(0)
    if first:
        ctx.init_running(0)
    else:
        ctx.stage_b_launch(0)
    return ctx.collect(0)


@pytest.mark.parametrize("curve", CURVES)
def test_fold_step_against_python_integers(L, oracle, spec, curve):
    """one step at a small shape, checked without oracle.c: T, z1 and E1 read back from the device against big-integer
    arithmetic on the CSR rows and the witnesses, the commitments against spec.msm_naive"""
    field, base, p, pb = _fields(spec, curve)
    ctx, o, mats, n_w, glue_fn, bases = _host_ctx(L, oracle, spec, curve, seed=2000 + curve, free=250, glue=40, lin_rows=120)
    rows = len(mats[0][0]) - 1
    W1, X1 = _witness(spec, curve, n_w, glue_fn, seed=1)
    W2, X2 = _witness(spec, curve, n_w, glue_fn, seed=3)
    rec1 = _host_step(ctx, o, pb, W1, X1, first=True)
    rec2 = _host_step(ctx, o, pb, W2, X2, first=False)
    b = ints(bases)
    pts = list(zip(b[0::2], b[1::2]))
    z1, z2 = ints(W1) + [1] + X1, ints(W2) + [1] + X2
    rowlists = []
    for rp, col, val in mats:
        v = ints(val)
        rowlists.append([[(int(col[k]), v[k]) for k in range(int(rp[i]), int(rp[i + 1]))] for i in range(rows)])

    def mv(z):
        return [[sum(z[c] * x for c, x in r) % p for r in m] for m in rowlists]
    (a1, b1, c1), (a2, b2, c2) = mv(z1), mv(z2)
    T = [(a1[i] * b2[i] + a2[i] * b1[i] - c2[i] - c1[i]) % p for i in range(rows)]
    assert all((a1[i] * b1[i] - c1[i]) % p == 0 for i in range(rows))
    comm_W1, comm_W2 = spec.msm_naive(curve, pts, ints(W1)), spec.msm_naive(curve, pts, ints(W2))
    comm_T = spec.msm_naive(curve, pts, T)
    r, h = spec.ro_squeeze(base, spec.nifs_absorb_list(PP, comm_W2, X2, comm_T))
    assert _same_point(rec1.comm_W, comm_W1)
    assert _same_point(rec2.comm_W, comm_W2) and _same_point(rec2.comm_T, comm_T)
    assert int.from_bytes(rec2.r.tobytes(), "little") == r and int.from_bytes(rec2.ro_hash.tobytes(), "little") == h
    assert _same_point(rec2.running_comm_W, spec.ec_add(comm_W1, spec.ec_mul(r, comm_W2, pb), pb))
    assert _same_point(rec2.running_comm_E, spec.ec_mul(r, comm_T, pb))
    assert _unmont(spec, field, ctx.read_device(0, L._capi.FOLD_BUF_T)) == T
    assert _unmont(spec, field, ctx.read_device(0, L._capi.FOLD_BUF_Z1)) == [(x + r * y) % p for x, y in zip(z1, z2)]
    assert _unmont(spec, field, ctx.read_device(0, L._capi.FOLD_BUF_E1)) == [r * t % p for t in T]
    assert ctx.check_running() == (0, True, True)


@pytest.mark.parametrize("curve", CURVES)
def test_edge_steps(L, oracle, spec, curve):
    """the identity commitments the sponge absorbs as (0, 0, 1), and public IO at the top of the field:
    step 1 folds the very instance the chain started from (T = 0: comm_T = identity, comm_E += r O), step 2 is the all-zero
    witness (comm_W2 = identity), steps 3 and 4 carry X2 near p.  The first instance's witness has every Montgomery form
    near p, so that its A z, B z, C z -- kept by the fold from then on -- come from the largest products; the device's
    relaxed-R1CS check runs after every step."""
    field, base, p, pb = _fields(spec, curve)
    ctx, o, mats, n_w, glue_fn, bases = _host_ctx(L, oracle, spec, curve, seed=3000 + curve, free=300, glue=33, lin_rows=66)
    W0, X0 = _witness(spec, curve, n_w, glue_fn, seed=5, mont_top=True)
    rec = _host_step(ctx, o, pb, W0, X0, first=True)
    assert _same_point(rec.comm_W, o.init_running(W0, X0)["comm_W"])
    steps = [(W0, X0), _witness(spec, curve, n_w, glue_fn, seed=7, zero=True),
             _witness(spec, curve, n_w, glue_fn, seed=9, X=[p - 1, (p + 1) // 2]),
             _witness(spec, curve, n_w, glue_fn, seed=11, X=[p - 2, p - 1])]
    for s, (W, X) in enumerate(steps, start=1):
        rec = _host_step(ctx, o, pb, W, X, first=False)
        want = o.prove_step(W, X)
        if s == 1:
            assert want["comm_T"] is None and not any(ints(want["T"])) and not rec.comm_T.any()
            assert o.comm_E is None and not rec.running_comm_E.any()
        if s == 2:
            assert want["comm_W"] is None and not rec.comm_W.any()
        _check_record(rec, want, o, s)
        assert ctx.check_running() == (0, True, True), f"step {s}"
    _check_final(ctx, o)


# ------------------------------------------------------------------------------------------------------------------ set_ro
CHALLENGE_BITS = (1, 31, 32, 33, 64, 127, 128, 129, 250)


def _pattern(rng, n, k):
    if n == 1:
        return [(nifs.RO_T_INF, nifs.RO_W_INF, nifs.RO_W_X)[k % 3]]
    kinds = list(rng.permutation(7)) + list(rng.integers(0, 7, size=n - 7))
    return [int(x) for x in kinds]


@pytest.mark.parametrize("curve", CURVES)
def test_set_ro_patterns_and_challenge_widths(L, oracle, spec, curve):
    """lurk_fold_ctx_set_ro: absorb patterns of 1, 9 and 24 elements with the identity flags among them, and every
    challenge width where the word masking of the squeezed element changes; out-of-range arguments are refused and leave
    the pattern as it was"""
    field, base, p, pb = _fields(spec, curve)
    ctx, o, mats, n_w, glue_fn, bases = _host_ctx(L, oracle, spec, curve, seed=4000 + curve, free=80, glue=14, lin_rows=24)
    rng = np.random.default_rng(curve)
    W0, X0 = _witness(spec, curve, n_w, glue_fn, seed=13)
    _host_step(ctx, o, pb, W0, X0, first=True)
    o.init_running(W0, X0)
    k = 0
    for bits in CHALLENGE_BITS:
        for n in (1, 9, 24):
            kinds = _pattern(rng, n, k)
            consts = ints(random_elements(base, 24, seed=100 + k, shape="edge"))
            if k == 0:
                W, X = W0, X0                              # T = 0: comm_T is the identity
            else:
                W, X = _witness(spec, curve, n_w, glue_fn, seed=200 + k, zero=k % 7 == 3)
            ctx.set_ro(kinds, bits)
            rec = _host_step(ctx, o, pb, W, X, first=False, consts=consts)
            want = o.prove_step(W, X, challenge_bits=bits, ro_kinds=kinds, ro_consts=consts)
            assert want["r"] < 1 << bits
            _check_record(rec, want, o, f"{k} (n_absorb {n}, {bits} bits)")
            k += 1
    for bad_kinds, bad_bits in (([], 128), ([0] * 25, 128), ([1], 0), ([1], 251), ([0, 7], 128), ([-1], 128)):
        with pytest.raises(L.LurkError) as e:
            ctx.set_ro(bad_kinds, bad_bits)
        assert e.value.code == L._capi.ERR_ARG
    W, X = _witness(spec, curve, n_w, glue_fn, seed=999)
    rec = _host_step(ctx, o, pb, W, X, first=False, consts=consts)
    _check_record(rec, o.prove_step(W, X, challenge_bits=bits, ro_kinds=kinds, ro_consts=consts), o, "after refused calls")
    _check_final(ctx, o)


# ---------------------------------------------------------------------------------------------------- stand-alone helpers
def _dev(arr):
    import torch
    return torch.from_numpy(np.ascontiguousarray(arr)).cuda()


@pytest.mark.parametrize("field", [0, 1, 2, 3])
def test_fold_helpers_real_shapes(L, spec, field):
    """lurk_spmv_csr_dev, lurk_cross_term_dev and lurk_axpy_dev on real row shapes and edge operands, against Python
    integers"""
    import torch
    lib = L._capi.lib()
    p = spec.FIELD_MODULUS[field]
    rng = np.random.default_rng(field)
    mats, n_w, _ = nifs.real_shape_step_circuit(rng, p, 2, 600, 40, 60)
    n = n_w + 3
    z = random_elements(field, n, seed=1, shape="edge")
    zi = ints(z)
    dz = _dev(_mont(spec, field, z))
    for rp, col, val in mats:
        rows = len(rp) - 1
        d_rp, d_col, d_val = _dev(rp), _dev(col), _dev(_mont(spec, field, val))
        y = torch.empty(rows * 32, dtype=torch.uint8, device="cuda")
        L._capi.check(lib.lurk_spmv_csr_dev(field, d_rp.data_ptr(), d_col.data_ptr(), d_val.data_ptr(), rows, dz.data_ptr(), y.data_ptr(), None))
        v = ints(val)
        want = [sum(v[k] * zi[int(col[k])] for k in range(int(rp[i]), int(rp[i + 1]))) % p for i in range(rows)]
        assert _unmont(spec, field, y.cpu().numpy()) == want
    m = 3000
    a, b = random_elements(field, m, seed=2, shape="edge"), random_elements(field, m, seed=3, shape="edge")
    ai, bi = ints(a), ints(b)
    da, db = _dev(_mont(spec, field, a)), _dev(_mont(spec, field, b))
    out = torch.empty_like(da)
    for r in edge_values(field):
        L._capi.check(lib.lurk_axpy_dev(field, da.data_ptr(), db.data_ptr(), L._capi.np_ptr(_mont(spec, field, pack([r]))), m, out.data_ptr(), None))
        assert _unmont(spec, field, out.cpu().numpy()) == [(x + r * y) % p for x, y in zip(ai, bi)], f"r = {r:#x}"
    v = [random_elements(field, m, seed=10 + k, shape="edge") for k in range(6)]
    vi = [ints(x) for x in v]
    dv = [_dev(_mont(spec, field, x)) for x in v]
    t = torch.empty_like(dv[0])
    for u1, u2 in ((1, 1), (p - 1, 1), (0, p - 1), (ints(random_elements(field, 1, 4, "edge"))[0], (p + 1) // 2)):
        L._capi.check(lib.lurk_cross_term_dev(field, *[x.data_ptr() for x in dv], L._capi.np_ptr(_mont(spec, field, pack([u1]))),
                                              L._capi.np_ptr(_mont(spec, field, pack([u2]))), m, t.data_ptr(), None))
        want = [(vi[0][i] * vi[4][i] + vi[3][i] * vi[1][i] - u1 * vi[5][i] - u2 * vi[2][i]) % p for i in range(m)]
        assert _unmont(spec, field, t.cpu().numpy()) == want, f"u1 = {u1:#x}, u2 = {u2:#x}"


def test_spmv_long_row_list_overflow(L, oracle, spec):
    """more than 4096 rows longer than 1024 non-zeros: the rows past the long-row list's capacity are walked by the thread
    that met them (fold.cu, spmv_kernel), the listed ones by a CTA each; against oracle.spmv"""
    import torch
    lib = L._capi.lib()
    field = 2
    rng = np.random.default_rng(77)
    n = 6000
    lens = np.concatenate([rng.integers(1025, 1100, size=4300), rng.integers(0, 10, size=3000)])
    lens = lens[rng.permutation(lens.size)]
    rows = lens.size
    assert (lens > 1024).sum() > 4096
    row_ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    nnz = int(row_ptr[-1])
    col = rng.integers(0, n, size=nnz).astype(np.uint32)
    val = random_elements(field, nnz, seed=5)
    z = random_elements(field, n, seed=6, shape="edge")
    d_rp, d_col, d_val, dz = _dev(row_ptr), _dev(col), _dev(val), _dev(_mont(spec, field, z))
    L._capi.check(lib.lurk_convert_dev(field, d_val.data_ptr(), nnz, L.FMT_MONTGOMERY, d_val.data_ptr(), None))
    y = torch.empty(rows * 32, dtype=torch.uint8, device="cuda")
    L._capi.check(lib.lurk_spmv_csr_dev(field, d_rp.data_ptr(), d_col.data_ptr(), d_val.data_ptr(), rows, dz.data_ptr(), y.data_ptr(), None))
    L._capi.check(lib.lurk_convert_dev(field, y.data_ptr(), rows, L.FMT_CANONICAL, y.data_ptr(), None))
    assert np.array_equal(y.cpu().numpy(), oracle.spmv(field, row_ptr, col, val, z, nthreads=8))
