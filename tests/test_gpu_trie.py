"""The trie coprocessor's lookup and insert witnesses on the GPU (csrc/trie.cu) against the oracle's restatement
(tests/trie_gadget_oracle.py), byte for byte: host and device batches, both formats, every field, H = 85 and H = 1..3 at
call counts around a warp and one past the pick kernel's grid-stride boundary; the goldens G1-G5 and G10 in
device-written blocks; every inconsistent path refused with its call and level; scatter at non-contiguous offsets; two
host threads at once; and fold contexts whose step circuits are the oracle's R1CS of lookup and insert calls, on Nova
(BN254 and Pallas) and on SuperNova with the two circuits at two circuit indices."""
import json
import os
import random
import threading

import numpy as np
import pytest
import torch

import trie_gadget_oracle as T
from oracle import nifs
from util import ints, pack

pytestmark = pytest.mark.gpu
FIELDS = [0, 1, 2, 3]
OPS = [T.LOOKUP, T.INSERT]
R = 1 << 256
DISTINCT = 4
_CACHE = {}
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_goldens.json")))["poseidon_digests"]


def _sets(field, op, H):
    """DISTINCT consistent calls (keys 0, p - 1 and random, over a trie with two inserted keys) and their oracle blocks
    as (DISTINCT, block, 32) uint8, canonical"""
    key = (field, op, H)
    if key not in _CACHE:
        p = T.spec.FIELD_MODULUS[field]
        rng = random.Random(1000 * field + 10 * H + op)
        t = T.SpecTrie(field, H)
        for k in (rng.randrange(p), rng.randrange(p)):
            t.insert_inputs(k, rng.randrange(p))
        keys = [0, p - 1] + [rng.randrange(p) for _ in range(DISTINCT - 2)]
        calls = [t.insert_inputs(k, rng.randrange(p)) if op == T.INSERT else t.lookup_inputs(k) for k in keys]
        blocks = np.stack([pack(T.witness(field, op, c)).reshape(-1, 32) for c in calls])
        _CACHE[key] = (calls, blocks)
    return _CACHE[key]


def _fmt(field, vals, fmt):
    p = T.spec.FIELD_MODULUS[field]
    return pack([v * R % p if fmt else v for v in vals])


def _mont(field, blocks):
    p = T.spec.FIELD_MODULUS[field]
    cache = {}
    return pack([cache.setdefault(v, v * R % p) for v in ints(blocks.reshape(-1))]).reshape(blocks.shape)


def _expected(field, op, H, fmt):
    calls, blocks = _sets(field, op, H)
    key = (field, op, H, fmt)
    if key not in _CACHE:
        _CACHE[key] = torch.from_numpy(_mont(field, blocks) if fmt else blocks).cuda()
    return calls, _CACHE[key]


def _pick(count, seed):
    return np.random.default_rng(seed).integers(0, DISTINCT, size=count)


def _inputs(field, calls, pick, fmt):
    return np.concatenate([_fmt(field, calls[k], fmt) for k in pick])


def _chk(L, rc):
    L._capi.check(rc)


def _grid_boundary_calls(H):
    """calls at which the pick kernel's items (H + 1 per call) first exceed one pass of its grid: SMs x 2 CTAs x 128"""
    return torch.cuda.get_device_properties(0).multi_processor_count * 2 * 128 // (H + 1) + 1


def _run_both(L, field, op, H, fmt, calls, want, pick):
    lib = L._capi.lib()
    count = len(pick)
    blk = L.trie_witness_block(field, op, H)
    src = _inputs(field, calls, pick, fmt)
    host = L.trie_witness_batch(field, op, H, src, fmt=fmt)
    exp = want[torch.from_numpy(pick).cuda()]
    assert torch.equal(torch.from_numpy(host).cuda().view(count, blk, 32), exp), f"host batch, count {count}"
    d_in = torch.from_numpy(src).cuda()
    out = torch.full((count * blk * 32,), 0xA5, dtype=torch.uint8, device="cuda")
    _chk(L, lib.lurk_trie_witness_batch_dev(field, op, H, d_in.data_ptr(), count, out.data_ptr(), fmt, None))
    torch.cuda.synchronize()
    assert torch.equal(out.view(count, blk, 32), exp), f"device batch, count {count}"


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("H", [1, 2, 3])
@pytest.mark.parametrize("fmt", [0, 1])
def test_small_heights_match_the_oracle(L, field, op, H, fmt):
    calls, want = _expected(field, op, H, fmt)
    assert want.shape[1] == L.trie_witness_block(field, op, H)
    for count in (1, 31, 32, 33):
        _run_both(L, field, op, H, fmt, calls, want, _pick(count, count + 7 * H + field))


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("fmt", [0, 1])
def test_standard_height_matches_the_oracle(L, field, op, fmt):
    calls, want = _expected(field, op, 85, fmt)
    _run_both(L, field, op, 85, fmt, calls, want, np.array([0, 3, 1], dtype=np.int64))


@pytest.mark.parametrize("field,op,H", [(0, T.LOOKUP, 1), (1, T.INSERT, 1), (2, T.LOOKUP, 3), (3, T.INSERT, 3)])
def test_past_the_grid_stride_boundary(L, field, op, H):
    lib = L._capi.lib()
    fmt = field % 2
    calls, want = _expected(field, op, H, fmt)
    blk = L.trie_witness_block(field, op, H)
    count = _grid_boundary_calls(H)
    pick = _pick(count, field)
    d_in = torch.from_numpy(_inputs(field, calls, pick, fmt)).cuda()
    out = torch.empty((count, blk, 32), dtype=torch.uint8, device="cuda")
    _chk(L, lib.lurk_trie_witness_batch_dev(field, op, H, d_in.data_ptr(), count, out.data_ptr(), fmt, None))
    torch.cuda.synchronize()
    assert torch.equal(out, want[torch.from_numpy(pick).cuda()])


def test_goldens_in_device_written_blocks(L):
    """an empty StandardTrie (PoseidonCache on the GPU): G1..G4 are the digests of levels 84..81 and G5 of level 0; the
    insert 123 -> 456 ends in G10, and a lookup of 123 afterwards selects 456"""
    g = {k: int(v["hex"], 16) for k, v in GOLD.items()}
    field, H = 0, 85
    S = T.slot_len(field)
    t = L.StandardTrie()
    root0 = t.root
    blk = ints(L.trie_witness_batch(field, L.TRIE_LOOKUP, H, pack(L.lookup_inputs(root0, 123, t.prove_lookup(123)))))
    for level, name in ((84, "G1"), (83, "G2"), (82, "G3"), (81, "G4"), (0, "G5")):
        assert blk[T.level_at(field, H, level) + S - 1] == g[name], name
    proof, inserted = t.prove_insert(123, 456)
    assert inserted
    blk = ints(L.trie_witness_batch(field, L.TRIE_INSERT, H, pack(L.insert_inputs(root0, 123, 456, proof))))
    assert blk[-1] == g["G10"] == t.root
    blk = ints(L.trie_witness_batch(field, L.TRIE_LOOKUP, H, pack(L.lookup_inputs(t.root, 123, t.prove_lookup(123)))))
    assert blk[0] == g["G10"] and blk[-1] == 456


@pytest.mark.parametrize("field", [0, 2])
def test_inconsistent_paths_are_refused(L, field):
    H = 3
    p = T.spec.FIELD_MODULUS[field]
    for op in OPS:
        calls, _ = _sets(field, op, H)
        first = 3 if op == T.INSERT else 2

        def refused(call, pos, delta):
            cs = [list(c) for c in calls]
            cs[call][pos] = (cs[call][pos] + delta) % p
            with pytest.raises(L.LurkError) as e:
                L.trie_witness_batch(field, op, H, np.concatenate([pack(c) for c in cs]))
            assert e.value.code == L._capi.ERR_ARG
            return str(e.value)

        assert "call 2 level 0" in refused(2, 0, 1)                      # the root
        key = calls[1][1]
        k1 = T.path_index(key, H, 1)
        other = first + 8 * 1 + (k1 + 1) % 8                             # an element level 1 does not select
        assert "call 1 level 1" in refused(1, other, 5)
        k0 = T.path_index(calls[3][1], H, 0)
        assert "call 3 level 0" in refused(3, first + k0, 1)              # level 0's preimage no longer hashes to the root
        if op == T.INSERT:
            msg = refused(0, 2, 1)                                        # the value: only the new leaf disagrees
            assert f"call 0 level {H - 1}" in msg and "value" in msg
            new_first = first + 8 * H
            msg = refused(2, new_first + T.path_index(calls[2][1], H, 0), 1)   # new level 0's selection
            assert "call 2 level 0" in msg and "new path" in msg


def test_inputs_not_below_p_are_refused(L):
    p = T.spec.FIELD_MODULUS[0]
    calls, _ = _sets(0, T.LOOKUP, 1)
    bad = list(calls[0])
    bad[5] = p
    with pytest.raises(L.LurkError) as e:
        L.trie_witness_batch(0, T.LOOKUP, 1, pack(bad))
    assert e.value.code == L._capi.ERR_RANGE


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("op", OPS)
def test_scatter_leaves_everything_else_untouched(L, field, op):
    lib = L._capi.lib()
    fmt, H = 1, 2
    calls, want = _expected(field, op, H, fmt)
    blk = L.trie_witness_block(field, op, H)
    count = 33
    gaps = np.random.default_rng(field + op).integers(0, 50, size=count)
    order = np.random.default_rng(op).permutation(count)            # blocks land out of call order
    offs = np.zeros(count, dtype=np.uint64)
    pos = 3
    for k in order:
        offs[k] = pos
        pos += blk + int(gaps[k])
    total = pos + 11
    pick = _pick(count, 99 + field)
    d_in = torch.from_numpy(_inputs(field, calls, pick, fmt)).cuda()
    W = torch.full((total, 32), 0x5C, dtype=torch.uint8, device="cuda")
    d_off = torch.from_numpy(offs.astype(np.int64)).cuda()
    _chk(L, lib.lurk_trie_witness_scatter_dev(field, op, H, d_in.data_ptr(), count, d_off.data_ptr(), W.data_ptr(), fmt, None))
    torch.cuda.synchronize()
    mask = torch.zeros(total, dtype=torch.bool, device="cuda")
    for k in range(count):
        o = int(offs[k])
        assert torch.equal(W[o:o + blk], want[int(pick[k])]), f"block {k}"
        mask[o:o + blk] = True
    assert bool((W[~mask] == 0x5C).all())


def test_two_host_threads(L):
    results, errors = {}, []
    jobs = ((0, T.LOOKUP, 3), (2, T.INSERT, 2))

    def run(field, op, H):
        try:
            calls, blocks = _sets(field, op, H)
            pick = _pick(40, field)
            got = L.trie_witness_batch(field, op, H, _inputs(field, calls, pick, 0))
            results[(field, op, H)] = np.array_equal(got.reshape(40, -1, 32), blocks[pick])
        except Exception as ex:      # noqa: BLE001 -- reported below
            errors.append(ex)

    for j in jobs:
        _sets(*j)
    ts = [threading.Thread(target=run, args=j) for j in jobs]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors and results == {j: True for j in jobs}


# ---------------------------------------------------------------------------------------------- fold contexts
GLUE = 4          # per frame: root, key, value, not_dummy
BASE_FIELD = {0: 1, 2: 3}   # witness field -> the commitment curve's base field (BN254 G1: Fq, Pallas: Fp)


def _circuit(L, oracle, curve, field, op, H, frames, bases=None):
    blk = L.trie_witness_block(field, op, H)
    per = GLUE + blk
    n_w, n_x = frames * per, 2
    A, B, Cm = [], [], []
    for f in range(frames):
        a, b, c = T.r1cs_rows(field, op, H, f * per + GLUE, f * per, f * per + 1, f * per + 3, n_w)
        A += a; B += b; Cm += c
    mats = [nifs.rows_to_csr(A), nifs.rows_to_csr(B), nifs.rows_to_csr(Cm)]
    return dict(mats=mats, n_w=n_w, n_x=n_x, per=per, rows=len(A), frames=frames, op=op, H=H, field=field)


def _context(L, c, curve, ck, depth=1):
    ctx = L.NovaFoldContext(curve, ck, c["n_w"], c["n_x"], c["mats"], depth=depth)
    bi = ctx.add_trie_batch(c["op"], c["H"], [f * c["per"] + GLUE for f in range(c["frames"])])
    ctx.set_spans([(0, GLUE, c["per"], c["frames"])])
    return ctx, bi


def _step_calls(c, trie, rng):
    """one step's calls (each frame one call on the shared trie) -> (glue per frame, inputs per frame, W)"""
    p = T.spec.FIELD_MODULUS[c["field"]]
    glue, ins, W = [], [], []
    for _ in range(c["frames"]):
        key, value = rng.randrange(p), rng.randrange(p)
        x = trie.insert_inputs(key, value) if c["op"] == T.INSERT else trie.lookup_inputs(key)
        g = [x[0], key, value if c["op"] == T.INSERT else 0, 1]
        glue.append(g)
        ins.append(x)
        W += g + T.witness(c["field"], c["op"], x)
    return glue, ins, W


def _fill(ctx, b, bi, glue, ins, X2, resident, p, c):
    ctx.host_buffer(b, -2)[:] = pack(X2)
    ro = np.zeros((24, 32), dtype=np.uint8)
    for pos, v in ((4, X2[0]), (5, X2[1])):
        ro[pos] = pack([v])
    ctx.host_buffer(b, -3)[:] = ro.reshape(-1)
    flat_in = [x for s in ins for x in s]
    flat_glue = [x for g in glue for x in g]
    if not resident:
        ctx.host_buffer(b, bi)[:] = pack(flat_in)
        ctx.host_buffer(b, -1)[:] = pack(flat_glue)
        return
    ctx.sync()
    ctx.device_view(b, bi).copy_(torch.from_numpy(pack([x * R % p for x in flat_in])).cuda())
    w2 = ctx.device_view(b, -4).view(-1, 32)
    for f, g in enumerate(glue):
        w2[f * c["per"]:f * c["per"] + GLUE] = torch.from_numpy(pack([x * R % p for x in g]).reshape(-1, 32)).cuda()
    w2[c["n_w"] + 1:c["n_w"] + 1 + c["n_x"]] = torch.from_numpy(pack([x * R % p for x in X2]).reshape(-1, 32)).cuda()
    # the step's RO constants, Montgomery form in the commitment curve's base field
    q = T.spec.FIELD_MODULUS[BASE_FIELD[c["field"]]]
    ro = [0] * 24
    ro[4], ro[5] = X2
    ctx.device_view(b, -3).copy_(torch.from_numpy(pack([x * R % q for x in ro])).cuda())
    torch.cuda.synchronize()


@pytest.mark.parametrize("curve,field", [(0, 0), (2, 2)])
@pytest.mark.parametrize("op", OPS)
def test_nova_fold_with_trie_blocks(L, oracle, curve, field, op):
    """four steps of two calls each (the last with device-resident inputs); the fresh W of every step is the oracle's and
    the folded instance satisfies the relaxed R1CS, on the context and on the oracle"""
    H = 2
    c = _circuit(L, oracle, curve, field, op, H, frames=2)
    p = T.spec.FIELD_MODULUS[field]
    bases = oracle.gen_bases(curve, max(c["n_w"], c["rows"]))
    ck = L.CommitmentKey(curve, bases)
    ctx, bi = _context(L, c, curve, ck)
    o = nifs.NovaOracle(curve, bases, c["mats"], c["n_w"], c["n_x"])
    rng = random.Random(5 + op + curve)
    trie = T.SpecTrie(field, H)
    for step in range(4):
        glue, ins, W = _step_calls(c, trie, rng)
        X2 = [rng.randrange(1 << 64), rng.randrange(1 << 64)]     # below both fields of the cycle
        _fill(ctx, 0, bi, glue, ins, X2, step == 3, p, c)
        if step == 3:
            ctx.stage_a(0, resident=True)
        else:
            ctx.stage_a(0)
        got = [v * pow(R, -1, p) % p for v in ints(ctx.read_device(0, -4))[:c["n_w"]]]
        assert got == W, f"step {step}: fresh W"
        if step == 0:
            ctx.init_running(0)
            o.init_running(pack(W), X2)
        else:
            ctx.stage_b_launch(0)
            o.prove_step(pack(W), X2)
        ctx.collect(0)
    run = ctx.get_running()
    assert np.array_equal(run["W"], o.W) and np.array_equal(run["E"], o.E)
    assert o.bad_rows(run["W"], run["E"], ints(run["u"])[0], ints(run["X"])) == 0
    assert ctx.check_running() == (0, True, True)
    ctx.close()


def test_supernova_lookup_and_insert_circuits(L, oracle):
    """SuperNova with the insert circuit at index 0 and the lookup circuit at index 1, stepped alternately on one trie:
    both running instances stay satisfied"""
    curve, field, H = 0, 0, 2
    p = T.spec.FIELD_MODULUS[field]
    cs = [_circuit(L, oracle, curve, field, T.INSERT, H, frames=1), _circuit(L, oracle, curve, field, T.LOOKUP, H, frames=1)]
    bases = oracle.gen_bases(curve, max(max(c["n_w"], c["rows"]) for c in cs))
    ck = L.CommitmentKey(curve, bases)
    ctxs = [L.NovaFoldContext(curve, ck, c["n_w"], c["n_x"], c["mats"], depth=2) for c in cs]
    nivc = L.SuperNovaFoldContext(ctxs)
    bis = [nivc.add_trie_batch(i, c["op"], H, [GLUE]) for i, c in enumerate(cs)]
    for ctx, c in zip(ctxs, cs):
        ctx.set_spans([(0, GLUE, c["per"], 1)])
    orc = [nifs.NovaOracle(curve, bases, c["mats"], c["n_w"], c["n_x"]) for c in cs]
    started = [False, False]
    rng = random.Random(77)
    trie = T.SpecTrie(field, H)
    for s, ci in enumerate([0, 1, 0, 1, 1, 0]):
        c = cs[ci]
        glue, ins, W = _step_calls(c, trie, rng)
        X2 = [rng.randrange(p), rng.randrange(p)]
        b = nivc._next[ci]
        _fill(ctxs[ci], b, bis[ci], glue, ins, X2, False, p, c)
        assert nivc.stage_a(ci) == b
        nivc.fold(ci, b)
        nivc.collect(ci, b)
        if not started[ci]:
            orc[ci].init_running(pack(W), X2)
            started[ci] = True
        else:
            orc[ci].prove_step(pack(W), X2)
    for ci, ctx in enumerate(ctxs):
        run = ctx.get_running()
        assert np.array_equal(run["W"], orc[ci].W) and np.array_equal(run["E"], orc[ci].E), f"circuit {ci}"
        assert orc[ci].bad_rows(run["W"], run["E"], ints(run["u"])[0], ints(run["X"])) == 0
        assert ctx.check_running() == (0, True, True)
