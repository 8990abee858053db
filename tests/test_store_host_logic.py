"""CPU tests of the HOST logic of the store, trie and slot mirrors (interning, children-first flattening into lurk_dag_node
tables, commitments) against the reference's goldens.  There is no GPU here, so the device entry points the mirrors
call are replaced -- in this test module only -- by a stand-in that hands the very same buffers to the oracle; what
is under test is everything the mirror does before and after that call.  The same expressions run against the real
library in tests/test_gpu_dag_fold.py."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_dag_fold import _StoreExprs
from util import GOLDEN


class _OracleBackedLib:
    """stand-in for liblurk_b200 exposing only lurk_dag_hash and lurk_poseidon_hash_batch with the C-ABI's argument order"""

    def __init__(self, oracle):
        self.o = oracle
        self.dag_calls = 0

    @staticmethod
    def _view(ptr, nbytes):
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(nbytes,)) if nbytes else np.zeros(0, np.uint8)

    def lurk_dag_hash(self, field, nodes, n, atoms, n_atoms, out):
        self.dag_calls += 1
        nodes_a = self._view(nodes, n * self.o.DAG_NODE.itemsize).view(self.o.DAG_NODE)
        self._view(out, n * 32)[:] = self.o.dag_hash(field, nodes_a, self._view(atoms, n_atoms * 32))
        return 0

    def lurk_poseidon_hash_batch(self, field, arity, pre, n, out):
        self._view(out, n * 32)[:] = self.o.poseidon_hash_batch(field, arity, self._view(pre, n * arity * 32))
        return 0

    def lurk_poseidon_witness_batch(self, field, arity, pre, n, blocks, fmt):
        assert fmt == 0
        w = self.o.poseidon_witness_batch(field, arity, self._view(pre, n * arity * 32))
        self._view(blocks, w.size)[:] = w
        return 0

    def lurk_bitdecomp_witness_batch(self, field, vals, n, blocks, fmt):
        assert fmt == 0
        w = self.o.bitdecomp_witness_batch(field, self._view(vals, n * 32))
        self._view(blocks, w.size)[:] = w
        return 0

    def __getattr__(self, name):
        # host-only entry points (block sizes, constants) need no GPU: the real library answers them
        if name in ("lurk_poseidon_witness_block", "lurk_bitdecomp_witness_block", "lurk_poseidon_constants", "lurk_last_error"):
            return getattr(self._real, name)
        raise AttributeError(f"{name}: a device entry point this CPU test does not stand in for")


@pytest.fixture()
def HL(monkeypatch, oracle):
    import lurk_beta_b200 as L
    from lurk_beta_b200 import _capi
    fake = _OracleBackedLib(oracle)
    fake._real = _capi.lib()
    monkeypatch.setattr(_capi, "lib", lambda: fake)
    L._fake = fake
    return L


def test_claim_golden_through_store_flattening(HL):
    e = _StoreExprs(HL)
    expr = e.lst([e.sym("lurk", "+"), e.num(1), e.num(1)])
    claim = e.claim(expr, e.env0, e.num(2), e.env0)
    assert e.s.hide(0, claim) == GOLDEN["G11"]
    assert HL._fake.dag_calls == 1                      # the whole claim DAG went down in one call
    assert e.s.hide(0, claim) == GOLDEN["G11"] and HL._fake.dag_calls == 1   # z_cache hit, nothing re-hashed


def test_functional_commitment_goldens_through_store_flattening(HL):
    e = _StoreExprs(HL)
    s = e.s
    pair = e.cons(e.num(13), e.num(21))
    assert s.hide(0, pair) == GOLDEN["G13"] and s.hide(12345, pair) == GOLDEN["G14"]
    assert s.open(GOLDEN["G14"]) == (12345, pair)
    x, plus, mul = e.sym("lurk", "user", "x"), e.sym("lurk", "+"), e.sym("lurk", "*")
    body = e.lst([plus, e.lst([mul, e.num(3), e.lst([mul, x, x])]), e.lst([plus, e.lst([mul, e.num(9), x]), e.num(2)])])
    fun = s.intern_tuple4([e.lst([x]), body, e.env0, s.intern_atom(e.NIL, 0)], e.FUN)
    comm = s.hide(0, fun)
    assert comm == GOLDEN["G16"]
    env = s.intern_compact([e.sym("lurk", "user", "f"), fun, e.env0], e.ENV)
    expr = e.lst([e.lst([e.sym("lurk", "open"), e.num(comm)]), e.num(5)])
    # children hashed by the earlier calls (the Fun, symbol paths) travel as extra digests, not as nodes
    assert s.hide(0, e.claim(expr, env, e.num(122), e.env0)) == GOLDEN["G17"]


def test_hydrate_queue_matches_on_demand_hashing(HL):
    """hydrate_z_cache over the interning-ordered queue (store_core.rs:266-269) and on-demand hash_ptr give equal digests"""
    a, b = _StoreExprs(HL), _StoreExprs(HL)
    mk = lambda e: e.lst([e.sym("lurk", "user", "abc"), e.num(7), e.lst([e.num(1), e.key("k")])])
    pa, pb = mk(a), mk(b)
    a.s.hydrate_z_cache()
    assert not a.s.dehydrated and a.s.z_cache[pa[1]] == b.s.hash_ptr(pb)[1]


def test_random_dags_match_recursive_hashing(HL, oracle):
    """random hash-consed DAGs (all five node kinds, shared sub-terms, several hydration calls so that later batches refer to
    earlier digests) through the mirror's flattening == plain recursive hashing with the oracle"""
    import random
    from util import ints, pack
    rng = random.Random(0x6c75726b)
    H = lambda pre: ints(oracle.poseidon_hash_batch(0, len(pre), pack(pre)))[0]
    for trial in range(4):
        s = HL.StoreCore(HL.FIELD_BN254_FR)
        ptrs, want = [], {}                      # ptr -> digest by direct recursion

        def digest(p):
            return want[p] if p[1][0] != "atom" else s.fetch_digest(p[1][1])

        for i in range(12):
            v = rng.randrange(1 << 200)
            p = s.intern_atom(rng.randrange(15), v)
            ptrs.append(p)
        for step in range(120):
            kind = rng.choice(["tuple2", "tuple3", "tuple4", "compact"])
            tag = rng.randrange(15)
            k = {"tuple2": 2, "tuple3": 3, "tuple4": 4, "compact": 3}[kind]
            ch = [rng.choice(ptrs[-30:] if rng.random() < 0.7 else ptrs) for _ in range(k)]
            p = getattr(s, "intern_" + kind)(ch, tag)
            if kind == "compact":
                want[p] = H([digest(ch[0]), ch[1][0], digest(ch[1]), digest(ch[2])])
            else:
                want[p] = H([x for c in ch for x in (c[0], digest(c))])
            ptrs.append(p)
            if step % 37 == 36:                  # hydrate part-way: later nodes refer to already cached digests
                s.hydrate_z_cache()
        probe = [p for p in ptrs if p[1][0] != "atom"]
        rng.shuffle(probe)
        for p in probe[:40]:
            assert s.hash_ptr(p) == (p[0], want[p])
        s.hydrate_z_cache()
        assert all(s.z_cache[p[1]] == want[p] for p in probe)
        # commitments on top (hash3 of secret, tag, digest)
        p = probe[0]
        assert s.hide(77, p) == H([77, p[0], want[p]])


def test_trie_mirror_goldens_and_lookup_witnesses(HL, oracle):
    """trie coprocessor mirror (src/coprocessor/trie/mod.rs): empty roots G1..G5, root after insert G10, lookups, and the 85
    arity-8 slot witnesses of one lookup circuit handed over as ONE batch"""
    from util import pack
    pc = HL.PoseidonCache(HL.FIELD_BN254_FR)
    small = HL.Trie(pc, 8, 3)
    assert [small.empty_root_for_height(h) for h in (1, 2, 3)] == [GOLDEN["G1"], GOLDEN["G2"], GOLDEN["G3"]]
    assert small.path(500) == [7, 6, 4]                                  # test_path, trie/mod.rs
    t = HL.StandardTrie(pc)
    assert t.empty_root() == GOLDEN["G5"]
    assert t.lookup(123) is None
    assert t.insert(123, 456) and t.root == GOLDEN["G10"]
    assert t.lookup(123) == 456 and t.lookup(124) is None
    assert not t.insert(123, 456)                                        # same value: root unchanged
    w = t.lookup_circuit_witnesses(123)
    pre = pack([x for p in t.prove_lookup_at_path(t.path(123)) for x in p])
    assert w.size == 85 * 396 * 32 and np.array_equal(w, oracle.poseidon_witness_batch(0, 8, pre))
    with pytest.raises(KeyError, match="MissingPreimage"):
        HL.StandardTrie(pc, root=12345).lookup(1)


def test_generate_slots_witnesses_order_and_dummies(HL, oracle):
    """frame order is preserved, one batch per slot type, all `None` slots of a type share the zero-preimage witness
    (src/lem/multiframe.rs:520-592)"""
    from util import ints, pack
    S = HL.SlotType
    slots = [(S.Hash4, [1, 2, 3, 4]), (S.Hash4, None), (S.Hash8, list(range(8))), (S.Commitment, [9, 4, 7]), (S.BitDecomp, [5]),
             (S.Hash4, None), (S.Hash8, None), (S.BitDecomp, None), (S.Hash4, [4, 3, 2, 1])]
    got = HL.generate_slots_witnesses(0, slots)
    assert len(got) == len(slots)
    for (st, pre), blk in zip(slots, got):
        a = st.preimg_size()
        row = pack(pre if pre is not None else [0] * a)
        want = oracle.bitdecomp_witness_batch(0, row) if st is S.BitDecomp else oracle.poseidon_witness_batch(0, a, row)
        assert np.array_equal(blk, want), (st, pre)
        assert blk.size == HL.compute_witness_size(st, 0) * 32
    assert got[1] is not got[0] and np.array_equal(got[1], got[5])
    assert ints(got[0])[:4] == [1, 2, 3, 4] and ints(got[8])[:4] == [4, 3, 2, 1]     # block = preimage | aux | digest
    with pytest.raises(ValueError):
        HL.generate_slots_witnesses(0, [(S.Hash4, [1, 2, 3])])


def test_chained_commitment_goldens_through_store_flattening(HL):
    """G18..G21 through the store mirror: nested compact Env nodes, a Rec (tuple4 digest under another tag) and a Comm-tagged
    output, hashed in a handful of lurk_dag_hash calls that reuse earlier digests"""
    REC, COMM = 13, 8
    e = _StoreExprs(HL)
    s = e.s
    counter, x, add = e.sym("lurk", "user", "counter"), e.sym("lurk", "user", "x"), e.sym("lurk", "user", "add")
    let, plus, cons_, commit = e.sym("lurk", "let"), e.sym("lurk", "+"), e.sym("lurk", "cons"), e.sym("lurk", "commit")
    body = e.lst([let, e.lst([e.lst([counter, e.lst([plus, counter, x])])]),
                  e.lst([cons_, counter, e.lst([commit, e.lst([add, counter])])])])
    foo = s.intern_atom(e.NIL, 0)
    fun2 = s.intern_tuple4([e.lst([counter, x]), body, e.env0, foo], e.FUN)
    rec = (REC, fun2[1])                                        # cast(result, Expr::Rec): same node, other tag
    rec_env = s.intern_compact([add, rec, e.env0], e.ENV)

    def head(c):
        env = s.intern_compact([counter, e.num(c), rec_env], e.ENV)
        return s.hide(0, s.intern_tuple4([e.lst([x]), body, env, foo], e.FUN))

    c0, c1, c2 = head(0), head(9), head(21)
    assert (c0, c1, c2) == (GOLDEN["G18"], GOLDEN["G19"], GOLDEN["G20"])
    expr = e.lst([e.lst([e.sym("lurk", "open"), e.num(c0)]), e.num(9)])
    out = e.cons(e.num(9), s.intern_atom(COMM, c1))
    assert s.hide(0, e.claim(expr, e.env0, out, e.env0)) == GOLDEN["G21"]


def test_hydration_plan_routes_chains_to_the_cpu_and_wide_dags_to_the_gpu(L):
    """lurk_dag_hash_plan (host only): a 2000-deep cons chain is one dependent hash per level -- slower on the GPU than one
    CPU core -- so the plan keeps it on the caller's CPU path; a wide store
    goes to the GPU.  Malformed input is rejected as by lurk_dag_hash."""
    import ctypes as C
    import numpy as np
    from lurk_beta_b200 import _capi
    lib = _capi.lib()
    node_t = np.dtype([("kind", "u1"), ("reserved", "u1"), ("tag", "<u2", (4,)), ("child", "<u4", (4,))], align=True)
    n_atoms = 16
    chain = np.zeros(2000, dtype=node_t)
    chain["kind"] = 2
    chain["child"][:, 0] = np.maximum(n_atoms + np.arange(2000) - 1, 0)
    chain["child"][0, 0] = 0
    plan = _capi.DagPlan()
    _capi.check(lib.lurk_dag_hash_plan(_capi.np_ptr(chain), 2000, n_atoms, C.byref(plan)))
    assert (plan.nodes, plan.levels, plan.max_width, plan.use_gpu) == (2000, 2000, 1, 0)
    wide = np.zeros(1 << 16, dtype=node_t)
    wide["kind"] = 4
    wide["child"] = np.random.default_rng(0).integers(0, n_atoms, size=(1 << 16, 4))
    _capi.check(lib.lurk_dag_hash_plan(_capi.np_ptr(wide), 1 << 16, n_atoms, C.byref(plan)))
    assert (plan.levels, plan.max_width, plan.use_gpu) == (1, 1 << 16, 1)
    chain["child"][5, 0] = n_atoms + 9                      # forward reference
    assert lib.lurk_dag_hash_plan(_capi.np_ptr(chain), 2000, n_atoms, C.byref(plan)) == _capi.ERR_ORDER
