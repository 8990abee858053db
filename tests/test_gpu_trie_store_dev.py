"""The device-resident forms of the trie store (lurk_trie_ctx_apply_dev / _register_dev, trie.DeviceTrie.apply_dev /
register_dev), whose batch is planned on the GPU, against the host form on a twin context and against the host mirror
`Trie`: results, proof bytes in both formats and node counts, on all four fields at H = 1, 2, 3 and 85; versions,
forks from stored roots, chains continued across batches that mix both forms; batch sizes around a CTA and the digest
launch's 8192-sponge boundary; 10^5 random operations.  Every refusal class at the first, a middle and the last operation
it can sit at gives the host form's code and operation, and leaves the store, the node count and the caller's buffers
as they were, in both formats.  Also: inputs still being written on the caller's stream (with the insert count that
sizes the proofs read there too), register_dev, the witness kernel fed from apply_dev's proofs, two host threads, and
the Python checks of the caller's tensors (exact proof-buffer sizes, the store's device)."""
import random
import re
import threading

import numpy as np
import pytest
import torch

from oracle import spec
from test_gpu_trie_store import INS, LOOK, OracleHash, _dense, _fmt_ops, _from, _split, _to, gen_ops, mirror
from util import ints, pack

pytestmark = pytest.mark.gpu
SENTINEL = 0xA5


def dev_ops(ops, roots=True, values=True):
    """(kinds, prev, roots, keys, values) CUDA tensors of ops (ints as given, so elements >= p stay unreduced)"""
    n = len(ops)
    col = lambda k: torch.from_numpy(pack([int(o[k]) for o in ops]).reshape(n, 32)).cuda() if n else torch.empty((0, 32), dtype=torch.uint8, device="cuda")
    kinds = torch.tensor([o[0] for o in ops], dtype=torch.int32, device="cuda")
    prev = torch.tensor([o[1] for o in ops], dtype=torch.int64, device="cuda")
    return kinds, prev, col(2) if roots else None, col(3), col(4) if values else None


def run_dev(dt, ops, fmt=0):
    """apply_dev on ops given as ints (converted to fmt) -> (results as canonical ints, lookup proofs, insert proofs)"""
    field = dt.field_id
    res, look, ins = dt.apply_dev(*dev_ops(_fmt_ops(field, ops, fmt)), fmt=fmt)
    torch.cuda.synchronize()
    return _from(field, ints(res.cpu().numpy()), fmt), look, ins


def run_host(dt, ops, fmt=0):
    field = dt.field_id
    res, look, ins = dt.apply(_fmt_ops(field, ops, fmt), fmt=fmt)
    torch.cuda.synchronize()
    return _from(field, res, fmt), look, ins


def same(a, b):
    """two (results, lookup proofs, insert proofs) are equal byte for byte"""
    assert a[0] == b[0], "results"
    assert torch.equal(a[1].reshape(-1), b[1].reshape(-1)), "lookup proofs"
    assert torch.equal(a[2].reshape(-1), b[2].reshape(-1)), "insert proofs"


def against_mirror(field, got, want, fmt):
    assert got[0] == want[0], "results against the mirror"
    for proofs, exp, name in ((got[1], want[1], "lookup"), (got[2], want[2], "insert")):
        exp_b = torch.from_numpy(pack(_to(field, [x for call in exp for x in call], fmt))).cuda()
        assert torch.equal(proofs.reshape(-1), exp_b), f"{name} proofs against the mirror"


def twins(L, field, H, capacity):
    return L.DeviceTrie(field, H, capacity=capacity), L.DeviceTrie(field, H, capacity=capacity)


def both(host, dev, ops, fmt=0, want=None):
    """the same batch through apply on `host` and apply_dev on `dev`: equal outputs and node counts (and the mirror's)"""
    a, b = run_host(host, ops, fmt), run_dev(dev, ops, fmt)
    same(a, b)
    assert host.node_count == dev.node_count
    if want is not None:
        against_mirror(host.field_id, b, want, fmt)
    return b


@pytest.mark.parametrize("field", [0, 1, 2, 3])
@pytest.mark.parametrize("H", [1, 2, 3, 85])
def test_apply_dev_matches_apply_and_the_mirror(L, field, H):
    """two batches, the second starting chains from roots the first produced, in both formats"""
    p = spec.FIELD_MODULUS[field]
    rng = random.Random(100 * field + H)
    if H == 85:
        stem = rng.randrange(p >> 3) << 3
        keys = [stem + c for c in range(8)] + [rng.randrange(p) for _ in range(6)]
        key, value, n = (lambda: rng.choice(keys)), (lambda: rng.choice([0, 5, rng.randrange(p)])), 250
    else:
        (key, value), n = _dense(rng, field, H), 1500
    hashc, shared = OracleHash(field), {}
    empty = L.Trie(hashc, 8, H, inverse_cache=shared).root
    ops1 = gen_ops(rng, n, key, value, [empty], p_chain=0.02)
    want1 = mirror(L, hashc, shared, H, ops1)
    produced = [r for (k, *_), r in zip(ops1, want1[0]) if k == INS]
    ops2 = gen_ops(rng, n, key, value, [empty] + rng.sample(produced, 10), p_chain=0.05)
    want2 = mirror(L, hashc, shared, H, ops2)
    for fmt in (0, 1):
        host, dev = twins(L, field, H, 1 << 16)
        both(host, dev, ops1, fmt, want1)
        both(host, dev, ops2, fmt, want2)
        host.close(), dev.close()


def test_versions_forks_and_lookups_of_earlier_versions(L):
    field, H = 0, 2
    hashc, shared = OracleHash(field), {}
    e = L.Trie(hashc, 8, H, inverse_cache=shared).root
    ops = [(INS, -1, e, 1, 10), (INS, 0, 0, 2, 20), (INS, 1, 0, 1, 11), (LOOK, 0, 0, 1, 0), (LOOK, 1, 0, 2, 0), (LOOK, 2, 0, 1, 0),
           (INS, -1, e, 1, 30), (INS, -1, e, 1, 40), (LOOK, 6, 0, 1, 0), (LOOK, 7, 0, 1, 0), (LOOK, 0, 0, 2, 0), (INS, 6, 0, 9, 50)]
    want = mirror(L, hashc, shared, H, ops)
    assert [want[0][i] for i in (3, 4, 5, 8, 9, 10)] == [10, 20, 11, 30, 40, 0]
    host, dev = twins(L, field, H, 1024)
    both(host, dev, ops, 0, want)
    # forks from stored roots the first batch produced, and lookups of them
    ops2 = [(INS, -1, want[0][2], 2, 21), (INS, -1, want[0][2], 2, 22), (LOOK, 0, 0, 1, 0), (LOOK, 1, 0, 2, 0), (LOOK, -1, want[0][11], 9, 0),
            (LOOK, -1, want[0][0], 2, 0)]
    want2 = mirror(L, hashc, shared, H, ops2)
    assert want2[0][2:] == [11, 22, 50, 0]
    both(host, dev, ops2, 1, want2)


def test_chains_continued_across_batches_that_mix_both_forms(L):
    """one batch of 3000 operations against the same operations cut into batches applied alternately by apply and
    apply_dev on one context"""
    field, H = 1, 3
    rng = random.Random(5)
    key, value = _dense(rng, field, H)
    hashc, shared = OracleHash(field), {}
    e = L.Trie(hashc, 8, H, inverse_cache=shared).root
    ops = gen_ops(rng, 3000, key, value, [e], p_chain=0.01)
    want = mirror(L, hashc, shared, H, ops)
    whole = L.DeviceTrie(field, H, capacity=1 << 16)
    full = run_host(whole, ops)
    against_mirror(field, full, want, 0)
    mixed = L.DeviceTrie(field, H, capacity=1 << 16)
    rs, ls, is_ = [], [], []
    for k, batch in enumerate(_split(ops, full[0], sorted(rng.sample(range(1, 3000), 9)))):
        r, lo, i = (run_dev if k % 2 else run_host)(mixed, batch)
        rs += r
        ls.append(lo.reshape(-1))
        is_.append(i.reshape(-1))
    assert rs == full[0] and torch.equal(torch.cat(ls), full[1].reshape(-1)) and torch.equal(torch.cat(is_), full[2].reshape(-1))
    assert mixed.node_count == whole.node_count


def test_batch_sizes(L):
    """1 and a CTA (128) +- 1 inserts, and 8191 / 8192 / 8193: the arity-8 digest launch's warp kernel takes up to 8192
    sponges"""
    field, H = 2, 1
    hashc, shared = OracleHash(field), {}
    e = L.Trie(hashc, 8, H, inverse_cache=shared).root
    rng = random.Random(3)
    p = spec.FIELD_MODULUS[field]
    for n in (1, 127, 128, 129, 8191, 8192, 8193):
        # all inserts, in a few chains, so the number of hashes per level is n
        ops, last = [], {}
        for i in range(n):
            c = rng.randrange(4)
            ops.append((INS, last.get(c, -1), e, rng.randrange(16), rng.randrange(p)))
            last[c] = i
        want = mirror(L, hashc, shared, H, ops)
        host, dev = twins(L, field, H, n * H + 16)
        both(host, dev, ops, 0, want)
        host.close(), dev.close()


def test_a_hundred_thousand_random_operations(L):
    field, H, n = 0, 85, 100_000
    p = spec.FIELD_MODULUS[field]
    rng = random.Random(17)
    stems = [rng.randrange(p >> 3) << 3 for _ in range(64)]
    key = lambda: rng.choice(stems) + rng.randrange(8) if rng.random() < 0.5 else rng.randrange(p)
    value = lambda: rng.randrange(p)
    host, dev = twins(L, field, H, 6_000_000)
    ops = gen_ops(rng, n, key, value, [host.empty_root()], p_chain=0.001)
    both(host, dev, ops)
    both(host, dev, ops[:2000], 1)
    host.close(), dev.close()


# ------------------------------------------------------------------------------------------------------------- refusals
def _raw(L, dt, ops, dev, roots=True, values=True, fmt=0):
    """one call of lurk_trie_ctx_apply (dev False) or _apply_dev with every output pre-filled with SENTINEL -> (code,
    operation named or None, outputs unchanged)"""
    lib, per_l, per_i = L._capi.lib(), 2 + 8 * dt.height, 3 + 16 * dt.height
    n, n_ins = len(ops), sum(1 for o in ops if o[0] == INS)
    look = torch.full(((n - n_ins) * per_l * 32 + 32,), SENTINEL, dtype=torch.uint8, device="cuda")
    ins = torch.full((n_ins * per_i * 32 + 32,), SENTINEL, dtype=torch.uint8, device="cuda")
    if dev:
        k, pv, r, key, v = dev_ops(ops, roots, values)
        res = torch.full((n, 32), SENTINEL, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        rc = lib.lurk_trie_ctx_apply_dev(dt._ctx, n, k.data_ptr(), pv.data_ptr(), r.data_ptr() if r is not None else None, key.data_ptr(),
                                         v.data_ptr() if v is not None else None, fmt, res.data_ptr(), look.data_ptr(), ins.data_ptr(), None)
        res = res.cpu().numpy()
    else:
        ptr = L._capi.np_ptr
        kinds = np.array([o[0] for o in ops], dtype=np.int32)
        prev = np.array([o[1] for o in ops], dtype=np.int64)
        r, key, v = (pack([int(o[c]) for o in ops]) for c in (2, 3, 4))
        res = np.full(n * 32, SENTINEL, dtype=np.uint8)
        rc = lib.lurk_trie_ctx_apply(dt._ctx, n, ptr(kinds), ptr(prev), ptr(r) if roots else None, ptr(key), ptr(v) if values else None, fmt,
                                     ptr(res), look.data_ptr(), ins.data_ptr(), None)
    torch.cuda.synchronize()
    msg = lib.lurk_last_error().decode()
    m = re.search(r"trie operation (\d+):", msg)
    untouched = bool((res == SENTINEL).all()) and bool((look == SENTINEL).all()) and bool((ins == SENTINEL).all())
    return rc, int(m.group(1)) if m else None, untouched, msg


def _base(e, n=12):
    """a valid batch: two chains from e, lookups of their versions, a lookup of e; inserts at 0 and n - 1"""
    ops = [(INS, -1, e, 1, 10), (LOOK, 0, 0, 1, 0), (INS, 0, 0, 2, 20), (LOOK, -1, e, 3, 0), (INS, 2, 0, 3, 30), (INS, -1, e, 4, 40),
           (LOOK, 4, 0, 2, 0), (INS, 5, 0, 5, 50), (LOOK, 2, 0, 1, 0), (INS, 4, 0, 6, 60), (LOOK, 7, 0, 5, 0), (INS, 9, 0, 7, 70)]
    return ops[:n]


def _inject(cls, ops, pos, p, e, top_d):
    """ops with refusal class `cls` at operation pos (every earlier operation left valid), or None where it cannot sit"""
    ops = list(ops)
    k, prev, root, key, val = ops[pos]
    if cls == "kind":
        ops[pos] = (2, prev, root, key, val)
    elif cls == "prev_ahead":
        ops[pos] = (k, pos, root, key, val)
    elif cls == "prev_below":
        ops[pos] = (k, -2, root, key, val)
    elif cls == "prev_lookup":
        looks = [j for j in range(pos) if ops[j][0] == LOOK]
        if not looks:
            return None
        ops[pos] = (k, looks[-1], root, key, val)
    elif cls == "fork":
        # an insert j that an insert between j and pos already continued
        cont = [ops[j][1] for j in range(pos) if ops[j][0] == INS and ops[j][1] >= 0]
        if not cont:
            return None
        ops[pos] = (INS, cont[0], 0, key, 7)
    elif cls == "root":
        ops[pos] = (k, -1, p, key, val)
    elif cls == "key":
        ops[pos] = (k, prev, root, p + 1, val)
    elif cls == "value":
        ops[pos] = (INS, -1, e, key, p)
    elif cls == "missing_root":
        ops[pos] = (k, -1, 12345, key, val)
    elif cls == "missing_node":
        ops[pos] = (k, -1, top_d, 0, val)
    return ops


CLASSES = ["kind", "prev_ahead", "prev_below", "prev_lookup", "fork", "root", "key", "value", "missing_root", "missing_node"]


def _after(L, host, dev, e, counts):
    """the store and node counts are as before, and a follow-up batch gives the same on both"""
    assert (host.node_count, dev.node_count) == counts
    both(host, dev, [(INS, -1, e, 9, 90), (LOOK, 0, 0, 9, 0), (LOOK, -1, e, 9, 0)])


def test_every_refusal_matches_the_host_form(L):
    field, H = 0, 2
    p = spec.FIELD_MODULUS[field]
    hashc = OracleHash(field)
    host, dev = twins(L, field, H, 4096)
    e = host.empty_root()
    orphan_child = hashc.compute_hash([9] * 8)
    top_d = host.register([[orphan_child] + [0] * 7])[0]
    assert dev.register([[orphan_child] + [0] * 7])[0] == top_d
    checked = 0
    for cls in CLASSES:
        base = _base(e)
        places = [pos for pos in range(len(base)) if _inject(cls, base, pos, p, e, top_d) is not None]
        for pos in sorted({places[0], places[len(places) // 2], places[-1]}):
            ops = _inject(cls, base, pos, p, e, top_d)
            counts = (host.node_count, dev.node_count)
            a, b = _raw(L, host, ops, False), _raw(L, dev, ops, True)
            want_rc = L._capi.ERR_RANGE if cls.startswith("missing") else L._capi.ERR_ARG
            assert a[:2] == (want_rc, pos), (cls, pos, a[3])
            assert b[:3] == (want_rc, pos, True), (cls, pos, b[3])
            assert a[2], (cls, pos)
            _after(L, host, dev, e, counts)
            checked += 1
    assert checked >= 25
    # Montgomery input: reduction is checked on the bytes as given, before the conversion (which would reduce them)
    R = 1 << 256
    e_m = e * R % p
    for cls in ("root", "key", "value"):
        base = _fmt_ops(field, _base(e), 1)
        places = [pos for pos in range(len(base)) if _inject(cls, base, pos, p, e_m, None) is not None]
        for pos in sorted({places[0], places[len(places) // 2], places[-1]}):
            ops = _inject(cls, base, pos, p, e_m, None)
            counts = (host.node_count, dev.node_count)
            a, b = _raw(L, host, ops, False, fmt=1), _raw(L, dev, ops, True, fmt=1)
            assert a[:2] == (L._capi.ERR_ARG, pos) and b[:3] == (L._capi.ERR_ARG, pos, True) and cls in b[3], (cls, pos, a[3], b[3])
            _after(L, host, dev, e, counts)
    ok = _fmt_ops(field, _base(e), 1)
    assert _raw(L, dev, ok, True, fmt=1)[0] == 0 and _raw(L, host, ok, False, fmt=1)[0] == 0
    # NULL roots (read by operation 0, whose prev is always -1) and NULL values (read by the one insert)
    for ops, roots, values, pos in ((_base(e), False, True, 0),
                                    ([(LOOK, -1, e, 1, 0)] * 5 + [(INS, -1, e, 2, 3)] + [(LOOK, -1, e, 1, 0)] * 5, True, False, 5),
                                    ([(INS, -1, e, 2, 3)] + [(LOOK, -1, e, 1, 0)] * 5, True, False, 0),
                                    ([(LOOK, -1, e, 1, 0)] * 5 + [(INS, -1, e, 2, 3)], True, False, 5)):
        counts = (host.node_count, dev.node_count)
        a, b = _raw(L, host, ops, False, roots, values), _raw(L, dev, ops, True, roots, values)
        assert a[:2] == b[:2] == (L._capi.ERR_ARG, pos), (a[3], b[3])
        assert b[2] and ("roots" if not roots else "values") in b[3], b[3]
        _after(L, host, dev, e, counts)
    # two errors in one batch: the earlier operation wins, whatever the classes
    for (c1, p1), (c2, p2) in ((("key", 3), ("kind", 8)), (("kind", 3), ("key", 8)), (("fork", 6), ("prev_ahead", 9)),
                               (("missing_root", 2), ("missing_root", 7))):
        ops = _inject(c2, _inject(c1, _base(e), p1, p, e, top_d), p2, p, e, top_d)
        a, b = _raw(L, host, ops, False), _raw(L, dev, ops, True)
        assert a[:2] == b[:2] and a[1] == p1 and b[2], (c1, c2, a[3], b[3])
    # a missing root before an argument error: the argument error wins, as on the host
    ops = _inject("kind", _inject("missing_root", _base(e), 1, p, e, top_d), 10, p, e, top_d)
    a, b = _raw(L, host, ops, False), _raw(L, dev, ops, True)
    assert a[:2] == b[:2] == (L._capi.ERR_ARG, 10), (a[3], b[3])
    _after(L, host, dev, e, (host.node_count, dev.node_count))


def test_capacity_refusals(L):
    """the first insert that does not fit is named, at the first, a middle and the last insert; a per-operation error
    at a later index than the overflow wins over it"""
    field, H = 3, 2
    p = spec.FIELD_MODULUS[field]
    ins_at = [i for i, o in enumerate(_base(0)) if o[0] == INS]
    assert ins_at == [0, 2, 4, 5, 7, 9, 11]
    for r in (0, 3, 6):    # the insert rank that no longer fits: operations 0, 5 and 11
        cap = H + H * r + (H - 1)
        host, dev = twins(L, field, H, cap)
        e = host.empty_root()
        a, b = _raw(L, host, _base(e), False), _raw(L, dev, _base(e), True)
        assert a[:2] == b[:2] == (L._capi.ERR_ARG, ins_at[r]), (a[3], b[3])
        assert b[2] and "capacity" in b[3] and host.node_count == dev.node_count == H
        if r < 6:
            ops = _inject("key", _base(e), 11, p, e, None)
        else:     # the overflowing insert moves to operation 10, a bad kind follows it
            ops = _base(e)[:10] + [_base(e)[11], (2, -1, e, 1, 0)]
        a, b = _raw(L, host, ops, False), _raw(L, dev, ops, True)
        assert a[:2] == b[:2] == (L._capi.ERR_ARG, 11) and b[2], (a[3], b[3])
        assert host.node_count == dev.node_count == H
        # what fits still applies
        if ins_at[r]:
            both(host, dev, _base(e)[:ins_at[r]])
        host.close(), dev.close()


# ---------------------------------------------------------------------------------------------------- the rest of the ABI
def test_inputs_written_on_the_callers_stream(L):
    """apply_dev and register_dev read inputs that a non-blocking stream is still writing, behind a spin of ~50 ms"""
    from test_gpu_stream_order import Streams, ordered
    st = Streams()
    try:
        field, H = 2, 3
        rng = random.Random(9)
        key, value = _dense(rng, field, H)
        e = L.DeviceTrie(field, H, 64).empty_root()
        real = gen_ops(rng, 400, key, value, [e])
        kinds = [o[0] for o in real]
        # the poison set: the same kinds and prev (so the proof buffers fit), other keys and values
        poison = [(k, pv, r, (kk + 1) % 8, (v + 3) % 1000) for k, pv, r, kk, v in real]
        real_t, poison_t = dev_ops(real), dev_ops(poison)
        bufs = [torch.empty_like(t) for t in real_t]
        n, n_ins = len(real), kinds.count(INS)
        res = torch.empty((n, 32), dtype=torch.uint8, device="cuda")
        look = torch.empty((n - n_ins, 2 + 8 * H, 32), dtype=torch.uint8, device="cuda")
        ins = torch.empty((n_ins, 3 + 16 * H, 32), dtype=torch.uint8, device="cuda")
        counts = []

        def call(stream):
            dt = L.DeviceTrie(field, H, 1 << 14)
            dt.apply_dev(*bufs, results=res, lookup_out=look, insert_out=ins, stream=stream)
            counts.append(dt.node_count)
            dt.close()
            return None

        ordered(st, "lurk_trie_ctx_apply_dev", call, list(zip(bufs, real_t, poison_t)), outputs=[res, look, ins])
        host = L.DeviceTrie(field, H, 1 << 14)
        r, lk, it = run_host(host, real)
        assert ints(res.cpu().numpy()) == r and torch.equal(look, lk) and torch.equal(ins, it)

        pre = torch.from_numpy(pack([rng.randrange(1000) for _ in range(64 * 8)]).reshape(64, 8, 32)).cuda()
        pre_poison = torch.from_numpy(pack([rng.randrange(1000) for _ in range(64 * 8)]).reshape(64, 8, 32)).cuda()
        buf, dig = torch.empty_like(pre), torch.empty((64, 32), dtype=torch.uint8, device="cuda")

        def reg(stream):
            dt = L.DeviceTrie(field, H, 1 << 10)
            dt.register_dev(buf, digests_out=dig, stream=stream)
            dt.close()
            return None

        ordered(st, "lurk_trie_ctx_register_dev", reg, [(buf, pre, pre_poison)], outputs=[dig])
        assert ints(dig.cpu().numpy()) == host.register([ints(x) for x in pre.cpu().numpy()])
    finally:
        st.close()


def test_insert_count_is_read_on_the_callers_stream(L):
    """only `stream` given: the insert count that sizes the proofs apply_dev allocates is read behind the caller's work
    on that stream.  Until the delayed copy, kinds say every operation is an insert (so an early count would size the
    lookup proofs given below wrongly and be refused, and would only over-size the insert proofs)."""
    from test_gpu_stream_order import Streams
    st = Streams()
    try:
        field, H = 0, 3
        rng = random.Random(31)
        key, value = _dense(rng, field, H)
        host = L.DeviceTrie(field, H, 1 << 14)
        e = host.empty_root()
        real = gen_ops(rng, 600, key, value, [e])
        early = [(INS, -1, e, k, v) for _, _, _, k, v in real]
        n, n_ins = len(real), sum(1 for o in real if o[0] == INS)
        assert 0 < n_ins < n
        bufs = dev_ops(early)
        real_t = dev_ops(real)
        look = torch.empty((n - n_ins, 2 + 8 * H, 32), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        dt = L.DeviceTrie(field, H, 1 << 14)
        with torch.cuda.stream(st.S):
            torch.cuda._sleep(st.spin)
            for b, t in zip(bufs, real_t):
                b.copy_(t)
        res, look2, ins = dt.apply_dev(*bufs, lookup_out=look, stream=st.S.cuda_stream)
        assert st.S.query(), "apply_dev returned before its stream's work was done"
        torch.cuda.synchronize()
        assert look2 is look and tuple(ins.shape) == (n_ins, 3 + 16 * H, 32)
        want = run_host(host, real)
        assert ints(res.cpu().numpy()) == want[0] and torch.equal(look, want[1]) and torch.equal(ins, want[2])
    finally:
        st.close()


@pytest.mark.parametrize("fmt", [0, 1])
def test_register_dev_equals_register(L, fmt):
    field, H = 1, 3
    rng = random.Random(11)
    hashc, shared = OracleHash(field), {}
    t = L.Trie(hashc, 8, H, inverse_cache=shared)
    for _ in range(40):
        t.insert(rng.randrange(8 ** H), rng.randrange(1000))
    pres = list(shared.values())
    a, b = twins(L, field, H, 4096)
    want = a.register([_to(field, pre, fmt) for pre in pres], fmt=fmt)
    dev_pre = torch.from_numpy(pack([x for pre in pres for x in _to(field, pre, fmt)]).reshape(-1, 8, 32)).cuda()
    got = b.register_dev(dev_pre, fmt=fmt)
    torch.cuda.synchronize()
    assert ints(got.cpu().numpy()) == want
    assert _from(field, want, fmt) == list(shared.keys())
    assert a.node_count == b.node_count == len(shared)
    # a node already stored is not added again; then both stores answer the same batch
    b.register_dev(dev_pre[:5], fmt=fmt)
    assert b.node_count == len(shared)
    ops = gen_ops(rng, 300, lambda: rng.randrange(8 ** H), lambda: rng.randrange(1000), [t.root])
    both(a, b, ops, 0, mirror(L, hashc, shared, H, ops))


def test_register_dev_refuses_an_unreduced_element(L):
    field = 2
    p = spec.FIELD_MODULUS[field]
    dt = L.DeviceTrie(field, 2, 1024)
    pres = [[1] * 8, [2] * 8, [3] * 5 + [p] + [4] * 2, [p + 1] * 8]
    with pytest.raises(L.LurkError) as err:
        dt.register_dev(torch.from_numpy(pack([x for pre in pres for x in pre]).reshape(-1, 8, 32)).cuda())
    assert err.value.code == L._capi.ERR_ARG and "preimage 2 element 5" in str(err.value), str(err.value)
    assert dt.node_count == 2
    with pytest.raises(L.LurkError) as err:
        L._capi.check(L._capi.lib().lurk_trie_ctx_register(dt._ctx, L._capi.np_ptr(pack([x for pre in pres for x in pre])), 4, None, 0))
    assert "preimage 2 element 5" in str(err.value)


def test_witness_kernel_from_apply_dev_proofs(L):
    """lurk_trie_witness_batch_dev on apply_dev's proofs equals the oracle's blocks of the mirror's inputs"""
    import trie_gadget_oracle as T
    field, H = 3, 3
    rng = random.Random(21)
    key, value = _dense(rng, field, H)
    hashc, shared = OracleHash(field), {}
    e = L.Trie(hashc, 8, H, inverse_cache=shared).root
    ops = gen_ops(rng, 200, key, value, [e])
    want = mirror(L, hashc, shared, H, ops)
    dt = L.DeviceTrie(field, H, capacity=4096)
    for fmt in (0, 1):
        _, look, ins = run_dev(dt, ops, fmt)
        for op, proofs, exp in ((LOOK, look, want[1]), (INS, ins, want[2])):
            blk = L.trie_witness_block(field, op, H)
            out = torch.empty(len(exp) * blk * 32, dtype=torch.uint8, device="cuda")
            L._capi.check(L._capi.lib().lurk_trie_witness_batch_dev(field, op, H, proofs.data_ptr(), len(exp), out.data_ptr(), fmt, None))
            torch.cuda.synchronize()
            oracle_blocks = pack([x for c in exp for x in T.witness(field, op, c)])
            got = out.cpu().numpy()
            if fmt:
                got = pack(_from(field, ints(got), 1))
            assert np.array_equal(got, oracle_blocks), (op, fmt)


def test_two_host_threads(L):
    errors, done = [], {}

    def run(field, H, seed):
        try:
            rng = random.Random(seed)
            key, value = _dense(rng, field, H)
            hashc, shared = OracleHash(field), {}
            roots = [L.Trie(hashc, 8, H, inverse_cache=shared).root]
            dt = L.DeviceTrie(field, H, capacity=1 << 14)
            for _ in range(3):
                ops = gen_ops(rng, 1000, key, value, roots)
                want = mirror(L, hashc, shared, H, ops)
                res, _, _ = dt.apply_dev(*dev_ops(ops))
                assert ints(res.cpu().numpy()) == want[0]
                roots = [r for (k, *_), r in zip(ops, want[0]) if k == INS][-5:]
            done[seed] = True
        except Exception as exc:   # noqa: BLE001 - reported by the main thread
            errors.append(repr(exc))

    threads = [threading.Thread(target=run, args=(f, h, s)) for f, h, s in ((0, 3, 1), (2, 2, 2))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors and done == {1: True, 2: True}, errors


def test_caller_tensors_are_checked(L):
    dt = L.DeviceTrie(0, 2, capacity=256)
    e = dt.empty_root()
    k, pv, r, key, v = dev_ops([(INS, -1, e, 1, 2), (LOOK, 0, 0, 1, 0)])
    for bad in (dict(kinds=k.long()), dict(prev=pv.int()), dict(keys=key[:1]), dict(roots=r.cpu()), dict(values=torch.cat([v, v], 1)[:, ::2]),
                dict(results=torch.empty((2, 31), dtype=torch.uint8, device="cuda")),
                dict(insert_out=torch.empty((1, 3 + 16 * 2 - 1, 32), dtype=torch.uint8, device="cuda"))):
        args = dict(kinds=k, prev=pv, roots=r, keys=key, values=v)
        args.update(bad)
        with pytest.raises(ValueError):
            dt.apply_dev(**args)
    assert dt.node_count == 2
    res, look, ins = dt.apply_dev(k, pv, r, key, v)
    assert ints(res.cpu().numpy())[1] == 2 and dt.node_count == 4
    # proof buffers must hold exactly the batch's proofs: one short or one over is refused, also when both are given
    ops = [(INS, -1, e, 1, 2), (LOOK, 0, 0, 1, 0), (INS, 0, 0, 2, 3), (LOOK, 2, 0, 2, 0), (LOOK, -1, e, 1, 0)]
    args = dev_ops(ops)
    per_l, per_i = 2 + 8 * 2, 3 + 16 * 2
    proofs = lambda c, per: torch.full((c, per, 32), SENTINEL, dtype=torch.uint8, device="cuda")
    for look_c, ins_c in ((2, 2), (3, 1), (4, 2), (3, 3), (2, None), (None, 1), (4, None), (None, 3)):
        with pytest.raises(ValueError, match="lookup_out" if look_c not in (3, None) else "insert_out"):
            dt.apply_dev(*args, lookup_out=None if look_c is None else proofs(look_c, per_l),
                         insert_out=None if ins_c is None else proofs(ins_c, per_i))
    assert dt.node_count == 4
    look, ins = proofs(3, per_l), proofs(2, per_i)
    res, look2, ins2 = dt.apply_dev(*args, lookup_out=look, insert_out=ins)
    # operation 0 rebuilds the version the first batch made (1 -> 2 from e), already stored: only operation 2 adds nodes
    assert look2 is look and ins2 is ins and ints(res.cpu().numpy())[3] == 3 and dt.node_count == 6
    # the store's device: a tensor on another device than the one the store was built on is refused
    dt._device = torch.cuda.current_device() + 1
    with pytest.raises(ValueError, match="built on"):
        dt.apply_dev(*args)
    with pytest.raises(ValueError, match="built on"):
        dt.register_dev(torch.zeros((1, 8, 32), dtype=torch.uint8, device="cuda"))
    assert dt.node_count == 6
