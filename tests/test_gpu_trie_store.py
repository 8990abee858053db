"""The device trie store (csrc/trie_store.cu, trie.DeviceTrie) against the host mirror `Trie` run sequentially over one
shared inverse cache, byte for byte: every result and every written proof, on all four fields, canonical and
Montgomery, at H = 1..3 (dense keys: overwrites, repeated keys, unchanged values, absent keys) and H = 85 (keys that
share all but their last chunk); versions, forks from stored roots and chains continued in later batches; batching
does not change anything at 10^5 operations; the goldens; batch sizes around a warp and past the Poseidon launch's
shape boundaries; register; MissingPreimage; the witness kernel and a Nova fold fed from the written proofs; two host
threads.  The mirror hashes with the oracle's C Poseidon, so it shares no device code with what it checks."""
import json
import os
import random
import threading

import numpy as np
import pytest
import torch

from oracle import capi as oracle_capi, spec
from util import ints, pack

pytestmark = pytest.mark.gpu
R = 1 << 256
FIELDS = [0, 1, 2, 3]
LOOK, INS = 0, 1
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_goldens.json")))["poseidon_digests"]


class OracleHash:
    """the mirror's PoseidonCache: arity-8 digests from the oracle's C Poseidon, memoised"""

    def __init__(self, field):
        self.field_id, self.memo = field, {}

    def compute_hash(self, preimage):
        key = tuple(int(x) for x in preimage)
        if key not in self.memo:
            self.memo[key] = ints(oracle_capi.poseidon_hash_batch(self.field_id, len(key), pack(key)))[0]
        return self.memo[key]


def mirror(L, hashc, shared, H, ops):
    """the sequential loop of include/lurk_b200.h: results, lookup inputs, insert inputs (ints)"""
    res, look, ins = [], [], []
    for kind, prev, root, key, value in ops:
        r = root if prev < 0 else res[prev]
        t = L.Trie(hashc, 8, H, root=r, inverse_cache=shared)
        if kind == LOOK:
            res.append(t.lookup_aux(key))
            look.append(L.lookup_inputs(r, key, t.prove_lookup(key)))
        else:
            proof, _ = t.prove_insert(key, value)
            res.append(t.root)
            ins.append(L.insert_inputs(r, key, value, proof))
    return res, look, ins


def gen_ops(rng, n, key, value, roots, p_look=0.5, p_chain=0.05):
    """n operations in program order: chains from the given stored roots, lookups of any earlier version, lookups of
    stored roots"""
    ops, chains = [], []
    for i in range(n):
        if not chains or rng.random() < p_chain:
            if rng.random() < 0.7:
                ops.append((INS, -1, rng.choice(roots), key(), value()))
                chains.append([i])
            else:
                ops.append((LOOK, -1, rng.choice(roots), key(), 0))
            continue
        ch = rng.choice(chains)
        if rng.random() < p_look:
            ops.append((LOOK, rng.choice(ch), 0, key(), 0))
        else:
            ops.append((INS, ch[-1], 0, key(), value()))
            ch.append(i)
    return ops


def _to(field, vals, fmt):
    p = spec.FIELD_MODULUS[field]
    return [v * R % p if fmt else v for v in vals]


def _from(field, vals, fmt):
    p = spec.FIELD_MODULUS[field]
    inv = pow(R, -1, p)
    return [v * inv % p if fmt else v for v in vals]


def _fmt_ops(field, ops, fmt):
    return [(k, pr, *_to(field, [r, key, v], fmt)) for k, pr, r, key, v in ops]


def check(L, dt, field, ops, want, fmt):
    res, look, ins = dt.apply(_fmt_ops(field, ops, fmt), fmt=fmt)
    torch.cuda.synchronize()
    assert _from(field, res, fmt) == want[0], "results"
    for got, exp, name in ((look, want[1], "lookup"), (ins, want[2], "insert")):
        exp_b = torch.from_numpy(pack(_to(field, [x for call in exp for x in call], fmt))).cuda()
        assert torch.equal(got.reshape(-1), exp_b), f"{name} proofs"


def _dense(rng, field, H):
    p = spec.FIELD_MODULUS[field]
    span = min(8 ** H, 12)
    vals = [0, 1, 7, p - 1, rng.randrange(p)]
    # keys: a dense window of paths, some with bits above 3H (they share the low bits), and p - 1
    keys = [rng.choice([k, k + (1 << (3 * H)), p - 1]) for k in range(span)]
    return (lambda: rng.choice(keys)), (lambda: rng.choice(vals))


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("H", [1, 2, 3])
def test_small_heights_match_the_mirror(L, field, H):
    """two batches of 2000 dense operations; the second starts chains from roots the first produced"""
    rng = random.Random(10 * field + H)
    key, value = _dense(rng, field, H)
    hashc, shared = OracleHash(field), {}
    empty = L.Trie(hashc, 8, H, inverse_cache=shared).root
    ops1 = gen_ops(rng, 2000, key, value, [empty], p_chain=0.02)
    want1 = mirror(L, hashc, shared, H, ops1)
    produced = [r for (k, *_), r in zip(ops1, want1[0]) if k == INS]
    ops2 = gen_ops(rng, 2000, key, value, [empty] + rng.sample(produced, 20), p_chain=0.05)
    want2 = mirror(L, hashc, shared, H, ops2)
    for fmt in (0, 1):
        dt = L.DeviceTrie(field, H, capacity=1 << 16)
        assert dt.empty_root() == empty and dt.node_count == H
        check(L, dt, field, ops1, want1, fmt)
        check(L, dt, field, ops2, want2, fmt)
        dt.close()


@pytest.mark.parametrize("field", FIELDS)
def test_standard_height_matches_the_mirror(L, field):
    """H = 85: random keys and keys that differ only in their last chunk, both formats"""
    p = spec.FIELD_MODULUS[field]
    rng = random.Random(85 + field)
    stem = rng.randrange(p >> 3) << 3
    keys = [stem + c for c in range(8)] + [rng.randrange(p) for _ in range(6)]
    key, value = (lambda: rng.choice(keys)), (lambda: rng.choice([0, 5, rng.randrange(p)]))
    hashc, shared = OracleHash(field), {}
    empty = L.Trie(hashc, 8, 85, inverse_cache=shared).root
    ops = gen_ops(rng, 300, key, value, [empty], p_chain=0.03)
    want = mirror(L, hashc, shared, 85, ops)
    for fmt in (0, 1):
        dt = L.DeviceTrie(field, 85, capacity=1 << 16)
        check(L, dt, field, ops, want, fmt)
        dt.close()


def test_versions_and_forks(L):
    """lookups of older versions of one chain, three chains forked from one stored root, and a chain continued in the
    next batch from a root the first one produced"""
    field, H = 0, 2
    hashc, shared = OracleHash(field), {}
    e = L.Trie(hashc, 8, H, inverse_cache=shared).root
    ops = [(INS, -1, e, 1, 10), (INS, 0, 0, 2, 20), (INS, 1, 0, 1, 11), (LOOK, 0, 0, 1, 0), (LOOK, 1, 0, 2, 0), (LOOK, 2, 0, 1, 0),
           (INS, -1, e, 1, 30), (INS, -1, e, 1, 40), (LOOK, 6, 0, 1, 0), (LOOK, 7, 0, 1, 0), (LOOK, 0, 0, 2, 0), (INS, 6, 0, 9, 50)]
    want = mirror(L, hashc, shared, H, ops)
    assert [want[0][i] for i in (3, 4, 5, 8, 9, 10)] == [10, 20, 11, 30, 40, 0]
    dt = L.DeviceTrie(field, H, capacity=1024)
    check(L, dt, field, ops, want, 0)
    ops2 = [(INS, -1, want[0][2], 2, 21), (LOOK, 0, 0, 1, 0), (LOOK, 0, 0, 2, 0), (LOOK, -1, want[0][11], 9, 0)]
    want2 = mirror(L, hashc, shared, H, ops2)
    assert want2[0][1:] == [11, 21, 50]
    check(L, dt, field, ops2, want2, 1)


def _split(ops, res, cuts):
    """the same operations cut into batches at `cuts`: a prev in an earlier batch becomes that insert's root"""
    out, start = [], 0
    for end in list(cuts) + [len(ops)]:
        batch = []
        for k, prev, root, key, v in ops[start:end]:
            if 0 <= prev < start:
                prev, root = -1, res[prev]
            elif prev >= start:
                prev -= start
            batch.append((k, prev, root, key, v))
        out.append(batch)
        start = end
    return out


def test_batching_does_not_change_results(L):
    """10^5 mixed operations at H = 85 in one batch, in random batches, and the first 300 one per batch"""
    field, H, n = 0, 85, 100_000
    p = spec.FIELD_MODULUS[field]
    rng = random.Random(7)
    stems = [rng.randrange(p >> 3) << 3 for _ in range(64)]
    key = lambda: rng.choice(stems) + rng.randrange(8) if rng.random() < 0.5 else rng.randrange(p)
    value = lambda: rng.randrange(p)
    first = L.DeviceTrie(field, H, capacity=6_000_000)
    ops = gen_ops(rng, n, key, value, [first.empty_root()], p_chain=0.001)
    res, look, ins = first.apply(ops)
    look, ins = look.reshape(-1), ins.reshape(-1)

    def run(batches):
        dt = L.DeviceTrie(field, H, capacity=6_000_000)
        rs, ls, is_ = [], [], []
        for b in batches:
            r, lo, i = dt.apply(b)
            rs += r
            ls.append(lo.reshape(-1))
            is_.append(i.reshape(-1))
        count = dt.node_count
        dt.close()
        return rs, torch.cat(ls), torch.cat(is_), count

    cuts = sorted(rng.sample(range(1, n), 6))
    rs, ls, is_, count = run(_split(ops, res, cuts))
    assert rs == res and torch.equal(ls, look) and torch.equal(is_, ins)
    assert count == first.node_count
    m = 300
    rs, ls, is_, _ = run(_split(ops[:m], res, range(1, m)))
    assert rs == res[:m] and torch.equal(ls, look[:ls.numel()]) and torch.equal(is_, ins[:is_.numel()])
    first.close()


def test_goldens(L):
    """G1..G4 are the empty roots of heights 1..4 and G5 that of 85; insert 123 -> 456 into the empty StandardTrie
    ends in G10, and a lookup of 123 then returns 456"""
    g = {k: int(v["hex"], 16) for k, v in GOLD.items()}
    for h, name in ((1, "G1"), (2, "G2"), (3, "G3"), (4, "G4"), (85, "G5")):
        assert L.DeviceTrie(0, h, capacity=256).empty_root() == g[name], name
    dt = L.DeviceTrie(0, 85, capacity=1024)
    res, _, ins = dt.apply([(INS, -1, g["G5"], 123, 456), (LOOK, 0, 0, 123, 0)])
    assert res == [g["G10"], 456]
    assert ints(ins.cpu().numpy()[0, :3])  == [g["G5"], 123, 456]
    assert dt.node_count == 85 + 85


def _boundary_sizes(L):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    # 1, a warp +- 1, and one past each of the arity-8 digest launch's shape boundaries (warp kernel up to 8192 sponges,
    # a persistent grid from SMs x 192)
    return [1, 31, 32, 33, 8193, sms * 192 + 1]


def test_batch_size_boundaries(L):
    field, H = 2, 1
    hashc, shared = OracleHash(field), {}
    e = L.Trie(hashc, 8, H, inverse_cache=shared).root
    rng = random.Random(3)
    p = spec.FIELD_MODULUS[field]
    for n in _boundary_sizes(L):
        # all inserts, so the number of hashes per level is n
        ops = [(INS, -1 if i == 0 else i - 1, e, rng.randrange(16), rng.randrange(p)) for i in range(n)]
        want = mirror(L, hashc, shared, H, ops)
        dt = L.DeviceTrie(field, H, capacity=n * H + 16)
        check(L, dt, field, ops, want, 0)
        dt.close()


def test_register_a_host_trie(L):
    field, H = 1, 3
    rng = random.Random(11)
    hashc, shared = OracleHash(field), {}
    t = L.Trie(hashc, 8, H, inverse_cache=shared)
    for _ in range(40):
        t.insert(rng.randrange(8 ** H), rng.randrange(1000))
    dt = L.DeviceTrie(field, H, capacity=4096)
    digests = dt.register(list(shared.values()))
    assert digests == list(shared.keys())
    assert dt.node_count == len(shared)            # the empty roots are among them: nothing is stored twice
    assert dt.register([_to(field, pre, 1) for pre in list(shared.values())[:5]], fmt=1) == _to(field, list(shared.keys())[:5], 1)
    assert dt.node_count == len(shared)
    ops = gen_ops(rng, 300, lambda: rng.randrange(8 ** H), lambda: rng.randrange(1000), [t.root])
    want = mirror(L, hashc, shared, H, ops)
    check(L, dt, field, ops, want, 0)


def test_missing_preimage(L):
    """a missing root and a missing node are refused naming the first operation; the store is left as it was"""
    field, H = 0, 2
    hashc, shared = OracleHash(field), {}
    e = L.Trie(hashc, 8, H, inverse_cache=shared).root
    dt = L.DeviceTrie(field, H, capacity=1024)
    good = [(INS, -1, e, 3, 4), (LOOK, 0, 0, 3, 0)]
    want = mirror(L, hashc, shared, H, good)
    check(L, dt, field, good, want, 0)
    count = dt.node_count
    # a node whose child is not stored: register only the top of a path built on the host
    orphan_child = hashc.compute_hash([9] * 8)
    top = [orphan_child] + [0] * 7
    (top_d,) = dt.register([top])
    count += 1
    for ops, bad, what in (([(LOOK, -1, e, 1, 0), (INS, -1, 12345, 1, 2), (LOOK, -1, 999, 1, 0)], 1, 12345),
                           ([(INS, -1, e, 0, 5), (LOOK, 0, 0, 0, 0), (INS, 0, 0, 1, 6), (LOOK, -1, top_d, 0, 0)], 3, orphan_child)):
        with pytest.raises(L.LurkError) as err:
            dt.apply(ops)
        assert err.value.code == L._capi.ERR_RANGE
        assert f"operation {bad}:" in str(err.value) and f"{what:064x}" in str(err.value), str(err.value)
        assert dt.node_count == count
    # the next batch is as if the failed calls never happened
    ops = [(INS, -1, want[0][0], 5, 6), (LOOK, 0, 0, 3, 0), (LOOK, -1, e, 3, 0)]
    want = mirror(L, hashc, shared, H, ops)
    check(L, dt, field, ops, want, 0)


def test_witness_kernel_from_written_proofs(L):
    """lurk_trie_witness_batch_dev on apply's outputs equals lurk_trie_witness_batch on the mirror's inputs"""
    field, H = 3, 3
    rng = random.Random(21)
    key, value = _dense(rng, field, H)
    hashc, shared = OracleHash(field), {}
    e = L.Trie(hashc, 8, H, inverse_cache=shared).root
    ops = gen_ops(rng, 200, key, value, [e])
    want = mirror(L, hashc, shared, H, ops)
    dt = L.DeviceTrie(field, H, capacity=4096)
    for fmt in (0, 1):
        _, look, ins = dt.apply(_fmt_ops(field, ops, fmt), fmt=fmt)
        for op, proofs, exp in ((LOOK, look, want[1]), (INS, ins, want[2])):
            blk = L.trie_witness_block(field, op, H)
            host = L.trie_witness_batch(field, op, H, pack(_to(field, [x for c in exp for x in c], fmt)), fmt=fmt)
            out = torch.empty(len(exp) * blk * 32, dtype=torch.uint8, device="cuda")
            L._capi.check(L._capi.lib().lurk_trie_witness_batch_dev(field, op, H, proofs.data_ptr(), len(exp), out.data_ptr(), fmt, None))
            torch.cuda.synchronize()
            assert torch.equal(out.cpu(), torch.from_numpy(host)), (op, fmt)


def test_nova_fold_with_proofs_from_the_device_trie(L, oracle):
    """a BN254 Nova fold context with a lookup batch and an insert batch: stage A from resident inputs written by
    write_trie_batch gives the same fold records as the same steps staged from the host"""
    import test_gpu_trie as TG
    import trie_gadget_oracle as T
    field, curve, H, frames = 0, 0, 2, 2
    p = spec.FIELD_MODULUS[field]
    cs = {op: TG._circuit(L, oracle, curve, field, op, H, frames=frames) for op in (LOOK, INS)}
    for op, c in cs.items():
        bases = oracle.gen_bases(curve, max(c["n_w"], c["rows"]))
        ck = L.CommitmentKey(curve, bases)
        records = []
        for resident in (False, True):
            ctx, bi = TG._context(L, c, curve, ck)
            dt = L.DeviceTrie(field, H, capacity=4096)
            root = dt.empty_root()
            rng = random.Random(40 + op)
            recs = []
            for step in range(3):
                keys = [rng.randrange(64) for _ in range(frames)]
                vals = [rng.randrange(p) for _ in range(frames)]
                if op == INS:
                    ops = [(INS, -1 if f == 0 else f - 1, root, keys[f], vals[f]) for f in range(frames)]
                else:
                    ops = [(LOOK, -1, root, keys[f], 0) for f in range(frames)]
                X2 = [rng.randrange(1 << 64), rng.randrange(1 << 64)]
                ctx.sync()
                if resident:
                    res = L.write_trie_batch(dt, ctx, 0, bi, ops)
                    torch.cuda.synchronize()
                    ins = None
                else:
                    res, lk, isr = dt.apply(ops)
                    ins = [ints(t.cpu().numpy()) for t in (lk if op == LOOK else isr)]
                roots_before = [o[2] if o[1] < 0 else res[o[1]] for o in ops]
                glue = [[roots_before[f], keys[f], vals[f] if op == INS else 0, 1] for f in range(frames)]
                if resident:
                    TG._fill(ctx, 0, bi, glue, [[0] * T.n_inputs(op, H)] * frames, X2, False, p, c)
                    ctx.sync()
                    w2 = ctx.device_view(0, -4).view(-1, 32)
                    for f, g in enumerate(glue):
                        w2[f * c["per"]:f * c["per"] + TG.GLUE] = torch.from_numpy(pack([x * R % p for x in g]).reshape(-1, 32)).cuda()
                    w2[c["n_w"] + 1:c["n_w"] + 1 + c["n_x"]] = torch.from_numpy(pack([x * R % p for x in X2]).reshape(-1, 32)).cuda()
                    q = spec.FIELD_MODULUS[TG.BASE_FIELD[field]]
                    ro = [0] * 24
                    ro[4], ro[5] = X2
                    ctx.device_view(0, -3).copy_(torch.from_numpy(pack([x * R % q for x in ro])).cuda())
                    torch.cuda.synchronize()
                    ctx.stage_a(0, resident=True)
                else:
                    TG._fill(ctx, 0, bi, glue, ins, X2, False, p, c)
                    ctx.stage_a(0)
                if step == 0:
                    ctx.init_running(0)
                else:
                    ctx.stage_b_launch(0)
                rec = ctx.collect(0)
                recs.append((rec.comm_W.tobytes(), rec.comm_T.tobytes(), rec.r.tobytes(), rec.running_comm_W.tobytes()))
                if op == INS:
                    root = res[-1]
            run = ctx.get_running()
            recs.append((run["W"].tobytes(), run["E"].tobytes()))
            assert ctx.check_running() == (0, True, True)
            records.append(recs)
            ctx.close()
            dt.close()
        assert records[0] == records[1], f"op {op}"


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
                res, _, _ = dt.apply(ops)
                assert res == want[0]
                roots = [r for (k, *_), r in zip(ops, res) if k == INS][-5:]
            done[seed] = True
        except Exception as exc:   # noqa: BLE001 - reported by the main thread
            errors.append(repr(exc))

    threads = [threading.Thread(target=run, args=(f, h, s)) for f, h, s in ((0, 3, 1), (2, 2, 2))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors and done == {1: True, 2: True}, errors


def test_caller_buffers_are_checked(L):
    """apply refuses a proof buffer of the wrong size, type or device before any device write"""
    dt = L.DeviceTrie(0, 2, capacity=256)
    e = dt.empty_root()
    ops = [(INS, -1, e, 1, 2), (LOOK, 0, 0, 1, 0)]
    per_l, per_i = 2 + 8 * 2, 3 + 16 * 2
    good_l = torch.empty((1, per_l, 32), dtype=torch.uint8, device="cuda")
    for bad in (torch.empty((1, per_i - 1, 32), dtype=torch.uint8, device="cuda"),
                torch.empty((per_i * 8,), dtype=torch.int32, device="cuda"),
                torch.empty((1, per_i, 32), dtype=torch.uint8)):
        with pytest.raises(ValueError):
            dt.apply(ops, lookup_out=good_l, insert_out=bad)
    assert dt.node_count == 2
    res, look, ins = dt.apply(ops, lookup_out=good_l)
    assert res[1] == 2 and look is good_l and dt.node_count == 4
