"""GPU parity for S1/S3: CUDA Poseidon digests, slot witnesses and bit-decomposition witnesses, through the C ABI,
bit-exact against the oracle.  Model: the reference's sequential-vs-parallel witness equivalence test
(src/lem/multiframe.rs:1019-1125)."""
import numpy as np
import pytest

from util import GOLDEN, TAG_NUM, ints, pack, random_elements

pytestmark = pytest.mark.gpu
FIELDS = [0, 1, 2, 3]
ARITIES = [3, 4, 6, 8]


def test_golden_digests_through_c_abi(L):
    pc = L.PoseidonCache(L.FIELD_BN254_FR)
    d = pc.hash8([0] * 8)
    assert d == GOLDEN["G1"]
    seq = [d]
    for _ in range(84):
        seq.append(pc.hash8([seq[-1]] * 8))
    assert (seq[1], seq[2], seq[3], seq[84]) == (GOLDEN["G2"], GOLDEN["G3"], GOLDEN["G4"], GOLDEN["G5"])
    assert pc.hash3([0, TAG_NUM, 0]) == GOLDEN["G6"]
    assert pc.hash3([0, TAG_NUM, 123]) == GOLDEN["G7"]
    assert pc.compute_hash([0, TAG_NUM, 123]) == GOLDEN["G7"]
    with pytest.raises(ValueError):
        pc.compute_hash([1, 2])            # unsupported arity (reference panics, src/hash.rs:26)


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("arity", ARITIES)
@pytest.mark.parametrize("shape", ["uniform", "lem"])
def test_digest_parity_small_batch(L, oracle, spec, field, arity, shape):
    n = 257                                    # ragged: not a multiple of the warp / CTA size
    pre = random_elements(field, n * arity, seed=1000 * field + 10 * arity + len(shape), shape=shape)
    p = spec.FIELD_MODULUS[field]
    pre[:arity * 32] = 0                                          # all-zero preimage (dummy slot)
    pre[arity * 32:2 * arity * 32] = pack([p - 1] * arity)        # maximum elements
    got = L.PoseidonCache(field).hash_batch_bytes(arity, pre)
    want = oracle.poseidon_hash_batch(field, arity, pre, mode=1, nthreads=8)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("field,arity", [(0, 8), (0, 4), (2, 8), (2, 4), (1, 3), (3, 6)])
def test_digest_parity_throughput_path(L, oracle, field, arity):
    # large enough for the persistent one-CTA-per-SM launch shape with a second grid-stride pass (arity 3/4: 512 threads per
    # SM, 6/8: 384); oracle on 8 threads takes seconds
    import torch
    n = torch.cuda.get_device_properties(0).multi_processor_count * 512 + 77
    pre = random_elements(field, n * arity, seed=55 + field + arity)
    got = L.PoseidonCache(field).hash_batch_bytes(arity, pre)
    want = oracle.poseidon_hash_batch(field, arity, pre, mode=1, nthreads=8)
    assert np.array_equal(got, want)


def test_digest_montgomery_entry_point(L, oracle, spec):
    field, arity, n = 0, 4, 100
    p = spec.FIELD_MODULUS[field]
    pre = random_elements(field, n * arity, seed=4)
    mont = pack([x * (1 << 256) % p for x in ints(pre)])
    out = np.zeros(n * 32, dtype=np.uint8)
    L._capi.check(L._capi.lib().lurk_poseidon_hash_batch_mont(field, arity, L._capi.np_ptr(mont), n, L._capi.np_ptr(out)))
    want = ints(oracle.poseidon_hash_batch(field, arity, pre))
    assert [x * pow(1 << 256, -1, p) % p for x in ints(out)] == want


def test_empty_and_errors(L, spec):
    pc = L.PoseidonCache(0)
    assert pc.hash_batch_bytes(8, np.zeros(0, dtype=np.uint8)).size == 0
    bad = pack([spec.FIELD_MODULUS[0]] + [0] * 7)       # not reduced: from_repr would fail (src/field.rs:76-81)
    with pytest.raises(L.LurkError) as e:
        pc.hash_batch_bytes(8, bad)
    assert e.value.code == L._capi.ERR_RANGE
    with pytest.raises(ValueError):
        pc.hash_batch_bytes(5, np.zeros(5 * 32, dtype=np.uint8))


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("arity", ARITIES)
def test_slot_witness_parity(L, oracle, field, arity):
    st = {3: L.SlotType.Commitment, 4: L.SlotType.Hash4, 6: L.SlotType.Hash6, 8: L.SlotType.Hash8}[arity]
    n = 67
    pre = random_elements(field, n * arity, seed=31 * field + arity, shape="lem")
    pre[:arity * 32] = 0
    got = L.slot_witness_batch_bytes(field, st, pre)
    want = oracle.poseidon_witness_batch(field, arity, pre, nthreads=8)
    assert L.compute_witness_size(st, field) == oracle.witness_block(field, arity)
    assert np.array_equal(got, want)


def test_slot_witness_montgomery_format(L, oracle, spec):
    field, arity, n = 0, 4, 9
    p = spec.FIELD_MODULUS[field]
    pre = random_elements(field, n * arity, seed=77)
    mont = pack([x * (1 << 256) % p for x in ints(pre)])
    got = L.slot_witness_batch_bytes(field, L.SlotType.Hash4, mont, fmt=L.FMT_MONTGOMERY)
    want = ints(oracle.poseidon_witness_batch(field, arity, pre))
    assert [x * pow(1 << 256, -1, p) % p for x in ints(got)] == want


@pytest.mark.parametrize("field", FIELDS)
def test_bitdecomp_witness_parity(L, oracle, spec, field):
    p = spec.FIELD_MODULUS[field]
    vals = pack([0, 1, p - 1, p >> 1, (1 << 64) - 1])
    vals = np.concatenate([vals, random_elements(field, 200, seed=8), random_elements(field, 60, seed=9, shape="witness")])
    got = L.slot_witness_batch_bytes(field, L.SlotType.BitDecomp, vals)
    want = oracle.bitdecomp_witness_batch(field, vals, nthreads=4)
    assert L.compute_witness_size(L.SlotType.BitDecomp, field) == oracle.bitdecomp_size(field)
    assert np.array_equal(got, want)


def test_generate_slots_witnesses_frame_layout(L, oracle):
    # one frame of the universal step circuit: 14 hash4, 0 hash6, 6 hash8, 1 commitment, 3 bit-decomp
    # (src/lem/eval.rs:1960-1964), mostly dummy slots
    ST = L.SlotType
    rnd = lambda k, seed: ints(random_elements(0, k, seed=seed, shape="lem"))
    slots = [(ST.Hash4, rnd(4, 1))] + [(ST.Hash4, None)] * 12 + [(ST.Hash4, rnd(4, 2))]
    slots += [(ST.Hash8, rnd(8, 3))] + [(ST.Hash8, None)] * 5 + [(ST.Commitment, None)]
    slots += [(ST.BitDecomp, rnd(1, 4)), (ST.BitDecomp, None), (ST.BitDecomp, None)]
    blocks = L.generate_slots_witnesses(0, slots)
    assert sum(b.size for b in blocks) == 7808 * 32          # src/lem/multiframe.rs:503-516 + eval.rs:1966
    for (st, pre), blk in zip(slots, blocks):
        pre = pre if pre is not None else [0] * st.preimg_size()
        if st is ST.BitDecomp:
            want = oracle.bitdecomp_witness_batch(0, pack(pre))
        else:
            want = oracle.poseidon_witness_batch(0, st.preimg_size(), pack(pre))
        assert np.array_equal(blk, want)


def test_slot_witness_chunked_host_pipeline(L, oracle):
    # > 48 MB of witness output: the host-buffer entry point streams chunks through its pinned staging slots
    field, arity, n = 0, 8, 9000
    pre = random_elements(field, n * arity, seed=123, shape="lem")
    got = L.slot_witness_batch_bytes(field, L.SlotType.Hash8, pre)
    assert got.size == n * 396 * 32
    assert np.array_equal(got, oracle.poseidon_witness_batch(field, arity, pre, nthreads=8))
    # a bad element in the last chunk is still reported
    bad = pre.copy()
    bad[-32:] = 0xff
    with pytest.raises(L.LurkError) as e:
        L.slot_witness_batch_bytes(field, L.SlotType.Hash8, bad)
    assert e.value.code == L._capi.ERR_RANGE


def test_concurrent_callers(L, oracle):
    """the seams are called from rayon workers and the witness thread concurrently (src/proof/nova.rs:297-326):
    every entry point must be re-entrant"""
    import threading
    jobs = [(0, 4, 3000, 1), (0, 8, 2000, 2), (2, 4, 2500, 3), (0, 3, 1000, 4), (0, 4, 200_000, 5), (2, 8, 1500, 6)]
    results, errors = {}, []

    def work(k, field, arity, n, seed):
        try:
            pre = random_elements(field, n * arity, seed=seed)
            pc = L.PoseidonCache(field)
            for _ in range(3):
                results[k] = (pre, pc.hash_batch_bytes(arity, pre))
        except Exception as ex:       # noqa: BLE001
            errors.append(ex)

    threads = [threading.Thread(target=work, args=(k, *j)) for k, j in enumerate(jobs)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for k, (field, arity, n, _seed) in enumerate(jobs):
        pre, got = results[k]
        m = min(n, 3000)
        assert np.array_equal(got[:m * 32], oracle.poseidon_hash_batch(field, arity, pre[:m * arity * 32], nthreads=4))


def test_slot_witness_scatter_into_frame_layout(L, oracle):
    """in-place form: blocks land at caller-given element offsets of the step witness -- the reference's layout is
    per frame [slot blocks | LEM body aux] (src/lem/multiframe.rs:635-712), 9119 elements per frame on BN256"""
    import torch
    lib, chk = L._capi.lib(), L._capi.check
    field, frames, frame_len = 0, 5, 9119
    W = torch.full((frames * frame_len * 32,), 0xAB, dtype=torch.uint8, device="cuda")
    base = 0
    expected = np.full(frames * frame_len * 32, 0xAB, dtype=np.uint8).reshape(frames, frame_len, 32)
    for arity, per_frame in ((4, 14), (8, 6), (3, 1)):
        n = frames * per_frame
        blk = oracle.witness_block(field, arity)
        pre = random_elements(field, n * arity, seed=arity, shape="lem")
        offs = (np.arange(frames, dtype=np.uint64)[:, None] * frame_len + base + np.arange(per_frame, dtype=np.uint64)[None, :] * blk).reshape(-1)
        d_pre, d_off = torch.from_numpy(pre).cuda(), torch.from_numpy(offs).cuda()
        chk(lib.lurk_poseidon_witness_scatter_dev(field, arity, d_pre.data_ptr(), n, W.data_ptr(), d_off.data_ptr(), L.FMT_CANONICAL, None))
        want = oracle.poseidon_witness_batch(field, arity, pre, nthreads=4).reshape(frames, per_frame * blk, 32)
        expected[:, base:base + per_frame * blk] = want
        base += per_frame * blk
    vals = random_elements(field, frames * 3, seed=77, shape="witness")
    bd = oracle.bitdecomp_size(field)
    offs = (np.arange(frames, dtype=np.uint64)[:, None] * frame_len + base + np.arange(3, dtype=np.uint64)[None, :] * bd).reshape(-1)
    d_v, d_off = torch.from_numpy(vals).cuda(), torch.from_numpy(offs).cuda()
    chk(lib.lurk_bitdecomp_witness_scatter_dev(field, d_v.data_ptr(), frames * 3, W.data_ptr(), d_off.data_ptr(), L.FMT_CANONICAL, None))
    expected[:, base:base + 3 * bd] = oracle.bitdecomp_witness_batch(field, vals).reshape(frames, 3 * bd, 32)
    base += 3 * bd
    assert base == 7808
    got = W.cpu().numpy().reshape(frames, frame_len, 32)
    assert np.array_equal(got, expected)           # includes: the 1311 body-aux elements of every frame are untouched
