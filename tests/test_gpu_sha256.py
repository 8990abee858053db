"""The SHA-256 coprocessor's witness on the GPU (csrc/sha256.cu) against the oracle's restatement of bellpepper's gadget
(tests/sha256_gadget_oracle.py), byte for byte: host and device batches and the scatter form, both formats, n = 1..4
on every field, call counts around a warp and one past the kernel's grid-stride boundary (SMs x 8 CTAs); scatter at
non-contiguous offsets; two host threads at once; and a fold context whose step circuit holds the gadget's constraints
as R1CS rows, folding steps whose SHA-256 blocks the context writes into W itself."""
import ctypes as C
import random
import threading

import numpy as np
import pytest
import torch

import sha256_gadget_oracle as G
from oracle import nifs
from util import ints, pack

pytestmark = pytest.mark.gpu
FIELDS = [0, 1, 2, 3]
R = 1 << 256
DISTINCT = 5
_CACHE = {}


def _sets(spec, field, n):
    """DISTINCT input sets (zeros, p - 1, random) and their oracle blocks as (DISTINCT, block, 32) uint8, canonical"""
    if (field, n) not in _CACHE:
        p = spec.FIELD_MODULUS[field]
        rng = random.Random(100 * field + n)
        sets = [[0] * (2 * n), [p - 1] * (2 * n)] + [[rng.randrange(p) for _ in range(2 * n)] for _ in range(DISTINCT - 2)]
        blocks = np.stack([pack(G.witness(field, s)).reshape(-1, 32) for s in sets])
        _CACHE[(field, n)] = (sets, blocks)
    return _CACHE[(field, n)]


def _fmt_bytes(spec, field, vals, fmt):
    p = spec.FIELD_MODULUS[field]
    return pack([v * R % p if fmt else v for v in vals])


def _mont_blocks(spec, field, blocks):
    p = spec.FIELD_MODULUS[field]
    flat = ints(blocks.reshape(-1))
    cache = {}
    return pack([cache.setdefault(v, v * R % p) for v in flat]).reshape(blocks.shape)


def _expected(spec, field, n, fmt):
    sets, blocks = _sets(spec, field, n)
    key = (field, n, fmt)
    if key not in _CACHE:
        _CACHE[key] = torch.from_numpy(_mont_blocks(spec, field, blocks) if fmt else blocks).cuda()
    return sets, _CACHE[key]


def _calls(count, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, DISTINCT, size=count)


def _inputs(spec, field, sets, pick, fmt):
    return np.concatenate([_fmt_bytes(spec, field, sets[k], fmt) for k in pick])


def _chk(L, rc):
    L._capi.check(rc)


def _grid_boundary():
    return torch.cuda.get_device_properties(0).multi_processor_count * 8


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("n", [1, 2, 3, 4])
@pytest.mark.parametrize("fmt", [0, 1])
def test_batches_match_the_oracle(L, spec, field, n, fmt):
    lib = L._capi.lib()
    sets, want = _expected(spec, field, n, fmt)
    blk = L.witness_block(field, n)
    assert want.shape[1] == blk
    for count in (1, 31, 32, 33):
        pick = _calls(count, count + 7 * n + field)
        src = _inputs(spec, field, sets, pick, fmt)
        host = L.sha256_witness_batch(field, n, src, fmt=fmt)
        exp = want[torch.from_numpy(pick).cuda()]
        assert torch.equal(torch.from_numpy(host).cuda().view(count, blk, 32), exp), f"host batch, count {count}"
        d_in = torch.from_numpy(src).cuda()
        out = torch.full((count * blk * 32,), 0xA5, dtype=torch.uint8, device="cuda")
        _chk(L, lib.lurk_sha256_witness_batch_dev(field, n, d_in.data_ptr(), count, out.data_ptr(), fmt, None))
        torch.cuda.synchronize()
        assert torch.equal(out.view(count, blk, 32), exp), f"device batch, count {count}"


def test_large_n_after_a_smaller_large_n(L, spec):
    """n >= 10 needs more than 48 KB of shared memory per CTA: n = 10 first, then larger n up to LURK_SHA256_MAX_N in the
    same process -- the opt-in must cover every n, not only the first one launched"""
    field = 0
    p = spec.FIELD_MODULUS[field]
    rng = random.Random(1234)
    for n, count in ((10, 2), (12, 2), (32, 1)):
        sets = [[rng.randrange(p) for _ in range(2 * n)] for _ in range(count)]
        want = np.concatenate([pack(G.witness(field, s)) for s in sets])
        assert L.witness_block(field, n) * 32 * count == want.size
        got = L.sha256_witness_batch(field, n, np.concatenate([pack(s) for s in sets]))
        assert np.array_equal(got, want), f"n = {n}"


@pytest.mark.parametrize("field", FIELDS)
def test_past_the_grid_stride_boundary(L, spec, field):
    """one CTA per call once there are SMs x 8 calls or more: the first calls past the grid wrap round the grid-stride loop"""
    lib = L._capi.lib()
    n, fmt = 1, field % 2
    sets, want = _expected(spec, field, n, fmt)
    blk = L.witness_block(field, n)
    count = _grid_boundary() + 1
    pick = _calls(count, field)
    d_in = torch.from_numpy(_inputs(spec, field, sets, pick, fmt)).cuda()
    out = torch.empty((count, blk, 32), dtype=torch.uint8, device="cuda")
    _chk(L, lib.lurk_sha256_witness_batch_dev(field, n, d_in.data_ptr(), count, out.data_ptr(), fmt, None))
    torch.cuda.synchronize()
    assert torch.equal(out, want[torch.from_numpy(pick).cuda()])


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("n", [1, 2])
def test_scatter_leaves_everything_else_untouched(L, spec, field, n):
    lib = L._capi.lib()
    fmt = 1
    sets, want = _expected(spec, field, n, fmt)
    blk = L.witness_block(field, n)
    count = 33
    gaps = np.random.default_rng(field + n).integers(0, 50, size=count)
    order = np.random.default_rng(n).permutation(count)           # blocks land out of call order
    offs = np.zeros(count, dtype=np.uint64)
    pos = 3
    for k in order:
        offs[k] = pos
        pos += blk + int(gaps[k])
    total = pos + 11
    pick = _calls(count, 99 + field)
    d_in = torch.from_numpy(_inputs(spec, field, sets, pick, fmt)).cuda()
    W = torch.full((total, 32), 0x5C, dtype=torch.uint8, device="cuda")
    d_off = torch.from_numpy(offs.astype(np.int64)).cuda()
    _chk(L, lib.lurk_sha256_witness_scatter_dev(field, n, d_in.data_ptr(), count, d_off.data_ptr(), W.data_ptr(), fmt, None))
    torch.cuda.synchronize()
    mask = torch.zeros(total, dtype=torch.bool, device="cuda")
    for k in range(count):
        o = int(offs[k])
        assert torch.equal(W[o:o + blk], want[int(pick[k])]), f"block {k}"
        mask[o:o + blk] = True
    assert bool((W[~mask] == 0x5C).all())


def test_inputs_not_below_p_are_refused(L, spec):
    p = spec.FIELD_MODULUS[0]
    with pytest.raises(L.LurkError) as e:
        L.sha256_witness_batch(0, 1, pack([5, p]))
    assert e.value.code == L._capi.ERR_RANGE


def test_two_host_threads(L, spec):
    results, errors = {}, []

    def run(field, n):
        try:
            sets, blocks = _sets(spec, field, n)
            pick = _calls(40, field)
            got = L.sha256_witness_batch(field, n, _inputs(spec, field, sets, pick, 0))
            results[(field, n)] = np.array_equal(got.reshape(40, -1, 32), blocks[pick])
        except Exception as ex:      # noqa: BLE001 -- reported below
            errors.append(ex)

    for f, n in ((0, 1), (2, 2)):
        _sets(spec, f, n)
    ts = [threading.Thread(target=run, args=a) for a in ((0, 1), (2, 2))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors and results == {(0, 1): True, (2, 2): True}


def test_fold_context_folds_steps_with_sha256_blocks(L, spec, oracle):
    """sha256_ivc-like step on BN254: frames of [2n inputs | the call's block]; the inputs come through the glue span,
    the blocks from the context's SHA-256 batch; the R1CS rows are the gadget's constraints.  Four steps, the last with
    device-resident inputs; the fresh W of every step is the oracle's, and the folded instance satisfies the relation."""
    field, curve, n, frames = 0, 0, 1, 2
    p = spec.FIELD_MODULUS[field]
    blk = L.witness_block(field, n)
    per = 2 * n + blk
    n_w, n_x = frames * per, 2
    A, B, Cm = [], [], []
    for f in range(frames):
        a, b, c = G.r1cs_rows(field, n, f * per + 2 * n, f * per, n_w)
        A += a; B += b; Cm += c
    mats = [nifs.rows_to_csr(A), nifs.rows_to_csr(B), nifs.rows_to_csr(Cm)]
    rows = len(A)
    bases = oracle.gen_bases(curve, max(n_w, rows))
    ck = L.CommitmentKey(curve, bases)
    ctx = L.NovaFoldContext(curve, ck, n_w, n_x, mats, depth=1)
    bi = ctx.add_sha256_batch(n, [f * per + 2 * n for f in range(frames)])
    ctx.set_spans([(0, 2 * n, per, frames)])
    o = nifs.NovaOracle(curve, bases, mats, n_w, n_x)
    rng = random.Random(5)
    for step in range(4):
        ins = [[rng.randrange(p) for _ in range(2 * n)] for _ in range(frames)]
        if step == 1:
            ins[0] = [p - 1] * (2 * n)
        W = []
        for s in ins:
            W += s + G.witness(field, s)
        X2 = [rng.randrange(p), rng.randrange(p)]
        ctx.host_buffer(0, -2)[:] = pack(X2)
        ro = np.zeros((24, 32), dtype=np.uint8)
        for pos, v in ((4, X2[0]), (5, X2[1])):
            ro[pos] = pack([v])
        ctx.host_buffer(0, -3)[:] = ro.reshape(-1)
        flat = [x for s in ins for x in s]
        if step < 3:
            ctx.host_buffer(0, bi)[:] = pack(flat)
            ctx.host_buffer(0, -1)[:] = pack(flat)
            ctx.stage_a(0)
        else:
            # device-resident inputs: the batch's device buffer and the glue columns of W2, Montgomery form
            ctx.sync()
            mont = pack([x * R % p for x in flat])
            ctx.device_view(0, bi).copy_(torch.from_numpy(mont).cuda())
            w2 = ctx.device_view(0, -4).view(-1, 32)
            for f in range(frames):
                w2[f * per:f * per + 2 * n] = torch.from_numpy(mont[64 * n * f:64 * n * (f + 1)].reshape(-1, 32)).cuda()
            x2m = pack([x * R % p for x in X2]).reshape(-1, 32)
            w2[n_w + 1:n_w + 1 + n_x] = torch.from_numpy(x2m).cuda()
            torch.cuda.synchronize()
            ctx.stage_a(0, resident=True)
        got = [v * pow(R, -1, p) % p for v in ints(ctx.read_device(0, -4))[:n_w]]
        assert got == W, f"step {step}: fresh W"
        if step == 0:
            ctx.init_running(0)
            o.init_running(pack(W), X2)
        else:
            ctx.stage_b_launch(0)
        ctx.collect(0)
    run = ctx.get_running()
    assert o.bad_rows(run["W"], run["E"], ints(run["u"])[0], ints(run["X"])) == 0
    assert ctx.check_running() == (0, True, True)
    ctx.close()
