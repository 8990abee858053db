"""GPU parity of the Poseidon kernels in every launch shape `launch_arity` (csrc/poseidon_kernel.cuh) picks, bit for bit
against the oracle: the warp-per-sponge latency shape, the thread-per-sponge medium shape with CTAs of 32, 64 and 128, and
the persistent throughput shape including its second grid-stride pass.  Each shape runs in digest and witness mode, with
canonical and Montgomery inputs, on preimages that reach the top of the field.  Also: scattered witness blocks, the host
entry point's tail chunk, DAG levels wider than the latency shape, bit decomposition in both formats, and the fold context
at rc = 600 frames, where the hash4 batch of a step lands in the medium shape."""
import json
import re

import numpy as np
import pytest

from util import ints, pack, random_elements

pytestmark = pytest.mark.gpu
FIELDS = [0, 1, 2, 3]
ARITIES = [3, 4, 6, 8]
LATENCY_MAX = 8192            # launch_arity: batches up to this size run the warp-per-sponge kernel
R = 1 << 256


def big_cta(arity):
    """CTA width of the throughput shape (the thread-per-sponge kernel's __launch_bounds__)"""
    return 384 if arity >= 6 else 512


def launch_shape(n, arity, sms):
    """(kernel, CTA width) that launch_arity picks for a batch of n sponges on a device with `sms` SMs"""
    big = big_cta(arity)
    if n >= sms * big // 2:
        return "poseidon_kernel", big
    if n <= LATENCY_MAX:
        return "poseidon_warp_kernel", 128
    return "poseidon_kernel", 128 if n >= sms * 128 else 64 if n >= sms * 64 else 32


def sweep(arity, sms):
    """{label: batch size}: the edges of every launch shape.  `second_pass` has more sponges than the persistent grid has
    threads, so some threads hash a second sponge."""
    big, per_warp = big_cta(arity), 32 // (arity + 1)
    return {"one": 1, "warp": per_warp, "warp+1": per_warp + 1, "latency_max": LATENCY_MAX, "cta32": LATENCY_MAX + 1,
            "cta64": sms * 64, "cta128": sms * big // 2 - 1, "throughput": sms * big // 2, "second_pass": sms * big + 77}


def expected_shape(label, arity):
    """the shape each sweep label claims to reach"""
    if label in ("one", "warp", "warp+1", "latency_max"):
        return "poseidon_warp_kernel", 128
    return "poseidon_kernel", {"cta32": 32, "cta64": 64, "cta128": 128}.get(label, big_cta(arity))


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def preimages(spec, field, arity, n, seed):
    """n preimages whose elements are drawn half from the `edge` shape (the top of the field, Montgomery-top operands,
    0, 1, p-1, ...) and half from `lem` (tags and values); row 0 is all zero, rows 1 and n-1 are all p-1"""
    p = spec.FIELD_MODULUS[field]
    rng = np.random.default_rng(seed)
    pool = random_elements(field, 4096, seed=seed, shape="edge").reshape(-1, 32)
    out = random_elements(field, n * arity, seed=seed + 1, shape="lem").reshape(-1, 32)
    pick = rng.random(n * arity) < 0.5
    out[pick] = pool[rng.integers(0, len(pool), size=int(pick.sum()))]
    out = out.reshape(n, arity * 32)
    out[0] = 0
    top = pack([p - 1] * arity)
    for row in {1, n - 1} - {0}:
        if row < n:
            out[row] = top
    return out.reshape(-1)


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _convert(L, field, t, n, fmt):
    """a fresh device buffer holding the n elements of t converted to `fmt` by the library's conversion kernel"""
    import torch
    out = torch.empty(n * 32, dtype=torch.uint8, device="cuda")
    L._capi.check(L._capi.lib().lurk_convert_dev(field, t.data_ptr(), n, fmt, out.data_ptr(), None))
    return out


def _check_mont_with_ints(spec, field, mont, canon):
    """Montgomery bytes against canonical bytes with Python integers: every element reduced, x R^-1 mod p equal"""
    p = spec.FIELD_MODULUS[field]
    rinv = pow(R, -1, p)
    got, want = ints(mont), ints(canon)
    assert all(g < p for g in got), "Montgomery element not reduced below p"
    assert [g * rinv % p for g in got] == want


def _sample_rows(rng, n, k):
    return np.unique(np.concatenate([[0, n - 1], rng.integers(0, n, size=k)])).astype(np.int64)


def test_sweep_reaches_every_launch_shape(L, sms, tmp_path):
    """every sweep size launches the kernel and CTA width it is labelled with, as the profiler sees it"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    lib = L._capi.lib()
    plan = [(arity, label, n) for arity in ARITIES for label, n in sweep(arity, sms).items()]
    nmax = max(n for _, _, n in plan)
    d_pre = torch.zeros(nmax * 8 * 32, dtype=torch.uint8, device="cuda")
    out = torch.empty(nmax * 32, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for arity, _, n in plan:
            L._capi.check(lib.lurk_poseidon_hash_batch_dev(0, arity, d_pre.data_ptr(), n, out.data_ptr(), L.FMT_CANONICAL, None))
            torch.cuda.synchronize()
    trace = tmp_path / "poseidon_shapes.json"
    prof.export_chrome_trace(str(trace))
    with open(trace) as f:
        events = json.load(f)["traceEvents"]
    kernels = sorted((e for e in events if e.get("cat") == "kernel" and "poseidon" in e.get("name", "")), key=lambda e: e["ts"])
    assert len(kernels) == len(plan), [e["name"] for e in kernels]
    seen = set()
    for (arity, label, n), e in zip(plan, kernels):
        name = re.search(r"\b(poseidon_warp_kernel|poseidon_kernel)<", e["name"]).group(1)
        got = (name, e["args"]["block"][0])
        assert got == expected_shape(label, arity), f"arity {arity}: sweep size {label} = {n} launches {got}"
        assert got == launch_shape(n, arity, sms), f"arity {arity}: n = {n}: the mirror of launch_arity is stale"
        if label in ("throughput", "second_pass"):
            assert e["args"]["grid"][0] == sms, "the throughput shape is one persistent CTA per SM"
        seen.add((big_cta(arity), got))
    for big in (384, 512):
        assert {s for b, s in seen if b == big} == {("poseidon_warp_kernel", 128), ("poseidon_kernel", 32), ("poseidon_kernel", 64),
                                                     ("poseidon_kernel", 128), ("poseidon_kernel", big)}
    assert sweep(4, sms)["second_pass"] > sms * big_cta(4) and sweep(8, sms)["second_pass"] > sms * big_cta(8)


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("arity", ARITIES)
def test_digests_every_launch_shape(L, oracle, spec, sms, field, arity):
    import torch
    lib = L._capi.lib()
    sizes = sweep(arity, sms)
    nmax = sizes["second_pass"]
    pre = preimages(spec, field, arity, nmax, seed=100 * field + arity)
    want = _dev(oracle.poseidon_hash_batch(field, arity, pre, nthreads=8))
    d_pre = _dev(pre)
    d_mont = _convert(L, field, d_pre, nmax * arity, L.FMT_MONTGOMERY)
    rng = np.random.default_rng(field + 10 * arity)
    rows = torch.from_numpy(_sample_rows(rng, nmax * arity, 200)).cuda()
    _check_mont_with_ints(spec, field, d_mont.view(-1, 32)[rows].cpu().numpy(), d_pre.view(-1, 32)[rows].cpu().numpy())
    out = torch.empty((nmax + 1) * 32, dtype=torch.uint8, device="cuda")
    for fmt, src in ((L.FMT_CANONICAL, d_pre), (L.FMT_MONTGOMERY, d_mont)):
        for label, n in sizes.items():
            out.fill_(0xA5)
            L._capi.check(lib.lurk_poseidon_hash_batch_dev(field, arity, src.data_ptr(), n, out.data_ptr(), fmt, None))
            what = f"{label} n={n} fmt={fmt}"
            assert bool((out[n * 32:(n + 1) * 32] == 0xA5).all()), f"{what}: wrote past the last digest"
            got = out[:n * 32] if fmt == L.FMT_CANONICAL else _convert(L, field, out, n, L.FMT_CANONICAL)
            assert torch.equal(got, want[:n * 32]), what
            if fmt == L.FMT_MONTGOMERY:
                rows = torch.from_numpy(_sample_rows(rng, n, 32)).cuda()
                _check_mont_with_ints(spec, field, out[:n * 32].view(n, 32)[rows].cpu().numpy(), want[:n * 32].view(n, 32)[rows].cpu().numpy())


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("arity", ARITIES)
def test_witness_blocks_every_launch_shape(L, oracle, spec, sms, field, arity):
    """whole blocks up to the throughput threshold; at the second-pass size the first CTA's blocks, the last 2 000 (every
    second-pass sponge) and a random sample"""
    import torch
    lib = L._capi.lib()
    sizes = sweep(arity, sms)
    half, nmax = sizes["throughput"], sizes["second_pass"]
    blk = oracle.witness_block(field, arity)
    assert L._capi.lib().lurk_poseidon_witness_block(field, arity) == blk
    pre = preimages(spec, field, arity, nmax, seed=1000 + 100 * field + arity)
    want = _dev(oracle.poseidon_witness_batch(field, arity, pre[:half * arity * 32], nthreads=8))
    rng = np.random.default_rng(7 * field + arity)
    sel = np.unique(np.concatenate([np.arange(big_cta(arity)), np.arange(nmax - 2000, nmax), rng.integers(0, nmax, size=500)]))
    want_sel = _dev(oracle.poseidon_witness_batch(field, arity, pre.reshape(nmax, -1)[sel], nthreads=8))
    d_pre = _dev(pre)
    d_mont = _convert(L, field, d_pre, nmax * arity, L.FMT_MONTGOMERY)
    out = torch.empty((nmax * blk + 1) * 32, dtype=torch.uint8, device="cuda")
    d_sel = torch.from_numpy(sel.astype(np.int64)).cuda()
    for fmt, src in ((L.FMT_CANONICAL, d_pre), (L.FMT_MONTGOMERY, d_mont)):
        for label, n in sizes.items():
            out.fill_(0xA5)
            L._capi.check(lib.lurk_poseidon_witness_batch_dev(field, arity, src.data_ptr(), n, out.data_ptr(), fmt, None))
            what = f"{label} n={n} fmt={fmt}"
            assert bool((out[n * blk * 32:(n * blk + 1) * 32] == 0xA5).all()), f"{what}: wrote past the last block"
            if n <= half:
                got, ref = out[:n * blk * 32], want[:n * blk * 32]
            else:
                got, ref = out[:n * blk * 32].view(n, blk * 32)[d_sel].reshape(-1), want_sel
            m = got.numel() // 32
            canon = got if fmt == L.FMT_CANONICAL else _convert(L, field, got, m, L.FMT_CANONICAL)
            assert torch.equal(canon, ref), what
            if fmt == L.FMT_MONTGOMERY:
                k = got.numel() // (blk * 32)
                rows = torch.from_numpy(_sample_rows(rng, k, 6)).cuda()
                _check_mont_with_ints(spec, field, got.view(k, blk * 32)[rows].cpu().numpy(), ref.view(k, blk * 32)[rows].cpu().numpy())
    del out, want, want_sel
    torch.cuda.empty_cache()


@pytest.mark.parametrize("field", [0, 2])
@pytest.mark.parametrize("arity", [4, 8])
@pytest.mark.parametrize("shape", ["medium", "throughput"])
def test_witness_scatter_permuted_offsets(L, oracle, spec, sms, field, arity, shape):
    """blocks land at a shuffled permutation of slot positions with three-element gaps; the gaps keep their canary bytes"""
    import torch
    n = 8400 if shape == "medium" else sms * big_cta(arity) // 2 + 1000
    kernel, cta = launch_shape(n, arity, sms)
    assert kernel == "poseidon_kernel" and (cta < big_cta(arity)) == (shape == "medium")
    blk, gap = oracle.witness_block(field, arity), 3
    stride = blk + gap
    rng = np.random.default_rng(field + arity)
    perm = rng.permutation(n)
    offs = (1 + perm * stride).astype(np.uint64)                  # element 0 of the buffer is a canary too
    pre = preimages(spec, field, arity, n, seed=2000 + field + arity)
    total = 1 + n * stride
    expected = np.full((total, 32), 0xAB, dtype=np.uint8)
    expected[1:].reshape(n, stride, 32)[perm, :blk] = oracle.poseidon_witness_batch(field, arity, pre, nthreads=8).reshape(n, blk, 32)
    W = torch.full((total * 32,), 0xAB, dtype=torch.uint8, device="cuda")
    d_pre, d_off = _dev(pre), _dev(offs)
    L._capi.check(L._capi.lib().lurk_poseidon_witness_scatter_dev(field, arity, d_pre.data_ptr(), n, W.data_ptr(), d_off.data_ptr(),
                                                                  L.FMT_CANONICAL, None))
    assert torch.equal(W, _dev(expected.reshape(-1)))


@pytest.mark.parametrize("field,arity", [(0, 4), (2, 8)])
def test_host_entry_point_tail_chunk(L, oracle, spec, sms, field, arity):
    """lurk_poseidon_hash_batch cuts its input into chunks of 48 MB of input + output: one full chunk (throughput shape)
    and a remainder in the medium shape"""
    chunk = (48 << 20) // (arity * 32 + 32)
    rest = sms * 64 + 5
    assert launch_shape(chunk, arity, sms) == ("poseidon_kernel", big_cta(arity))
    assert launch_shape(rest, arity, sms) in (("poseidon_kernel", 32), ("poseidon_kernel", 64), ("poseidon_kernel", 128))
    n = chunk + rest
    pre = preimages(spec, field, arity, n, seed=3000 + field + arity)
    out = np.zeros(n * 32, dtype=np.uint8)
    L._capi.check(L._capi.lib().lurk_poseidon_hash_batch(field, arity, L._capi.np_ptr(pre), n, L._capi.np_ptr(out)))
    assert np.array_equal(out, oracle.poseidon_hash_batch(field, arity, pre, nthreads=8))


@pytest.mark.parametrize("field", [0, 2])
def test_wide_dag_levels(L, oracle, sms, field):
    """store hydration hashes in Montgomery form, one batch per (level, arity): level 0 is a throughput-sized TUPLE2 (H4)
    batch and a medium COMMITMENT (H3) batch over edge atoms, level 1 a CTA-32 TUPLE4 (H8) batch and a throughput TUPLE3
    (H6) batch, level 2 a COMPACT (H4) batch; tags cover all of u16"""
    TUPLE2, TUPLE3, TUPLE4, COMPACT, COMMITMENT = 2, 3, 4, 5, 6
    rng = np.random.default_rng(40 + field)
    n_atoms = 4096
    atoms = random_elements(field, n_atoms, seed=41 + field, shape="edge")
    levels = [[(TUPLE2, 4, sms * 256 + 77), (COMMITMENT, 3, sms * 128 + 11)],
              [(TUPLE4, 8, LATENCY_MAX + 101), (TUPLE3, 6, sms * 192 + 33)],
              [(COMPACT, 4, 3000)]]
    assert [launch_shape(n, a, sms) for lvl in levels for _, a, n in lvl] == [
        ("poseidon_kernel", 512), ("poseidon_kernel", 128), ("poseidon_kernel", 32), ("poseidon_kernel", 384), ("poseidon_warp_kernel", 128)]
    total = sum(n for lvl in levels for _, _, n in lvl)
    nodes = np.zeros(total, dtype=oracle.DAG_NODE)
    nodes["tag"] = rng.integers(0, 0x10000, size=(total, 4))
    nodes["tag"][::97] = 0xffff
    first, prev = 0, None              # prev: (first, count) of the previous level's nodes
    for lvl in levels:
        count = sum(n for _, _, n in lvl)
        kinds = np.concatenate([np.full(n, k, dtype=np.uint8) for k, _, n in lvl])
        nodes["kind"][first:first + count] = kinds[rng.permutation(count)]
        child = rng.integers(0, n_atoms + first, size=(count, 4)) if prev else rng.integers(0, n_atoms, size=(count, 4))
        if prev:   # child 0 or 1 (every kind hashes both) lies on the previous level: the node is on this one
            child[np.arange(count), rng.integers(0, 2, size=count)] = n_atoms + prev[0] + rng.integers(0, prev[1], size=count)
        nodes["child"][first:first + count] = child
        prev = (first, count)
        first += count
    out = np.zeros(total * 32, dtype=np.uint8)
    L._capi.check(L._capi.lib().lurk_dag_hash(field, L._capi.np_ptr(nodes), total, L._capi.np_ptr(atoms), n_atoms, L._capi.np_ptr(out)))
    assert np.array_equal(out, oracle.dag_hash(field, nodes, atoms))


@pytest.mark.parametrize("field", FIELDS)
def test_bitdecomp_blocks_both_formats(L, oracle, spec, field):
    import torch
    lib = L._capi.lib()
    n = 5 * 128 + 37                                         # five CTAs and a ragged tail
    vals = random_elements(field, n, seed=60 + field, shape="edge")
    blk = oracle.bitdecomp_size(field)
    want = oracle.bitdecomp_witness_batch(field, vals, nthreads=8)
    p = spec.FIELD_MODULUS[field]
    for fmt in (L.FMT_CANONICAL, L.FMT_MONTGOMERY):
        src = _dev(vals if fmt == L.FMT_CANONICAL else pack([x * R % p for x in ints(vals)]))
        out = torch.full(((n * blk + 1) * 32,), 0xA5, dtype=torch.uint8, device="cuda")
        L._capi.check(lib.lurk_bitdecomp_witness_batch_dev(field, src.data_ptr(), n, out.data_ptr(), fmt, None))
        assert bool((out[n * blk * 32:] == 0xA5).all()), f"fmt={fmt}: wrote past the last block"
        got = out[:n * blk * 32]
        if fmt == L.FMT_CANONICAL:
            assert np.array_equal(got.cpu().numpy(), want)
        else:
            assert np.array_equal(_convert(L, field, got, n * blk, L.FMT_CANONICAL).cpu().numpy(), want)
            _check_mont_with_ints(spec, field, got.cpu().numpy(), want)


class _LazyInts:
    """W[i] as a Python integer, decoded on demand (glue definitions read a few columns of a multi-million-element W)"""

    def __init__(self, W):
        self.W = W

    def __getitem__(self, i):
        return int.from_bytes(self.W[i].tobytes(), "little")


def test_fold_rc600_medium_hash4_batch(L, oracle, spec, sms):
    """the reference's bench configuration rc = 600: 600 frames of 14 hash4, 6 hash8, 1 commitment and 3 bit-decomposition
    slots.  Stage A writes 8 400 hash4 blocks in the medium shape from canonical, then from Montgomery inputs, and builds
    the all-dummy witness D from zeros with the same kernel; W2 must equal the oracle's, commit(W2) = commit(W2 - D) +
    commit(D) must equal a direct commitment, and the folded instance must satisfy the relaxed R1CS."""
    import torch
    from oracle import nifs
    from test_gpu_fold_pipeline import CURVE, FIELD, _fill, _layout, _mont_bytes
    frames, glue = 600, 4
    kernel, cta = launch_shape(14 * frames, 4, sms)
    assert kernel == "poseidon_kernel" and cta < big_cta(4), "the hash4 batch of one step is not medium-shaped"
    rng = np.random.default_rng(600)
    p = spec.FIELD_MODULUS[FIELD]
    lay = _layout(oracle, frames, glue)
    mats, n_w, glue_fn = nifs.synthetic_step_circuit(rng, frames, lay["slot_elems"], glue, 4)
    rows = len(mats[0][0]) - 1
    ck = L.CommitmentKey(CURVE, L.synthetic_bases(CURVE, max(n_w, rows)))
    ctx = L.NovaFoldContext(CURVE, ck, n_w, 2, mats, depth=2, fmt=L.FMT_CANONICAL)
    bi = {a: ctx.add_slot_batch(a, lay["offs"][a]) for a, _ in lay["slots"]}
    bi[0] = ctx.add_slot_batch(0, lay["offs"][0])
    ctx.set_spans([(lay["slot_elems"], glue, lay["per"], frames)])
    pp = 0x600

    def step(seed):
        pre = {}
        for a, n in lay["slots"]:
            x = preimages(spec, FIELD, a, n, seed=seed + a).reshape(n, a * 32)
            x[rng.random(n) < 0.6] = 0                                 # most slots are dummies
            pre[a] = x.reshape(-1)
        bd = random_elements(FIELD, lay["nbd"], seed=seed, shape="edge")
        W = np.zeros((n_w, 32), dtype=np.uint8)
        for a, n in lay["slots"]:
            blk = lay["blocks"][a]
            W[lay["offs"][a].astype(np.int64)[:, None] + np.arange(blk)] = oracle.poseidon_witness_batch(FIELD, a, pre[a], nthreads=8).reshape(n, blk, 32)
        bdb = lay["bd_block"]
        W[lay["offs"][0].astype(np.int64)[:, None] + np.arange(bdb)] = oracle.bitdecomp_witness_batch(FIELD, bd, nthreads=8).reshape(-1, bdb, 32)
        gv = glue_fn(_LazyInts(W), p)
        for dst, v in gv.items():
            W[dst] = np.frombuffer(int(v).to_bytes(32, "little"), dtype=np.uint8)
        glue_dense = pack([gv[f * lay["per"] + lay["slot_elems"] + g] for f in range(frames) for g in range(glue)])
        X2 = [int(rng.integers(1, 2**62)) * int(rng.integers(1, 2**62)) for _ in range(2)]
        return dict(pre=pre, bd=bd, glue=glue_dense, X2=X2, W2=W.reshape(-1))

    def check_w2(b, W2):
        z2 = ctx.read_device(b, L._capi.FOLD_BUF_W2)[:n_w * 32]
        canon = _convert(L, FIELD, _dev(z2), n_w, L.FMT_CANONICAL)
        assert torch.equal(canon, _dev(W2)), f"buffer {b}: W2"
        sample = _sample_rows(rng, n_w, 2000)
        _check_mont_with_ints(spec, FIELD, z2.reshape(n_w, 32)[sample], W2.reshape(n_w, 32)[sample])

    st = step(6000)
    _fill(ctx, 0, lay, st, pp, bi)
    ctx.stage_a(0)
    check_w2(0, st["W2"])
    ctx.init_running(0)
    rec = ctx.collect(0)
    assert np.array_equal(rec.comm_W, ck.commit(st["W2"])), "comm_W of the canonical step"

    st = step(7000)
    _fill(ctx, 1, lay, st, pp, bi, mont=lambda x, base=False: _mont_bytes(spec, x, field=1 if base else 0))
    ctx.stage_a(1, fmt=L.FMT_MONTGOMERY)
    check_w2(1, st["W2"])
    ctx.stage_b_launch(1)
    rec = ctx.collect(1)
    assert np.array_equal(rec.comm_W, ck.commit(st["W2"])), "comm_W of the Montgomery step"
    assert ctx.check_running() == (0, True, True)
    ctx.close()
    ck.close()
