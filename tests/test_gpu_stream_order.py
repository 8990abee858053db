"""The ordering contract of the C ABI (include/lurk_b200.h, "Threading"): a `*_dev` call reads its inputs in the order of the caller's
stream and, when it says it returns when done, leaves nothing of its own work behind it.  Several calls fork side streams from the
caller's stream and join them back (HyperKZG, IPA, compress, recursive verify); the fold context runs on streams of its own.

Every other GPU test hands these calls inputs that are already complete, so a missing cudaStreamWaitEvent or an early return would pass
there.  Here the caller's stream S is non-blocking and, before each call, runs a spin of about 50 ms and only then the copy of the real
inputs into the buffers the call reads.  Until that copy the buffers hold another valid input set, so a call that reads early answers for
those; output buffers start as 0xA5 bytes (not below any of the four moduli), so a call that returns early leaves them behind.  Each result
must equal, byte for byte, the same call's result on inputs made complete beforehand (the path the other tests pin to the oracle), and
the cheap calls are also checked against Python integers or the oracle.  The spin ends by itself: nothing here waits on a condition that
could fail to come."""
import ctypes as C
import hashlib

import numpy as np
import pytest

from test_gpu_compress import cchal
from test_gpu_spartan_chain import challenge
from util import ints, pack, random_elements

pytestmark = pytest.mark.gpu

POISON = 0xA5
SPIN_MS = 50.0
N = 1 << 16          # element-wise calls and witness generators: the call's own work outlasts its launch
N_PROVE = 1 << 18    # provers
CUDA_STREAM_NON_BLOCKING = 1


def _cudart():
    """the CUDA runtime library torch has loaded into this process"""
    import torch
    torch.cuda.init()
    with open("/proc/self/maps") as f:
        paths = sorted({line.split()[-1] for line in f if "libcudart.so" in line})
    return C.CDLL(paths[0] if paths else "libcudart.so.12")


def _stream_flags(rt, handle):
    flags = C.c_uint()
    assert rt.cudaStreamGetFlags(C.c_void_p(handle), C.byref(flags)) == 0
    return flags.value


class Streams:
    """S: the caller's non-blocking stream; S2: a second one for reading the outputs of calls that return when done; spin: the cycle
    count of torch.cuda._sleep that lasts about SPIN_MS"""

    def __init__(self):
        import torch
        rt = _cudart()
        self._own = []
        self.S, self.S2 = self._non_blocking(torch, rt), self._non_blocking(torch, rt)
        for s in (self.S, self.S2):
            assert _stream_flags(rt, s.cuda_stream) & CUDA_STREAM_NON_BLOCKING
        cycles = 1 << 22
        torch.cuda._sleep(cycles)
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        torch.cuda._sleep(cycles)
        t1.record()
        t1.synchronize()
        self.spin = int(cycles * SPIN_MS / t0.elapsed_time(t1))

    def _non_blocking(self, torch, rt):
        s = torch.cuda.Stream()
        if _stream_flags(rt, s.cuda_stream) & CUDA_STREAM_NON_BLOCKING:
            return s
        h = C.c_void_p()
        assert rt.cudaStreamCreateWithFlags(C.byref(h), CUDA_STREAM_NON_BLOCKING) == 0
        self._own.append((rt, h))
        return torch.cuda.ExternalStream(h.value)

    def close(self):
        import torch
        torch.cuda.synchronize()
        for rt, h in self._own:
            rt.cudaStreamDestroy(h)


@pytest.fixture(scope="module")
def st():
    s = Streams()
    yield s
    s.close()


def _norm(x):
    """host results as plain comparable values"""
    import torch
    if isinstance(x, dict):
        return {k: _norm(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [_norm(v) for v in x]
    if isinstance(x, np.ndarray):
        return x.tobytes()
    if isinstance(x, torch.Tensor):
        return x.cpu().numpy().tobytes()
    return x


def ordered(st, name, call, inputs, outputs=(), reads=None, asynchronous=False, null_stream=False):
    """call(stream handle) -> host results.  inputs: [(buffer the call reads, real contents, poison contents)], device tensors; outputs:
    device buffers the call writes (0xA5 before it); reads: device buffers compared afterwards (default: outputs).  Runs the call on
    complete real inputs, on complete poison inputs (must differ), then behind the delayed producer on S (null_stream: on the legacy
    default stream, with stream = NULL).  Asserts whether the call returned before its work was done, and returns the settled results."""
    import torch
    prod = torch.cuda.default_stream() if null_stream else st.S
    handle = 0 if null_stream else st.S.cuda_stream
    reads = list(outputs) if reads is None else list(reads)

    def prepare(which):
        for buf, real, poison in inputs:
            buf.copy_(real if which == "real" else poison)
        for o in outputs:
            o.fill_(POISON)
        torch.cuda.synchronize()

    def settled(which):
        prepare(which)
        host = _norm(call(handle))
        torch.cuda.synchronize()
        return host, [r.cpu().numpy().tobytes() for r in reads]

    want = settled("real")
    if inputs:
        assert settled("poison") != want, f"{name}: the poison inputs give the same answer, so an early read would go unseen"
    prepare("poison")
    with torch.cuda.stream(prod):
        torch.cuda._sleep(st.spin)
        for buf, real, _ in inputs:
            buf.copy_(real)
    host = _norm(call(handle))          # host outputs are used as soon as the call returns
    busy = not prod.query()
    reader = prod if asynchronous else st.S2
    with torch.cuda.stream(reader):
        got = [r.clone() for r in reads]
    reader.synchronize()
    got = [g.cpu().numpy().tobytes() for g in got]
    torch.cuda.synchronize()
    assert busy == asynchronous, f"{name}: {'returned only after' if asynchronous else 'returned before'} its stream's work was done"
    assert host == want[0], f"{name}: host outputs differ from the settled call's (an early read of the inputs)"
    for k, (g, w) in enumerate(zip(got, want[1])):
        if g != w:
            left = sum(1 for i in range(0, len(g), 32) if g[i:i + 32] == bytes([POISON]) * 32)
            pytest.fail(f"{name}: device output {k} differs from the settled call's ({left} elements still 0xA5)")
    return want


# ---------------------------------------------------------------------------------------------------------------- device data
def _lib():
    from lurk_beta_b200 import _capi
    return _capi.lib()


def _chk(rc):
    from lurk_beta_b200 import _capi
    _capi.check(rc)


def dev_canonical(buf):
    import torch
    return torch.from_numpy(np.ascontiguousarray(buf, dtype=np.uint8)).cuda()


def dev_mont(field, canon):
    """device tensor of the Montgomery forms of canonical elements (converted on the device, settled)"""
    import torch
    t = dev_canonical(canon)
    _chk(_lib().lurk_convert_dev(field, t.data_ptr(), t.numel() // 32, 1, t.data_ptr(), None))
    torch.cuda.synchronize()
    return t


def real_and_poison(field, n, seed, mont=True):
    """(buffer, real, poison): two different uniform input sets of n elements"""
    make = (lambda c: dev_mont(field, c)) if mont else dev_canonical
    real, poison = make(random_elements(field, n, seed)), make(random_elements(field, n, seed + 7919))
    return (real.clone(), real, poison)


def p_of(field):
    from oracle import spec
    return spec.FIELD_MODULUS[field]


def from_mont(field, buf):
    p = p_of(field)
    rinv = pow(1 << 256, -1, p)
    return [x * rinv % p for x in ints(np.frombuffer(buf, dtype=np.uint8))]


def elems_at(buf, idx):
    """the bytes of elements idx of a buffer of 32-byte elements"""
    a = np.frombuffer(buf, dtype=np.uint8).reshape(-1, 32)
    return a[np.asarray(idx, dtype=np.int64)].reshape(-1)


def sample(n, k=64, seed=0):
    return sorted(set([0, n - 1] + list(np.random.default_rng(seed).integers(0, n, size=k))))


def empty(n_elems):
    import torch
    return torch.empty(n_elems * 32, dtype=torch.uint8, device="cuda")


FIELDS = [0, 1, 2, 3]
CURVES = [0, 1, 2, 3]


# ---------------------------------------------------------------------------------------------------------------- element-wise calls
@pytest.mark.parametrize("field", FIELDS)
def test_convert_axpy_spmv_cross_term(st, field):
    p, R = p_of(field), 1 << 256
    lib = _lib()
    # lurk_convert_dev: canonical -> Montgomery into another buffer
    x = real_and_poison(field, N, 1, mont=False)
    out = empty(N)
    _, (got,) = ordered(st, "lurk_convert_dev", lambda s: _chk(lib.lurk_convert_dev(field, x[0].data_ptr(), N, 1, out.data_ptr(), C.c_void_p(s))),
                        [x], [out], asynchronous=True)
    xi, gi = ints(x[1].cpu().numpy()), ints(np.frombuffer(got, dtype=np.uint8))
    assert all(gi[i] == xi[i] * R % p for i in sample(N))
    # lurk_axpy_dev
    a, b = real_and_poison(field, N, 2), real_and_poison(field, N, 3)
    r = random_elements(field, 1, 4)
    r_mont = pack([ints(r)[0] * R % p])
    _, (got,) = ordered(st, "lurk_axpy_dev", lambda s: _chk(lib.lurk_axpy_dev(field, a[0].data_ptr(), b[0].data_ptr(), r_mont.ctypes.data, N,
                                                                              out.data_ptr(), C.c_void_p(s))), [a, b], [out], asynchronous=True)
    ai, bi, yi = from_mont(field, a[1].cpu().numpy().tobytes()), from_mont(field, b[1].cpu().numpy().tobytes()), from_mont(field, got)
    assert all(yi[i] == (ai[i] + ints(r)[0] * bi[i]) % p for i in sample(N))
    # lurk_spmv_csr_dev: one non-zero per row, at a random column
    rng = np.random.default_rng(field)
    row_ptr = dev_canonical(np.arange(N + 1, dtype=np.uint64).view(np.uint8))
    cols = rng.integers(0, N, size=N).astype(np.uint32)
    col = dev_canonical(cols.view(np.uint8))
    val = dev_mont(field, random_elements(field, N, 5))
    z = real_and_poison(field, N, 6)
    _, (got,) = ordered(st, "lurk_spmv_csr_dev", lambda s: _chk(lib.lurk_spmv_csr_dev(field, row_ptr.data_ptr(), col.data_ptr(), val.data_ptr(), N,
                                                                                      z[0].data_ptr(), out.data_ptr(), C.c_void_p(s))),
                        [z], [out], asynchronous=True)
    vi, zi, yi = from_mont(field, val.cpu().numpy().tobytes()), from_mont(field, z[1].cpu().numpy().tobytes()), from_mont(field, got)
    assert all(yi[i] == vi[i] * zi[int(cols[i])] % p for i in sample(N))
    # lurk_cross_term_dev
    v = [real_and_poison(field, N, 10 + k) for k in range(6)]
    u1, u2 = ints(random_elements(field, 2, 16))
    u1m, u2m = pack([u1 * R % p]), pack([u2 * R % p])
    _, (got,) = ordered(st, "lurk_cross_term_dev",
                        lambda s: _chk(lib.lurk_cross_term_dev(field, *[t[0].data_ptr() for t in v], u1m.ctypes.data, u2m.ctypes.data, N, out.data_ptr(),
                                                               C.c_void_p(s))), v, [out], asynchronous=True)
    vi = [from_mont(field, t[1].cpu().numpy().tobytes()) for t in v]
    ti = from_mont(field, got)
    assert all(ti[i] == (vi[0][i] * vi[4][i] + vi[3][i] * vi[1][i] - u1 * vi[5][i] - u2 * vi[2][i]) % p for i in sample(N))


@pytest.mark.parametrize("field", FIELDS)
def test_ntt_forward_and_inverse(st, field):
    from oracle import spec
    lib = _lib()
    s = spec.TWO_ADICITY[field]
    for log_n in sorted({min(4, s), min(16, s)}):
        n = 1 << log_n
        for inverse in (0, 1):
            a = real_and_poison(field, n, 20 + inverse)
            _, (got,) = ordered(st, f"lurk_ntt_dev(log_n {log_n}, inverse {inverse})",
                                lambda s: _chk(lib.lurk_ntt_dev(field, a[0].data_ptr(), log_n, inverse, C.c_void_p(s))), [a], reads=[a[0]],
                                asynchronous=True)
            if log_n <= 4:
                assert from_mont(field, got) == spec.ntt_naive(field, from_mont(field, a[1].cpu().numpy().tobytes()), inverse=bool(inverse))


@pytest.mark.parametrize("field", FIELDS)
def test_eq_evals_and_ipa_fold_scalars(st, field):
    from oracle import sumcheck as osc
    from lurk_beta_b200 import spartan
    p, lib = p_of(field), _lib()
    # lurk_eq_evals_dev reads no device input: only the early return is observable
    tau = ints(random_elements(field, 16, 30))
    out = empty(N)
    _, (got,) = ordered(st, "lurk_eq_evals_dev", lambda s: spartan.eq_evals(field, tau, out.data_ptr(), stream=s), [], [out], asynchronous=True)
    want = osc.eq_evals(tau, p)
    gi = from_mont(field, got)
    assert all(gi[i] == want[i] for i in sample(N))
    # lurk_ipa_fold_scalars_dev, in place on 2N elements
    a = real_and_poison(field, 2 * N, 31)
    x, y = ints(random_elements(field, 2, 32))
    _, (got,) = ordered(st, "lurk_ipa_fold_scalars_dev", lambda s: spartan.ipa_fold_scalars(field, a[0].data_ptr(), 2 * N, x, y, stream=s), [a],
                        reads=[a[0]], asynchronous=True)
    ai, gi = from_mont(field, a[1].cpu().numpy().tobytes()), from_mont(field, got)
    assert all(gi[i] == (x * ai[i] + y * ai[i + N]) % p for i in sample(N))


def key_on_device(curve, n, label):
    """a from_label key of n points, affine Montgomery, on the device (settled)"""
    import torch
    buf = torch.empty(n * 64, dtype=torch.uint8, device="cuda")
    _chk(_lib().lurk_ck_generate_dev(curve, label, len(label), n, buf.data_ptr(), None))
    torch.cuda.synchronize()
    return buf


@pytest.mark.parametrize("curve", CURVES)
def test_ipa_fold_bases(st, curve):
    from lurk_beta_b200 import spartan
    real, poison = key_on_device(curve, 2 * N, b"stream-order real"), key_on_device(curve, 2 * N, b"stream-order poison")
    g = (real.clone(), real, poison)
    x, y = ints(random_elements(curve, 2, 40))
    ordered(st, "lurk_ipa_fold_bases_dev", lambda s: spartan.ipa_fold_bases(curve, g[0].data_ptr(), 2 * N, x, y, stream=s), [g], reads=[g[0]],
            asynchronous=True)


def diagonal_shape(n_w, rows):
    """CSR over z = (W, u, X) with n_x = 2, one non-zero (1) per row: A = C = column of W[i], B = column of W[i + 1] (of W[0] for the last
    row), so that the cross term A z1 B z2 + A z2 B z1 - u1 C z2 - u2 C z1 is non-zero on every row"""
    i = np.arange(rows, dtype=np.uint64) % n_w
    rp = np.arange(rows + 1, dtype=np.uint64)
    one = np.zeros((rows, 32), dtype=np.uint8)
    one[:, 0] = 1
    one = one.reshape(-1)
    a = (rp, i.astype(np.uint32), one)
    b = (rp, ((i + 1) % n_w).astype(np.uint32), one)
    return [a, b, a]


@pytest.mark.parametrize("field", FIELDS)
def test_spartan_eval_table(st, field):
    from lurk_beta_b200 import spartan
    ctx = spartan.SpartanContext(field, diagonal_shape(N, N), N, 2)
    eq = real_and_poison(field, 1 << ctx.log_rows, 50)
    out = empty(2 * ctx.num_vars)
    r = ints(random_elements(field, 1, 51))[0]
    ordered(st, "lurk_spartan_eval_table_dev", lambda s: ctx.eval_table(eq[0].data_ptr(), r, out.data_ptr(), stream=s), [eq], [out], asynchronous=True)


# ---------------------------------------------------------------------------------------------------------------- witness generators
@pytest.mark.parametrize("field", FIELDS)
def test_poseidon_and_bitdecomp_witnesses(st, field, oracle):
    lib = _lib()
    for arity in (4, 8):
        pre = real_and_poison(field, N * arity, 60 + arity, mont=False)
        out = empty(N)
        _, (got,) = ordered(st, f"lurk_poseidon_hash_batch_dev(arity {arity})",
                            lambda s: _chk(lib.lurk_poseidon_hash_batch_dev(field, arity, pre[0].data_ptr(), N, out.data_ptr(), 0, C.c_void_p(s))),
                            [pre], [out], asynchronous=True)
        assert got == oracle.poseidon_hash_batch(field, arity, pre[1].cpu().numpy(), nthreads=8).tobytes()
    count = 1 << 12
    perm = np.random.default_rng(field).permutation(count).astype(np.uint64)
    for arity in (3, 8, 0):
        blk = lib.lurk_poseidon_witness_block(field, arity) if arity else lib.lurk_bitdecomp_witness_block(field)
        pre = real_and_poison(field, count * max(arity, 1), 70 + arity, mont=False)
        out, base = empty(count * blk), empty(count * blk)
        offs = dev_canonical((perm * blk).view(np.uint8))
        what = f"arity {arity}" if arity else "bit decomposition"
        if arity:
            batch = lambda s: _chk(lib.lurk_poseidon_witness_batch_dev(field, arity, pre[0].data_ptr(), count, out.data_ptr(), 0, C.c_void_p(s)))
            scatter = lambda s: _chk(lib.lurk_poseidon_witness_scatter_dev(field, arity, pre[0].data_ptr(), count, base.data_ptr(), offs.data_ptr(), 0,
                                                                           C.c_void_p(s)))
        else:
            batch = lambda s: _chk(lib.lurk_bitdecomp_witness_batch_dev(field, pre[0].data_ptr(), count, out.data_ptr(), 0, C.c_void_p(s)))
            scatter = lambda s: _chk(lib.lurk_bitdecomp_witness_scatter_dev(field, pre[0].data_ptr(), count, base.data_ptr(), offs.data_ptr(), 0,
                                                                            C.c_void_p(s)))
        _, (dense,) = ordered(st, f"witness batch ({what})", batch, [pre], [out], asynchronous=True)
        _, (placed,) = ordered(st, f"witness scatter ({what})", scatter, [pre], [base], asynchronous=True)
        d = np.frombuffer(dense, dtype=np.uint8).reshape(count, blk * 32)
        assert np.array_equal(np.frombuffer(placed, dtype=np.uint8).reshape(count, blk * 32)[perm.astype(np.int64)], d)


@pytest.mark.parametrize("field", FIELDS)
def test_sha256_and_trie_witnesses(st, field):
    lib = _lib()
    cases = [("sha256", 2, 64, 2 * 2), ("trie lookup", 0, 256, 2 + 8 * 4), ("trie insert", 1, 128, 3 + 16 * 4)]
    for name, arg, count, per in cases:
        if name == "sha256":
            blk = lib.lurk_sha256_witness_block(field, arg)
        else:
            blk = lib.lurk_trie_witness_block(field, arg, 4)
        assert blk
        inp = real_and_poison(field, count * per, 80 + count, mont=False)
        perm = np.random.default_rng(count).permutation(count).astype(np.uint64)
        offs = dev_canonical((perm * blk).view(np.uint8))
        out, base = empty(count * blk), empty(count * blk)
        if name == "sha256":
            batch = lambda s: _chk(lib.lurk_sha256_witness_batch_dev(field, arg, inp[0].data_ptr(), count, out.data_ptr(), 0, C.c_void_p(s)))
            scatter = lambda s: _chk(lib.lurk_sha256_witness_scatter_dev(field, arg, inp[0].data_ptr(), count, offs.data_ptr(), base.data_ptr(), 0,
                                                                         C.c_void_p(s)))
        else:
            batch = lambda s: _chk(lib.lurk_trie_witness_batch_dev(field, arg, 4, inp[0].data_ptr(), count, out.data_ptr(), 0, C.c_void_p(s)))
            scatter = lambda s: _chk(lib.lurk_trie_witness_scatter_dev(field, arg, 4, inp[0].data_ptr(), count, offs.data_ptr(), base.data_ptr(), 0,
                                                                       C.c_void_p(s)))
        _, (dense,) = ordered(st, f"{name} witness batch", batch, [inp], [out], asynchronous=True)
        _, (placed,) = ordered(st, f"{name} witness scatter", scatter, [inp], [base], asynchronous=True)
        d = np.frombuffer(dense, dtype=np.uint8).reshape(count, blk * 32)
        assert np.array_equal(np.frombuffer(placed, dtype=np.uint8).reshape(count, blk * 32)[perm.astype(np.int64)], d)


@pytest.mark.parametrize("curve", CURVES)
def test_hash_to_curve_batch(st, curve):
    import torch
    lib = _lib()
    msg_len = 32
    rng = np.random.default_rng(curve)
    real = torch.from_numpy(rng.integers(0, 256, size=N * msg_len, dtype=np.uint8)).cuda()
    poison = torch.from_numpy(rng.integers(0, 256, size=N * msg_len, dtype=np.uint8)).cuda()
    m = (real.clone(), real, poison)
    out = torch.empty(N * 64, dtype=torch.uint8, device="cuda")
    _, (got,) = ordered(st, "lurk_hash_to_curve_batch_dev",
                        lambda s: _chk(lib.lurk_hash_to_curve_batch_dev(curve, b"stream-order", m[0].data_ptr(), msg_len, N, out.data_ptr(), 0,
                                                                        C.c_void_p(s))), [m], [out], asynchronous=True)
    from lurk_beta_b200 import commit
    k = sample(N, 8)
    msgs = real.cpu().numpy().reshape(N, msg_len)[k]
    want = commit.hash_to_curve_batch(curve, "stream-order", msgs.reshape(-1), msg_len)
    assert np.array_equal(np.frombuffer(got, dtype=np.uint8).reshape(N, 64)[k].reshape(-1), np.asarray(want).reshape(-1))


# ---------------------------------------------------------------------------------------------------------------- MSM
@pytest.mark.parametrize("curve", CURVES)
def test_msm_run_and_launch_on_a_context_and_its_clone(st, curve):
    import lurk_beta_b200 as L
    ck = L.CommitmentKey.setup(curve, b"stream-order msm", N)
    sc = real_and_poison(curve, N, 90)
    ordered(st, "lurk_msm_ctx_run_dev", lambda s: ck.commit_device(sc[0].data_ptr(), N, stream=s), [sc])
    clone = ck.clone()
    sc2 = real_and_poison(curve, N, 91)

    def launch(s):
        ck.launch_device(sc[0].data_ptr(), N, stream=s)
        clone.launch_device(sc2[0].data_ptr(), N, stream=s)

    # launch + finish on both contexts at once; finish returns the point, so the call as a whole returns when done
    want = ordered(st, "lurk_msm_ctx_launch_dev + _finish", lambda s: (launch(s), [ck.finish(), clone.finish()])[1], [sc, sc2])
    # launch alone returns before the commitments are done
    import torch
    for buf, _, poison in (sc, sc2):
        buf.copy_(poison)
    torch.cuda.synchronize()
    with torch.cuda.stream(st.S):
        torch.cuda._sleep(st.spin)
        for buf, real, _ in (sc, sc2):
            buf.copy_(real)
    launch(st.S.cuda_stream)
    busy = not st.S.query()
    got = _norm([ck.finish(), clone.finish()])
    assert busy, "lurk_msm_ctx_launch_dev returned only after its stream's work was done"
    assert got == want[0]


# ---------------------------------------------------------------------------------------------------------------- calls that return when done
def fs(field):
    """a Fiat-Shamir stand-in: challenge(round, message) -> element"""
    p = p_of(field)
    return lambda rnd, msg: int.from_bytes(hashlib.sha256(rnd.to_bytes(4, "little") + bytes(msg)).digest(), "little") % p


def settled_ip(field, a, b, n):
    from lurk_beta_b200 import spartan
    return spartan.inner_product(field, a.data_ptr(), b.data_ptr(), n)


@pytest.mark.parametrize("field", FIELDS)
def test_inner_product_and_sumcheck_provers(st, field):
    from lurk_beta_b200 import spartan
    p = p_of(field)
    a, b = real_and_poison(field, N, 100), real_and_poison(field, N, 101)
    want = ordered(st, "lurk_inner_product_dev", lambda s: spartan.inner_product(field, a[0].data_ptr(), b[0].data_ptr(), N, stream=s), [a, b])
    ai, bi = from_mont(field, a[1].cpu().numpy().tobytes()), from_mont(field, b[1].cpu().numpy().tobytes())
    assert want[0] == sum(x * y for x, y in zip(ai, bi)) % p
    l1, l2 = 18, 16
    polys = [real_and_poison(field, 1 << l1, 110 + k) for k in range(2)] + [real_and_poison(field, 1 << l2, 120 + k) for k in range(2)]
    c1 = settled_ip(field, polys[0][1], polys[1][1], 1 << l1)
    c2 = settled_ip(field, polys[2][1], polys[3][1], 1 << l2)
    ordered(st, "lurk_sumcheck_prove_dev", lambda s: spartan.sumcheck_prove(field, spartan.QUAD, [t[0].data_ptr() for t in polys[:2]], l1, c1, fs(field),
                                                                            stream=s), polys[:2])
    ordered(st, "lurk_sumcheck_prove_batch_dev",
            lambda s: spartan.sumcheck_prove_batch(field, spartan.QUAD, [([t[0].data_ptr() for t in polys[:2]], l1), ([t[0].data_ptr() for t in polys[2:]], l2)],
                                                   [c1, c2], [1, 5], fs(field), stream=s), polys)
    joint = empty(1 << l1)
    pts = [ints(random_elements(field, l, 130 + l)) for l in (l1, l2)]
    ordered(st, "lurk_batch_eval_reduce_dev",
            lambda s: spartan.batch_eval_reduce(field, [(polys[0][0].data_ptr(), l1, pts[0], 3), (polys[2][0].data_ptr(), l2, pts[1], 4)], fs(field),
                                                d_joint_ptr=joint.data_ptr(), stream=s)[:5], [polys[0], polys[2]], [joint])


def affine_of(buf64):
    v = ints(buf64)
    return (v[0], v[1])


def point_of(buf96):
    v = ints(buf96)
    return (v[0], v[1]) if v[2] else None


def point_of_mont(curve, buf96):
    """(x, y) of a 96-byte point in Montgomery form (base field of curve k: field k ^ 1)"""
    x, y, z = from_mont(curve ^ 1, np.asarray(buf96).tobytes())
    return (x, y) if z else None


@pytest.mark.parametrize("null", [False, True], ids=["stream", "null-stream"])
@pytest.mark.parametrize("curve", CURVES)
def test_ipa_prove_and_verify(st, curve, null):
    import lurk_beta_b200 as L
    from lurk_beta_b200 import spartan
    log_n = 16
    n = 1 << log_n
    ck = L.CommitmentKey.setup(curve, b"stream-order ipa", n)
    ck_c = affine_of(L.synthetic_bases(curve, 1, start=5))
    a, b = real_and_poison(curve, n, 140), real_and_poison(curve, n, 141)
    comm = point_of_mont(curve, ck.commit_device(a[1].data_ptr(), n))
    c = settled_ip(curve, a[1], b[1], n)
    proof, _ = ordered(st, "lurk_ipa_prove_dev", lambda s: spartan.ipa_prove(curve, ck, ck_c, a[0].data_ptr(), b[0].data_ptr(), log_n, fs(curve), stream=s),
                       [a, b], null_stream=null)
    Ls, Rs, a_final, _ = proof
    verdict, _ = ordered(st, "lurk_ipa_verify_dev", lambda s: spartan.ipa_verify(curve, ck, ck_c, comm, c, b[0].data_ptr(), log_n, Ls, Rs, a_final, fs(curve),
                                                                                 stream=s), [b], null_stream=null)
    assert verdict[0] is True


@pytest.mark.parametrize("null", [False, True], ids=["stream", "null-stream"])
@pytest.mark.parametrize("curve", CURVES)
def test_hyperkzg_prove(st, curve, null):
    import lurk_beta_b200 as L
    from lurk_beta_b200 import spartan
    l = 18
    g = affine_of(L.synthetic_bases(curve, 1))
    ck = L.CommitmentKey.powers_of_tau(curve, g, 0x1234567 + curve, 1 << l)
    poly = real_and_poison(curve, 1 << l, 150)
    point = ints(random_elements(curve, l, 151))
    ordered(st, "lurk_hyperkzg_prove_dev", lambda s: spartan.hyperkzg_prove(curve, ck, poly[0].data_ptr(), point, fs(curve), stream=s), [poly],
            null_stream=null)


_SHAPES = {}


def shape(field, log_rows):
    """a Spartan context on diagonal_shape with n_w = rows = 2^log_rows"""
    from lurk_beta_b200 import spartan
    key = (field, log_rows)
    if key not in _SHAPES:
        n = 1 << log_rows
        _SHAPES[key] = spartan.SpartanContext(field, diagonal_shape(n, n), n, 2)
    return _SHAPES[key]


def instance(field, log_rows, seed):
    """(z, E) of a running instance of shape(field, log_rows), each (buffer, real, poison)"""
    n = 1 << log_rows
    return real_and_poison(field, n + 3, seed), real_and_poison(field, n, seed + 1)


@pytest.mark.parametrize("field", FIELDS)
def test_spartan_prove_and_prove_batch(st, field):
    from lurk_beta_b200 import spartan
    big, small = shape(field, 18), shape(field, 16)
    z, E = instance(field, 18, 160)
    z2, E2 = instance(field, 16, 170)
    joint = empty(big.joint_len)
    ordered(st, "lurk_spartan_prove_dev", lambda s: big.prove(z[0].data_ptr(), E[0].data_ptr(), challenge, d_joint_ptr=joint.data_ptr(), stream=s),
            [z, E], [joint])
    ordered(st, "lurk_spartan_prove_batch_dev",
            lambda s: spartan.spartan_prove_batch([big, small], [(z[0].data_ptr(), E[0].data_ptr()), (z2[0].data_ptr(), E2[0].data_ptr())], challenge,
                                                  d_joint_ptr=joint.data_ptr(), stream=s), [z, E, z2, E2], [joint])


@pytest.mark.parametrize("null", [False, True], ids=["stream", "null-stream"])
@pytest.mark.parametrize("field", FIELDS)
def test_recursive_verify(st, field, null):
    import lurk_beta_b200 as L
    n = 1 << 18
    sh = shape(field, 18)
    ck = L.CommitmentKey.setup(field, b"stream-order recursive", n)      # curve k's scalar field is field k
    z, E = instance(field, 18, 180)
    cw, ce = point_of_mont(field, ck.commit_device(z[1].data_ptr(), n)), point_of_mont(field, ck.commit_device(E[1].data_ptr(), n))
    (acc, verdicts), _ = ordered(st, "lurk_recursive_verify_dev",
                                 lambda s: L.recursive.recursive_verify([dict(shape=sh, ck=ck, z=z[0].data_ptr(), E=E[0].data_ptr(), comm_W=cw, comm_E=ce)],
                                                                        stream=s), [z, E], null_stream=null)
    assert verdicts[0]["comm_W_ok"] and verdicts[0]["comm_E_ok"] and verdicts[0]["bad_rows"] > 0


@pytest.mark.parametrize("null", [False, True], ids=["stream", "null-stream"])
@pytest.mark.parametrize("curves", [(0, 1), (2, 3)], ids=["bn254-grumpkin", "pallas-vesta"])
def test_compress_prove(st, curves, null):
    """the secondary's z and E are written on the caller's stream just before the call: its worker stream must follow that work"""
    import lurk_beta_b200 as L
    log_rows = 18
    f1, f2 = curves
    keys = [L.CommitmentKey.setup(c, b"stream-order compress", 2 << log_rows) for c in curves]
    pcs = [("ipa", keys[k], affine_of(L.synthetic_bases(curves[k], 1, start=9))) for k in range(2)]
    cctx = L.compress.CompressContext(shape(f1, log_rows), shape(f2, log_rows), pcs[0], pcs[1])
    z, E = instance(f1, log_rows, 190)
    z2, E2 = instance(f2, log_rows, 200)
    ordered(st, "lurk_compress_prove_dev",
            lambda s: cctx.prove([(z[0].data_ptr(), E[0].data_ptr(), None, None)], (z2[0].data_ptr(), E2[0].data_ptr(), None, None), cchal, stream=s),
            [z, E, z2, E2], null_stream=null)
    cctx.close()


# ---------------------------------------------------------------------------------------------------------------- the fold context
# The fold context runs on streams of its own, created non-blocking, and takes no stream argument.  Its device buffers are ordered for a
# caller by its calls: LURK_FOLD_BUF_Z1 / _E1 (the running instance) and LURK_FOLD_BUF_T by lurk_fold_ctx_collect, LURK_FOLD_BUF_W2 after a
# stage A by lurk_fold_ctx_sync alone; inputs a caller places in W2 for LURK_FOLD_INPUTS_RESIDENT must be complete before stage A.
LOG_FOLD = 22


@pytest.fixture(scope="module")
def fold(L):
    """a BN254 fold context of 2^22 rows and 2^22 witness columns on diagonal_shape, its key, and a verifier-only shape of the same
    matrices for lurk_recursive_verify_dev"""
    n = 1 << LOG_FOLD
    mats = diagonal_shape(n, n)
    ck = L.CommitmentKey.setup(0, b"stream-order fold", n)
    fctx = L.NovaFoldContext(0, ck, n, 2, mats, depth=1)
    fctx.set_spans([(0, n, n, 1)])
    fx = dict(n=n, ck=ck, fctx=fctx, shape=L.spartan.SpartanContext.verifier(0, mats, n, 2), steps=0, z1=None)
    yield fx
    fctx.close()


def fold_stage(L, fx, seed):
    """stage A of a fresh instance with a random W and X from the host buffers; returns (W, X) as canonical bytes"""
    fctx, n = fx["fctx"], fx["n"]
    W, X = random_elements(0, n, seed), random_elements(0, 2, seed + 1)
    fctx.host_buffer(0, L._capi.FOLD_BUF_GLUE)[:] = W
    fctx.host_buffer(0, L._capi.FOLD_BUF_X2)[:] = X
    fctx.host_buffer(0, L._capi.FOLD_BUF_RO)[:] = 0
    fctx.stage_a(0)
    return W, X


def fold_step(L, fx, seed):
    """one step (init_running first, then folds) and its record; fx["z1"] keeps the running z before the step (canonical bytes)"""
    W, X = fold_stage(L, fx, seed)
    if fx["steps"] == 0:
        fx["fctx"].init_running(0)
    else:
        fx["fctx"].stage_b_launch(0)
    fx["steps"] += 1
    fx["fresh"] = (W, X)
    return fx["fctx"].collect(0)


def running_instance(L, fx, rec):
    fctx = fx["fctx"]
    return dict(shape=fx["shape"], ck=fx["ck"], z=fctx.device_buffer(0, L._capi.FOLD_BUF_Z1)[0], E=fctx.device_buffer(0, L._capi.FOLD_BUF_E1)[0],
                comm_W=point_of(rec.running_comm_W), comm_E=point_of(rec.running_comm_E))


def test_collect_makes_the_running_instance_readable(L, fold):
    """right after lurk_fold_ctx_collect, a copy of Z1 and E1 on a fresh non-blocking stream equals them after lurk_fold_ctx_sync, and
    lurk_recursive_verify_dev on another fresh stream gives the verdicts it gives after the sync -- after init_running and after a fold"""
    import torch
    fctx = fold["fctx"]
    z1, e1 = fctx.device_view(0, L._capi.FOLD_BUF_Z1), fctx.device_view(0, L._capi.FOLD_BUF_E1)
    for step in ("init_running", "fold"):
        copy_stream, verify_stream = torch.cuda.Stream(), torch.cuda.Stream()
        rec = fold_step(L, fold, 300 + 10 * fold["steps"])
        with torch.cuda.stream(copy_stream):
            z_now, e_now = z1.clone(), e1.clone()
        verdict_now = L.recursive.recursive_verify([running_instance(L, fold, rec)], stream=verify_stream.cuda_stream)
        fctx.sync()
        copy_stream.synchronize()
        torch.cuda.synchronize()
        assert torch.equal(z_now, z1), f"{step}: Z1 read right after collect differs from Z1 after the sync"
        assert torch.equal(e_now, e1), f"{step}: E1 read right after collect differs from E1 after the sync"
        verdict_after = L.recursive.recursive_verify([running_instance(L, fold, rec)])
        assert verdict_now == verdict_after, step
        v = verdict_after[1][0]
        assert v["comm_W_ok"] and v["comm_E_ok"], step


def test_T_after_stage_b_is_ordered_by_collect(L, fold):
    """right after collect, LURK_FOLD_BUF_T read on a fresh stream is the cross term of the step, against Python integers on sampled rows"""
    import torch
    fctx, n = fold["fctx"], fold["n"]
    if fold["steps"] == 0:
        fold_step(L, fold, 400)
    z1_before = fctx.read_device(0, L._capi.FOLD_BUF_Z1)
    t = fctx.device_view(0, L._capi.FOLD_BUF_T)
    s = torch.cuda.Stream()
    fold_step(L, fold, 410)
    with torch.cuda.stream(s):
        t_now = t.clone()
    s.synchronize()
    fctx.sync()
    assert torch.equal(t_now, t), "T read right after collect differs from T after the sync"
    p = p_of(0)
    rows = sample(n - 1, 256, seed=1) + [n - 1]
    cols = rows + [(i + 1) % n for i in rows] + [n]
    z1 = dict(zip(cols, from_mont(0, elems_at(z1_before, cols))))
    W2 = fold["fresh"][0]
    ti = from_mont(0, elems_at(t_now.cpu().numpy(), rows))
    for i, t_i in zip(rows, ti):
        a2, b2 = ints(elems_at(W2, [i, (i + 1) % n]))
        a1, b1 = z1[i], z1[(i + 1) % n]
        assert t_i == (a1 * b2 + a2 * b1 - z1[n] * a2 - a1) % p, i
        assert t_i != 0, i


def test_W2_after_stage_a_is_ordered_by_sync(L, fold):
    """after stage A and lurk_fold_ctx_sync, LURK_FOLD_BUF_W2 holds (W, 1, X) of the staged inputs in Montgomery form"""
    fctx, n = fold["fctx"], fold["n"]
    W, X = fold_stage(L, fold, 500)
    fctx.sync()
    z2 = fctx.device_view(0, L._capi.FOLD_BUF_W2).cpu().numpy()
    rows = sample(n, 256, seed=2)
    assert from_mont(0, elems_at(z2, rows)) == ints(elems_at(W, rows))
    assert from_mont(0, elems_at(z2, [n, n + 1, n + 2])) == [1] + ints(X)
    # the staged buffer is then folded, so that the context is left with nothing pending
    if fold["steps"] == 0:
        fctx.init_running(0)
    else:
        fctx.stage_b_launch(0)
    fold["steps"] += 1
    fctx.collect(0)


def test_resident_inputs_complete_before_stage_a(L, fold):
    """a caller writes z2 into LURK_FOLD_BUF_W2 on its own non-blocking stream and completes it (the context's streams do not know the
    caller's stream) before stage A with LURK_FOLD_INPUTS_RESIDENT: the step commits to exactly those inputs"""
    import torch
    fctx, n = fold["fctx"], fold["n"]
    if fold["steps"] == 0:
        fold_step(L, fold, 600)
    W, X = random_elements(0, n, 610), random_elements(0, 2, 611)
    z2 = dev_mont(0, np.concatenate([W, pack([1]), X]))
    fctx.sync()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        fctx.device_view(0, L._capi.FOLD_BUF_W2).copy_(z2)
    s.synchronize()
    fctx.stage_a(0, resident=True)
    fctx.stage_b_launch(0)
    fold["steps"] += 1
    rec = fctx.collect(0)
    assert np.array_equal(rec.comm_W, fold["ck"].commit(W)), "comm_W of the resident W2"
