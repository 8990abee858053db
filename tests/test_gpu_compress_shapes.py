"""The compress-side kernels checked exactly past their grid-stride and sweep-level boundaries, on operands from the whole field.

Every N4 kernel is grid-stride with a capped grid, so below a size that depends on the SM count each thread runs its loop once; the
HyperKZG witness polynomials climb one up-sweep / down-sweep level per factor of KZG_SEG; the IPA verifier's tensor tables split the
index into 8-bit groups.  The launch-shape model below restates those formulas, the sizes are derived from it for the device's SM
count, and every test asserts that its size reaches the shape it claims, so that a later constant change fails a test instead of
quietly moving it back below its boundary.  tests/test_oracle_compress_shapes.py checks the model for 114 and 132 SMs.

References, all exact:
  * sum-check: the multithreaded C port of the oracle prover (oracle.capi.sumcheck_prove); batched: oracle/sumcheck.py prove_batch;
  * eq table: closed forms (one-hot for a Boolean tau, 2^-l for tau = 1/2, entries summing to 1, the product formula at sampled and
    wrap-boundary indices);
  * IPA: keys of known discrete logarithm, G_i = [beta^i] g and ck_c = [gamma] g: the folded key's logarithms fold in the scalar field, so
    L_j = [<a_lo, d_hi> + c_L gamma] g and R_j alike cost one scalar multiplication each; the verifier's ck_hat = [<d, s>] g;
  * HyperKZG: bit-exact against oracle/kzg.py up to 2^16; above, the known-beta closed form with the fold chain and every polynomial
    evaluation done by the C oracle's axpy (P(u) = (E + u O)(u^2) halves the length per call);
  * batch_eval_reduce: tests/batched_oracle.py.
Every entry point that takes a format runs in both: canonical and Montgomery scalars in and out of the call."""
import ctypes as C
import functools
import hashlib
import itertools
import operator
import os

import numpy as np
import pytest

import batched_oracle as bo
from oracle import kzg, sumcheck as sc
from util import ints, montgomery_top, pack, random_elements

pytestmark = pytest.mark.gpu

# csrc/sc_scratch.cuh: sc_grid -- grid <= 4 CTAs per SM; 256 threads for sc_round_kernel, dot_kernel, poly_combine_kernel (sumcheck_impl.cuh)
# and ipa_fold_scalars_kernel, ipa_weighted_kernel, ipa_weights_update_kernel, ipa_s_kernel (ipa.cu)
SC_CTAS_PER_SM, SC_BLOCK = 4, 256
# csrc/ipa.cu: ipa_fold_bases_kernel, 128 threads, sized by sc_grid
IPA_BASES_BLOCK = 128
# csrc/sumcheck_impl.cuh: eq_kernel, 128 threads, 2^LOW outputs per thread with LOW = min(l, 4) (one CTA below l = 4); SC_MAX_INSTANCES
EQ_BLOCK, EQ_LOW_MAX = 128, 4
SC_MAX_INSTANCES = 60
# csrc/kzg.cu: kzg_grid -- grid <= 8 CTAs per SM of 256 threads; KZG_CHUNK = 256 * KZG_SEG elements per kzg_eval_chunk_kernel CTA
KZG_CTAS_PER_SM, KZG_BLOCK = 8, 256
# csrc/kzg.cuh
KZG_SEG = 32
KZG_CHUNK = 256 * KZG_SEG
# csrc/tensor.cuh
TENSOR_GROUP_BITS = 8


# ------------------------------------------------------------------------------------------------------------------ launch-shape model
def grid(n, block, per_sm, sms):
    """sc_grid / kzg_grid: ceil(n / block) CTAs, at least 1, at most per_sm per SM"""
    return max(1, min(-(-n // block), per_sm * sms))


def sweeps(n, block, per_sm, sms):
    """grid-stride iterations of the busiest thread over n items"""
    return max(1, -(-n // (grid(n, block, per_sm, sms) * block)))


def tensor_groups(l):
    return -(-l // TENSOR_GROUP_BITS) if l else 1


def kzg_lens(l):
    """kzg_witness_polys: level lengths n, ceil(n / 32), .. down to <= KZG_SEG; K = len - 1 levels above level 0"""
    lens = [1 << l]
    while lens[-1] > KZG_SEG:
        lens.append(-(-lens[-1] // KZG_SEG))
    return lens


class Shapes:
    """the launch shapes of the compress-side kernels on a device with `sms` SMs"""

    def __init__(self, sms):
        self.sms = sms
        self.sc_cap = SC_CTAS_PER_SM * SC_BLOCK * sms            # items one sc_grid launch covers in one sweep
        self.bases_cap = SC_CTAS_PER_SM * IPA_BASES_BLOCK * sms
        self.sc_wrap = next(l for l in range(1, 40) if self.sc_round_sweeps(l, 0) >= 2)
        self.eq_wrap = next(l for l in range(1, 33) if self.eq_sweeps(l) >= 2)
        self.combine_wrap = next(m for m in range(1, 40) if self.sc_sweeps(1 << m) >= 2)

    def sc_sweeps(self, n):
        return sweeps(n, SC_BLOCK, SC_CTAS_PER_SM, self.sms)

    def sc_round_sweeps(self, l, j):
        """round j of an l-variable sum-check: 2^(l - 1 - j) index pairs (the bind of round j's challenge rides in round j + 1)"""
        return self.sc_sweeps(1 << (l - 1 - j))

    def eq_low(self, l):
        return min(l, EQ_LOW_MAX)

    def eq_threads(self, l):
        groups = 1 << (l - self.eq_low(l))
        return EQ_BLOCK * (1 if l < EQ_LOW_MAX else grid(groups, EQ_BLOCK, SC_CTAS_PER_SM, self.sms))

    def eq_sweeps(self, l):
        return max(1, -(-(1 << (l - self.eq_low(l))) // self.eq_threads(l)))

    def bases_sweeps(self, half):
        return sweeps(half, IPA_BASES_BLOCK, SC_CTAS_PER_SM, self.sms)

    def kzg_sweeps(self, n):
        return sweeps(n, KZG_BLOCK, KZG_CTAS_PER_SM, self.sms)

    def kzg_levels(self, l):
        return len(kzg_lens(l)) - 1

    @staticmethod
    def kzg_chunks(l):
        return -(-(1 << l) // KZG_CHUNK)

    # ---- the sizes the tests run
    def sumcheck_sizes(self):
        return [self.sc_wrap - 1, self.sc_wrap, self.sc_wrap + 1]

    def eq_sizes(self):
        return list(range(EQ_LOW_MAX + 2)) + [self.eq_wrap - 1, self.eq_wrap, self.eq_wrap + 1, 24]

    def inner_product_sizes(self):
        c = self.sc_cap
        return [1, 255, 256, 257, c - 1, c, c + 1, 2 * c + 3, 1 << 22]

    def pow2_around(self, cap):
        """the largest power of two <= cap and the next one"""
        below = 1 << (cap.bit_length() - 1)
        return [below, 2 * below]

    def fold_scalar_halves(self):
        return self.pow2_around(self.sc_cap)

    def fold_bases_halves(self):
        return self.pow2_around(self.bases_cap)

    def ipa_reach(self, log_n):
        """what an IPA proof of 2^log_n reaches: sweeps of the round-0 inner products and fold, of the weighted / weights-update passes
        over the whole key, and the verifier's s pass; tensor groups of the verifier"""
        n = 1 << log_n
        return dict(dot=self.sc_sweeps(n // 2), fold=self.sc_sweeps(n // 2), weighted=self.sc_sweeps(n), s=self.sc_sweeps(n), groups=tensor_groups(log_n))

    def kzg_reach(self, l):
        """K, the chunks of P_0 and the sweeps of the level-0 up / down sweeps, the batch kernel and the first fold"""
        n = 1 << l
        return dict(K=self.kzg_levels(l), chunks=self.kzg_chunks(l), sweep0=self.kzg_sweeps(-(-n // KZG_SEG)), batch=self.kzg_sweeps(n),
                    fold=self.kzg_sweeps(n // 2))

    def batch_eval_m(self):
        return self.combine_wrap


HYPERKZG_EXACT = [10, 11, 13, 14, 16]
HYPERKZG_KNOWN_BETA = [21, 24]
IPA_LOG_N = [17, 19]


@functools.lru_cache(maxsize=None)
def shapes():
    import torch
    return Shapes(torch.cuda.get_device_properties(0).multi_processor_count)


# ------------------------------------------------------------------------------------------------------------------------- plumbing
def lib(L):
    return L._capi.lib()


NTHREADS = max(1, min(16, os.cpu_count() or 1))


class Codec:
    """field elements of one call in the format `fmt`: canonical ints <-> the 32-byte words the C ABI takes and returns"""

    def __init__(self, L, p, fmt):
        self.p, self.fmt = p, fmt
        self.mont = fmt == L.FMT_MONTGOMERY
        self.R = (1 << 256) % p
        self.Ri = pow(self.R, -1, p)

    def enc(self, x):
        return x * self.R % self.p if self.mont else x % self.p

    def dec(self, w):
        assert w < self.p, "an unreduced word"
        return w * self.Ri % self.p if self.mont else w

    def words(self, vals):
        return pack([self.enc(v) for v in vals]) if len(vals) else np.zeros(32, dtype=np.uint8)

    def ints(self, buf, count=None):
        v = [self.dec(w) for w in ints(buf)]
        return v if count is None else v[:count]

    def point(self, b96):
        """x | y | z (z = one, or all zero for the identity) -> (x, y) or None"""
        w = ints(b96)
        if w[2] == 0:
            assert w[0] == 0 and w[1] == 0
            return None
        assert self.dec(w[2]) == 1
        return (self.dec(w[0]), self.dec(w[1]))

    def point_words(self, P):
        return np.zeros(96, dtype=np.uint8) if P is None else self.words([P[0], P[1], 1])


def callback(L, codec_out, challenge, errors, decode):
    """a lurk_challenge_fn: the message decoded by decode(round, bytes), challenge(round, decoded) -> canonical int, returned in
    codec_out's format"""
    def cb(user, rnd, msg, msg_len, out):
        try:
            r = challenge(rnd, decode(rnd, C.string_at(msg, msg_len)))
            for i, byte in enumerate(int(codec_out.enc(r)).to_bytes(32, "little")):
                out[i] = byte
            return 0
        except Exception as e:          # never unwind through the C frames
            errors.append(e)
            return 1
    return L._capi.CHALLENGE_FN(cb)


def dec_elems(codec, msg):
    return codec.ints(np.frombuffer(msg, dtype=np.uint8))


def dec_points(codec, msg):
    return [codec.point(np.frombuffer(msg[i:i + 96], dtype=np.uint8)) for i in range(0, len(msg), 96)]


def run(L, rc, errors):
    if errors:
        raise errors[0]
    L._capi.check(rc)


def convert(L, field, t, fmt):
    """a device tensor of elements converted in place into `fmt`"""
    L._capi.check(lib(L).lurk_convert_dev(field, C.c_void_p(t.data_ptr()), t.numel() // 32, fmt, C.c_void_p(t.data_ptr()), None))
    return t


def to_device(L, field, canon_buf):
    """canonical host elements -> Montgomery device tensor"""
    import torch
    return convert(L, field, torch.from_numpy(np.ascontiguousarray(canon_buf, dtype=np.uint8).reshape(-1)).cuda(), L.FMT_MONTGOMERY)


def to_host(L, field, t):
    """Montgomery device tensor -> canonical host bytes"""
    return convert(L, field, t.clone(), L.FMT_CANONICAL).cpu().numpy()


def digest(rnd, vals, tag=b""):
    data = tag + bytes([rnd % 256]) + b"".join(int(v).to_bytes(32, "little") for v in vals)
    return int.from_bytes(hashlib.sha256(data).digest() + hashlib.sha256(data + b"x").digest(), "little")


def special_challenge(p, special, tag=b""):
    """challenge(round, values): the values chosen in `special` in their rounds, a hash of the message otherwise"""
    return lambda rnd, vals: special[rnd] % p if rnd in special else digest(rnd, vals, tag) % p


FMTS = [0, 1]     # FMT_CANONICAL, FMT_MONTGOMERY


# ------------------------------------------------------------------------------------------------------------------------- sum-check
@functools.lru_cache(maxsize=8)
def edge_polys(field, l):
    return tuple(random_elements(field, 1 << l, seed=1000 * field + 10 * l + k, shape="edge") for k in range(4))


@functools.lru_cache(maxsize=2)
def degenerate_polys(spec, field, l, kind, shapes_):
    """(name, polys as canonical bytes, claim) of the degenerate sets"""
    p = spec.FIELD_MODULUS[field]
    n, k = 1 << l, (2 if kind == "quad" else 4)
    z = np.zeros(n * 32, dtype=np.uint8)
    full = lambda v: np.tile(pack([v]), n)
    # one-hot at the first index pair of round 0's second grid-stride sweep, in the high half
    hot = n // 2 + min(shapes_.sc_cap, n // 2 - 1)
    tops = [montgomery_top(p, j) for j in range(k)]
    onehot = []
    for j in range(k):
        b = z.copy()
        b[32 * hot:32 * hot + 32] = pack([tops[j]])
        onehot.append(b)
    consts = [(p + 1) // 2, p - 1, montgomery_top(p, 0), 2][:k]
    tau = ints(random_elements(field, l, seed=l, shape="edge"))
    eq = pack(sc.eq_evals(tau, p))
    edge = list(edge_polys(field, l))
    comb = sc.comb_quad if kind == "quad" else sc.comb_cubic
    return [("zero", [z] * k, 0),
            ("minus_one", [full(p - 1)] * k, n * comb(*([p - 1] * k), p) % p),
            ("one_hot", onehot, comb(*tops, p)),
            ("constant", [full(c) for c in consts], n * comb(*consts, p) % p),
            ("eq_tau", [eq] + edge[1:k], p - 3)]


def sumcheck_dev(L, field, kind, bufs, l, claim, challenge, fmt):
    """lurk_sumcheck_prove_dev with the claim, round messages, challenges and final evaluations in `fmt`; returns them canonical"""
    p = int.from_bytes(L.spartan.field_modulus(field), "little")
    cd = Codec(L, p, fmt)
    k, deg1 = (2, 3) if kind == "quad" else (4, 4)
    dev = [to_device(L, field, b) for b in bufs]
    ptrs = (C.c_void_p * k)(*[C.c_void_p(d.data_ptr()) for d in dev])
    rounds = np.zeros(max(1, l) * deg1 * 32, dtype=np.uint8)
    chal = np.zeros(max(1, l) * 32, dtype=np.uint8)
    fin = np.zeros(k * 32, dtype=np.uint8)
    errors = []
    cb = callback(L, cd, challenge, errors, lambda rnd, msg: dec_elems(cd, msg))
    rc = lib(L).lurk_sumcheck_prove_dev(field, L.spartan.QUAD if kind == "quad" else L.spartan.CUBIC, ptrs, l, L._capi.np_ptr(cd.words([claim])), cb, None,
                                        L._capi.np_ptr(rounds), L._capi.np_ptr(chal), L._capi.np_ptr(fin), fmt, None)
    run(L, rc, errors)
    ev = cd.ints(rounds)
    heads = [to_host(L, field, d[:32]) for d in dev]          # bound in place: slot 0 holds the final evaluation
    return [ev[i * deg1:(i + 1) * deg1] for i in range(l)], cd.ints(chal, l), cd.ints(fin), [ints(h)[0] for h in heads]


def check_sumcheck(L, oracle, spec, field, kind, bufs, l, claim, fmt):
    p = spec.FIELD_MODULUS[field]
    chal = special_challenge(p, {1: 0, 2: 1, 3: p - 1}, b"sc")
    want = oracle.sumcheck_prove(field, kind, bufs, l, claim, chal, nthreads=NTHREADS)
    rounds, rs, fin, heads = sumcheck_dev(L, field, kind, bufs, l, claim, chal, fmt)
    assert rs[1:4] == [0, 1, p - 1]
    for j in range(l):
        assert rounds[j] == want[0][j], (kind, l, j)
    assert rs == want[1] and fin == want[2] and heads == want[2]


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("kind", ["quad", "cubic"])
@pytest.mark.parametrize("at", [-1, 0, 1])
def test_sumcheck_edge_around_wrap(L, oracle, spec, at, kind, fmt):
    """field 0 at l = wrap - 1, wrap, wrap + 1 (wrap: the first size whose round 0 runs two grid-stride sweeps), every round, challenge
    and final evaluation bit for bit; challenges 0, 1 and p - 1 in rounds 1 .. 3"""
    S = shapes()
    l = S.sc_wrap + at
    assert (S.sc_round_sweeps(l, 0) >= 2) == (at >= 0)
    if at == 1:
        assert S.sc_round_sweeps(l, 0) >= 2 and S.sc_round_sweeps(l, 1) >= 2
    check_sumcheck(L, oracle, spec, 0, kind, list(edge_polys(0, l))[:2 if kind == "quad" else 4], l, spec.FIELD_MODULUS[0] - 2, fmt)


@pytest.mark.parametrize("kind", ["quad", "cubic"])
@pytest.mark.parametrize("field", [1, 2, 3])
def test_sumcheck_edge_other_fields_at_wrap(L, oracle, spec, field, kind):
    S = shapes()
    l = S.sc_wrap
    assert S.sc_round_sweeps(l, 0) >= 2
    check_sumcheck(L, oracle, spec, field, kind, list(edge_polys(field, l))[:2 if kind == "quad" else 4], l, 12345, FMTS[field % 2])


@pytest.mark.parametrize("kind", ["quad", "cubic"])
@pytest.mark.parametrize("case", ["zero", "minus_one", "one_hot", "constant", "eq_tau"])
def test_sumcheck_degenerate_at_wrap(L, oracle, spec, case, kind):
    """all zero, all p - 1, one-hot in round 0's second sweep, constants, and A = eq(tau) as in the outer sum-check"""
    S = shapes()
    l = S.sc_wrap
    assert S.sc_round_sweeps(l, 0) >= 2
    name, bufs, claim = next(c for c in degenerate_polys(spec, 0, l, kind, S) if c[0] == case)
    check_sumcheck(L, oracle, spec, 0, kind, bufs, l, claim, FMTS[len(case) % 2])


def sumcheck_batch_dev(L, field, kind, insts, claims, coeffs, challenge, fmt):
    """lurk_sumcheck_prove_batch_dev in `fmt`.  insts: [(canonical bufs, rounds)].  Returns (rounds, challenges, finals) canonical."""
    p = int.from_bytes(L.spartan.field_modulus(field), "little")
    cd = Codec(L, p, fmt)
    k, deg1 = (2, 3) if kind == "quad" else (4, 4)
    n = len(insts)
    dev = [to_device(L, field, b) for bufs, _ in insts for b in bufs]
    ptrs = (C.c_void_p * (n * k))(*[C.c_void_p(d.data_ptr()) for d in dev])
    nr = (C.c_int * n)(*[r for _, r in insts])
    mx = max(r for _, r in insts)
    rounds = np.zeros(max(1, mx) * deg1 * 32, dtype=np.uint8)
    chal = np.zeros(max(1, mx) * 32, dtype=np.uint8)
    fin = np.zeros(n * k * 32, dtype=np.uint8)
    errors = []
    cb = callback(L, cd, challenge, errors, lambda rnd, msg: dec_elems(cd, msg))
    rc = lib(L).lurk_sumcheck_prove_batch_dev(field, L.spartan.QUAD if kind == "quad" else L.spartan.CUBIC, n, ptrs, nr,
                                              L._capi.np_ptr(cd.words(claims)), L._capi.np_ptr(cd.words(coeffs)), cb, None, L._capi.np_ptr(rounds),
                                              L._capi.np_ptr(chal), L._capi.np_ptr(fin), fmt, None)
    run(L, rc, errors)
    ev, fi = cd.ints(rounds), cd.ints(fin)
    return [ev[i * deg1:(i + 1) * deg1] for i in range(mx)], cd.ints(chal, mx), [fi[i * k:(i + 1) * k] for i in range(n)]


def check_batch(L, spec, field, kind, sizes, fmt, seed):
    p = spec.FIELD_MODULUS[field]
    k = 2 if kind == "quad" else 4
    bufs = [[random_elements(field, 1 << l, seed=seed + 10 * i + j, shape="edge") for j in range(k)] for i, l in enumerate(sizes)]
    polys = [[ints(b) for b in inst] for inst in bufs]
    claims = ints(random_elements(field, len(sizes), seed=seed + 1, shape="edge"))
    coeffs = ints(random_elements(field, len(sizes), seed=seed + 2, shape="edge"))
    chal = special_challenge(p, {0: p - 1, 2: 0, 3: 1}, b"batch")
    want = sc.prove_batch(polys, kind, claims, coeffs, chal, p)
    got = sumcheck_batch_dev(L, field, kind, list(zip(bufs, sizes)), claims, coeffs, chal, fmt)
    assert got[0] == want[0] and got[1] == want[1] and got[2] == want[2]


@pytest.mark.parametrize("fmt", FMTS)
def test_batched_sumcheck_across_wrap(L, spec, fmt):
    """one instance at the wrap size, the others joining in rounds on both sides of it: its round 0 sweeps twice, the instance of
    wrap - 1 rounds joins in round 1 with one sweep"""
    S = shapes()
    sizes = [S.sc_wrap, S.sc_wrap - 1, 9, 1, 0]
    assert S.sc_round_sweeps(sizes[0], 0) >= 2 and S.sc_round_sweeps(sizes[1], 0) == 1
    check_batch(L, spec, 0, "quad", sizes, fmt, seed=70)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("kind", ["quad", "cubic"])
def test_batched_sumcheck_max_instances(L, spec, kind, fmt):
    """SC_MAX_INSTANCES instances, several of them without rounds"""
    sizes = [(i * 7) % 11 if i % 6 else 0 for i in range(SC_MAX_INSTANCES)]
    assert len(sizes) == SC_MAX_INSTANCES and sizes.count(0) >= 5
    check_batch(L, spec, 2, kind, sizes, fmt, seed=80)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("kind", ["quad", "cubic"])
def test_batched_sumcheck_no_rounds(L, spec, kind, fmt):
    """every instance of 0 rounds: max_rounds = 0, the final evaluations are the single elements"""
    check_batch(L, spec, 0, kind, [0] * 7, fmt, seed=90)


# ------------------------------------------------------------------------------------------------------------------------- eq table
def eq_dev(L, field, tau, fmt):
    """lurk_eq_evals_dev with tau and the table in `fmt`; returns the device tensor"""
    import torch
    p = int.from_bytes(L.spartan.field_modulus(field), "little")
    cd = Codec(L, p, fmt)
    out = torch.empty((1 << len(tau)) * 32, dtype=torch.uint8, device="cuda")
    L._capi.check(lib(L).lurk_eq_evals_dev(field, L._capi.np_ptr(cd.words(tau)), len(tau), C.c_void_p(out.data_ptr()), fmt, None))
    torch.cuda.synchronize()
    return out


def eq_at_index(tau, i, p):
    l = len(tau)
    v = 1
    for j, t in enumerate(tau):
        v = v * (t if (i >> (l - 1 - j)) & 1 else 1 - t) % p
    return v


def eq_wrap_indices(S, l):
    """the first and last outputs of the first and last thread of every grid-stride sweep"""
    low = S.eq_low(l)
    T = S.eq_threads(l)
    groups = 1 << (l - low)
    idx = set()
    for s in range(S.eq_sweeps(l) + 1):
        for g in (s * T - 1, s * T, s * T + 1):
            if 0 <= g < groups:
                idx |= {g << low, (g << low) + (1 << low) - 1}
    return sorted(idx)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("field", [0, 2])
def test_eq_table(L, spec, field, fmt):
    import torch
    S = shapes()
    p = spec.FIELD_MODULUS[field]
    cd = Codec(L, p, fmt)
    sizes = S.eq_sizes()
    assert {S.eq_low(l) for l in sizes} == set(range(EQ_LOW_MAX + 1))
    assert S.eq_sweeps(S.eq_wrap - 1) == 1 and S.eq_sweeps(S.eq_wrap) >= 2 and S.eq_sweeps(24) >= 4
    rng = np.random.default_rng(field + 7 * fmt)
    one_m = torch.from_numpy(np.tile(pack([(1 << 256) % p]), 1 << 24)).cuda()     # ones, Montgomery
    for l in sizes:
        n = 1 << l
        tau = ints(random_elements(field, l, seed=l, shape="edge"))
        t = eq_dev(L, field, tau, fmt)
        if l <= EQ_LOW_MAX + 1:
            assert cd.ints(t.cpu().numpy()) == sc.eq_evals(tau, p), l
            continue
        # general tau: the product formula at the wrap boundaries and a seeded sample, the entries sum to 1
        idx = eq_wrap_indices(S, l) + [int(i) for i in rng.integers(0, n, size=64)] + [n - 1]
        rows = t.view(-1, 32)
        host = np.stack([rows[i].cpu().numpy() for i in idx])
        assert cd.ints(host) == [eq_at_index(tau, i, p) for i in idx], l
        tm = t if fmt == L.FMT_MONTGOMERY else convert(L, field, t.clone(), L.FMT_MONTGOMERY)
        assert L.spartan.inner_product(field, tm.data_ptr(), one_m.data_ptr(), n) == 1, l
        del tm
        # Boolean tau: one-hot at the index tau spells
        spelled = int(rng.integers(0, n))
        t = eq_dev(L, field, [(spelled >> (l - 1 - j)) & 1 for j in range(l)], fmt)
        nz = (t.view(-1, 32) != 0).any(dim=1).nonzero().flatten().tolist()
        assert nz == [spelled] and cd.ints(t.view(-1, 32)[spelled].cpu().numpy()) == [1], l
        # tau_j = 1/2: the constant 2^-l
        half = (p + 1) // 2
        t = eq_dev(L, field, [half] * l, fmt)
        want = torch.from_numpy(cd.words([pow(half, l, p)])).cuda()
        assert bool((t.view(-1, 32) == want).all()), l
        del t


# ------------------------------------------------------------------------------------------------------------------------- inner product
def periodic(field, p, kind, n, period, seed):
    """(canonical bytes of n elements, the block's ints): one block of `period` elements repeated"""
    if kind == "minus_one":
        block = [p - 1]
    elif kind == "montgomery_top":
        block = [montgomery_top(p, k) for k in range(period)]
    else:
        block = ints(random_elements(field, period, seed=seed, shape="edge"))
    return np.tile(pack(block), -(-n // len(block)))[:32 * n], block


def ip_dev(L, field, da, db, n, fmt):
    p = int.from_bytes(L.spartan.field_modulus(field), "little")
    out = np.zeros(32, dtype=np.uint8)
    L._capi.check(lib(L).lurk_inner_product_dev(field, C.c_void_p(da.data_ptr()), C.c_void_p(db.data_ptr()), n, L._capi.np_ptr(out), fmt, None))
    return Codec(L, p, fmt).ints(out)[0]


@pytest.mark.parametrize("field", [0, 2])
def test_inner_product_around_grid_cap(L, spec, field):
    """n around cap = 1024 SMs (one sweep of dot_kernel's capped grid) up to 2^22; operands all p - 1 (the result is n mod p), elements
    whose Montgomery form is near p, and the edge shape, with periods 4099 / 4093 so that no sweep sees the same values in the same lanes"""
    S = shapes()
    p = spec.FIELD_MODULUS[field]
    sizes = S.inner_product_sizes()
    assert [S.sc_sweeps(n) for n in sizes[4:7]] == [1, 1, 2] and S.sc_sweeps(sizes[7]) == 3 and S.sc_sweeps(sizes[8]) >= 4
    N = max(sizes)
    for kind in ("minus_one", "montgomery_top", "edge"):
        ha, A = periodic(field, p, kind, N, 4099, seed=field)
        hb, B = periodic(field, p, kind, N, 4093, seed=field + 1)
        da, db = to_device(L, field, ha), to_device(L, field, hb)
        for i, n in enumerate(sizes):
            want = sum(map(operator.mul, itertools.islice(itertools.cycle(A), n), itertools.islice(itertools.cycle(B), n))) % p
            if kind == "minus_one":
                assert want == n % p
            assert ip_dev(L, field, da, db, n, FMTS[i % 2]) == want, (kind, n)
        del da, db


# ------------------------------------------------------------------------------------------------------------------------- IPA folds
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("field", [1, 2])
def test_ipa_fold_scalars_around_cap(L, oracle, spec, field, fmt):
    S = shapes()
    p = spec.FIELD_MODULUS[field]
    cd = Codec(L, p, fmt)
    halves = S.fold_scalar_halves()
    assert [S.sc_sweeps(h) for h in halves] == [1, 2]
    x = ints(random_elements(field, 1, seed=5, shape="edge"))[0] or 3
    for half in halves:
        a = random_elements(field, 2 * half, seed=half, shape="edge")
        lo, hi = a[:32 * half], a[32 * half:]
        for fx, fy in ((0, 0), (1, 0), (0, 1), (1, 1), (p - 1, 1), (x, x)):
            d = to_device(L, field, a)
            L._capi.check(lib(L).lurk_ipa_fold_scalars_dev(field, C.c_void_p(d.data_ptr()), 2 * half, L._capi.np_ptr(cd.words([fx])),
                                                           L._capi.np_ptr(cd.words([fy])), fmt, None))
            want = oracle.axpy(field, oracle.axpy(field, np.zeros_like(lo), lo, pack([fx]), NTHREADS), hi, pack([fy]), NTHREADS)
            got = to_host(L, field, d)
            assert np.array_equal(got[:32 * half], want), (half, fx, fy)
            assert np.array_equal(got[32 * half:], hi), "the high half is not the kernel's to write"


RELATIONS = ("P=Q", "P=-Q", "Q=2P")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("curve", [1, 2])
def test_ipa_fold_bases_around_cap(L, spec, curve, fmt):
    """G' = x G_lo + y G_hi on a powers-of-tau key whose pairs at the sweep boundaries (and a few more) are made P = Q, P = -Q and Q = [2]P,
    so that ipa_fold_point doubles in P + Q, meets the identity and adds equal points; every index is checked where (x, y) makes the
    result a copy, the boundaries and a seeded sample elsewhere through the discrete logs"""
    import torch
    S = shapes()
    Cv = spec.CURVES[curve]
    pb, q = spec.FIELD_MODULUS[Cv["base"]], spec.FIELD_MODULUS[Cv["scalar"]]
    cd = Codec(L, q, fmt)
    g = Cv["gen"]
    halves = S.fold_bases_halves()
    assert [S.bases_sweeps(h) for h in halves] == [1, 2]
    x = ints(random_elements(Cv["scalar"], 1, seed=9, shape="edge"))[0] or 3
    beta = ints(random_elements(Cv["scalar"], 1, seed=curve))[0]
    rng = np.random.default_rng(curve + 2 * fmt)
    for half in halves:
        n = 2 * half
        ck = L.CommitmentKey.powers_of_tau(curve, g, beta, n)
        key = to_host(L, Cv["base"], ck._bases[:64 * n]).reshape(n, 64).copy()
        dlog = {}
        T = grid(half, IPA_BASES_BLOCK, SC_CTAS_PER_SM, S.sms) * IPA_BASES_BLOCK
        designed = sorted({i for i in (0, 1, T - 1, T, T + 1, half - 1, half - 2, half - 3) if 0 <= i < half})
        for k, i in enumerate(designed):
            P = (ints(key[i, :32])[0], ints(key[i, 32:])[0])
            rel = RELATIONS[k % 3]
            Q = P if rel == "P=Q" else (P[0], pb - P[1]) if rel == "P=-Q" else spec.ec_add(P, P, pb)
            key[half + i] = pack([Q[0], Q[1]])
            dlog[half + i] = (pow(beta, i, q) * {"P=Q": 1, "P=-Q": -1, "Q=2P": 2}[rel]) % q
        sample = sorted(set(designed) | {int(i) for i in rng.integers(0, half, size=40)})
        lg = lambda j: dlog.get(j, pow(beta, j, q))
        for fx, fy in ((0, 0), (1, 0), (0, 1), (1, 1), (q - 1, 1), (x, x)):
            d = to_device(L, Cv["base"], key.reshape(-1))
            L._capi.check(lib(L).lurk_ipa_fold_bases_dev(curve, C.c_void_p(d.data_ptr()), n, L._capi.np_ptr(cd.words([fx])),
                                                         L._capi.np_ptr(cd.words([fy])), fmt, None))
            got = to_host(L, Cv["base"], d).reshape(n, 64)
            assert np.array_equal(got[half:], key[half:])
            if (fx, fy) == (0, 0):
                assert not got[:half].any()
                continue
            if (fx, fy) in ((1, 0), (0, 1)):
                assert np.array_equal(got[:half], key[:half] if fx else key[half:]), (half, fx, fy)
                continue
            for i in sample:
                P = spec.ec_mul((fx * lg(i) + fy * lg(half + i)) % q, g, pb)
                assert got[i].tobytes() == pack([P[0], P[1]] if P else [0, 0]).tobytes(), (half, fx, fy, i)
            del d
        del ck
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------------- IPA prove / verify
def ipa_prove_dev(L, curve, ck, gc, da, db, log_n, challenge, fmt):
    """lurk_ipa_prove_dev in `fmt`; challenge(round, (L, R)) -> int.  Returns (Ls, Rs, a_final, b_final) canonical."""
    from oracle import spec
    Cv = spec.CURVES[curve]
    cb_, cs = Codec(L, spec.FIELD_MODULUS[Cv["base"]], fmt), Codec(L, spec.FIELD_MODULUS[Cv["scalar"]], fmt)
    Lb, Rb = np.zeros(max(1, log_n) * 96, dtype=np.uint8), np.zeros(max(1, log_n) * 96, dtype=np.uint8)
    af, bf = np.zeros(32, dtype=np.uint8), np.zeros(32, dtype=np.uint8)
    errors = []
    cb = callback(L, cs, challenge, errors, lambda rnd, msg: dec_points(cb_, msg))
    rc = lib(L).lurk_ipa_prove_dev(curve, ck._ctx, L._capi.np_ptr(cb_.words(list(gc))), C.c_void_p(da.data_ptr()), C.c_void_p(db.data_ptr()), log_n, cb,
                                   None, L._capi.np_ptr(Lb), L._capi.np_ptr(Rb), L._capi.np_ptr(af), L._capi.np_ptr(bf), fmt, None)
    run(L, rc, errors)
    pts = lambda b: [cb_.point(b[96 * j:96 * j + 96]) for j in range(log_n)]
    return pts(Lb), pts(Rb), cs.ints(af)[0], cs.ints(bf)[0]


def ipa_verify_dev(L, curve, ck, gc, comm, c, db, log_n, Ls, Rs, a_final, challenge, fmt):
    from oracle import spec
    Cv = spec.CURVES[curve]
    cb_, cs = Codec(L, spec.FIELD_MODULUS[Cv["base"]], fmt), Codec(L, spec.FIELD_MODULUS[Cv["scalar"]], fmt)
    Lb = np.concatenate([cb_.point_words(P) for P in Ls])
    Rb = np.concatenate([cb_.point_words(P) for P in Rs])
    hat, bh = np.zeros(96, dtype=np.uint8), np.zeros(32, dtype=np.uint8)
    acc = C.c_int(-1)
    errors = []
    cb = callback(L, cs, challenge, errors, lambda rnd, msg: dec_points(cb_, msg))
    rc = lib(L).lurk_ipa_verify_dev(curve, ck._ctx, L._capi.np_ptr(cb_.words(list(gc))), L._capi.np_ptr(cb_.point_words(comm)), L._capi.np_ptr(cs.words([c])),
                                    C.c_void_p(db.data_ptr()), log_n, L._capi.np_ptr(Lb), L._capi.np_ptr(Rb), L._capi.np_ptr(cs.words([a_final])), cb, None,
                                    C.byref(acc), L._capi.np_ptr(hat), L._capi.np_ptr(bh), fmt, None)
    run(L, rc, errors)
    return bool(acc.value), cb_.point(hat), cs.ints(bh)[0]


def ipa_challenge(q, special):
    def f(rnd, pts):
        if rnd in special:
            return special[rnd] % q
        flat = [c for P in pts for c in (P or (0, 0))]
        return 1 + digest(rnd, flat, b"ipa") % (q - 1)
    return f


def ipa_case(L, spec, curve, log_n, fmt, special):
    import torch
    S = shapes()
    Cv = spec.CURVES[curve]
    field, pb, q = Cv["scalar"], spec.FIELD_MODULUS[Cv["base"]], spec.FIELD_MODULUS[Cv["scalar"]]
    n = 1 << log_n
    g = Cv["gen"]
    beta, gamma = ints(random_elements(field, 2, seed=100 + curve + log_n))
    gc = spec.ec_mul(gamma, g, pb)
    ck = L.CommitmentKey.powers_of_tau(curve, g, beta, n)
    a_h = random_elements(field, n, seed=log_n, shape="witness")
    b_h = random_elements(field, n, seed=log_n + 1, shape="edge")
    a, b = ints(a_h), ints(b_h)
    d = [1] * n
    for i in range(1, n):
        d[i] = d[i - 1] * beta % q
    chal = ipa_challenge(q, special)
    db = to_device(L, field, b_h)
    keep = db.clone()
    Ls, Rs, a_fin, b_fin = ipa_prove_dev(L, curve, ck, gc, to_device(L, field, a_h), db, log_n, chal, fmt)
    comm = spec.ec_mul(sc.inner_product(a, d, q), g, pb)
    c = sc.inner_product(a, b, q)
    pt = lambda s: spec.ec_mul(s % q, g, pb)
    for j in range(log_n):
        h = len(a) // 2
        cl, cr = sc.inner_product(a[:h], b[h:], q), sc.inner_product(a[h:], b[:h], q)
        eL, eR = sc.inner_product(a[:h], d[h:], q), sc.inner_product(a[h:], d[:h], q)
        assert Ls[j] == pt(eL + cl * gamma) and Rs[j] == pt(eR + cr * gamma), (curve, log_n, j)
        r = chal(j, [Ls[j], Rs[j]])
        ri = pow(r, -1, q)
        a = [(r * x + ri * y) % q for x, y in zip(a[:h], a[h:])]
        b = [(ri * x + r * y) % q for x, y in zip(b[:h], b[h:])]
        d = [(ri * x + r * y) % q for x, y in zip(d[:h], d[h:])]
    assert (a_fin, b_fin) == (a[0], b[0])
    ok, ck_hat, b_hat = ipa_verify_dev(L, curve, ck, gc, comm, c, keep, log_n, Ls, Rs, a_fin, chal, fmt)
    assert ok and ck_hat == pt(d[0]) and b_hat == b[0]
    bad = list(Ls)
    bad[log_n // 2] = spec.ec_add(bad[log_n // 2], g, pb)
    assert not ipa_verify_dev(L, curve, ck, gc, comm, c, keep, log_n, bad, Rs, a_fin, chal, fmt)[0]
    del ck, db, keep
    torch.cuda.empty_cache()


@pytest.mark.parametrize("curve", [1, 2])
@pytest.mark.parametrize("log_n", IPA_LOG_N)
def test_ipa_prove_and_verify_known_dlog(L, spec, curve, log_n):
    """every L_j, R_j, a_final and b_final exact; the verifier accepts with ck_hat and b_hat exact and rejects a tampered L.  2^17: the
    verifier's tensor has 3 groups; 2^19: the round-0 inner products, fold and every weighted pass run >= 2 grid-stride sweeps"""
    S = shapes()
    reach = S.ipa_reach(log_n)
    assert reach["groups"] == 3 if log_n == 17 else reach["groups"] >= 3
    if log_n == max(IPA_LOG_N):
        assert min(reach["dot"], reach["fold"], reach["weighted"], reach["s"]) >= 2, reach
    ipa_case(L, spec, curve, log_n, FMTS[(curve + log_n) % 2], {})


def test_ipa_challenges_one_and_minus_one(L, spec):
    """r = 1 and r = p - 1, where r = 1 / r"""
    ipa_case(L, spec, 1, min(IPA_LOG_N), L.FMT_MONTGOMERY, {0: 1, 1: -1, 5: 1, 9: -1})


# ------------------------------------------------------------------------------------------------------------------------- HyperKZG
def hyperkzg_dev(L, curve, ck, d_poly, point, challenge, fmt):
    """lurk_hyperkzg_prove_dev in `fmt`; challenge(round, values) with round 0 = commitments, 1 = evaluations, 2 = witness commitments.
    Returns (com, v, w) canonical."""
    from oracle import spec
    Cv = spec.CURVES[curve]
    cb_, cs = Codec(L, spec.FIELD_MODULUS[Cv["base"]], fmt), Codec(L, spec.FIELD_MODULUS[Cv["scalar"]], fmt)
    l = len(point)
    com = np.zeros(max(1, l - 1) * 96, dtype=np.uint8)
    w = np.zeros(3 * 96, dtype=np.uint8)
    v = np.zeros(3 * l * 32, dtype=np.uint8)
    errors = []
    cb = callback(L, cs, challenge, errors, lambda rnd, msg: dec_elems(cs, msg) if rnd == 1 else dec_points(cb_, msg))
    rc = lib(L).lurk_hyperkzg_prove_dev(curve, ck._ctx, C.c_void_p(d_poly.data_ptr()), L._capi.np_ptr(cs.words(point)), l, cb, None,
                                        L._capi.np_ptr(com), L._capi.np_ptr(w), L._capi.np_ptr(v), fmt, None)
    run(L, rc, errors)
    vi = cs.ints(v)
    return [cb_.point(com[96 * j:96 * j + 96]) for j in range(l - 1)], [vi[t * l:(t + 1) * l] for t in range(3)], \
        [cb_.point(w[96 * j:96 * j + 96]) for j in range(3)]


class KzgChallenge:
    """round 0 (the commitments) -> r, or the fixed r; 1 (the evaluations) -> q; 2 (the witness commitments) -> ignored.  Records
    every round's values and answer."""

    def __init__(self, p, r=None):
        self.p, self.r, self.log, self.out = p, r, [], []

    def __call__(self, rnd, vals):
        self.log.append((rnd, vals))
        if rnd == 0 and self.r is not None:
            x = self.r % self.p
        else:
            flat = vals if rnd == 1 else [c for P in vals for c in (P or (0, 0))]
            x = digest(rnd, flat, b"kzg") % self.p
        self.out.append(x)
        return x


def oracle_values(vals_by_round):
    """oracle/kzg.py hands the challenge points and rows of v: flatten them as the GPU's messages decode"""
    rnd, msg = vals_by_round
    return msg if rnd != 1 else [e for row in msg for e in row]


@pytest.mark.parametrize("l", HYPERKZG_EXACT)
def test_hyperkzg_exact(L, oracle, spec, l):
    """bit-exact against oracle/kzg.py: K = 1 (l = 10, one partial chunk), K = 2 (l = 11; l = 13 exactly one KZG_CHUNK; l = 14 two chunks),
    K = 3 (l = 16, eight chunks)"""
    S = shapes()
    reach = S.kzg_reach(l)
    assert reach["K"] == {10: 1, 11: 2, 13: 2, 14: 2, 16: 3}[l] and reach["chunks"] == max(1, (1 << l) // KZG_CHUNK)
    if l == 13:
        assert (1 << l) == KZG_CHUNK
    run_hyperkzg_exact(L, oracle, spec, l, None, FMTS[l % 2])


@pytest.mark.parametrize("r", [0, 1, -1])
def test_hyperkzg_degenerate_r(L, oracle, spec, r):
    """r in {0, 1, p - 1}: u = (r, -r, r^2) with repeated or zero points, at l = 11 (K = 2)"""
    assert shapes().kzg_levels(11) == 2
    run_hyperkzg_exact(L, oracle, spec, 11, r, FMTS[r % 2])


def run_hyperkzg_exact(L, oracle, spec, l, r, fmt):
    curve, field = 0, 0
    p = spec.FIELD_MODULUS[field]
    n = 1 << l
    bases = oracle.gen_bases(curve, n, start=11)
    ck = L.CommitmentKey(curve, bases)
    Ph = random_elements(field, n, seed=l, shape="edge")
    x = ints(random_elements(field, l, seed=60 + l, shape="edge"))
    chal = KzgChallenge(p, r)
    com, v, w = hyperkzg_dev(L, curve, ck, to_device(L, field, Ph), x, chal, fmt)

    def commit(f):
        vv = ints(oracle.msm(curve, bases[:64 * len(f)], pack(f), nthreads=NTHREADS))
        return (vv[0], vv[1]) if vv[2] else None
    ochal = KzgChallenge(p, r)
    want = kzg.prove(curve, commit, ints(Ph), x, lambda rnd, msg: ochal(rnd, oracle_values((rnd, msg))))
    assert chal.log == ochal.log
    assert com == want["com"] and v == want["v"] and w == want["w"]


def poly_eval_c(oracle, field, f, u):
    """f(u) for f in the coefficient basis (canonical bytes, power-of-two length): (E + u O)(u^2), halving per axpy"""
    p = oracle.spec.FIELD_MODULUS[field]
    f = np.ascontiguousarray(f).reshape(-1, 32)
    while len(f) > 1:
        pairs = f.reshape(-1, 64)
        f = oracle.axpy(field, pairs[:, :32], pairs[:, 32:], pack([u]), NTHREADS).reshape(-1, 32)
        u = u * u % p
    return ints(f)[0]


@pytest.mark.parametrize("l", HYPERKZG_KNOWN_BETA)
def test_hyperkzg_known_beta(L, oracle, spec, l):
    """K = 4 at l = 21; at l = 24 the level-0 up- and down-sweeps and the batch kernel run several grid-stride sweeps.  The key is
    beta^i g: every commitment is [f(beta)] g for the polynomial the protocol defines, every evaluation is the polynomial's, and each
    witness commitment is [(B(beta) - B(u_t)) / (beta - u_t)] g"""
    import torch
    S = shapes()
    reach = S.kzg_reach(l)
    assert reach["K"] >= 4
    if l == 24:
        assert min(reach["sweep0"], reach["batch"], reach["fold"]) >= 2, reach
    curve, field = 0, 0
    Cv = spec.CURVES[curve]
    pb, p = spec.FIELD_MODULUS[Cv["base"]], spec.FIELD_MODULUS[field]
    n = 1 << l
    g = spec.ec_mul(4242, Cv["gen"], pb)
    beta = ints(random_elements(field, 1, seed=l))[0]
    ck = L.CommitmentKey.powers_of_tau(curve, g, beta, n)
    Ph = random_elements(field, n, seed=l + 1, shape="witness")
    x = ints(random_elements(field, l, seed=l + 2, shape="edge"))
    chal = KzgChallenge(p)
    dP = to_device(L, field, Ph)
    com, v, w = hyperkzg_dev(L, curve, ck, dP, x, chal, FMTS[l % 2])
    del dP, ck
    torch.cuda.empty_cache()
    # the fold chain P_{i+1} = even + x_{l-1-i} (odd - even), by the C oracle
    polys = [Ph.reshape(-1, 32)]
    for i in range(l - 1):
        pairs = polys[-1].reshape(-1, 64)
        diff = oracle.axpy(field, pairs[:, 32:], pairs[:, :32], pack([p - 1]), NTHREADS)
        polys.append(oracle.axpy(field, pairs[:, :32], diff, pack([x[l - 1 - i]]), NTHREADS).reshape(-1, 32))
    at_beta = [poly_eval_c(oracle, field, f, beta) for f in polys]
    assert com == [spec.ec_mul(s, g, pb) for s in at_beta[1:]]
    r, q = chal.out[0], chal.out[1]
    u = [r, (-r) % p, r * r % p]
    assert v == [[poly_eval_c(oracle, field, f, ut) for f in polys] for ut in u]
    Bbeta = sum(pow(q, j, p) * s for j, s in enumerate(at_beta)) % p
    ws = [(Bbeta - sum(pow(q, j, p) * v[t][j] for j in range(l))) * pow(beta - u[t], -1, p) % p for t in range(3)]
    assert w == [spec.ec_mul(s, g, pb) for s in ws]


# ------------------------------------------------------------------------------------------------------------------------- batch_eval_reduce
def batch_eval_dev(L, field, claims, challenge, fmt):
    """lurk_batch_eval_reduce_dev in `fmt`.  claims: [(device tensor, num_vars, point, eval)].  Returns canonical
    (rounds, r, claims_left, weights, joint_eval) and the joint polynomial (canonical host bytes)."""
    import torch
    p = int.from_bytes(L.spartan.field_modulus(field), "little")
    cd = Codec(L, p, fmt)
    n = len(claims)
    nv = [c[1] for c in claims]
    m = max(nv)
    joint = torch.empty((1 << m) * 32, dtype=torch.uint8, device="cuda")
    ptrs = (C.c_void_p * n)(*[C.c_void_p(c[0].data_ptr()) for c in claims])
    nvs = (C.c_int * n)(*nv)
    pts = cd.words([x for c in claims for x in c[2]])
    ev = cd.words([c[3] for c in claims])
    rounds, r = np.zeros(max(1, m) * 3 * 32, dtype=np.uint8), np.zeros(max(1, m) * 32, dtype=np.uint8)
    left, w, je = np.zeros(n * 32, dtype=np.uint8), np.zeros(n * 32, dtype=np.uint8), np.zeros(32, dtype=np.uint8)
    errors = []
    cb = callback(L, cd, challenge, errors, lambda rnd, msg: dec_elems(cd, msg))
    rc = lib(L).lurk_batch_eval_reduce_dev(field, n, ptrs, nvs, L._capi.np_ptr(pts), L._capi.np_ptr(ev), cb, None, L._capi.np_ptr(rounds), L._capi.np_ptr(r),
                                           L._capi.np_ptr(left), L._capi.np_ptr(w), L._capi.np_ptr(je), C.c_void_p(joint.data_ptr()), fmt, None)
    run(L, rc, errors)
    ri = cd.ints(rounds)
    return ([ri[3 * j:3 * j + 3] for j in range(m)], cd.ints(r, m), cd.ints(left), cd.ints(w), cd.ints(je)[0]), to_host(L, field, joint)


@pytest.mark.parametrize("fmt", FMTS)
def test_batch_eval_reduce_across_wrap(L, spec, fmt):
    """m = the first size where poly_combine_kernel runs two grid-stride sweeps; claims of 2^m, 2^(m - 1) (one sweep), and shorter ones"""
    S = shapes()
    field = 0
    p = spec.FIELD_MODULUS[field]
    m = S.batch_eval_m()
    assert S.sc_sweeps(1 << m) >= 2 and S.sc_sweeps(1 << (m - 1)) == 1
    nv = [m - 1, m, 5, 1]
    bufs = [random_elements(field, 1 << k, seed=200 + i, shape="edge") for i, k in enumerate(nv)]
    polys = [ints(b) for b in bufs]
    points = [ints(random_elements(field, k, seed=300 + i, shape="edge")) for i, k in enumerate(nv)]
    evals = [sc.mle_eval(P, x, p) for P, x in zip(polys, points)]
    chal = special_challenge(p, {2: 0, 3: 1, 4: p - 1}, b"be")
    want = bo.batch_eval_reduce(polys, points, evals, chal, p)
    dev = [to_device(L, field, b) for b in bufs]
    got, joint = batch_eval_dev(L, field, [(d, k, x, e) for d, k, x, e in zip(dev, nv, points, evals)], chal, fmt)
    assert got == (want["rounds"], want["r"], want["claims_left"], want["weights"], want["joint_eval"])
    assert ints(joint) == want["joint"]
    assert bo.batch_eval_verify(got[0], points, evals, got[2], chal, p) == (got[1], got[4], got[3])
