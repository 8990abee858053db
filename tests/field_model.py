"""A word-for-word restatement of csrc/field.cuh's limb algorithms that records which carries and branches each operand takes.

The device code keeps its carries in the condition-code register between separate asm statements, and several of them are reached
only by operands nobody feeds by chance (a carry that needs a 128-bit run of ones, the 3rd or 4th conditional subtraction of a lazy
dot product that needs m close to 2^256).  The model below runs the same 32-bit word operations on numpy arrays of operands (one
lane per operand, the carry flag an array too) and returns, beside the value, a boolean array per named event:

  merge_carry     carry of even[0] + odd[1] at the start of a row of the Montgomery product (mad_row_redc)
  cmad_n_carry    carry of the row product cmad_n(even, a, bi) into odd[7]
  mod0_carry      carry of the m*p row cmad_mod<0>(even, mi) into odd[7]
  mod1_carry      carry out of cmad_mod<1>(odd, mi), which the code drops: must never happen
  addc_overflow   a carry lost by an addc without carry-out (odd[7], r[7], t[16], the counters): must never happen
  final_sub       the conditional subtraction of the product / sum taken
  sub_borrow      a - b borrowed (p added back)
  ce0..ce4 co0..co3   a pending carry counter of WideAcc non-zero at reduce()
  round1..round4  the k-th conditional subtraction of redc17 taken
  unreduced       redc17 returned a value >= p (ROUNDS too small for the operands): must never happen with the bounds respected
  inv_zero inv_no_loop inv_exit_u inv_exit_w inv_halve_odd   inv_vartime's early exits, loop exits and the + p of halve

Operand builders at the bottom reach each event; tests/test_field_model.py checks the model against Python integers and that the
builders reach every event the model can reach.  Montgomery operands are raw words: the element x is stored as x * 2^256 mod p.
"""
import numpy as np

from oracle import spec

MASK = np.uint64(0xffffffff)
R = 1 << 256
FIELDS = (0, 1, 2, 3)


class Field:
    def __init__(self, fid):
        self.fid = fid
        self.p = p = spec.FIELD_MODULUS[fid]
        self.mod = [(p >> (32 * i)) & 0xffffffff for i in range(8)]
        self.m0 = (-pow(p, -1, 1 << 32)) % (1 << 32)
        self.rinv = pow(R, -1, p)

    def mont(self, x):
        return x * R % self.p

    def unmont(self, x):
        return x * self.rinv % self.p


def to_words(vals):
    """(n, 8) uint64 array of 32-bit words from Python integers < 2^256"""
    b = b"".join(int(v).to_bytes(32, "little") for v in vals)
    return np.frombuffer(b, dtype="<u4").reshape(-1, 8).astype(np.uint64)


def from_words(w):
    w = np.asarray(w, dtype=np.uint64).reshape(-1, 8)
    b = w.astype("<u4").tobytes()
    return [int.from_bytes(b[i:i + 32], "little") for i in range(0, len(b), 32)]


class _Run:
    """the carry flag and the events of one vectorised call"""

    def __init__(self, n):
        self.n = n
        self.cf = np.zeros(n, dtype=np.uint64)
        self.ev = {}

    def hit(self, name, mask):
        mask = np.asarray(mask, dtype=bool)
        self.ev[name] = self.ev.get(name, np.zeros(self.n, dtype=bool)) | mask

    # PTX add/sub with the condition code
    def add_cc(self, a, b):
        s = a + b
        self.cf = s >> np.uint64(32)
        return s & MASK

    def addc_cc(self, a, b):
        s = a + b + self.cf
        self.cf = s >> np.uint64(32)
        return s & MASK

    def addc(self, a, b, wraps=False):
        s = a + b + self.cf
        if not wraps:
            self.hit("addc_overflow", (s >> np.uint64(32)) != 0)
        return s & MASK

    def sub_cc(self, a, b):
        self.cf = (a < b).astype(np.uint64)
        return (a - b) & MASK

    def subc_cc(self, a, b):
        d = b + self.cf
        c = (a < d).astype(np.uint64)
        r = (a - d) & MASK
        self.cf = c
        return r

    def subc00(self):
        return self.cf != 0           # subc(0, 0) != 0: the chain borrowed

    def mad_lo_cc(self, a, b, c):
        return self.add_cc((a * b) & MASK, c)

    def madc_lo_cc(self, a, b, c):
        return self.addc_cc((a * b) & MASK, c)

    def madc_hi_cc(self, a, b, c):
        return self.addc_cc((a * b) >> np.uint64(32), c)

    def madc_hi(self, a, b, c):
        return self.addc((a * b) >> np.uint64(32), c)


def _col(w, i):
    return w[:, i].copy()


ZERO = np.uint64(0)


# ------------------------------------------------------------------------------------------------- Fe::operator* and friends
def _cmad_n(c, acc, off, a, bi):
    """acc[off..off+7] += (a[0], a[2], a[4], a[6]) * bi, one carry chain (a: list of 4 word arrays)"""
    acc[off] = c.mad_lo_cc(a[0], bi, acc[off])
    acc[off + 1] = c.madc_hi_cc(a[0], bi, acc[off + 1])
    for j in (2, 4, 6):
        acc[off + j] = c.madc_lo_cc(a[j // 2], bi, acc[off + j])
        acc[off + j + 1] = c.madc_hi_cc(a[j // 2], bi, acc[off + j + 1])


def _cmad_mod(F, c, acc, off, which, mi):
    _cmad_n(c, acc, off, [np.uint64(F.mod[which + j]) for j in (0, 2, 4, 6)], mi)


def _mad_row_redc(F, c, first, even, odd, ae, ao, bi):
    if first:
        for j in range(4):
            odd[2 * j], odd[2 * j + 1] = (ao[j] * bi) & MASK, (ao[j] * bi) >> np.uint64(32)
            even[2 * j], even[2 * j + 1] = (ae[j] * bi) & MASK, (ae[j] * bi) >> np.uint64(32)
    else:
        even[0] = c.add_cc(even[0], odd[1])
        c.hit("merge_carry", c.cf != 0)
        for j in (0, 2, 4):                                     # madc_n_rshift
            odd[j] = c.madc_lo_cc(ao[j // 2], bi, odd[j + 2])
            odd[j + 1] = c.madc_hi_cc(ao[j // 2], bi, odd[j + 3])
        odd[6] = c.madc_lo_cc(ao[3], bi, ZERO)
        odd[7] = c.madc_hi(ao[3], bi, ZERO)
        _cmad_n(c, even, 0, ae, bi)
        c.hit("cmad_n_carry", c.cf != 0)
        odd[7] = c.addc(odd[7], ZERO)
    mi = (even[0] * np.uint64(F.m0)) & MASK
    _cmad_mod(F, c, odd, 0, 1, mi)
    c.hit("mod1_carry", c.cf != 0)
    _cmad_mod(F, c, even, 0, 0, mi)
    c.hit("mod0_carry", c.cf != 0)
    odd[7] = c.addc(odd[7], ZERO)


def _final_sub(F, c, v, name="final_sub"):
    t = [c.sub_cc(v[0], np.uint64(F.mod[0]))] + [None] * 7
    for i in range(1, 8):
        t[i] = c.subc_cc(v[i], np.uint64(F.mod[i]))
    borrow = c.subc00()
    c.hit(name, ~borrow)
    return [np.where(borrow, v[i], t[i]) for i in range(8)]


def _stack(v):
    return np.stack(v, axis=1)


def mul(F, a, b, c=None):
    """Montgomery product a b / 2^256 mod p of (n, 8) word arrays; returns (words, events)"""
    own = c is None
    c = c or _Run(a.shape[0])
    ae = [_col(a, i) for i in (0, 2, 4, 6)]
    ao = [_col(a, i) for i in (1, 3, 5, 7)]
    even, odd = [None] * 8, [None] * 8
    _mad_row_redc(F, c, True, even, odd, ae, ao, _col(b, 0))
    _mad_row_redc(F, c, False, odd, even, ae, ao, _col(b, 1))
    for i in (2, 4, 6):
        _mad_row_redc(F, c, False, even, odd, ae, ao, _col(b, i))
        _mad_row_redc(F, c, False, odd, even, ae, ao, _col(b, i + 1))
    r = [None] * 8
    r[0] = c.add_cc(even[0], odd[1])
    for i in range(1, 7):
        r[i] = c.addc_cc(even[i], odd[i + 1])
    r[7] = c.addc(even[7], ZERO)
    r = _final_sub(F, c, r)
    return _stack(r), (c.ev if own else None)


def add(F, a, b, c=None):
    own = c is None
    c = c or _Run(a.shape[0])
    r = [c.add_cc(a[:, 0], b[:, 0])] + [None] * 7
    for i in range(1, 7):
        r[i] = c.addc_cc(a[:, i], b[:, i])
    r[7] = c.addc(a[:, 7], b[:, 7])
    r = _final_sub(F, c, r)
    return _stack(r), (c.ev if own else None)


def sub(F, a, b, c=None):
    own = c is None
    c = c or _Run(a.shape[0])
    r = [c.sub_cc(a[:, 0], b[:, 0])] + [None] * 7
    for i in range(1, 8):
        r[i] = c.subc_cc(a[:, i], b[:, i])
    borrow = c.subc00()
    c.hit("sub_borrow", borrow)
    m = [np.where(borrow, np.uint64(F.mod[i]), ZERO) for i in range(8)]
    r[0] = c.add_cc(r[0], m[0])
    for i in range(1, 7):
        r[i] = c.addc_cc(r[i], m[i])
    r[7] = c.addc(r[7], m[7], wraps=True)       # a - b + 2^256 + p: the carry out is the 2^256 the borrow lent
    return _stack(r), (c.ev if own else None)


def final_sub(F, a):
    """Fe::final_sub on raw 256-bit words (any value < 2^256) and Fe::is_reduced"""
    c = _Run(a.shape[0])
    r = _final_sub(F, c, [_col(a, i) for i in range(8)])
    reduced = ~c.ev["final_sub"]
    return _stack(r), reduced, c.ev


# ------------------------------------------------------------------------------------------------- WideAcc and redc17
def redc17(F, c, t, rounds):
    r = [np.zeros(c.n, dtype=np.uint64) for _ in range(9)]
    for i in range(8):
        mi = (t[i] * np.uint64(F.m0)) & MASK
        _cmad_mod(F, c, t, i, 0, mi)
        r[i] = c.addc(r[i], ZERO)
        _cmad_mod(F, c, t, i + 1, 1, mi)
        r[i + 1] = c.addc(r[i + 1], ZERO)
    t[8] = c.add_cc(t[8], r[0])
    for k in range(1, 8):
        t[8 + k] = c.addc_cc(t[8 + k], r[k])
    t[16] = c.addc(t[16], r[8])
    pre = [t[8 + k].copy() for k in range(9)]
    for rnd in range(rounds):
        d = [c.sub_cc(t[8], np.uint64(F.mod[0]))] + [None] * 8
        for k in range(1, 8):
            d[k] = c.subc_cc(t[8 + k], np.uint64(F.mod[k]))
        d[8] = c.subc_cc(t[16], ZERO)
        borrow = c.subc00()
        c.hit("round%d" % (rnd + 1), ~borrow)
        for k in range(9):
            t[8 + k] = np.where(borrow, t[8 + k], d[k])
    out = _stack([t[8 + k] for k in range(8)])
    c.hit("unreduced", (t[16] != 0) | ~_is_reduced(F, out))
    return out, pre


def _is_reduced(F, w):
    c = _Run(w.shape[0])
    _final_sub(F, c, [_col(w, i) for i in range(8)])
    return ~c.ev["final_sub"]


def dot(F, A, B, rounds=3):
    """WideAcc: sum_k A[:, k] B[:, k] / 2^256 mod p through mul_acc and reduce<rounds>.  A, B: (n, k, 8) word arrays.
    Returns (words, events, pre) with pre the 9-word value before the conditional subtractions."""
    n, k = A.shape[0], A.shape[1]
    c = _Run(n)
    e = [np.zeros(n, dtype=np.uint64) for _ in range(17)]
    o = [np.zeros(n, dtype=np.uint64) for _ in range(16)]
    ce = [np.zeros(n, dtype=np.uint64) for _ in range(5)]
    co = [np.zeros(n, dtype=np.uint64) for _ in range(4)]
    for q in range(k):
        ae = [A[:, q, i] for i in (0, 2, 4, 6)]
        ao = [A[:, q, i] for i in (1, 3, 5, 7)]
        for I in range(8):
            bi = B[:, q, I]
            if I % 2 == 0:
                _cmad_n(c, e, I, ae, bi)
                ce[I // 2] = c.addc(ce[I // 2], ZERO)
                _cmad_n(c, o, I, ao, bi)
                co[I // 2] = c.addc(co[I // 2], ZERO)
            else:
                _cmad_n(c, e, I + 1, ao, bi)
                ce[(I + 1) // 2] = c.addc(ce[(I + 1) // 2], ZERO)
                _cmad_n(c, o, I - 1, ae, bi)
                co[(I - 1) // 2] = c.addc(co[(I - 1) // 2], ZERO)
    for i in range(5):
        c.hit("ce%d" % i, ce[i] != 0)
    for i in range(4):
        c.hit("co%d" % i, co[i] != 0)
    e[8] = c.add_cc(e[8], ce[0]); e[9] = c.addc_cc(e[9], ZERO)
    e[10] = c.addc_cc(e[10], ce[1]); e[11] = c.addc_cc(e[11], ZERO)
    e[12] = c.addc_cc(e[12], ce[2]); e[13] = c.addc_cc(e[13], ZERO)
    e[14] = c.addc_cc(e[14], ce[3]); e[15] = c.addc_cc(e[15], ZERO)
    e[16] = c.addc(e[16], ce[4])
    o[8] = c.add_cc(o[8], co[0]); o[9] = c.addc_cc(o[9], ZERO)
    o[10] = c.addc_cc(o[10], co[1]); o[11] = c.addc_cc(o[11], ZERO)
    o[12] = c.addc_cc(o[12], co[2]); o[13] = c.addc_cc(o[13], ZERO)
    o[14] = c.addc_cc(o[14], co[3]); o[15] = c.addc(o[15], ZERO)
    t = [None] * 17
    t[0] = e[0]
    t[1] = c.add_cc(e[1], o[0])
    for q in range(2, 16):
        t[q] = c.addc_cc(e[q], o[q - 1])
    t[16] = c.addc(e[16], o[15])
    out, pre = redc17(F, c, t, rounds)
    return out, c.ev, from_words_wide(pre)


def from_words_wide(pre):
    return [sum(int(pre[k][i]) << (32 * k) for k in range(9)) for i in range(len(pre[0]))]


# ------------------------------------------------------------------------------------------------- Fe::inv_vartime
def inv_vartime(F, x):
    """binary extended Euclid on the raw Montgomery value x (a Python int); returns (x^-1 in Montgomery form, events, iterations)"""
    p, ev = F.p, set()
    if x == 0:
        return 0, {"inv_zero"}, 0
    u, w, x1, x2, it = x, p, 1, 0, 0

    def halve(v):
        if v & 1:
            ev.add("inv_halve_odd")
            v += p
        return v >> 1

    if u == 1:
        ev.add("inv_no_loop")
    while u != 1 and w != 1:
        it += 1
        while not u & 1:
            u >>= 1
            x1 = halve(x1)
        while not w & 1:
            w >>= 1
            x2 = halve(x2)
        if u >= w:
            u, x1 = u - w, (x1 - x2) % p
        else:
            w, x2 = w - u, (x2 - x1) % p
    ev.add("inv_exit_u" if u == 1 else "inv_exit_w")
    xr = x1 if u == 1 else x2
    r3, _ = mul(F, to_words([F.mont(F.mont(1))]), to_words([F.mont(F.mont(1))]))   # rr() * rr() = R^3 mod p
    out, _ = mul(F, to_words([xr]), r3)
    return from_words(out)[0], ev, it


# ------------------------------------------------------------------------------------------------- operand builders
def chosen_products(F, rng, count=8):
    """(a, b) raw Montgomery pairs whose Montgomery product is a chosen value: 0, 1, p - 1, p - 2, 2^j, R mod p and values with runs of
    0xffffffff words (b = target * R / a)"""
    p = F.p
    targets = [0, 1, 2, p - 1, p - 2, p - 3, (p - 1) // 2, (p + 1) // 2, R % p, F.rinv]
    targets += [1 << j for j in (31, 32, 63, 64, 127, 128, 191, 192, 223, 224, p.bit_length() - 2, p.bit_length() - 1) if (1 << j) < p]
    for lo, hi in ((0, 4), (4, 8), (0, 7), (1, 8), (2, 6), (0, 8)):
        targets.append(sum(0xffffffff << (32 * i) for i in range(lo, hi)) % p)
    targets += [(p - 1 - s) for s in (1 << 32, 1 << 64, (1 << 128) - 1)]
    a_vals = [1, 2, p - 1, p - 2, R % p, F.mont(1), F.mont(p - 1)] + [int(rng.integers(1, 1 << 62)) * int(rng.integers(1, 1 << 62)) % p
                                                                        for _ in range(count)]
    pairs = []
    for t in targets:
        for a in a_vals:
            pairs.append((a, t * R * pow(a, -1, p) % p))
    return pairs


def word_patterns(F, rng, count):
    """raw values < p with words drawn from {0, 1, 0xffffffff, 0xfffffffe, 0x80000000, 0x7fffffff, the modulus' own words, random}"""
    p = F.p
    pool = np.array([0, 1, 0xffffffff, 0xfffffffe, 0x80000000, 0x7fffffff] + F.mod, dtype=np.uint64)
    out = []
    while len(out) < count:
        w = pool[rng.integers(0, len(pool), size=(count, 8))]
        rand = rng.integers(0, 1 << 32, size=(count, 8), dtype=np.uint64)
        w = np.where(rng.random((count, 8)) < 0.25, rand, w)
        out += [v for v in from_words(w) if v < p]
    return out[:count]


def near_top(F, rng, count, span=1 << 64):
    """raw Montgomery values p - 1 - s for small s"""
    return [F.p - 1 - int(s) for s in rng.integers(0, span, size=count, dtype=np.uint64)]


def edge_values(F):
    p = F.p
    vals = [0, 1, 2, 3, p - 1, p - 2, p - 3, (p - 1) // 2, (p + 1) // 2, R % p, F.rinv, F.mont(1), F.mont(p - 1), F.mont(2)]
    vals += [(1 << j) % p for j in range(0, 256, 31)] + [((1 << j) - 1) % p for j in (32, 64, 96, 128, 160, 192, 224, 253, 254)]
    vals += [sum(0xffffffff << (32 * i) for i in range(lo, hi)) % p for lo, hi in ((0, 4), (4, 8), (0, 7), (1, 8), (3, 5), (0, 8))]
    return sorted(set(vals))


def random_below(F, rng, count):
    """uniform raw values in [0, p)"""
    p, bits = F.p, F.p.bit_length()
    out = []
    while len(out) < count:
        w = rng.integers(0, 1 << 32, size=(2 * count, 8), dtype=np.uint64)
        w[:, 7] &= np.uint64((1 << (bits - 224)) - 1)
        out += [v for v in from_words(w) if v < p]
    return out[:count]


def dot_at_round(F, k, rnd, rng, tries=4000):
    """k pairs (A, B) of raw Montgomery values whose WideAcc reduction takes conditional subtraction `rnd` (the value before the
    subtractions is >= rnd p), or None when no such pair of lists exists.  The value is (T + m p) / 2^256 with T = sum A_i B_i and
    m = -T / p mod 2^256; it is largest for T close to k (p - 1)^2 and m close to 2^256.  First a search over operands p - 1 - s (s
    below 2^64); when that needs m within ~2^128 of 2^256 (Pasta at k = 4, 8, 12) a construction: T = k (p - 1)^2 - D with
    m = 2^256 - 1 - s fixes D mod 2^256, D = r0 + j 2^256 picks j so that D = (u + 1)(p - 1) + v (p - 2) with small u, v, and the
    last two pairs become (p - 1, p - 1 - u), (p - 2, p - 1 - v)."""
    p = F.p
    if k * (p - 1) ** 2 + (R - 1) * p < rnd * p * R:
        return None
    A = np.array([near_top(F, rng, k, 1 << 64) for _ in range(tries)], dtype=object)
    B = np.array([near_top(F, rng, k, 1 << 64) for _ in range(tries)], dtype=object)
    for i in range(tries):
        T = sum(int(x) * int(y) for x, y in zip(A[i], B[i]))
        m = (-T * pow(p, -1, R)) % R
        if (T + m * p) >> 256 >= rnd * p:
            return [int(x) for x in A[i]], [int(y) for y in B[i]]
    # Q = r p exactly: with a_i = p - alpha_i, b_i = p - beta_i and sum alpha_i beta_i = p, T = 0 mod p and m = r 2^256 - k p + S - 1,
    # S = sum (alpha_i + beta_i); m < 2^256 asks S <= k p - (r - 1) 2^256.  One pair near sqrt(p) carries the product, the others
    # are (1, rho - (k - 2)) and (1, 1).
    from math import isqrt
    budget = k * p - (rnd - 1) * R
    if k < 2 or budget < 2 * isqrt(p):
        return None
    # with alpha = isqrt(p) - j, p mod alpha is about (j^2 + p - isqrt(p)^2) mod alpha: small near j^2 + p - isqrt(p)^2 = c alpha
    s0 = isqrt(p)
    e0 = p - s0 * s0
    starts = [0] + [isqrt(c * s0 - e0) for c in range(1, 8) if c * s0 > e0]
    for j in (j0 + d for j0 in starts for d in range(-2048, 2048)):
        alpha = s0 - j
        if j < 0 or alpha < 2:
            continue
        beta, rho = divmod(p, alpha)
        S = alpha + beta + 1 + (rho - (k - 2)) + 2 * (k - 2)
        if rho >= k - 1 and S <= budget and beta < p:
            al = [alpha, 1] + [1] * (k - 2)
            be = [beta, rho - (k - 2)] + [1] * (k - 2)
            return [p - x for x in al], [p - y for y in be]
    return None


# ------------------------------------------------------------------------------------------------- cases of the operation harness
# operation numbers of tests/csrc/field_dev_test.cu
OPS = ("mul", "sqr", "add", "sub", "neg", "dbl", "pow5", "inv", "inv_vartime", "from_canonical", "to_canonical", "final_sub",
       "is_reduced", "mul_sub_mul", "ipa_fold", "dot", "dot4", "csr_row")
# "dot" is WideAcc::reduce() with its default ROUNDS (3), "dot4" reduce<4>
OP = {name: i for i, name in enumerate(OPS)}
# WideAcc::reduce's comment: ROUNDS = 3 is enough for k <= 11 products on Pasta (p / 2^256 = 0.25) and k <= 15 on BN254 (0.19)
REDUCE3_MAX_K = {0: 15, 1: 15, 2: 11, 3: 11}
ARITY = {"mul": 2, "add": 2, "sub": 2, "mul_sub_mul": 4, "ipa_fold": 4}


def expected(F, op, args):
    """the operation on raw words, from Python integers (Montgomery operands stay in Montgomery form)"""
    p, ri = F.p, F.rinv
    a = args[0]
    if op == "mul":
        return a * args[1] * ri % p
    if op == "sqr":
        return a * a * ri % p
    if op == "add":
        return (a + args[1]) % p
    if op == "sub":
        return (a - args[1]) % p
    if op == "neg":
        return -a % p
    if op == "dbl":
        return 2 * a % p
    if op == "pow5":
        return pow(a, 5, p) * pow(ri, 4, p) % p
    if op in ("inv", "inv_vartime"):
        return pow(a, -1, p) * R * R % p if a % p else 0
    if op == "from_canonical":
        return a * R % p
    if op == "to_canonical":
        return a * ri % p
    if op == "final_sub":
        return a - p if a >= p else a
    if op == "is_reduced":
        return int(a < p)
    if op == "mul_sub_mul":
        return (a * args[1] - args[2] * args[3]) * ri % p
    if op == "ipa_fold":
        return (a * args[2] + args[1] * args[3]) * ri % p
    k = len(args) // 2
    return sum(x * y for x, y in zip(args[:k], args[k:])) * ri % p


def inversion_inputs(F):
    """0, 1, p - 1, 2^j, and raw Montgomery words 1 and 2^j (the early exit and the long runs of halvings)"""
    p, bits = F.p, F.p.bit_length()
    vals = [0, 1, 2, p - 1, p - 2, F.mont(1), F.mont(p - 1), F.mont(2), (p - 1) // 2, (p + 1) // 2]
    vals += [1 << j for j in range(bits - 1)] + [F.mont(1 << j) for j in range(0, bits - 1, 7)] + [(1 << j) - 1 for j in range(2, bits - 1, 9)]
    return sorted(set(v % p for v in vals))


def raw_boundaries(F):
    """unreduced 256-bit values around p and 2^256 for final_sub / is_reduced"""
    p = F.p
    vals = [0, 1, p - 2, p - 1, p, p + 1, p + 2, 2 * p - 1, 2 * p, R - 1, R - 2, R - p, (R - 1) // 2, p | 0xffffffff, p + (1 << 128)]
    if 3 * p < R:
        vals += [3 * p - 1, 3 * p]
    vals += [p + (1 << j) for j in range(0, 254, 17)] + [p - (1 << j) for j in range(0, 254, 17)]
    return sorted(set(v for v in vals if 0 <= v < R))


def constructed_cases(F, seed=0):
    """{op: list of argument tuples (raw words)} reaching the events of the model; dot products as {("dot", k): [(A + B)]}"""
    rng = np.random.default_rng(seed)
    edge = edge_values(F)
    pairs = chosen_products(F, rng) + [(x, y) for x in edge for y in edge]
    pairs += list(zip(word_patterns(F, rng, 2000), word_patterns(F, rng, 2000)))
    pairs += list(zip(near_top(F, rng, 300), near_top(F, rng, 300))) + list(zip(near_top(F, rng, 300), random_below(F, rng, 300)))
    unary = sorted(set(edge + [x for x, _ in pairs[:200]] + word_patterns(F, rng, 500) + near_top(F, rng, 200) + inversion_inputs(F)))
    quads = [tuple(int(edge[i]) for i in rng.integers(0, len(edge), size=4)) for _ in range(1500)]
    quads += [tuple(near_top(F, rng, 4)) for _ in range(300)] + [tuple(word_patterns(F, rng, 4)) for _ in range(300)]
    quads += [(F.p - 1,) * 4, (F.p - 1, F.p - 1, 1, 1), (0, 0, F.p - 1, F.p - 1)]
    cases = {op: [(x,) for x in unary] for op in ("sqr", "neg", "dbl", "pow5", "to_canonical", "from_canonical")}
    cases["inv"] = [(x,) for x in inversion_inputs(F)] + [(x,) for x in edge]
    cases["inv_vartime"] = [(x,) for x in sorted(set(unary))]
    for op in ("mul", "add", "sub"):
        cases[op] = pairs
    cases["final_sub"] = cases["is_reduced"] = [(x,) for x in raw_boundaries(F) + [x for x, _ in pairs[:300]]]
    cases["mul_sub_mul"] = cases["ipa_fold"] = quads
    for k in range(1, 16):
        rows = [[F.p - 1] * (2 * k), [0] * (2 * k), [1] * (2 * k)]
        for rnd in range(1, 5):
            d = dot_at_round(F, k, rnd, rng, tries=200)
            if d is not None:
                rows.append(d[0] + d[1])
        rows += [near_top(F, rng, 2 * k) for _ in range(48)] + [word_patterns(F, rng, 2 * k) for _ in range(48)]
        rows += [random_below(F, rng, 2 * k) for _ in range(16)]
        cases[("dot", k)] = [tuple(r) for r in rows]
    return cases


def model_events(F, cases):
    """union of the named events the model records over the constructed cases (and the dot results of reduce<3> and reduce<4>)"""
    seen, dots = set(), {}

    def take(ev):
        seen.update(name for name, m in ev.items() if m.any())

    for op in ("mul", "sqr", "add", "sub"):
        args = cases[op]
        a = to_words([t[0] for t in args])
        b = a if op == "sqr" else to_words([t[1] for t in args])
        take({"mul": mul, "sqr": mul, "add": add, "sub": sub}[op](F, a, b)[1])
    take(final_sub(F, to_words([t[0] for t in cases["final_sub"]]))[2])
    for (x,) in cases["inv_vartime"]:
        seen |= inv_vartime(F, x)[1]
    for key, rows in cases.items():
        if isinstance(key, tuple):
            k = key[1]
            A = np.stack([to_words([r[q] for r in rows]) for q in range(k)], axis=1)
            B = np.stack([to_words([r[k + q] for r in rows]) for q in range(k)], axis=1)
            for rounds in (3, 4):
                out, ev, pre = dot(F, A, B, rounds)
                dots[(k, rounds)] = (from_words(out), ev)
                if rounds == 4 or k <= REDUCE3_MAX_K[F.fid]:
                    take(ev)
    return seen, dots


def random_words(F, rng, n):
    """(n, 8) uint32 array of uniform raw values in [0, p), vectorised (rejection on the top word, then a word-wise compare with p)"""
    bits = F.p.bit_length()
    out = np.zeros((0, 8), dtype=np.uint32)
    while len(out) < n:
        w = rng.integers(0, 1 << 32, size=(n + n // 2 + 16, 8), dtype=np.uint64).astype(np.uint32)
        w[:, 7] &= np.uint32((1 << (bits - 224)) - 1)
        lt = np.zeros(len(w), dtype=bool)
        eq = np.ones(len(w), dtype=bool)
        for i in range(7, -1, -1):
            lt |= eq & (w[:, i] < np.uint32(F.mod[i]))
            eq &= w[:, i] == np.uint32(F.mod[i])
        out = np.concatenate([out, w[lt]])
    return out[:n]


def pack_cases(args):
    """uint8 buffer of argument tuples, 32 bytes per element, for fdt_run"""
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for t in args for v in t), dtype=np.uint8).copy()
