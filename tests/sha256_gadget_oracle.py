"""ORACLE (test infrastructure, NOT product code): from-spec restatement of the witness of the SHA-256 coprocessor's
circuit, `synthesize_sha256` (reference src/coprocessor/sha256.rs:27-64).

bellpepper is not in the reference tree; its gadgets are restated here from the public crate (the code bellman's
`gadgets::sha256`, `uint32::UInt32`, `boolean::{Boolean, AllocatedBit}` and `multipack::pack_bits` carry):

  * A Boolean is Constant(v), Is(bit) or Not(bit).  rotr / shr only move Booleans; shr shifts in Constant(false).
  * Boolean::xor: a constant operand returns the other operand or its not() and allocates nothing; otherwise one
    AllocatedBit::xor of the two underlying bits, wrapped in Not when exactly one operand was Not.
  * Boolean::and: nothing for constant operands; otherwise one of and / and_not / nor.
  * sha256_ch / sha256_maj: constant cases reduce to a copy or to a (possibly negated) and; otherwise ch is one
    cs.alloc, maj is `bc = b and c` then one cs.alloc.
  * UInt32::addmany over k operands: all-constant -> a constant; otherwise bitlen(k * (2^32 - 1)) AllocatedBit::alloc
    result bits, LSB first, 32 kept.  MultiEq packs constraints only.
  * sha256_compression_function: schedule i = 16..63 is s0 (two xors), s1 (two xors), addmany[w[i-16], s0, w[i-7], s1];
    rounds defer e = temp1 ++ [d] and a = temp1 ++ temp2 to the top of the next round (e before S1, a before S0);
    h0 / h4 extend the deferred lists with the IV word, h1..h3 / h5..h7 are 2-operand addmany.

One call with n pointers allocates, in order: to_bits_le_strict of every pointer's tag then hash (bellpepper-core,
restated in oracle/spec.py: bitdecomp_witness, whose values are used here), the gadget's aux over the bits (each
pointer's bits padded to a multiple of 8 with Constant(false), the whole vector reversed), pack_bits' element (the
first CAPACITY bits of the reversed digest) and allocate_constant's ExprTag::Num (src/circuit/gadgets/pointer.rs:97-108).

The aux ORDER is pinned by nothing in the reference (as for the Poseidon aux); the packed digest is pinned to the
reference's native compute_sha256 (sha256.rs:66-90) over standard SHA-256 (hashlib).
"""
import hashlib
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import spec  # noqa: E402

TAG_NUM = 4   # ExprTag::Num (reference src/tag.rs:42-47)

K = [0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5,
     0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174,
     0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da,
     0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967,
     0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
     0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,
     0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3,
     0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2]
IV = [0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19]

C0, C1 = ("c", 0), ("c", 1)


def capacity(field):
    return spec.FIELD_NUM_BITS[field] - 1


def compute_sha256(field, inputs):
    """the reference's native compute_sha256 (sha256.rs:66-90) over hashlib: inputs = [tag0, hash0, tag1, hash1, ...]"""
    msg = b"".join(int(x).to_bytes(32, "little") for x in inputs)[::-1]
    return int.from_bytes(hashlib.sha256(msg).digest(), "big") & ((1 << capacity(field)) - 1)


class _Gadget:
    """constraint system that records every aux's value and the relation bellpepper enforces on it"""

    def __init__(self, p):
        self.p = p
        self.aux, self.rel, self.lin = [], [], []

    def alloc(self, v, rel):
        self.aux.append(v)
        self.rel.append(rel)
        return len(self.aux) - 1

    def val(self, b):
        kind, x = b
        return x if kind == "c" else (self.aux[x] if kind == "is" else 1 - self.aux[x])

    # ---- Boolean
    @staticmethod
    def bnot(b):
        kind, x = b
        return ("c", 1 - x) if kind == "c" else (("not", x) if kind == "is" else ("is", x))

    def xor(self, a, b):
        if a == C0:
            return b
        if b == C0:
            return a
        if a == C1:
            return self.bnot(b)
        if b == C1:
            return self.bnot(a)
        x, y = a[1], b[1]
        k = self.alloc(self.aux[x] ^ self.aux[y], ("xor", x, y))
        return ("not", k) if (a[0] == "not") != (b[0] == "not") else ("is", k)

    def band(self, a, b):
        if a == C0 or b == C0:
            return C0
        if a == C1:
            return b
        if b == C1:
            return a
        # and / and_not / nor: the allocated bit is the Booleans' AND
        return ("is", self.alloc(self.val(a) & self.val(b), ("and", a, b)))

    def ch(self, a, b, c):
        v = (self.val(a) & self.val(b)) ^ ((1 - self.val(a)) & self.val(c))
        if a[0] == "c" and b[0] == "c" and c[0] == "c":
            return ("c", v)
        if a == C0:
            return c
        if b == C0:
            return self.band(self.bnot(a), c)
        if c == C0:
            return self.band(a, b)
        if c == C1:
            return self.bnot(self.band(a, self.bnot(b)))
        if b == C1:
            return self.bnot(self.band(self.bnot(a), self.bnot(c)))
        return ("is", self.alloc(v, ("ch", a, b, c)))

    def maj(self, a, b, c):
        va, vb, vc = self.val(a), self.val(b), self.val(c)
        v = (va & vb) ^ (va & vc) ^ (vb & vc)
        if a[0] == "c" and b[0] == "c" and c[0] == "c":
            return ("c", v)
        if a == C0:
            return self.band(b, c)
        if b == C0:
            return self.band(a, c)
        if c == C0:
            return self.band(a, b)
        if c == C1:
            return self.bnot(self.band(self.bnot(a), self.bnot(b)))
        if b == C1:
            return self.bnot(self.band(self.bnot(a), self.bnot(c)))
        if a == C1:
            return self.bnot(self.band(self.bnot(b), self.bnot(c)))
        bc = self.band(b, c)
        return ("is", self.alloc(v, ("maj", a, b, c, bc)))

    # ---- UInt32: 32 Booleans, LSB first
    def u32_value(self, u):
        return sum(self.val(b) << i for i, b in enumerate(u))

    @staticmethod
    def u32_const(v):
        return [("c", (v >> i) & 1) for i in range(32)]

    @staticmethod
    def rotr(u, by):
        return u[by:] + u[:by]

    @staticmethod
    def shr(u, by):
        return u[by:] + [C0] * by

    def u32_xor(self, a, b):
        return [self.xor(x, y) for x, y in zip(a, b)]

    def addmany(self, ops):
        assert 2 <= len(ops) <= 10
        total = sum(self.u32_value(u) for u in ops)
        if all(b[0] == "c" for u in ops for b in u):
            return self.u32_const(total & 0xFFFFFFFF)
        nbits = (len(ops) * 0xFFFFFFFF).bit_length()
        bits = [("is", self.alloc((total >> i) & 1, ("bool",))) for i in range(nbits)]
        self.lin.append(("sum", [b[1] for b in bits], [list(u) for u in ops]))
        return bits[:32]

    # ---- SHA-256
    def compression(self, block, cur):
        w = [list(reversed(block[32 * i:32 * i + 32])) for i in range(16)]     # UInt32::from_bits_be
        for i in range(16, 64):
            s0 = self.u32_xor(self.u32_xor(self.rotr(w[i - 15], 7), self.rotr(w[i - 15], 18)), self.shr(w[i - 15], 3))
            s1 = self.u32_xor(self.u32_xor(self.rotr(w[i - 2], 17), self.rotr(w[i - 2], 19)), self.shr(w[i - 2], 10))
            w.append(self.addmany([w[i - 16], s0, w[i - 7], s1]))

        def compute(m, others):
            return m[1] if m[0] == "concrete" else self.addmany(m[1] + others)

        a, b, c, d = ("concrete", cur[0]), cur[1], cur[2], cur[3]
        e, f, g, h = ("concrete", cur[4]), cur[5], cur[6], cur[7]
        for i in range(64):
            new_e = compute(e, [])
            s1 = self.u32_xor(self.u32_xor(self.rotr(new_e, 6), self.rotr(new_e, 11)), self.rotr(new_e, 25))
            ch = [self.ch(x, y, z) for x, y, z in zip(new_e, f, g)]
            temp1 = [h, s1, ch, self.u32_const(K[i]), w[i]]
            new_a = compute(a, [])
            s0 = self.u32_xor(self.u32_xor(self.rotr(new_a, 2), self.rotr(new_a, 13)), self.rotr(new_a, 22))
            maj = [self.maj(x, y, z) for x, y, z in zip(new_a, b, c)]
            h, g, f = g, f, new_e
            e = ("deferred", temp1 + [d])
            d, c, b = c, b, new_a
            a = ("deferred", temp1 + [s0, maj])
        h0 = compute(a, [cur[0]])
        h1 = self.addmany([cur[1], b])
        h2 = self.addmany([cur[2], c])
        h3 = self.addmany([cur[3], d])
        h4 = compute(e, [cur[4]])
        h5 = self.addmany([cur[5], f])
        h6 = self.addmany([cur[6], g])
        h7 = self.addmany([cur[7], h])
        return [h0, h1, h2, h3, h4, h5, h6, h7]

    def sha256(self, bits):
        assert len(bits) % 8 == 0
        padded = list(bits) + [C1]
        while (len(padded) + 64) % 512:
            padded.append(C0)
        padded += [("c", (len(bits) >> i) & 1) for i in reversed(range(64))]
        cur = [self.u32_const(v) for v in IV]
        for i in range(0, len(padded), 512):
            cur = self.compression(padded[i:i + 512], cur)
        return [b for u in cur for b in reversed(u)]                           # into_bits_be

    # ---- AllocatedNum::to_bits_le_strict; values from oracle/spec.py: bitdecomp_witness
    def to_bits_le_strict(self, field, j, x):
        values = iter(spec.bitdecomp_witness(field, x)[0][1:])
        b = self.p - 1
        result, current_run, last_run, found = [], [], None, False
        for i in reversed(range(256)):
            bb = (b >> i) & 1
            found |= bool(bb)
            if not found:
                continue
            if bb:
                k = self.alloc(next(values), ("bool",))
                current_run.append(k)
                result.append(k)
            else:
                if current_run:
                    if last_run is not None:
                        current_run.append(last_run)
                    cur = current_run[0]
                    for v in current_run[1:]:                          # kary_and
                        cur = self.alloc(next(values), ("and", ("is", cur), ("is", v)))
                    last_run, current_run = cur, []
                result.append(self.alloc(next(values), ("cond", last_run)))   # alloc_conditionally
        assert next(values, None) is None
        le = list(reversed(result))
        self.lin.append(("num", le, j))
        return [("is", k) for k in le]


def _run(field, inputs):
    p = spec.FIELD_MODULUS[field]
    g = _Gadget(p)
    bits = []
    for j, x in enumerate(inputs):        # per pointer: tag, then hash
        bits += g.to_bits_le_strict(field, j, int(x) % p)
        bits += [C0] * (-len(bits) % 8)
    digest = g.sha256(list(reversed(bits)))
    digest.reverse()
    packed = digest[:capacity(field)]
    g.alloc(sum(g.val(b) << i for i, b in enumerate(packed)) % p, ("pack", packed))
    g.alloc(TAG_NUM, ("const", TAG_NUM))
    return g


def witness(field, inputs):
    """the aux block of one synthesize_sha256 call: inputs = [tag0, hash0, ..., tag_{n-1}, hash_{n-1}] (ints < p)"""
    assert len(inputs) % 2 == 0 and inputs
    return _run(field, inputs).aux


_REL = {}


def relations(field, n):
    """(per-aux relations, linear relations) of one call with n pointers; they depend on (field, n) only"""
    if (field, n) not in _REL:
        g = _run(field, [0] * (2 * n))
        _REL[(field, n)] = (g.rel, g.lin)
    return _REL[(field, n)]


def block_len(field, n):
    return len(relations(field, n)[0])


def check(field, block, inputs):
    """evaluate every relation the circuit enforces on the block; returns the list of violated ones (empty = ok)"""
    p = spec.FIELD_MODULUS[field]
    n = len(inputs) // 2
    rel, lin = relations(field, n)
    if len(block) != len(rel):
        return ["length"]
    aux = [int(v) % p for v in block]

    def v(b):
        kind, x = b
        return x if kind == "c" else (aux[x] if kind == "is" else (1 - aux[x]) % p)

    bad = []
    for k, r in enumerate(rel):
        c = aux[k]
        t = r[0]
        if t == "bool":
            ok = c * (1 - c) % p == 0
        elif t == "cond":                  # (1 - last_run - a) * a = 0
            ok = (1 - aux[r[1]] - c) * c % p == 0
        elif t == "xor":                   # (2a) * b = a + b - c
            a, b = aux[r[1]], aux[r[2]]
            ok = (2 * a * b - (a + b - c)) % p == 0
        elif t == "and":                   # and / and_not / nor on the operands' linear forms
            ok = (v(r[1]) * v(r[2]) - c) % p == 0
        elif t == "ch":                    # a (b - c) = ch - c
            a, b, cc = v(r[1]), v(r[2]), v(r[3])
            ok = (a * (b - cc) - (c - cc)) % p == 0
        elif t == "maj":                   # (2bc - b - c) a = bc - maj
            a, b, cc, bc = v(r[1]), v(r[2]), v(r[3]), v(r[4])
            ok = ((2 * bc - b - cc) * a - (bc - c)) % p == 0
        elif t == "pack":                  # sum 2^i bit_i = packed
            ok = (sum(v(b) << i for i, b in enumerate(r[1])) - c) % p == 0
        elif t == "const":
            ok = (c - r[1]) % p == 0
        else:
            raise AssertionError(t)
        if not ok:
            bad.append((k, t))
    for r in lin:
        if r[0] == "sum":                  # addmany: sum of the operands = sum of the result bits
            lhs = sum(v(b) << i for u in r[2] for i, b in enumerate(u))
            rhs = sum(aux[k] << i for i, k in enumerate(r[1]))
        else:                              # to_bits_le_strict: the bits pack to the input
            lhs = sum(aux[k] << i for i, k in enumerate(r[1]))
            rhs = int(inputs[r[2]])
        if (lhs - rhs) % p:
            bad.append(r[:1])
    return bad


def r1cs_rows(field, n, aux_col, in_col, u_col):
    """the constraints bellpepper enforces on one call's block, as R1CS rows over z = (W, u, X): the block's aux k is
    column aux_col + k, input element j is column in_col + j, constants multiply u_col.  Returns (A, B, C), each a list
    of [(column, canonical coefficient)] per row."""
    p = spec.FIELD_MODULUS[field]
    rel, lin = relations(field, n)
    A, B, C = [], [], []

    def lc(terms):
        acc = {}
        for col, v in terms:
            acc[col] = (acc.get(col, 0) + v) % p
        return [(col, v) for col, v in acc.items() if v]

    def bl(b, coeff=1):
        kind, x = b
        if kind == "c":
            return [(u_col, coeff * x)]
        return [(aux_col + x, coeff)] if kind == "is" else [(u_col, coeff), (aux_col + x, -coeff)]

    def row(a, b, c):
        A.append(lc(a)); B.append(lc(b)); C.append(lc(c))

    one = [(u_col, 1)]
    for k, r in enumerate(rel):
        c = aux_col + k
        t = r[0]
        if t == "bool":
            row([(c, 1)], [(u_col, 1), (c, -1)], [])
        elif t == "cond":
            row([(u_col, 1), (aux_col + r[1], -1), (c, -1)], [(c, 1)], [])
        elif t == "xor":
            a, b = aux_col + r[1], aux_col + r[2]
            row([(a, 2)], [(b, 1)], [(a, 1), (b, 1), (c, -1)])
        elif t == "and":
            row(bl(r[1]), bl(r[2]), [(c, 1)])
        elif t == "ch":
            row(bl(r[2]) + bl(r[3], -1), bl(r[1]), [(c, 1)] + bl(r[3], -1))
        elif t == "maj":
            row(bl(r[4], 2) + bl(r[2], -1) + bl(r[3], -1), bl(r[1]), bl(r[4]) + [(c, -1)])
        elif t == "pack":
            row([t_ for i, b in enumerate(r[1]) for t_ in bl(b, 1 << i)], one, [(c, 1)])
        elif t == "const":
            row([(c, 1)], one, [(u_col, r[1])])
    for r in lin:
        if r[0] == "sum":
            row([t_ for u in r[2] for i, b in enumerate(u) for t_ in bl(b, 1 << i)], one, [(aux_col + k, 1 << i) for i, k in enumerate(r[1])])
        else:
            row([(aux_col + k, 1 << i) for i, k in enumerate(r[1])], one, [(in_col + r[2], 1)])
    return A, B, C
