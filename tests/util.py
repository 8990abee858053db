"""Shared helpers for the parity tests: seeded inputs in the shapes SURVEY.md 8(d) prescribes."""
import numpy as np

from oracle import spec

import json
import os

# reference golden digests, BN256 Fr (SURVEY.md 8(c)); the fixture cites the reference test each one comes from
with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_goldens.json")) as _f:
    REFERENCE = json.load(_f)
GOLDEN = {k: int(v["hex"], 16) for k, v in REFERENCE["poseidon_digests"].items()}
# ExprTag values used by the goldens (src/tag.rs): Nil=0, Cons=1, Sym=2, Fun=3, Num=4, Str=6, Char=7
TAG_SYM, TAG_NUM, TAG_STR, TAG_CHAR, TAG_NIL = 2, 4, 6, 7, 0


def edge_values(field_id):
    """the operands where modular arithmetic goes wrong: 0, 1, 2, p-1, p-2, (p-1)/2, (p+1)/2, 2^k and 2^k - 1 for the top
    bits, R mod p and R^-1 mod p (R = 2^256, the Montgomery radix), and the elements whose Montgomery form is p - 1, p - 2"""
    p = spec.FIELD_MODULUS[field_id]
    bits = p.bit_length()
    R = 1 << 256
    vals = [0, 1, 2, p - 1, p - 2, (p - 1) // 2, (p + 1) // 2, R % p, pow(R, -1, p), montgomery_top(p, 0), montgomery_top(p, 1)]
    for k in range(bits - 3, bits):
        vals += [(1 << k) % p, ((1 << k) - 1) % p]
    return sorted(set(vals))


def montgomery_top(p, k):
    """the element whose Montgomery form (x 2^256 mod p, what the kernels multiply) is p - 1 - k: operands like these make
    the largest products, the worst case of a lazy reduction"""
    return (p - 1 - k) * pow(1 << 256, -1, p) % p


def uniform_ints(rng, p, count):
    """`count` integers uniform over all of [0, p) (rejection sampling on bit_length(p) random bits)"""
    mask = (1 << p.bit_length()) - 1
    out = []
    while len(out) < count:
        raw = rng.integers(0, 256, size=(2 * (count - len(out)) + 8, 32), dtype=np.uint8)
        out += [x for x in (int.from_bytes(r.tobytes(), "little") & mask for r in raw) if x < p]
    return out[:count]


def random_elements(field_id, count, seed, shape="uniform"):
    """uint8 array of `count` canonical elements.
    uniform: uniform in [0, 2^(bits-1)) -- below p, so it never produces the top of the field ([2^(bits-1), p) is a
    third of BN254 Fr / Fq); the "edge" shape covers it.  lem: even positions are tags (u16), odd "uniform".
    witness: 40% in {0,1}, 10% < 2^16, 50% "uniform" (SURVEY.md 8(d) config 3 (ii)).
    edge: shuffled quarters: edge_values() in turn, uniform in [2^(bits-1), p), elements whose Montgomery form lies in the
    top sixteenth of [0, p), uniform over all of [0, p)."""
    p = spec.FIELD_MODULUS[field_id]
    rng = np.random.default_rng(seed)
    if shape == "edge":
        bits = p.bit_length()
        fixed = [edge_values(field_id)[i] for i in rng.permutation(len(edge_values(field_id)))]
        vals = [fixed[i % len(fixed)] for i in range(min(count, max(len(fixed), count // 4)))]
        half = 1 << (bits - 1)
        rest = count - len(vals)
        vals += [half + x for x in uniform_ints(rng, p - half, rest // 3)]
        vals += [montgomery_top(p, k) for k in uniform_ints(rng, p >> 4, rest // 3)]
        vals += uniform_ints(rng, p, count - len(vals))
        return pack([vals[i] for i in rng.permutation(count)]) if count else np.zeros(0, dtype=np.uint8)
    raw = rng.integers(0, 256, size=(count, 32), dtype=np.uint8)
    top_bits = p.bit_length() - 248
    raw[:, 31] &= (1 << (top_bits - 1)) - 1          # < 2^(bits-1) < p: uniform enough, always reduced
    if shape == "lem":
        tags = rng.integers(0, 0x3014, size=count).astype(np.uint16)
        even = np.arange(count) % 2 == 0
        raw[even] = 0
        raw[even, 0] = (tags[even] & 0xff).astype(np.uint8)
        raw[even, 1] = (tags[even] >> 8).astype(np.uint8)
    elif shape == "witness":
        u = rng.random(count)
        small = u < 0.4
        raw[small] = 0
        raw[small, 0] = rng.integers(0, 2, size=int(small.sum()), dtype=np.uint8)
        mid = (u >= 0.4) & (u < 0.5)
        raw[mid, 2:] = 0
    elif shape != "uniform":
        raise ValueError(shape)
    return raw.reshape(-1)


def ints(buf):
    b = np.ascontiguousarray(buf, dtype=np.uint8).tobytes()
    return [int.from_bytes(b[i:i + 32], "little") for i in range(0, len(b), 32)]


def pack(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint8).copy()
