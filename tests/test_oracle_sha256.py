"""CPU checks of the SHA-256 coprocessor's witness restatement (tests/sha256_gadget_oracle.py): its packed digest is the
reference's native compute_sha256 over standard SHA-256, its block satisfies every relation bellpepper enforces and a
single flipped aux violates one, and its length per (field, n) is what the library's schedule builds."""
import hashlib
import random

import pytest

import sha256_gadget_oracle as G

FIELDS = [0, 1, 2, 3]
# aux per call, by field id and n = 1..4 (n = 1: about the 45 000 boolean aux bench.py models per sha256_ivc frame)
BLOCK_LEN = {0: [45530, 72396, 99262, 126128], 1: [45550, 72436, 99322, 126208],
             2: [45421, 72178, 98935, 125692], 3: [45427, 72190, 98953, 125716]}


def test_hashlib_is_fips_180_4_sha256():
    # FIPS 180-4 / NIST example vectors: "abc" (one block) and the 448-bit message (two blocks)
    assert hashlib.sha256(b"abc").hexdigest() == "ba7816bf8f01cfea414140de5dae2223b00361a396177a9cb410ff61f20015ad"
    assert hashlib.sha256(b"abcdbcdecdefdefgefghfghighijhijkijkljklmklmnlmnomnopnopq").hexdigest() == \
        "248d6a61d20638b8e5c026930c3e6039a33ce45964ff2167f6ecedd419db06c1"


def _inputs(spec, field, n, kind, rng):
    p = spec.FIELD_MODULUS[field]
    if kind == "zeros":
        return [0] * (2 * n)
    if kind == "top":
        return [p - 1] * (2 * n)
    if kind == "tags":                     # ExprTag values as tags (Nil .. Prov), random hashes
        return [v for j in range(n) for v in (j % 15, rng.randrange(p))]
    return [rng.randrange(p) for _ in range(2 * n)]


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("n", [1, 2, 3, 4])
def test_packed_digest_is_compute_sha256(L, spec, field, n):
    rng = random.Random(field * 10 + n)
    co = L.Sha256Coprocessor(n)
    for kind in ("zeros", "top", "tags", "random"):
        ins = _inputs(spec, field, n, kind, rng)
        block = G.witness(field, ins)
        assert len(block) == BLOCK_LEN[field][n - 1]
        want = G.compute_sha256(field, ins)
        assert block[-2] == want == co.compute_sha256(field, list(zip(ins[0::2], ins[1::2]))), kind
        assert block[-1] == G.TAG_NUM
        assert G.check(field, block, ins) == [], kind


@pytest.mark.parametrize("field", FIELDS)
def test_a_flipped_aux_is_caught(spec, field):
    rng = random.Random(7 + field)
    ins = _inputs(spec, field, 1, "random", rng)
    block = G.witness(field, ins)
    rel, _ = G.relations(field, 1)
    kinds = {}
    for k, r in enumerate(rel):
        kinds.setdefault(r[0], []).append(k)
    picks = [rng.choice(ks) for ks in kinds.values()] + [rng.randrange(len(block)) for _ in range(20)]
    for k in picks:
        bad = list(block)
        bad[k] = (bad[k] ^ 1) if bad[k] in (0, 1) else bad[k] + 1
        assert G.check(field, bad, ins), f"aux {k} ({rel[k][0]}) flipped but every relation holds"


@pytest.mark.parametrize("field", FIELDS)
def test_r1cs_rows_hold_on_the_block(spec, field):
    rng = random.Random(field)
    p = spec.FIELD_MODULUS[field]
    ins = _inputs(spec, field, 1, "random", rng)
    block = G.witness(field, ins)
    z = list(ins) + block + [1]
    A, B, C = G.r1cs_rows(field, 1, len(ins), 0, len(z) - 1)
    dot = lambda r: sum(z[c] * v for c, v in r) % p
    assert all(dot(a) * dot(b) % p == dot(c) for a, b, c in zip(A, B, C))
    z[len(ins) + 1000] ^= 1
    assert not all(dot(a) * dot(b) % p == dot(c) for a, b, c in zip(A, B, C))


@pytest.mark.parametrize("field", FIELDS)
def test_library_block_lengths(L, field):
    assert [L.witness_block(field, n) for n in (1, 2, 3, 4)] == BLOCK_LEN[field]
    assert [G.block_len(field, n) for n in (1, 2, 3, 4)] == BLOCK_LEN[field]
