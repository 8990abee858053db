"""CPU checks of the trie coprocessor's witness restatement (tests/trie_gadget_oracle.py): the digests it writes are the
reference's goldens (G1-G5 on an empty StandardTrie lookup, G10 after inserting 123 -> 456), its blocks satisfy every
constraint the reference enforces and a flipped pick, bit or Poseidon aux violates one, and its block lengths are
D + 403 H (lookup) and D + 799 H (insert)."""
import json
import os
import random

import pytest

import trie_gadget_oracle as T

FIELDS = [0, 1, 2, 3]
D = {0: 354, 1: 364, 2: 298, 3: 301}     # the reference's lurk_bitdecomp_witness_block (multiframe.rs:495-498)
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_goldens.json")))["poseidon_digests"]


def _g(name):
    return int(GOLD[name]["hex"], 16)


def _digest(block, field, height, level, new=False):
    return block[T.level_at(field, height, level, new) + T.slot_len(field) - 1]


def test_standard_trie_goldens():
    field, H = 0, 85
    t = T.SpecTrie(field, H)
    ins = t.lookup_inputs(123)
    block = T.witness(field, T.LOOKUP, ins)
    for level, g in ((84, "G1"), (83, "G2"), (82, "G3"), (81, "G4"), (0, "G5")):
        assert _digest(block, field, H, level) == _g(g), g
    assert block[0] == _g("G5") and block[-1] == 0            # the empty trie holds 0 at every key
    ins = t.insert_inputs(123, 456)
    block = T.witness(field, T.INSERT, ins)
    assert block[-1] == _g("G10") == t.root
    assert _digest(block, field, H, 0, new=True) == _g("G10")
    assert T.check(field, T.INSERT, block, ins) == []
    ins = t.lookup_inputs(123)
    block = T.witness(field, T.LOOKUP, ins)
    assert block[0] == _g("G10") and block[-1] == 456
    assert T.check(field, T.LOOKUP, block, ins) == []


def _calls(field, op, H, rng, n=3):
    p = T.spec.FIELD_MODULUS[field]
    t = T.SpecTrie(field, H)
    keys = [rng.randrange(p) for _ in range(4)]
    for k in keys[:2]:
        t.insert_inputs(k, rng.randrange(p))
    out = []
    for i in range(n):
        k = keys[i % len(keys)]
        out.append(t.insert_inputs(k, rng.randrange(p)) if op == T.INSERT else t.lookup_inputs(k))
    return out


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("op", [T.LOOKUP, T.INSERT])
@pytest.mark.parametrize("H", [1, 2, 3, 85])
def test_relations_hold_and_catch_flips(field, op, H):
    rng = random.Random(1000 * field + 10 * H + op)
    p = T.spec.FIELD_MODULUS[field]
    assert T.block_len(field, op, H) == D[field] + (799 if op == T.INSERT else 403) * H
    ins = _calls(field, op, H, rng, n=1 if H == 85 else 3)
    for x in ins:
        block = T.witness(field, op, x)
        assert len(block) == T.block_len(field, op, H)
        assert T.check(field, op, block, x) == []
        assert T.check(field, op, block, x, not_dummy=0) == []
    x = ins[0]
    block = T.witness(field, op, x)
    S = T.slot_len(field)
    L = rng.randrange(H)
    base = T.level_at(field, H, L)
    flips = {"pick": base + S + rng.randrange(T.PICKS), "bit": 1 + rng.randrange(D[field] - 1),
             "poseidon aux": base + T.ARITY + rng.randrange(S - T.ARITY), "root": 0}
    if op == T.INSERT:
        flips["new poseidon aux"] = T.level_at(field, H, L, new=True) + T.ARITY + rng.randrange(S - T.ARITY)
    for what, k in flips.items():
        bad = list(block)
        bad[k] = (bad[k] + 1) % p
        assert T.check(field, op, bad, x), f"{what} (element {k}) flipped but every constraint holds"
    # implies_equal: a wrong supplied root is caught only when not_dummy is set
    wrong = [x[0] + 1] + list(x[1:])
    assert T.check(field, op, block, wrong) and not T.check(field, op, block, wrong, not_dummy=0)


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("op", [T.LOOKUP, T.INSERT])
def test_r1cs_rows_hold_on_the_block(spec, field, op):
    rng = random.Random(field + 7 * op)
    p = spec.FIELD_MODULUS[field]
    H = 2
    x = _calls(field, op, H, rng, n=1)[0]
    block = T.witness(field, op, x)
    z = [x[0], x[1], 1] + block + [1]                       # root, key, not_dummy, block, u
    A, B, C = T.r1cs_rows(field, op, H, 3, 0, 1, 2, len(z) - 1)
    dot = lambda r: sum(z[c] * v for c, v in r) % p        # noqa: E731
    ok = lambda: all(dot(a) * dot(b) % p == dot(c) for a, b, c in zip(A, B, C))   # noqa: E731
    assert len(A) == len(T.rows(field, op, H)[0]) and ok()
    z[3 + T.level_at(field, H, 1) + T.slot_len(field)] += 1   # the first pick of level 1
    assert not ok()


def test_nothing_ties_the_new_path_to_the_value():
    """the reference constrains the new preimages only through their hashes: a block over a new path that does not hold
    the value still satisfies every constraint"""
    field, H = 0, 2
    t = T.SpecTrie(field, H)
    x = t.insert_inputs(5, 77)
    y = list(x)
    first_new = 3 + 8 * H
    y[first_new + 8 * (H - 1) + T.path_index(5, H, H - 1)] = 78
    assert T.check(field, T.INSERT, T.witness(field, T.INSERT, y), y) == []
