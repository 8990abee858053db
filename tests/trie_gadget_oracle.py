"""ORACLE (test infrastructure, NOT product code): from-spec restatement of the witness of the trie coprocessor's lookup and
insert circuits (reference src/coprocessor/trie/mod.rs: synthesize_lookup_aux 118-156, synthesize_insert_aux 226-268,
synthesize_path 611-629, synthesize_lookup_at_path 668-714, synthesize_modify_value_at_path 846-880; gadgets
src/circuit/gadgets/constraints.rs: select / pick 334-391, implies_equal 681-691, enforce_equal 14-30).

One call allocates, in order (arity 8, height H, D = the field's bit-decomposition slot block):
  * allocated_root_value; implies_equal(not_dummy, root, allocated_root) enforces not_dummy * (root - allocated) = 0
    (enforce_implication_lc_zero) and allocates nothing;
  * the D - 1 aux of key.to_bits_le_strict (restated in sha256_gadget_oracle.py, values from oracle/spec.py); the bits
    are padded with Constant(false) to 255, and level L uses bits 3(H-1-L) .. +2, little-endian within the level;
  * per level L = 0..H-1: the 8 preimage elements, the arity-8 Poseidon witness (oracle/spec.py: slot_witness, Neptune's
    optimised schedule: per S-box x^2, x^4, x^5 + post-key, then the digest), `hashed == next` (digest * 1 = the root or
    the previous level's last pick), and select's 7 picks, most significant bit first, each
    (b - a) * bit = b - c with c = bit ? a : b, a = state[half + j], b = state[j];
  * insert only, per level L = H-1 down to 0: the 8 new preimage elements and their Poseidon witness.  Nothing ties the
    new preimages to the old path or to the value: the reference constrains them only through their hashes.
The Poseidon relations are written over the state's linear combinations of earlier aux, as the optimised schedule
forms them, and the digest as (its linear combination) * 1 = digest.  The Poseidon aux order and to_bits_le_strict's
order are pinned by nothing in the reference (as for the slot blocks); digests and preimages are pinned by G1-G5 and G10.

Root, key, value and not_dummy are inputs of the call (glue columns of the step)."""
import os
import sys

import sha256_gadget_oracle as SG

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import spec  # noqa: E402

LOOKUP, INSERT = 0, 1
ARITY, PICKS = 8, 7
KEY_BITS = 255                    # 3 x 85


def n_inputs(op, height):
    return 3 + 16 * height if op == INSERT else 2 + 8 * height


def slot_len(field):
    return ARITY + len(spec.hash_optimised(field, [0] * ARITY, True)[1]) + 1


def bitdecomp_len(field):
    return len(spec.bitdecomp_witness(field, 0)[0])


def block_len(field, op, height):
    D, S = bitdecomp_len(field), slot_len(field)
    return D + (S + PICKS) * height + (S * height if op == INSERT else 0)


def level_at(field, height, level, new=False):
    """block index of the first element (the preimage) of a level's slot block"""
    D, S = bitdecomp_len(field), slot_len(field)
    if not new:
        return D + (S + PICKS) * level
    return D + (S + PICKS) * height + S * (height - 1 - level)


def path_index(key, height, level):
    return (int(key) >> (3 * (height - 1 - level))) & 7


# ---------------------------------------------------------------------------------------------- witness
def witness(field, op, inputs):
    """the aux block of one call: inputs = lookup_inputs / insert_inputs (ints < p)"""
    p = spec.FIELD_MODULUS[field]
    first = 3 if op == INSERT else 2
    height = (len(inputs) - first) // (16 if op == INSERT else 8)
    assert len(inputs) == n_inputs(op, height)
    root, key = int(inputs[0]) % p, int(inputs[1]) % p
    block = [root] + spec.bitdecomp_witness(field, key)[0][1:]
    for L in range(height):
        pre = [int(x) % p for x in inputs[first + 8 * L:first + 8 * L + 8]]
        block += spec.slot_witness(field, pre)
        state = pre
        for hi in (2, 1, 0):
            bit = (path_index(key, height, L) >> hi) & 1
            half = len(state) // 2
            state = [state[half + j] if bit else state[j] for j in range(half)]
            block += state
    if op == INSERT:
        for L in reversed(range(height)):
            off = first + 8 * height + 8 * L
            block += spec.slot_witness(field, [int(x) % p for x in inputs[off:off + 8]])
    return block


# ---------------------------------------------------------------------------------------------- constraints
# A row is (A, B, C): lists of (column, coefficient); columns are ("w", block index), ("in", "root" | "key" | "nd") or "u".
_POSEIDON = {}


def _poseidon_rows(field):
    """rows of one arity-8 Poseidon witness over local columns ("p", j) (preimage) and ("a", k) (aux; k = 387 is the
    digest): the optimised schedule run on linear combinations"""
    if field in _POSEIDON:
        return _POSEIDON[field]
    P = spec.params(field, ARITY)
    p, t, rf, rp = P["p"], P["t"], P["rf"], P["rp"]
    c, mds, pre_m, sparse = P["compressed"], P["mds"], P["pre_sparse"], P["sparse"]
    rows, naux = [], [0]

    def lc_add(*terms):                            # terms: (lc, coefficient)
        out = {}
        for lc, k in terms:
            for col, v in lc.items():
                out[col] = (out.get(col, 0) + v * k) % p
        return {col: v for col, v in out.items() if v}

    def new_aux():
        naux[0] += 1
        return ("a", naux[0] - 1)

    def sbox(x, key):
        x2, x4, x5 = new_aux(), new_aux(), new_aux()
        rows.append((x, x, {x2: 1}))
        rows.append(({x2: 1}, {x2: 1}, {x4: 1}))
        rows.append(({x4: 1}, x, lc_add(({x5: 1}, 1), ({"u": 1}, -key))))
        return {x5: 1}

    def vm(s, M):
        return [lc_add(*[(s[i], M[i][j]) for i in range(t)]) for j in range(t)]

    s = [{"u": (P["domain_tag"] + c[0]) % p}] + [lc_add(({("p", j): 1}, 1), ({"u": 1}, c[j + 1])) for j in range(ARITY)]
    k = t
    half = rf // 2
    for r in range(half):
        s = [sbox(s[i], c[k + i]) for i in range(t)]
        k += t
        s = vm(s, pre_m if r == half - 1 else mds)
    for r in range(rp):
        s[0] = sbox(s[0], c[k])
        k += 1
        sp = sparse[r]
        s0 = lc_add(*[(s[i], sp["w_hat"][i]) for i in range(t)])
        s = [s0] + [lc_add((s[j], 1), (s[0], sp["v_rest"][j - 1])) for j in range(1, t)]
    for r in range(half - 1):
        s = [sbox(s[i], c[k + i]) for i in range(t)]
        k += t
        s = vm(s, mds)
    s = [sbox(s[i], 0) for i in range(t)]
    s = vm(s, mds)
    digest = new_aux()
    rows.append((s[1], {"u": 1}, {digest: 1}))
    assert naux[0] == slot_len(field) - ARITY
    _POSEIDON[field] = [tuple(list(lc.items()) for lc in row) for row in rows]
    return _POSEIDON[field]


_ROWS = {}


def rows(field, op, height):
    """(rows, kinds): every constraint the reference enforces on one call, and a name per row"""
    key_ = (field, op, height)
    if key_ in _ROWS:
        return _ROWS[key_]
    p = spec.FIELD_MODULUS[field]
    g = SG._Gadget(p)
    g.alloc(0, ("root",))
    bits = g.to_bits_le_strict(field, 0, 0)
    bits += [SG.C0] * (KEY_BITS - len(bits))
    out, kinds = [], []

    def w(k):
        return ("w", k)

    def bl(b):
        kind, x = b
        assert kind in ("is", "c")
        return [(w(x), 1)] if kind == "is" else ([("u", 1)] if x else [])

    def row(kind, a, b, c):
        out.append((a, b, c))
        kinds.append(kind)

    # implies_equal(not_dummy, root, allocated_root): not_dummy * (root - allocated) = 0
    row("root", [(("in", "nd"), 1)], [(("in", "root"), 1), (w(0), -1)], [])
    # to_bits_le_strict
    for k, r in enumerate(g.rel):
        if r[0] == "bool":
            row("bool", [(w(k), 1)], [("u", 1), (w(k), -1)], [])
        elif r[0] == "cond":
            row("cond", [("u", 1), (w(r[1]), -1), (w(k), -1)], [(w(k), 1)], [])
        elif r[0] == "and":
            row("and", bl(r[1]), bl(r[2]), [(w(k), 1)])
    for r in g.lin:
        row("pack", [(w(k), 1 << i) for i, k in enumerate(r[1])], [("u", 1)], [(("in", "key"), 1)])

    pos = [len(g.aux)]

    def poseidon():
        base = pos[0]
        loc = {**{("p", j): w(base + j) for j in range(ARITY)}, "u": "u"}
        for a, b, c in _poseidon_rows(field):
            m = [[(loc[col] if col in loc else w(base + ARITY + col[1]), v) for col, v in lc] for lc in (a, b, c)]
            row("poseidon", *m)
        pos[0] += slot_len(field)
        return base

    nxt = w(0)
    for L in range(height):
        base = poseidon()
        row("hashed == next", [(w(base + slot_len(field) - 1), 1)], [("u", 1)], [(nxt, 1)])
        state = [w(base + j) for j in range(ARITY)]
        chunk = bits[3 * (height - 1 - L):3 * (height - 1 - L) + 3]
        for bit in reversed(chunk):
            half = len(state) // 2
            new = []
            for j in range(half):
                c = w(pos[0])
                pos[0] += 1
                a_, b_ = state[half + j], state[j]
                row("pick", [(b_, 1), (a_, -1)], bl(bit), [(b_, 1), (c, -1)])
                new.append(c)
            state = new
        nxt = state[0]
    if op == INSERT:
        for _ in range(height):
            poseidon()
    assert pos[0] == block_len(field, op, height)
    _ROWS[key_] = (out, kinds)
    return _ROWS[key_]


def _lc_val(lc, z, p):
    return sum(z[col] * v for col, v in lc) % p


def check(field, op, block, inputs, not_dummy=1):
    """evaluate every constraint on the block; returns the violated rows as (row, kind) (empty = ok)"""
    p = spec.FIELD_MODULUS[field]
    first = 3 if op == INSERT else 2
    height = (len(inputs) - first) // (16 if op == INSERT else 8)
    rs, kinds = rows(field, op, height)
    if len(block) != block_len(field, op, height):
        return [(-1, "length")]
    z = {("w", k): int(v) % p for k, v in enumerate(block)}
    z.update({("in", "root"): int(inputs[0]) % p, ("in", "key"): int(inputs[1]) % p, ("in", "nd"): not_dummy, "u": 1})
    bad = []
    for i, (a, b, c) in enumerate(rs):
        if (_lc_val(a, z, p) * _lc_val(b, z, p) - _lc_val(c, z, p)) % p:
            bad.append((i, kinds[i]))
    return bad


def r1cs_rows(field, op, height, aux_col, root_col, key_col, nd_col, u_col):
    """the constraints as R1CS rows over z = (W, u, X): block element k is column aux_col + k, the call's root, key
    and not_dummy are columns root_col, key_col, nd_col; constants multiply u_col.  Returns (A, B, C), each a list of
    [(column, canonical coefficient)] per row."""
    p = spec.FIELD_MODULUS[field]
    cols = {("in", "root"): root_col, ("in", "key"): key_col, ("in", "nd"): nd_col, "u": u_col}
    rs, _ = rows(field, op, height)
    mats = ([], [], [])

    def col(c):
        return aux_col + c[1] if c[0] == "w" else cols[c]

    for r in rs:
        for m, lc in zip(mats, r):
            acc = {}
            for c, v in lc:
                acc[col(c)] = (acc.get(col(c), 0) + v) % p
            m.append([(c, v) for c, v in acc.items() if v])
    return mats


# ---------------------------------------------------------------------------------------------- a trie to draw calls from
class SpecTrie:
    """the reference's Trie (mod.rs) over oracle/spec.py's Poseidon: empty roots, path proofs and inserts, giving the
    inputs of lookup and insert calls"""

    def __init__(self, field, height):
        self.field, self.height = field, height
        self.children = {}
        self.empty = [0]
        for _ in range(height):
            self.empty.append(self._register([self.empty[-1]] * ARITY))
        self.root = self.empty[height]

    def _register(self, pre):
        d = spec.hash_optimised(self.field, list(pre))
        self.children[d] = tuple(pre)
        return d

    def proof(self, key):
        out, nxt = [], self.root
        for L in range(self.height):
            pre = self.children[nxt]
            out.append(pre)
            nxt = pre[path_index(key, self.height, L)]
        return out

    def lookup_inputs(self, key):
        return [self.root, key] + [x for pre in self.proof(key) for x in pre]

    def insert_inputs(self, key, value):
        """the call's inputs; the trie holds the value afterwards"""
        old = self.proof(key)
        new, v = [], value
        for L in reversed(range(self.height)):
            pre = list(old[L])
            pre[path_index(key, self.height, L)] = v
            v = self._register(pre)
            new.append(tuple(pre))
        new.reverse()
        ins = [self.root, key, value] + [x for pre in old for x in pre] + [x for pre in new for x in pre]
        self.root = v
        return ins
