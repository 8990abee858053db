"""
ORACLE (test infrastructure, NOT product code) -- from-spec Python restatement.

Pure-Python big-int restatement of the algorithms on the lurk-beta proving hot path.
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this.
It is slow on purpose (small cases only); the C restatement in oracle/oracle.c is the
fast checker and the CPU baseline.  The two are written independently and are checked
against each other and against the reference's golden vectors in tests/.

What it restates, with the reference call sites it follows:
  * Poseidon (Neptune `PoseidonConstants::new()` = Strength::Standard, HashType::MerkleTree)
      - reference call sites: src/hash.rs:61-72 (constants), src/hash.rs:180-203 (hashN)
      - neptune is a git dependency (argumentcomputer/neptune, branch dev; not in tree, no
        Cargo.lock).  Published algorithm restated here; pinned by the reference's own golden
        digests (SURVEY.md 8(c) G1..G11 plus G13..G27 from documented REPL examples and demo scripts,
        tests/golden/reference_goldens.json; src/coprocessor/trie/mod.rs:932-1010,
        src/lem/store.rs:1473, src/lem/tests/eval_tests.rs:1944,1955,3868).
  * Poseidon *witness* in Neptune's optimised-round order (src/lem/circuit.rs:212-247 call site)
      - aux count pinned by src/lem/multiframe.rs:991-1016 / store.rs:286-306; aux ORDER unpinned.
  * bit-decomposition slot witness (bellpepper-core 0.4 `AllocatedNum::to_bits_le_strict`,
    call site src/lem/circuit.rs:241-243) -- sizes pinned by src/lem/multiframe.rs:495-498.
  * short-Weierstrass a=0 group law + naive MSM (Arecibo `vartime_multiscalar_mul`; call sites
    src/proof/nova.rs:287,292) -- parity unpinned (no golden commitment in tree); group law is
    canonical so any correct MSM agrees after affine normalisation.
  * radix-2 NTT -- parity unpinned (no call site in the reference, SURVEY.md D4).
"""
import math

# ---------------------------------------------------------------- fields / curves
BN254_FR = 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001
BN254_FQ = 0x30644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd47
PALLAS_FP = 0x40000000000000000000000000000000224698fc094cf91b992d30ed00000001  # pallas base
PALLAS_FQ = 0x40000000000000000000000000000000224698fc0994a8dd8c46eb2100000001  # pallas scalar

# field ids follow include/lurk_b200.h
FIELD_MODULUS = {0: BN254_FR, 1: BN254_FQ, 2: PALLAS_FQ, 3: PALLAS_FP}
FIELD_NAME = {0: "bn254_fr", 1: "bn254_fq", 2: "pallas_fq", 3: "pallas_fp"}
FIELD_NUM_BITS = {0: 254, 1: 254, 2: 255, 3: 255}

# curve ids: (base field id, scalar field id, b, generator)
CURVES = {
    0: dict(name="bn254_g1", base=1, scalar=0, b=3, gen=(1, 2)),
    1: dict(name="grumpkin", base=0, scalar=1, b=BN254_FR - 17, gen=(1, 0x0000000000000002cf135e7506a45d632d270d45f1181294833fc48d823f272c)),
    2: dict(name="pallas", base=3, scalar=2, b=5, gen=(PALLAS_FP - 1, 2)),
    3: dict(name="vesta", base=2, scalar=3, b=5, gen=(PALLAS_FQ - 1, 2)),
}


# ---------------------------------------------------------------- Poseidon parameters
def round_numbers(t):
    """Neptune calc_round_numbers(t, security_margin=True): n=255, M=128 hard-coded."""
    n, M = 255.0, 128.0

    def secure(t, rf, rp):
        c = 6.0 if M <= (n - 3.0) * (t + 1.0) else 10.0
        rf_stat = c
        rf_interp = 0.43 * M + math.log2(t) - rp
        rf_grob1 = 0.21 * n - rp
        rf_grob2 = (0.14 * n - 1.0 - rp) / (t - 1.0)
        rf_max = max(math.ceil(rf_stat), math.ceil(rf_interp), math.ceil(rf_grob1), math.ceil(rf_grob2))
        return rf >= rf_max

    best = None
    for rp in range(1, 200):
        for rf in range(4, 101, 2):
            if secure(t, rf, rp):
                rf2 = rf + 2
                rp2 = math.ceil(1.075 * rp)
                cost = t * rf2 + rp2
                if best is None or cost < best[0] or (cost == best[0] and rf2 < best[1]):
                    best = (cost, rf2, rp2)
    return best[1], best[2]


class Grain:
    """Poseidon reference Grain LFSR as Neptune seeds it (sbox field = 1)."""

    def __init__(self, nbits, t, rf, rp):
        bits = []

        def push(v, n):
            for i in reversed(range(n)):
                bits.append((v >> i) & 1)

        push(1, 2)      # prime field
        push(1, 4)      # sbox id as Neptune writes it
        push(nbits, 12)
        push(t, 12)
        push(rf, 10)
        push(rp, 10)
        push((1 << 30) - 1, 30)
        assert len(bits) == 80
        self.s = bits
        for _ in range(160):
            self._next()

    def _next(self):
        s = self.s
        b = s[62] ^ s[51] ^ s[38] ^ s[23] ^ s[13] ^ s[0]
        s.pop(0)
        s.append(b)
        return b

    def bit(self):
        while True:
            a = self._next()
            b = self._next()
            if a:
                return b

    def elem(self, nbits, p):
        while True:
            v = 0
            for _ in range(nbits):
                v = (v << 1) | self.bit()
            if v < p:
                return v


def mat_mul(A, B, p):
    n, m, k = len(A), len(B[0]), len(B)
    return [[sum(A[i][x] * B[x][j] for x in range(k)) % p for j in range(m)] for i in range(n)]


def mat_inv(A, p):
    n = len(A)
    M = [row[:] + [1 if i == j else 0 for j in range(n)] for i, row in enumerate(A)]
    for c in range(n):
        piv = next(r for r in range(c, n) if M[r][c] % p)
        M[c], M[piv] = M[piv], M[c]
        inv = pow(M[c][c], p - 2, p)
        M[c] = [v * inv % p for v in M[c]]
        for r in range(n):
            if r != c and M[r][c]:
                f = M[r][c]
                M[r] = [(a - f * b) % p for a, b in zip(M[r], M[c])]
    return [row[n:] for row in M]


def vec_mat(v, M, p):
    """row vector times matrix (Neptune's convention: state <- state * M)."""
    t = len(v)
    return [sum(v[i] * M[i][j] for i in range(t)) % p for j in range(t)]


_PARAM_CACHE = {}


def params(field_id, arity):
    key = (field_id, arity)
    if key in _PARAM_CACHE:
        return _PARAM_CACHE[key]
    p = FIELD_MODULUS[field_id]
    t = arity + 1
    rf, rp = round_numbers(t)
    g = Grain(FIELD_NUM_BITS[field_id], t, rf, rp)
    rc = [g.elem(FIELD_NUM_BITS[field_id], p) for _ in range(t * (rf + rp))]
    mds = [[pow(i + t + j, p - 2, p) for j in range(t)] for i in range(t)]
    P = dict(p=p, t=t, arity=arity, rf=rf, rp=rp, rc=rc, mds=mds, domain_tag=(1 << arity) - 1)
    _optimise(P)
    _PARAM_CACHE[key] = P
    return P


def _optimise(P):
    """Neptune's optimised constants: compressed round keys, pre-sparse matrix, sparse factors."""
    p, t, rf, rp, rc, mds = P["p"], P["t"], P["rf"], P["rp"], P["rc"], P["mds"]
    half = rf // 2
    minv = mat_inv(mds, p)
    rnd = lambda r: rc[r * t:(r + 1) * t]

    comp = list(rnd(0))
    for i in range(half - 1):                      # rounds 1..half-1 folded behind the S-box of round i
        comp += vec_mat(rnd(i + 1), minv, p)
    # partial rounds, walked backwards
    acc = list(rnd(half + rp))                     # keys of the first full round after the partials
    partial_keys = []
    for i in range(rp):
        inv = vec_mat(acc, minv, p)
        partial_keys.append(inv[0])
        inv[0] = 0
        acc = [(a + b) % p for a, b in zip(rnd(half + rp - 1 - i), inv)]
    comp += vec_mat(acc, minv, p)                  # post-key of the last first-half full round
    comp += list(reversed(partial_keys))
    for i in range(1, half):
        comp += vec_mat(rnd(half + rp + i), minv, p)
    assert len(comp) == t * rf + rp
    P["compressed"] = comp

    # sparse factorisation  M = M' * M''
    cur = [row[:] for row in mds]
    sparse = []
    for _ in range(rp):
        hat = [row[1:] for row in cur[1:]]
        hat_inv = mat_inv(hat, p)
        w = [[cur[i][0]] for i in range(1, t)]
        w_hat = mat_mul(hat_inv, w, p)             # column
        m_prime = [[1] + [0] * (t - 1)] + [[0] + hat[i] for i in range(t - 1)]
        # M'' : first row = cur[0], first column below = w_hat, identity elsewhere
        sparse.append(dict(w_hat=[cur[0][0]] + [w_hat[i][0] for i in range(t - 1)], v_rest=cur[0][1:]))
        cur = mat_mul(mds, m_prime, p)
    P["pre_sparse"] = cur
    P["sparse"] = list(reversed(sparse))


# ---------------------------------------------------------------- Poseidon permutations
def hash_correct(field_id, preimage):
    """Textbook Poseidon: ARK, S-box, MDS per round; digest = state[1]."""
    P = params(field_id, len(preimage))
    p, t, rf, rp, rc, mds = P["p"], P["t"], P["rf"], P["rp"], P["rc"], P["mds"]
    s = [P["domain_tag"]] + [x % p for x in preimage]
    half = rf // 2
    for r in range(rf + rp):
        s = [(a + b) % p for a, b in zip(s, rc[r * t:(r + 1) * t])]
        if r < half or r >= half + rp:
            s = [pow(x, 5, p) for x in s]
        else:
            s[0] = pow(s[0], 5, p)
        s = vec_mat(s, mds, p)
    return s[1]


def hash_optimised(field_id, preimage, want_aux=False):
    """Neptune hash_optimized_static order.  Returns digest, or (digest, aux) where aux is the
    witness the circuit allocates per S-box: x^2, x^4, x^5 + post-key."""
    P = params(field_id, len(preimage))
    p, t, rf, rp = P["p"], P["t"], P["rf"], P["rp"]
    c, mds, pre, sparse = P["compressed"], P["mds"], P["pre_sparse"], P["sparse"]
    half = rf // 2
    aux = []
    s = [P["domain_tag"]] + [x % p for x in preimage]
    s = [(a + b) % p for a, b in zip(s, c[:t])]
    k = t

    def sbox(x, key):
        x2 = x * x % p
        x4 = x2 * x2 % p
        x5 = (x4 * x + key) % p
        aux.extend((x2, x4, x5))
        return x5

    for r in range(half):
        s = [sbox(s[i], c[k + i]) for i in range(t)]
        k += t
        s = vec_mat(s, pre if r == half - 1 else mds, p)
    for r in range(rp):
        s[0] = sbox(s[0], c[k])
        k += 1
        sp = sparse[r]
        s0 = sum(a * b for a, b in zip(s, sp["w_hat"])) % p
        s = [s0] + [(s[j] + s[0] * sp["v_rest"][j - 1]) % p for j in range(1, t)]
    for r in range(half - 1):
        s = [sbox(s[i], c[k + i]) for i in range(t)]
        k += t
        s = vec_mat(s, mds, p)
    s = [sbox(s[i], 0) for i in range(t)]
    s = vec_mat(s, mds, p)
    assert k == len(c)
    return (s[1], aux) if want_aux else s[1]


def slot_witness(field_id, preimage):
    """Slot block as the reference lays it out (src/lem/circuit.rs:264-299):
    preimage, then Poseidon aux, then digest."""
    d, aux = hash_optimised(field_id, preimage, True)
    return [x % FIELD_MODULUS[field_id] for x in preimage] + aux + [d]


# ---------------------------------------------------------------- Nova random oracle (Arecibo PoseidonRO)
# Arecibo (git dependency `nova`, branch dev, not in tree) instantiates its RO as neptune's SAFE sponge over
# PoseidonConstants<F, U24> = Sponge::api_constants(Strength::Standard): width 25, simplex mode, IO pattern
# [Absorb(n), Squeeze(1)], the squeezed element truncated to its low `num_bits` bits and re-read in the other
# field of the cycle.  Call sites in the reference: every `prove_step` (src/proof/nova.rs:286-293).  Restated
# from the public crates; no golden challenge exists in the reference => parity unpinned.
RO_RATE = 24


def sponge_io_tag(n_absorb, n_squeeze=1, domain_separator=0):
    """neptune sponge::api::IOPattern::value: polynomial hash in wrapping u128 with base 2^128 - 159"""
    mask = (1 << 128) - 1
    x = (0 - 159) & mask
    x_i, state = 1, 0
    for v in (n_absorb + (1 << 31), n_squeeze, domain_separator):
        x_i = x_i * x & mask
        state = (state + x_i * v) & mask
    return state


def poseidon_permute(field_id, state):
    """textbook permutation of a full state (width len(state)); Neptune constants of that width"""
    t = len(state)
    P = params(field_id, t - 1)
    p, rf, rp, rc, mds = P["p"], P["rf"], P["rp"], P["rc"], P["mds"]
    s = [x % p for x in state]
    half = rf // 2
    for r in range(rf + rp):
        s = [(a + b) % p for a, b in zip(s, rc[r * t:(r + 1) * t])]
        if r < half or r >= half + rp:
            s = [pow(x, 5, p) for x in s]
        else:
            s[0] = pow(s[0], 5, p)
        s = vec_mat(s, mds, p)
    return s


def ro_squeeze(base_field_id, absorbed, num_bits=128):
    """PoseidonRO::squeeze: capacity element = IO tag, absorbed elements in the rate, one permutation, element 1,
    low num_bits bits.  Returns (challenge integer, full squeezed element)."""
    assert 1 <= len(absorbed) <= RO_RATE
    p = FIELD_MODULUS[base_field_id]
    state = [sponge_io_tag(len(absorbed)) % p] + [a % p for a in absorbed] + [0] * (RO_RATE - len(absorbed))
    h = poseidon_permute(base_field_id, state)[1]
    return h & ((1 << num_bits) - 1), h


def nifs_absorb_list(pp_digest, comm_W2, X2, comm_T):
    """what Arecibo's NIFS::prove absorbs: pp digest, U2 = (comm_W, X), comm_T; points as (x, y, is_infinity)"""
    def pt(P):
        return [0, 0, 1] if P is None else [P[0], P[1], 0]
    return [pp_digest] + pt(comm_W2) + list(X2) + pt(comm_T)


# ---------------------------------------------------------------- bit decomposition slot
def bitdecomp_witness(field_id, x):
    """bellpepper-core AllocatedNum::to_bits_le_strict aux allocation order, preceded by the
    preimage element the slot allocates first (src/lem/circuit.rs:294-305).
    Returns (aux list, bits little-endian)."""
    p = FIELD_MODULUS[field_id]
    x %= p
    aux = [x]
    b = p - 1
    result = []
    last_run = None
    current_run = []
    found_one = False
    for i in reversed(range(256)):
        b_bit = (b >> i) & 1
        a_bit = (x >> i) & 1
        found_one |= bool(b_bit)
        if not found_one:
            assert a_bit == 0
            continue
        if b_bit:
            aux.append(a_bit)
            current_run.append(a_bit)
            result.append(a_bit)
        else:
            if current_run:
                if last_run is not None:
                    current_run.append(last_run)
                cur = current_run[0]
                for v in current_run[1:]:
                    cur = cur & v
                    aux.append(cur)          # AllocatedBit::and allocates its result
                last_run = cur
                current_run = []
            aux.append(a_bit)               # alloc_conditionally
            result.append(a_bit)
    assert not current_run
    return aux, list(reversed(result))


# ---------------------------------------------------------------- curves
def ec_add(P, Q, p):
    if P is None:
        return Q
    if Q is None:
        return P
    x1, y1 = P
    x2, y2 = Q
    if x1 == x2:
        if (y1 + y2) % p == 0:
            return None
        l = 3 * x1 * x1 * pow(2 * y1, p - 2, p) % p
    else:
        l = (y2 - y1) * pow(x2 - x1, p - 2, p) % p
    x3 = (l * l - x1 - x2) % p
    return x3, (l * (x1 - x3) - y1) % p


def ec_mul(k, P, p):
    """k P on y^2 = x^3 + b (a = 0): double-and-add in Jacobian coordinates, one inversion at the end"""
    if P is None or k == 0:
        return None
    x2, y2 = P
    X, Y, Z = 1, 1, 0                       # the identity
    for bit in bin(k)[2:]:
        if Z:                               # doubling (dbl-2009-l)
            A, B = X * X % p, Y * Y % p
            C = B * B % p
            D = 2 * ((X + B) ** 2 - A - C) % p
            E = 3 * A % p
            X3 = (E * E - 2 * D) % p
            Y, Z = (E * (D - X3) - 8 * C) % p, 2 * Y * Z % p
            X = X3
        if bit == "1":                      # mixed addition of the affine P (madd-2007-bl), with its special cases
            if not Z:
                X, Y, Z = x2, y2, 1
                continue
            Z2 = Z * Z % p
            U2, S2 = x2 * Z2 % p, y2 * Z * Z2 % p
            H, rr = (U2 - X) % p, (S2 - Y) % p
            if H == 0:
                if rr:
                    X, Y, Z = 1, 1, 0
                    continue
                A, B = X * X % p, Y * Y % p          # P + P: double
                C = B * B % p
                D = 2 * ((X + B) ** 2 - A - C) % p
                E = 3 * A % p
                X3 = (E * E - 2 * D) % p
                Y, Z = (E * (D - X3) - 8 * C) % p, 2 * Y * Z % p
                X = X3
                continue
            HH = H * H % p
            HHH = H * HH % p
            V = X * HH % p
            X3 = (rr * rr - HHH - 2 * V) % p
            Y, Z = (rr * (V - X3) - Y * HHH) % p, Z * H % p
            X = X3
    if not Z:
        return None
    zi = pow(Z, -1, p)
    zi2 = zi * zi % p
    return X * zi2 % p, Y * zi2 * zi % p


def msm_naive(curve_id, bases, scalars):
    """bases: list of (x,y) or None; scalars: ints.  Returns affine point or None."""
    C = CURVES[curve_id]
    p = FIELD_MODULUS[C["base"]]
    acc = None
    for P, k in zip(bases, scalars):
        if P is None or P == (0, 0):
            continue
        acc = ec_add(acc, ec_mul(k % FIELD_MODULUS[C["scalar"]], P, p), p)
    return acc


def on_curve(curve_id, P):
    C = CURVES[curve_id]
    p = FIELD_MODULUS[C["base"]]
    x, y = P
    return (y * y - x * x * x - C["b"]) % p == 0


# ---------------------------------------------------------------- NTT
TWO_ADICITY = {0: 28, 1: 1, 2: 32, 3: 32}
# multiplicative generators of the reference's field types (ff::PrimeField::MULTIPLICATIVE_GENERATOR): halo2curves bn256::Fr 7,
# bn256::Fq 3, pasta_curves Fp / Fq 5 -- so that 2^s-th roots equal their ROOT_OF_UNITY (checked in tests/test_oracle_golden.py)
MULT_GEN = {0: 7, 1: 3, 2: 5, 3: 5}


def root_of_unity(field_id, log_n):
    p = FIELD_MODULUS[field_id]
    s = TWO_ADICITY[field_id]
    assert log_n <= s
    w = pow(MULT_GEN[field_id], (p - 1) >> s, p)
    return pow(w, 1 << (s - log_n), p)


def ntt_naive(field_id, a, inverse=False):
    """O(n^2) DFT: out[k] = sum_j a[j] w^(jk), natural order in and out."""
    p = FIELD_MODULUS[field_id]
    n = len(a)
    w = root_of_unity(field_id, n.bit_length() - 1)
    if inverse:
        w = pow(w, p - 2, p)
    out = [sum(a[j] * pow(w, j * k, p) for j in range(n)) % p for k in range(n)]
    if inverse:
        ninv = pow(n, p - 2, p)
        out = [x * ninv % p for x in out]
    return out


# ---------------------------------------------------------------- byte helpers
def fe_to_bytes(x):
    return int(x).to_bytes(32, "little")


def fe_from_bytes(b):
    return int.from_bytes(b, "little")
