"""
ORACLE (test infrastructure, NOT product code) -- commitment-key generation (SURVEY.md 8(f) N3).

Restates what `public_params` (reference src/proof/nova.rs:196-216, supernova.rs:117-137) makes Arecibo do to obtain the
Pedersen commitment key: `R1CSShape::commitment_key` -> `CommitmentKey::setup(b"ck", n)` with
n = next_power_of_two(max(#constraints, #variables, ck_floor)) -> `DlogGroup::from_label(label, n)`:

    reader = SHAKE256(label).xof();  uniform_i = next 32 bytes of the stream, i = 0..n-1        (sequential)
    G_i = Curve::hash_to_curve("from_uniform_bytes")(uniform_i)  -> affine                     (independent per i)

Arecibo (git, branch dev), halo2curves 0.6.0 and pasta_curves 0.5.0 are NOT under the reference checkout (Cargo.toml:42,68,70-73);
this file restates their published algorithms:
  * hash_to_field: expand_message_xmd (RFC 9380 5.3.1) with BLAKE2b-512 (hash_length 64, empty personalisation),
    len_in_bytes 128, DST = domain_prefix || "-" || curve_id || "_XMD:BLAKE2b_" || method || "_RO_"; each 64-byte half is
    read big-endian and reduced mod p (both crates: reverse the bytes, `from_uniform_bytes` little-endian).
  * BN254 G1 / Grumpkin (halo2curves `svdw_hash_to_curve`): Shallue-van de Woestijne map, RFC 9380 6.6.1 / F.1, Z = 1 (what RFC
    9380 H.1 `find_z_svdw` returns for both curves; checked below), curve ids "bn256_g1" / "grumpkin_g1", method "SVDW".
  * Pallas / Vesta (pasta_curves `hashtocurve.rs`): simplified SWU (RFC 9380 6.6.2) onto the 3-isogenous curves iso-Pallas /
    iso-Vesta (Zcash protocol spec 5.4.9.8: b = 1265, Z = -13), the two points added there, then the isogeny; curve ids
    "pallas" / "vesta", method "SSWU".
    The 13 isogeny constants are DERIVED here (Velu's formulas for the unique rational order-3 subgroup, composed with the
    isomorphism (x, y) -> (x/9, y/27) onto y^2 = x^3 + 5) instead of being typed in; for Pallas the result equals the published
    pasta_curves ISOGENY_CONSTANTS (first: 0x0e38e38e...aaaaaaab = 1/9, last: p - 540).  iso-curve coefficients `a` are checked by
    the group order (an isogenous curve has the same number of points).

Parity: the Pasta hash_to_curve is PINNED by pasta_curves' own unit-test vectors (tests/golden/pasta_hash_to_curve_vectors.json: this file
reproduces hash_to_curve("z.cash:test") of "Trans rights now!" on Pallas and of "hello" on Vesta); the SVDW curves (halo2curves has property
tests only) and the way Arecibo feeds the SHAKE256 stream into it are UNPINNED against Arecibo's actual key (no golden point of the key exists in
the reference; SURVEY.md 8(c)).
Pinned pieces: SHAKE256 and BLAKE2b are Python's hashlib (the CUDA/C++ side has its own implementations, compared with these);
the group-order and on-curve checks; the isogeny constants.  tests/test_oracle_h2c.py holds those checks.

Only tests/, __graft_entry__.smoke() and the cpu_baseline legs (bench.py; the CPU-timing legs of tools/config_benches.py and
tools/compress_cpu_baseline.py, where the oracle is the thing timed BESIDE the product, never a checker inside it) may import this file.
"""
import hashlib

from . import spec

# curve ids follow include/lurk_b200.h
CURVE_H2C_ID = {0: "bn256_g1", 1: "grumpkin_g1", 2: "pallas", 3: "vesta"}
CURVE_H2C_METHOD = {0: "SVDW", 1: "SVDW", 2: "SSWU", 3: "SSWU"}
ISO_A = {
    2: 0x18354a2eb0ea8c9c49be2d7258370742b74134581a27a59f92bb4b0b657a014b,   # iso-Pallas
    3: 0x267f9b2ee592271a81639c4d96f787739673928c7d01b212c515ad7242eaa6b1,   # iso-Vesta
}
ISO_B = 1265
SSWU_Z = -13
SVDW_Z = 1


def base_modulus(curve_id):
    return spec.FIELD_MODULUS[spec.CURVES[curve_id]["base"]]


def curve_b(curve_id):
    return spec.CURVES[curve_id]["b"] % base_modulus(curve_id)


# ------------------------------------------------------------------------------------------------ field helpers
def sgn0(x):
    return x & 1


def is_square(x, p):
    return x == 0 or pow(x, (p - 1) // 2, p) == 1


def sqrt(x, p):
    """some square root of a square x (Tonelli-Shanks); callers fix the sign themselves"""
    if x == 0:
        return 0
    assert pow(x, (p - 1) // 2, p) == 1
    s, t = 0, p - 1
    while t % 2 == 0:
        s, t = s + 1, t // 2
    z = 2
    while pow(z, (p - 1) // 2, p) != p - 1:
        z += 1
    c, r, tt, m = pow(z, t, p), pow(x, (t + 1) // 2, p), pow(x, t, p), s
    while tt != 1:
        i, x2 = 0, tt
        while x2 != 1:
            x2, i = x2 * x2 % p, i + 1
        b = pow(c, 1 << (m - i - 1), p)
        r, c = r * b % p, b * b % p
        tt, m = tt * c % p, i
    assert r * r % p == x
    return r


def inv0(x, p):
    return pow(x, p - 2, p)


# ------------------------------------------------------------------------------------------------ hash_to_field
def dst_prime(curve_id, domain_prefix):
    dst = domain_prefix.encode() + b"-" + CURVE_H2C_ID[curve_id].encode() + b"_XMD:BLAKE2b_" + \
        CURVE_H2C_METHOD[curve_id].encode() + b"_RO_"
    assert len(dst) < 256
    return dst + bytes([len(dst)])


def hash_to_field(curve_id, domain_prefix, message):
    """two base-field elements; expand_message_xmd with BLAKE2b-512, ell = 2 (RFC 9380 5.3.1)"""
    p = base_modulus(curve_id)
    dp = dst_prime(curve_id, domain_prefix)

    def h(data):
        return hashlib.blake2b(data, digest_size=64).digest()

    b0 = h(bytes(128) + bytes(message) + bytes([0, 128, 0]) + dp)
    b1 = h(b0 + b"\x01" + dp)
    b2 = h(bytes(x ^ y for x, y in zip(b0, b1)) + b"\x02" + dp)
    return [int.from_bytes(b, "big") % p for b in (b1, b2)]


# ------------------------------------------------------------------------------------------------ affine group law, any a
def ec_add(P, Q, a, p):
    if P is None:
        return Q
    if Q is None:
        return P
    x1, y1 = P
    x2, y2 = Q
    if x1 == x2:
        if (y1 + y2) % p == 0:
            return None
        lam = (3 * x1 * x1 + a) * pow(2 * y1, -1, p) % p
    else:
        lam = (y2 - y1) * pow(x2 - x1, -1, p) % p
    x3 = (lam * lam - x1 - x2) % p
    return x3, (lam * (x1 - x3) - y1) % p


def ec_mul(k, P, a, p):
    R = None
    while k:
        if k & 1:
            R = ec_add(R, P, a, p)
        P = ec_add(P, P, a, p)
        k >>= 1
    return R


# ------------------------------------------------------------------------------------------------ SVDW (RFC 9380 6.6.1, F.1)
def svdw_constants(curve_id):
    p, A, B, Z = base_modulus(curve_id), 0, curve_b(curve_id), SVDW_Z % base_modulus(curve_id)
    gz = (Z * Z * Z + A * Z + B) % p
    h = (3 * Z * Z + 4 * A) % p
    c1 = gz
    c2 = (-Z) * pow(2, -1, p) % p
    c3 = sqrt((-gz * h) % p, p)
    if sgn0(c3) == 1:
        c3 = p - c3
    c4 = (-4 * gz) * pow(h, -1, p) % p
    return c1, c2, c3, c4


def svdw_z_is_valid(curve_id, Z):
    """criteria of RFC 9380 H.1 find_z_svdw"""
    p, A, B = base_modulus(curve_id), 0, curve_b(curve_id)
    g = lambda x: (x * x * x + A * x + B) % p
    h = (-(3 * Z * Z + 4 * A) * pow(4 * g(Z), -1, p)) % p if g(Z) else 0
    return g(Z) != 0 and h != 0 and is_square(h, p) and (is_square(g(Z), p) or is_square(g((-Z) * pow(2, -1, p) % p), p))


def svdw_map(curve_id, u):
    p, A, B, Z = base_modulus(curve_id), 0, curve_b(curve_id), SVDW_Z % base_modulus(curve_id)
    c1, c2, c3, c4 = svdw_constants(curve_id)
    g = lambda x: (x * x * x + A * x + B) % p
    tv1 = u * u % p * c1 % p
    tv2 = (1 + tv1) % p
    tv1 = (1 - tv1) % p
    tv3 = inv0(tv1 * tv2 % p, p)
    tv4 = u * tv1 % p * tv3 % p * c3 % p
    x1 = (c2 - tv4) % p
    e1 = is_square(g(x1), p)
    x2 = (c2 + tv4) % p
    e2 = is_square(g(x2), p) and not e1
    x3 = tv2 * tv2 % p * tv3 % p
    x3 = (x3 * x3 % p * c4 + Z) % p
    x = x1 if e1 else (x2 if e2 else x3)
    y = sqrt(g(x), p)
    if sgn0(u) != sgn0(y):
        y = (p - y) % p
    return x, y


# ------------------------------------------------------------------------------------------------ SSWU + 3-isogeny (Pasta)
def sswu_map(curve_id, u):
    """RFC 9380 6.6.2 on the iso-curve y^2 = x^3 + a x + b; returns an affine point of the ISO curve"""
    p, a, b, Z = base_modulus(curve_id), ISO_A[curve_id], ISO_B, SSWU_Z % base_modulus(curve_id)
    g = lambda x: (x * x * x + a * x + b) % p
    zu2 = Z * u * u % p
    ta = (zu2 * zu2 + zu2) % p
    tv1 = inv0(ta, p)
    x1 = (-b) * pow(a, -1, p) % p * (1 + tv1) % p
    if tv1 == 0:
        x1 = b * pow(Z * a % p, -1, p) % p
    if is_square(g(x1), p):
        x, y = x1, sqrt(g(x1), p)
    else:
        x = zu2 * x1 % p
        y = sqrt(g(x), p)
    if sgn0(u) != sgn0(y):
        y = (p - y) % p
    return x, y


def _roots(f, p):
    """roots in F_p of a polynomial (coefficients low -> high): gcd with x^p - x, then equal-degree splitting"""
    import random
    rnd = random.Random(1)

    def pmod(a, m):
        a = a[:]
        inv = pow(m[-1], -1, p)
        while len(a) >= len(m):
            c = a[-1] * inv % p
            if c:
                off = len(a) - len(m)
                for i, mi in enumerate(m):
                    a[off + i] = (a[off + i] - c * mi) % p
            a.pop()
        while len(a) > 1 and a[-1] == 0:
            a.pop()
        return a or [0]

    def pmul(a, b, m):
        r = [0] * (len(a) + len(b) - 1)
        for i, x in enumerate(a):
            for j, y in enumerate(b):
                r[i + j] = (r[i + j] + x * y) % p
        return pmod(r, m)

    def ppow(base, e, m):
        r = [1]
        while e:
            if e & 1:
                r = pmul(r, base, m)
            base = pmul(base, base, m)
            e >>= 1
        return r

    def pgcd(a, b):
        while len(b) > 1 or b[0] != 0:
            a, b = b, pmod(a, b)
        inv = pow(a[-1], -1, p)
        return [x * inv % p for x in a]

    def pdiv(a, m):
        a, q = a[:], [0] * (len(a) - len(m) + 1)
        inv = pow(m[-1], -1, p)
        while len(a) >= len(m):
            c = a[-1] * inv % p
            off = len(a) - len(m)
            q[off] = c
            for i, mi in enumerate(m):
                a[off + i] = (a[off + i] - c * mi) % p
            a.pop()
        return q

    xp = ppow([0, 1], p, f)
    xp = xp + [0] * (2 - len(xp))
    xp[1] = (xp[1] - 1) % p
    while len(xp) > 1 and xp[-1] == 0:
        xp.pop()
    g = pgcd(f, xp)
    out = []

    def split(h):
        if len(h) == 1:
            return
        if len(h) == 2:
            out.append((-h[0]) * pow(h[1], -1, p) % p)
            return
        while True:
            r = ppow([rnd.randrange(p), 1], (p - 1) // 2, h)
            r[0] = (r[0] - 1) % p
            d = pgcd(h, r)
            if 1 < len(d) < len(h):
                split(d)
                split(pdiv(h, d))
                return

    split(g)
    return sorted(out)


_ISO_CACHE = {}


def isogeny_constants(curve_id):
    """The 13 constants of pasta_curves' `iso_map` (WB2019 4.3 layout): x' = (c0 x^3 + c1 x^2 + c2 x + c3) / (x^2 + c4 x + c5),
    y' = y (c6 x^3 + c7 x^2 + c8 x + c9) / (x^3 + c10 x^2 + c11 x + c12), derived by Velu's formulas."""
    if curve_id in _ISO_CACHE:
        return _ISO_CACHE[curve_id]
    p, a, b = base_modulus(curve_id), ISO_A[curve_id], ISO_B
    # x-coordinates of the points of order 3: roots of the 3-division polynomial
    ks = _roots([(-a * a) % p, 12 * b % p, 6 * a % p, 0, 3], p)
    found = []
    for x0 in ks:
        y02 = (x0 ** 3 + a * x0 + b) % p
        gx = (3 * x0 * x0 + a) % p
        v, u0 = 2 * gx % p, 4 * y02 % p
        w = (u0 + x0 * v) % p
        A2, B2 = (a - 5 * v) % p, (b - 7 * w) % p
        if A2 != 0:
            continue
        u = pow(3, -1, p)                      # (x, y) -> (u^2 x, u^3 y) maps y^2 = x^3 + B2 onto y^2 = x^3 + u^6 B2
        if pow(u, 6, p) * B2 % p != curve_b(curve_id):
            continue
        N = [(u0 - v * x0) % p, (x0 * x0 + v) % p, (-2 * x0) % p, 1]        # x (x-x0)^2 + v (x-x0) + u0
        D = [x0 * x0 % p, (-2 * x0) % p, 1]
        Nd = [N[1], 2 * N[2] % p, 3 * N[3] % p]
        t = [0, 0, 0, 0]
        for i, c in enumerate(Nd):                                          # N'(x) (x - x0)
            t[i + 1] = (t[i + 1] + c) % p
            t[i] = (t[i] - c * x0) % p
        NY = [(t[i] - 2 * N[i]) % p for i in range(4)]                      # y' = y X'(x) for a normalised isogeny
        DY = [(-x0 ** 3) % p, 3 * x0 * x0 % p, (-3 * x0) % p, 1]
        u2, u3 = u * u % p, u * u * u % p
        found.append([u2 * N[3] % p, u2 * N[2] % p, u2 * N[1] % p, u2 * N[0] % p, D[1], D[0],
                      u3 * NY[3] % p, u3 * NY[2] % p, u3 * NY[1] % p, u3 * NY[0] % p, DY[2], DY[1], DY[0]])
    assert len(found) == 1, "expected exactly one rational 3-isogeny onto the target curve"
    _ISO_CACHE[curve_id] = found[0]
    return found[0]


def iso_map(curve_id, P):
    if P is None:
        return None
    p = base_modulus(curve_id)
    c = isogeny_constants(curve_id)
    x, y = P
    nx = (((c[0] * x + c[1]) * x + c[2]) * x + c[3]) % p
    dx = ((x + c[4]) * x + c[5]) % p
    ny = (((c[6] * x + c[7]) * x + c[8]) * x + c[9]) % p * y % p
    dy = (((x + c[10]) * x + c[11]) * x + c[12]) % p
    if dx == 0 or dy == 0:
        return None                       # the kernel of the isogeny
    return nx * pow(dx, -1, p) % p, ny * pow(dy, -1, p) % p


# ------------------------------------------------------------------------------------------------ hash_to_curve / from_label
def hash_to_curve(curve_id, domain_prefix, message):
    """affine (x, y) or None for the identity"""
    p = base_modulus(curve_id)
    u0, u1 = hash_to_field(curve_id, domain_prefix, message)
    if CURVE_H2C_METHOD[curve_id] == "SVDW":
        return ec_add(svdw_map(curve_id, u0), svdw_map(curve_id, u1), 0, p)
    r = ec_add(sswu_map(curve_id, u0), sswu_map(curve_id, u1), ISO_A[curve_id], p)
    return iso_map(curve_id, r)


def uniform_bytes(label, n):
    """the n 32-byte blocks `from_label` reads from SHAKE256(label)"""
    stream = hashlib.shake_256(bytes(label)).digest(32 * n)
    return [stream[32 * i:32 * i + 32] for i in range(n)]


def from_label(curve_id, label, n):
    """DlogGroup::from_label(label, n): n affine points, canonical integers; identity = (0, 0)"""
    out = []
    for ub in uniform_bytes(label, n):
        P = hash_to_curve(curve_id, "from_uniform_bytes", ub)
        out.append(P if P is not None else (0, 0))
    return out


def from_label_bytes(curve_id, label, n):
    """same as 64-byte x || y little-endian canonical records (the layout of include/lurk_b200.h)"""
    return b"".join(x.to_bytes(32, "little") + y.to_bytes(32, "little") for x, y in from_label(curve_id, label, n))


def ck_size(num_cons, num_vars, ck_floor=0):
    """R1CSShape::commitment_key: next_power_of_two(max(num_cons, num_vars, ck_floor))"""
    m = max(num_cons, num_vars, ck_floor, 1)
    return 1 << (m - 1).bit_length()
