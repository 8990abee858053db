"""
ORACLE (test infrastructure, NOT product code): Nova's non-interactive folding scheme on the CPU.

Restates what `RecursiveSNARK::new` / `prove_step` (reference call sites src/proof/nova.rs:286-293, supernova.rs:231-244)
do with one circuit's witness inside Arecibo's `NIFS::prove` (third-party git dependency `nova`, branch dev, not in
tree; public protocol, SURVEY.md Appendix B):
    comm_W2 = commit(W2);  T = Az1*Bz2 + Az2*Bz1 - u1 Cz2 - u2 Cz1;  comm_T = commit(T)
    r = RO(pp_digest, U2 = (comm_W2, X2), comm_T)        [oracle/spec.py: ro_squeeze, 128 bits]
    W <- W1 + r W2, E <- E1 + r T, u <- u1 + r, X <- X1 + r X2, comm_W <- comm_W1 + r comm_W2, comm_E <- comm_E1 + r comm_T
and the relaxed-R1CS satisfiability check a verifier of the folded instance performs.  Heavy vector work goes through
oracle/oracle.c, scalars and points through oracle/spec.py.  No golden NIFS transcript exists in the reference => the
challenge derivation is "parity unpinned"; satisfiability of the folded instance is the protocol-level property tested.

Only tests/, __graft_entry__.smoke() and bench.py's CPU legs may import this module.
"""
import numpy as np

from . import capi, spec


def ints(buf):
    b = np.ascontiguousarray(buf, dtype=np.uint8).tobytes()
    return [int.from_bytes(b[i:i + 32], "little") for i in range(0, len(b), 32)]


def pack(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint8).copy()


def point_of(buf96):
    x, y, z = ints(buf96)
    return None if z == 0 else (x, y)


def point_bytes(P):
    return pack([0, 0, 0]) if P is None else pack([P[0], P[1], 1])


# kinds of absorbed elements (include/lurk_b200.h, lurk_fold_ctx_set_ro): a per-step constant, or a coordinate / the identity
# flag of comm_W2 or comm_T
RO_CONST, RO_W_X, RO_W_Y, RO_W_INF, RO_T_X, RO_T_Y, RO_T_INF = range(7)
DEFAULT_RO_KINDS = (RO_CONST, RO_W_X, RO_W_Y, RO_W_INF, RO_CONST, RO_CONST, RO_T_X, RO_T_Y, RO_T_INF)


def ro_absorb_list(kinds, consts, comm_W2, comm_T):
    """the sponge input the fold context builds for an absorb pattern: element i is consts[i] for a CONST slot, else a
    coordinate or identity flag of comm_W2 / comm_T; the identity is absorbed as (0, 0, 1)"""
    def pt(P):
        return (0, 0, 1) if P is None else (P[0], P[1], 0)
    w, t = pt(comm_W2), pt(comm_T)
    pick = {RO_W_X: w[0], RO_W_Y: w[1], RO_W_INF: w[2], RO_T_X: t[0], RO_T_Y: t[1], RO_T_INF: t[2]}
    return [consts[i] if k == RO_CONST else pick[k] for i, k in enumerate(kinds)]


class NovaOracle:
    """one running instance of one circuit"""

    def __init__(self, curve_id, bases_w, mats, n_w, n_x, bases_t=None, nthreads=1, pp_digest=0):
        """mats: [(row_ptr, col, val canonical bytes)] x 3 over z = (W, u, X); bases: canonical affine bytes"""
        C = spec.CURVES[curve_id]
        self.curve_id, self.field, self.base_field = curve_id, C["scalar"], C["base"]
        self.p = spec.FIELD_MODULUS[self.field]
        self.pb = spec.FIELD_MODULUS[self.base_field]
        self.bases_w, self.bases_t = bases_w, bases_w if bases_t is None else bases_t
        self.mats, self.n_w, self.n_x, self.th, self.pp_digest = mats, n_w, n_x, nthreads, pp_digest
        self.rows = len(mats[0][0]) - 1
        self.W = self.E = self.u = self.X = self.comm_W = self.comm_E = None

    # ---- helpers
    def z(self, W, u, X):
        return np.concatenate([np.ascontiguousarray(W, dtype=np.uint8).reshape(-1), pack([u]), pack(X)])

    def mv(self, z):
        return [capi.spmv(self.field, rp, col, val, z, nthreads=self.th) for rp, col, val in self.mats]

    def commit_w(self, W):
        return point_of(capi.msm(self.curve_id, self.bases_w, W, nthreads=self.th))

    def commit_t(self, T):
        return point_of(capi.msm(self.curve_id, self.bases_t, T, nthreads=self.th))

    # ---- RecursiveSNARK::new
    def init_running(self, W2, X2):
        self.W = np.ascontiguousarray(W2, dtype=np.uint8).reshape(-1).copy()
        self.E = np.zeros(self.rows * 32, dtype=np.uint8)
        self.u, self.X = 1, [x % self.p for x in X2]
        self.comm_W, self.comm_E = self.commit_w(self.W), None
        return dict(comm_W=self.comm_W)

    def ro_consts(self, X2):
        """the CONST elements of the default absorb pattern, by position: pp digest at 0, X2 after comm_W2's 3 slots"""
        c = [self.pp_digest, 0, 0, 0] + [int(x) for x in X2]
        return c + [0] * (spec.RO_RATE - len(c))

    # ---- NIFS::prove + fold
    def prove_step(self, W2, X2, challenge_bits=128, ro_kinds=None, ro_consts=None):
        """ro_kinds: absorb pattern (FOLD_RO_* per absorbed element, as lurk_fold_ctx_set_ro takes it; None = Arecibo's
        NIFS::prove list); ro_consts: the CONST element of every position (None = ro_consts(X2))"""
        p = self.p
        W2 = np.ascontiguousarray(W2, dtype=np.uint8).reshape(-1)
        comm_W2 = self.commit_w(W2)
        az1, bz1, cz1 = self.mv(self.z(self.W, self.u, self.X))
        az2, bz2, cz2 = self.mv(self.z(W2, 1, X2))
        T = capi.cross_term(self.field, az1, bz1, cz1, az2, bz2, cz2, pack([self.u]), pack([1]), nthreads=self.th)
        comm_T = self.commit_t(T)
        if ro_kinds is None:
            absorbed = spec.nifs_absorb_list(self.pp_digest, comm_W2, X2, comm_T)
        else:
            absorbed = ro_absorb_list(ro_kinds, self.ro_consts(X2) if ro_consts is None else ro_consts, comm_W2, comm_T)
        r, h = spec.ro_squeeze(self.base_field, absorbed, challenge_bits)
        rb = pack([r])
        self.W = capi.axpy(self.field, self.W, W2, rb, nthreads=self.th)
        self.E = capi.axpy(self.field, self.E, T, rb, nthreads=self.th)
        self.u = (self.u + r) % p
        self.X = [(a + r * b) % p for a, b in zip(self.X, X2)]
        self.comm_W = spec.ec_add(self.comm_W, spec.ec_mul(r, comm_W2, self.pb), self.pb)
        self.comm_E = spec.ec_add(self.comm_E, spec.ec_mul(r, comm_T, self.pb), self.pb)
        return dict(comm_W=comm_W2, comm_T=comm_T, r=r, hash=h, T=T, absorbed=absorbed)

    # ---- verifier side
    def bad_rows(self, W=None, E=None, u=None, X=None):
        """rows of the relaxed R1CS equation (A z) o (B z) = u (C z) + E that do not hold"""
        W = self.W if W is None else W
        E = self.E if E is None else E
        u = self.u if u is None else u
        X = self.X if X is None else X
        az, bz, cz = (ints(v) for v in self.mv(self.z(W, u, X)))
        e = ints(E)
        p = self.p
        return sum(1 for a, b, c, d in zip(az, bz, cz, e) if (a * b - u * c - d) % p)

    def commitments_consistent(self, W=None, E=None, comm_W=None, comm_E=None):
        W = self.W if W is None else W
        E = self.E if E is None else E
        comm_W = self.comm_W if comm_W is None else comm_W
        comm_E = self.comm_E if comm_E is None else comm_E
        return self.commit_w(W) == comm_W, self.commit_t(E) == comm_E


def synthetic_step_circuit(rng, frames, slot_elems, glue, lin_rows, n_x=2):
    """Satisfiable-by-construction R1CS in the shape of a Lurk step circuit: per frame `slot_elems` slot-witness columns
    (any values), `glue` columns each DEFINED as (a . slots) * (b . slots) of the same frame -- the LEM body aux stand-in
    --, the same `glue` definitions restated with other coefficients, and `lin_rows` linear rows (a . z) * u = (a . z)
    that hold for every z (their cross term vanishes).  Columns: frame-major W, then u, then X.
    Returns (mats, n_w, glue_fn) where glue_fn(W2 bytes with slot columns filled, p) -> glue values per frame."""
    per = slot_elems + glue
    n_w = frames * per
    u_col = n_w
    A, B, Cm = [], [], []
    defs = []
    small = lambda: int(rng.integers(1, 7))
    for f in range(frames):
        base = f * per
        for g in range(glue):
            a = [(base + int(c), small()) for c in rng.choice(slot_elems, size=int(rng.integers(1, 4)), replace=False)]
            b = [(base + int(c), small()) for c in rng.choice(slot_elems, size=int(rng.integers(1, 3)), replace=False)]
            A.append(a); B.append(b); Cm.append([(base + slot_elems + g, 1)])
            defs.append((base + slot_elems + g, a, b))
        for g in range(glue):
            # the same definition restated with other coefficients: (l a . s)(m b . s) = l m glue_g -- keeps the system
            # satisfiable while most rows have a non-vanishing cross term, as in a real circuit
            dst, a, b = defs[len(defs) - glue + g]
            l, m = small(), small()
            A.append([(c, v * l) for c, v in a]); B.append([(c, v * m) for c, v in b]); Cm.append([(dst, l * m)])
        for _ in range(lin_rows):
            cols = [base + int(c) for c in rng.choice(per, size=int(rng.integers(1, 4)), replace=False)]
            if rng.random() < 0.3:
                cols.append(n_w + 1 + int(rng.integers(0, n_x)))          # touch the public IO too
            a = [(c, small()) for c in cols]
            A.append(a); B.append([(u_col, 1)]); Cm.append(list(a))

    def glue_fn(W_ints, p):
        out = {}
        for dst, a, b in defs:
            out[dst] = sum(W_ints[c] * v for c, v in a) * sum(W_ints[c] * v for c, v in b) % p
        return out

    return [rows_to_csr(A), rows_to_csr(B), rows_to_csr(Cm)], n_w, glue_fn


def rows_to_csr(rows):
    """[[(column, canonical coefficient)] per row] -> (row_ptr u64, col u32, val bytes)"""
    rp = np.zeros(len(rows) + 1, dtype=np.uint64)
    col, val = [], []
    for i, r in enumerate(rows):
        for c, v in r:
            col.append(c); val.append(v)
        rp[i + 1] = len(col)
    return rp, np.array(col, dtype=np.uint32), pack(val)


# non-zeros per row that the real-shape circuit produces: empty rows, the one-product fast path of the sparse products, the
# lazy-reduction group boundaries (8 products per group) on both sides, a 64-limb row, a 255-bit packing row and a long row
# (a Lurk step circuit's `u` and public-IO columns collect thousands of entries)
REAL_ROW_LENGTHS = (0, 1, 7, 8, 9, 15, 16, 17, 64, 255, 2000)


def real_shape_step_circuit(rng, p, frames, free, glue, lin_rows, n_x=2, row_lengths=REAL_ROW_LENGTHS):
    """Satisfiable-by-construction R1CS with the rows a real Lurk step circuit has and synthetic_step_circuit lacks.
    Per frame: `free` columns (slot witnesses or host values: any values), then `glue` columns, each DEFINED by a product
    row (a . z) * (b . z) = glue with u = 1 for a fresh instance; half of the definitions are restated with two more
    full-width factors.  Then `lin_rows` linear rows (a . z) * u = (a . z), which hold for every z, and two empty rows.
    Rows take their lengths from `row_lengths` in turn; the 255-term rows are bit packings sum 2^i b_i (coefficients 2^i mod
    p), a quarter of the others have only coefficients whose Montgomery form is near p, the rest mix small coefficients,
    p - 1 and full-width ones.  The a side of a product row and the linear rows also
    reference u and X; the b side only W columns, so that the all-zero witness satisfies the system for every X.
    Columns: frame-major W, then u, then X.  Returns (mats, n_w, glue_fn) where glue_fn(W ints with the free columns
    filled, X) -> {glue column: value} for a fresh instance."""
    per = free + glue
    n_w = frames * per
    u_col = n_w
    A, B, Cm, defs = [], [], [], []
    lengths = iter(row_lengths * (1 + (frames * (glue + lin_rows)) // len(row_lengths)))

    rinv = pow(1 << 256, -1, p)

    def coeff(k, i, mont_top=False):
        if k == 255:
            return pow(2, i, p)
        if mont_top:        # Montgomery form (c 2^256 mod p) near p: the largest products a lazy reduction group can hold
            return (p - 1 - int(rng.integers(0, 2**32))) * rinv % p
        kind = rng.random()
        return int(rng.integers(1, 37)) if kind < 0.4 else p - 1 if kind < 0.6 else int(rng.integers(0, 2**63)) * int(rng.integers(1, 2**63)) ** 3 % p

    def terms(pool, k):
        cols = rng.choice(pool, size=k, replace=k > len(pool))
        top = rng.random() < 0.25
        return [(int(c), coeff(k, i, top)) for i, c in enumerate(cols)]

    for f in range(frames):
        base = f * per
        free_cols = np.arange(base, base + free)
        for g in range(glue):
            k = next(lengths)
            a = terms(free_cols, k)
            if rng.random() < 0.4:
                a += [(u_col, coeff(0, 0)), (n_w + 1 + int(rng.integers(0, n_x)), coeff(0, 0))]
            b = terms(free_cols, int(rng.integers(1, 10)) if g % 2 else k)
            dst = base + free + g
            A.append(a); B.append(b); Cm.append([(dst, 1)])
            defs.append((dst, a, b))
            if g % 2 == 0:
                l, m = coeff(0, 0) or 1, coeff(0, 0) or 1
                A.append([(c, v * l % p) for c, v in a]); B.append([(c, v * m % p) for c, v in b]); Cm.append([(dst, l * m % p)])
        all_cols = np.concatenate([np.arange(base, base + per), [u_col], n_w + 1 + np.arange(n_x)])
        for _ in range(lin_rows):
            a = terms(all_cols, next(lengths))
            A.append(a); B.append([(u_col, 1)]); Cm.append(list(a))
        A += [[], []]; B += [[], [(base, 1)]]; Cm += [[], []]            # two empty rows: 0 * 0 = 0 and 0 * w = 0

    def glue_fn(W_ints, X):
        z = lambda c: W_ints[c] if c < n_w else 1 if c == u_col else X[c - n_w - 1]
        return {dst: sum(z(c) * v for c, v in a) * sum(z(c) * v for c, v in b) % p for dst, a, b in defs}

    return [rows_to_csr(A), rows_to_csr(B), rows_to_csr(Cm)], n_w, glue_fn
