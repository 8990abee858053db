"""
ORACLE (test infrastructure, NOT product code) -- sum-check prover / verifier and the inner-product argument's folding
steps (SURVEY.md 8(f) N4: `compress`, reference src/proof/nova.rs:341-356 -> Arecibo CompressedSNARK::prove ->
spartan::snark::RelaxedR1CSSNARK::prove -> SumcheckProof::{prove_cubic_with_additive_term, prove_quad} and
provider::ipa_pc::InnerProductArgument::prove).

Arecibo (git, branch dev) is NOT under the reference checkout; restated from the public crate (spartan/sumcheck.rs,
spartan/polys/{multilinear,eq,univariate}.rs, provider/ipa_pc.rs):
  * MultilinearPolynomial: evaluations Z[0 .. 2^l) over the boolean cube, index bit l-1 (the TOP bit) = first variable;
    bind_poly_var_top(r): Z[i] <- Z[i] + r (Z[i + n/2] - Z[i]) for i < n/2, length halves.
  * EqPolynomial(tau).evals(): table[i] = prod_j (tau_j if bit_j(i) else 1 - tau_j), tau_0 <-> top bit.
  * round of prove_quad: e0 = sum_i comb(A[i], B[i]); e2 = sum_i comb(2A[n/2+i] - A[i], ...); evals [e0, claim - e0, e2].
  * round of prove_cubic_with_additive_term, comb(a,b,c,d) = a (b c - d): e0, e2 as above and e3 at the point 3
    (3 hi - 2 lo); evals [e0, claim - e0, e2, e3].
  * the next claim is the round polynomial (Lagrange through 0..deg) evaluated at the challenge.
  * IPA round (n -> n/2): c_L = <a_lo, b_hi>, c_R = <a_hi, b_lo>, L = commit(a_lo; G_hi) + c_L Gc, R = commit(a_hi; G_lo) + c_R Gc,
    a' = a_lo r + a_hi r^-1, b' = b_lo r^-1 + b_hi r, G' = G_lo r^-1 + G_hi r.
The transcript (Keccak256Transcript: which bytes are absorbed, how a challenge is squeezed) is the CALLER's: the product takes the
challenge through a callback, the oracle through a Python function.

Parity: UNPINNED against Arecibo's proof bytes (the reference holds no proof fixture -- SURVEY.md 8(c): only prove -> verify round
trips).  Pinned by construction instead: the verifier below accepts what the GPU prover produced (round consistency + final
evaluation against independently evaluated multilinear extensions); the IPA fold keeps <a,b> and the commitment relation.

Only tests/, __graft_entry__.smoke() and the cpu_baseline legs (bench.py; the CPU-timing legs of tools/config_benches.py and
tools/compress_cpu_baseline.py, where the oracle is the thing timed BESIDE the product, never a checker inside it) may import this file.
"""
from . import spec


def eq_evals(tau, p):
    """EqPolynomial::evals: 2^len(tau) values, tau[0] is the top index bit"""
    out = [1]
    for t in tau:
        nxt = [0] * (2 * len(out))
        for i, v in enumerate(out):
            hi = v * t % p
            nxt[2 * i] = (v - hi) % p
            nxt[2 * i + 1] = hi
        out = nxt
    return out


def mle_eval(Z, r, p):
    """MultilinearPolynomial::evaluate: sum_i Z[i] eq(r, i)"""
    return sum(z * e for z, e in zip(Z, eq_evals(r, p))) % p


def bind_top(Z, r, p):
    n = len(Z) // 2
    return [(Z[i] + r * (Z[i + n] - Z[i])) % p for i in range(n)]


def comb_quad(a, b, p):
    return a * b % p


def comb_cubic(a, b, c, d, p):
    return a * (b * c - d) % p


def round_evals(polys, kind, p):
    """(e0, e2) for 'quad' (2 polynomials) or (e0, e2, e3) for 'cubic' (4 polynomials: A (B C - D))"""
    n = len(polys[0]) // 2
    comb = comb_quad if kind == "quad" else comb_cubic
    e0 = e2 = e3 = 0
    for i in range(n):
        lo = [P[i] for P in polys]
        hi = [P[n + i] for P in polys]
        p2 = [(2 * h - l) % p for l, h in zip(lo, hi)]
        e0 += comb(*lo, p)
        e2 += comb(*p2, p)
        if kind == "cubic":
            p3 = [(3 * h - 2 * l) % p for l, h in zip(lo, hi)]
            e3 += comb(*p3, p)
    return (e0 % p, e2 % p) if kind == "quad" else (e0 % p, e2 % p, e3 % p)


def uni_eval_from_evals(evals, x, p):
    """value at x of the polynomial of degree len(evals) - 1 through (0, evals[0]), (1, evals[1]), ..."""
    k = len(evals)
    total = 0
    for i in range(k):
        num, den = 1, 1
        for j in range(k):
            if j != i:
                num = num * (x - j) % p
                den = den * (i - j) % p
        total += evals[i] * num % p * pow(den, -1, p)
    return total % p


def prove(polys, kind, claim, challenge, p):
    """SumcheckProof::prove_quad / prove_cubic_with_additive_term.  challenge(round, evals) -> r.
    returns (round polynomials as evaluation lists, challenges, final evaluations of every polynomial, final claim)"""
    polys = [list(P) for P in polys]
    rounds, rs = [], []
    while len(polys[0]) > 1:
        e = round_evals(polys, kind, p)
        evals = [e[0], (claim - e[0]) % p] + list(e[1:])
        r = challenge(len(rounds), evals) % p
        rounds.append(evals)
        rs.append(r)
        claim = uni_eval_from_evals(evals, r, p)
        polys = [bind_top(P, r, p) for P in polys]
    return rounds, rs, [P[0] for P in polys], claim


def verify(rounds, rs, claim, degree, p):
    """SumcheckProof::verify: every round polynomial has the right degree and sums to the running claim over {0, 1};
    returns the final claim (to be compared with comb(final evaluations))"""
    for evals, r in zip(rounds, rs):
        if len(evals) != degree + 1 or (evals[0] + evals[1]) % p != claim % p:
            return None
        claim = uni_eval_from_evals(evals, r, p)
    return claim


def prove_batch(instances, kind, claims, coeffs, challenge, p):
    """SumcheckProof::prove_quad_batch / prove_cubic_with_additive_term_batch.  instances: list of polynomial lists (each instance
    2 or 4 polynomials of 2^nr_i elements).  Returns (rounds, challenges, final evaluations per instance, final claim)."""
    insts = [[list(P) for P in polys] for polys in instances]
    nr = [len(polys[0]).bit_length() - 1 for polys in insts]
    mx = max(nr)
    e = sum(c * (1 << (mx - n)) * cl for c, n, cl in zip(coeffs, nr, claims)) % p
    rounds, rs = [], []
    for rnd in range(mx):
        remaining = mx - rnd
        comb = None
        for i, polys in enumerate(insts):
            if remaining <= nr[i]:
                ev = round_evals(polys, kind, p)
            else:
                sc = (1 << (remaining - nr[i] - 1)) * claims[i] % p
                ev = (sc,) * (2 if kind == "quad" else 3)
            comb = [coeffs[i] * x % p for x in ev] if comb is None else [(a + coeffs[i] * x) % p for a, x in zip(comb, ev)]
        evals = [comb[0], (e - comb[0]) % p] + comb[1:]
        r = challenge(rnd, evals) % p
        rounds.append(evals)
        rs.append(r)
        e = uni_eval_from_evals(evals, r, p)
        for i, polys in enumerate(insts):
            if remaining <= nr[i]:
                insts[i] = [bind_top(P, r, p) for P in polys]
    return rounds, rs, [[P[0] for P in polys] for polys in insts], e


# ------------------------------------------------------------------------------------------------ inner-product argument
def inner_product(a, b, p):
    return sum(x * y for x, y in zip(a, b)) % p


def ipa_fold_scalars(a, x, y, p):
    """a'[i] = x a[i] + y a[i + n/2]"""
    n = len(a) // 2
    return [(x * a[i] + y * a[i + n]) % p for i in range(n)]


def ipa_fold_bases(curve_id, G, x, y):
    """G'[i] = x G[i] + y G[i + n/2]; points are affine (x, y) tuples or None"""
    n = len(G) // 2
    p = spec.FIELD_MODULUS[spec.CURVES[curve_id]["base"]]
    return [spec.ec_add(spec.ec_mul(x, G[i], p), spec.ec_mul(y, G[i + n], p), p) for i in range(n)]
