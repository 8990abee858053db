"""
ORACLE (test infrastructure, NOT product code) -- the KZG side of the BN256 path (SURVEY.md 8(f) N3 / N4).

Restates, from the public Arecibo crate (git, branch dev -- NOT under the reference checkout; provider/hyperkzg.rs, provider/kzg_commitment.rs,
provider/non_hiding_kzg.rs), what the reference's BN256 engine (`Bn256EngineKZG` with `hyperkzg::EvaluationEngine`, reference
src/proof/nova.rs:65-71) does with vectors:
  * key: UniversalKZGParam::gen_srs_for_testing -> powers_of_g[i] = beta^i g  (how beta and g come out of the label-seeded RNG is not
    restated: they are inputs here);
  * EvaluationEngine::prove(ck, _, transcript, _, hat_P, point, _):
      Phase 1  P_0 = hat_P;  P_{i+1}[j] = x[l-1-i] (P_i[2j+1] - P_i[2j]) + P_i[2j];  com = [commit(P_1), ..., commit(P_{l-1})]
      Phase 2  r = challenge(com);  u = [r, -r, r^2]
      Phase 3  v[t][j] = P_j(u_t) (polynomials in the coefficient basis: P_j[k] is the coefficient of X^k);  q = challenge(v);
               B = sum_j q^j P_j;  w_t = commit(h_t),  h_t = B(X) / (X - u_t):  h[i-1] = B[i] + h[i] u  (i = d-1 .. 1);  challenge(w).
The transcript is the caller's (callbacks).

Parity: UNPINNED against Arecibo's proof bytes.  Pinned by construction: with a key of KNOWN beta the commitments are commit(f) =
f(beta) g, so the KZG opening identity (beta - u) h(beta) = B(beta) - B(u) and the fold identities
P_{i+1}(u^2)-style checks of the verifier can be evaluated in the field -- `verify_known_beta` below does the verifier's algebra
without pairings.

Only tests/, __graft_entry__.smoke() and the cpu_baseline legs (bench.py; the CPU-timing legs of tools/config_benches.py and
tools/compress_cpu_baseline.py, where the oracle is the thing timed BESIDE the product, never a checker inside it) may import this file.
"""
from . import spec


def powers_of_tau(curve_id, g, beta, n):
    """[beta^i g for i < n] as affine tuples (None = identity)"""
    C = spec.CURVES[curve_id]
    pb, q = spec.FIELD_MODULUS[C["base"]], spec.FIELD_MODULUS[C["scalar"]]
    out, s = [], 1
    for _ in range(n):
        out.append(spec.ec_mul(s, g, pb) if s else None)
        s = s * beta % q
    return out


def poly_eval(f, u, p):
    r = 0
    for c in reversed(f):
        r = (r * u + c) % p
    return r


def witness_poly(f, u, p):
    h = [0] * len(f)
    for i in range(len(f) - 1, 0, -1):
        h[i - 1] = (f[i] + h[i] * u) % p
    return h


def fold_chain(P0, x, p):
    l = len(x)
    polys = [list(P0)]
    for i in range(l - 1):
        cur = polys[i]
        polys.append([(x[l - 1 - i] * (cur[2 * j + 1] - cur[2 * j]) + cur[2 * j]) % p for j in range(len(cur) // 2)])
    return polys


def prove(curve_id, commit, hat_P, point, challenge):
    """commit(f) -> point; challenge(round, message) -> int.  Returns dict(com, v, w, polys, B, u, q)."""
    p = spec.FIELD_MODULUS[spec.CURVES[curve_id]["scalar"]]
    l = len(point)
    polys = fold_chain(hat_P, point, p)
    com = [commit(f) for f in polys[1:]]
    r = challenge(0, com) % p
    u = [r, (-r) % p, r * r % p]
    v = [[poly_eval(f, ut, p) for f in polys] for ut in u]
    q = challenge(1, v) % p
    B = [0] * len(hat_P)
    qp = 1
    for f in polys:
        for k, c in enumerate(f):
            B[k] = (B[k] + qp * c) % p
        qp = qp * q % p
    hs = [witness_poly(B, ut, p) for ut in u]
    w = [commit(h) for h in hs]
    challenge(2, w)
    return dict(com=com, v=v, w=w, polys=polys, B=B, u=u, q=q, h=hs)


def verify_known_beta(curve_id, g, beta, C0_scalar, point, eval_, com_scalars, v, w_scalars, r, q):
    """The verifier's checks of EvaluationEngine::verify with every commitment replaced by its discrete log w.r.t. g
    (commit(f) = f(beta) g for the key beta^i g): (1) the fold consistency of the evaluations
    2 r v[2][i+1] = r (1 - x_{l-i-1}) (v[0][i] + v[1][i]) + x_{l-i-1} (v[0][i] - v[1][i]) with v[.][l] = eval;
    (2) the batched opening (beta - u_t) h_t(beta) = B(beta) - B(u_t) with B(beta) = sum_j q^j com_j, B(u_t) = sum_j q^j v[t][j]."""
    p = spec.FIELD_MODULUS[spec.CURVES[curve_id]["scalar"]]
    l = len(point)
    u = [r, (-r) % p, r * r % p]
    Y = [v[2][j] for j in range(l)] + [eval_ % p]
    for i in range(l):
        x = point[l - 1 - i]
        lhs = 2 * r * Y[i + 1] % p
        rhs = (r * (1 - x) * (v[0][i] + v[1][i]) + x * (v[0][i] - v[1][i])) % p
        if lhs != rhs:
            return False
    coms = [C0_scalar % p] + [c % p for c in com_scalars]
    Bbeta = sum(pow(q, j, p) * c for j, c in enumerate(coms)) % p
    for t in range(3):
        Bu = sum(pow(q, j, p) * v[t][j] for j in range(l)) % p
        if (beta - u[t]) * w_scalars[t] % p != (Bbeta - Bu) % p:
            return False
    return True
