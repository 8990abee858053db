"""Test oracle of the compressed verifier's HyperKZG points (tests/test_gpu_compress_verify.py), on top of oracle/kzg.py: under a key of
known beta every commitment is a scalar multiple of g, so the two G1 points of EvaluationEngine::verify's batched pairing check can be
computed as scalars and compared with what lurk_compress_verify hands its pairing callback."""
from oracle import spec


def verifier_points(curve_id, C0_scalar, com_scalars, v, w_scalars, r, q, d):
    """The two G1 points of the batched pairing check e(P, H) == e(Q, beta H), as discrete logs w.r.t. g under the key beta^i g: with
    B = sum_j q^j com_j (com_0 = C0), B(u_t) = sum_j q^j v[t][j] and u = (r, -r, r^2),
    P = sum_t d^t (B - B(u_t) + u_t w_t) and Q = sum_t d^t w_t.  The check holds exactly when P = beta Q."""
    p = spec.FIELD_MODULUS[spec.CURVES[curve_id]["scalar"]]
    u = [r % p, (-r) % p, r * r % p]
    coms = [C0_scalar % p] + [c % p for c in com_scalars]
    B = sum(pow(q, j, p) * c for j, c in enumerate(coms)) % p
    P = Q = 0
    for t in range(3):
        Bu = sum(pow(q, j, p) * v[t][j] for j in range(len(coms))) % p
        P = (P + pow(d, t, p) * (B - Bu + u[t] * w_scalars[t])) % p
        Q = (Q + pow(d, t, p) * w_scalars[t]) % p
    return P, Q
