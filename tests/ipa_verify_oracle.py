"""
ORACLE (test infrastructure, NOT product code) -- provider::ipa_pc::InnerProductArgument::verify, restated from the public Arecibo crate
(not under the reference checkout) on top of oracle/sumcheck.py and oracle/spec.py, with the transcript replaced by an explicit challenge
function as everywhere in the oracle:
  r_j = challenge(j, L_j | R_j);  s[i] = prod_j (bit_j(i) ? r_j : r_j^-1), bit 0 = the top bit of i;
  ck_hat = <s, G>;  b_hat = <b, s>;  P_hat = comm + c ck_c + sum_j (r_j^2 L_j + r_j^-2 R_j);
  accept iff a_hat ck_hat + a_hat b_hat ck_c == P_hat.
`msm(G, s)` is the caller's (oracle/spec.py: msm_naive for small keys, the C oracle's Pippenger for large ones).

Parity: UNPINNED against Arecibo's proof bytes; pinned by construction: it accepts what a pure-Python prover built from
oracle/sumcheck.py's ipa_fold_* steps produces and rejects tampered transcripts (tests/test_oracle_ipa_verify.py).
"""
from oracle import spec


def point_bytes(P):
    """(x, y) or None -> x | y | z (96 bytes, canonical), the message format of the IPA rounds"""
    vals = [0, 0, 0] if P is None else [P[0], P[1], 1]
    return b"".join(int(v).to_bytes(32, "little") for v in vals)


def tensor(rs, q):
    """s[i] = prod_j (bit_j(i) ? r_j : r_j^-1) with bit 0 the top bit"""
    s = [1]
    for r in rs:
        ri = pow(r, -1, q)
        s = [x * f % q for x in s for f in (ri, r)]
    return s


def ipa_verify(curve, G, ck_c, comm, c, b, Ls, Rs, a_hat, challenge, msm):
    """Returns (accepted, ck_hat, b_hat).  G: the first 2^len(Ls) bases; points (x, y) or None; challenge(round, bytes) -> int."""
    pb, q = spec.FIELD_MODULUS[spec.CURVES[curve]["base"]], spec.FIELD_MODULUS[spec.CURVES[curve]["scalar"]]
    add = lambda P, Q: spec.ec_add(P, Q, pb)
    mul = lambda k, P: spec.ec_mul(k % q, P, pb)
    rs = [challenge(j, point_bytes(Lj) + point_bytes(Rj)) % q for j, (Lj, Rj) in enumerate(zip(Ls, Rs))]
    s = tensor(rs, q)
    ck_hat = msm(G, s)
    b_hat = sum(x * y for x, y in zip(b, s)) % q
    P_hat = add(comm, mul(c, ck_c))
    for r, Lj, Rj in zip(rs, Ls, Rs):
        ri = pow(r, -1, q)
        P_hat = add(P_hat, add(mul(r * r, Lj), mul(ri * ri, Rj)))
    return add(mul(a_hat, ck_hat), mul(a_hat * b_hat, ck_c)) == P_hat, ck_hat, b_hat
