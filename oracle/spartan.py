"""
ORACLE (test infrastructure, NOT product code) -- the verifier's side of Spartan's relaxed-R1CS argument as Arecibo's
spartan::snark::RelaxedR1CSSNARK runs it inside `compress` (reference src/proof/nova.rs:341-373; Arecibo is not under
the reference checkout -- restated from the public crate, the transcript replaced by an explicit challenge function):

  z = (W padded to 2^t | u | X | 0 ..) of length 2^(t+1);  rows padded to 2^s
  outer sum-check (degree 3, claim 0) of  eq(tau, x) (Az(x) Bz(x) - u Cz(x) - E(x))                      -> r_x
  claims  Az(r_x), Bz(r_x), Cz(r_x), E(r_x);   r = challenge
  inner sum-check (degree 2, claim Az + r Bz + r^2 Cz) of  (A + r B + r^2 C)(r_x, y) z(y)                 -> r_y
  the verifier evaluates the matrices' multilinear extensions at (r_x, r_y) itself, z(r_y) = (1 - r_y0) W(r_y[1:]) + r_y0 (u, X)(r_y[1:]),
  and gets W(r_y[1:]) and E(r_x) from the polynomial commitment scheme.
`verify` does exactly those checks on a transcript produced by the GPU prover (lurk-beta_b200/spartan.py: RelaxedR1CSProver); the PCS
openings are checked separately (oracle/kzg.py, key of known beta).

Parity: UNPINNED against Arecibo's proof bytes; pinned by construction (the verifier accepts; a perturbed witness is rejected).
Only tests/, __graft_entry__.smoke() and the cpu_baseline legs (bench.py; the CPU-timing legs of tools/config_benches.py and
tools/compress_cpu_baseline.py, where the oracle is the thing timed BESIDE the product, never a checker inside it) may import this file.
"""
from . import sumcheck as sc


def col_map(col, n_w, num_vars):
    """column of the CSR matrices (over z = (W, u, X) contiguous) -> index in the padded z"""
    return col if col < n_w else num_vars + (col - n_w)


def matrices_eval(mats_rows, n_w, num_vars, rx, ry, p):
    """MLEs of A, B, C at (rx, ry); mats_rows: per matrix a list of rows, each a list of (col, value)"""
    eq_x, eq_y = sc.eq_evals(rx, p), sc.eq_evals(ry, p)
    out = []
    for rows in mats_rows:
        acc = 0
        for i, row in enumerate(rows):
            if row:
                acc += eq_x[i] * sum(v * eq_y[col_map(c, n_w, num_vars)] for c, v in row)
        out.append(acc % p)
    return out


def verify(mats_rows, n_w, num_vars, log_rows, u, X, proof, challenge, p):
    """proof: dict(outer_rounds, inner_rounds, claims=(Az, Bz, Cz, E at rx), eval_W); challenge(label, data) -> int.
    Returns (ok, rx, ry) -- eval_W at ry[1:] and claims[3] = E(rx) remain to be checked against the commitments."""
    tau = [challenge("tau", i) % p for i in range(log_rows)]
    rx = [challenge("outer", (i, ev)) % p for i, ev in enumerate(proof["outer_rounds"])]
    last = sc.verify(proof["outer_rounds"], rx, 0, 3, p)
    if last is None or len(rx) != log_rows:
        return False, None, None
    cA, cB, cC, cE = proof["claims"]
    eq_tau_rx = 1
    for t, r in zip(tau, rx):
        eq_tau_rx = eq_tau_rx * (t * r + (1 - t) * (1 - r)) % p
    if last != eq_tau_rx * (cA * cB - u * cC - cE) % p:
        return False, None, None
    r = challenge("inner_r", proof["claims"]) % p
    joint = (cA + r * cB + r * r * cC) % p
    ry = [challenge("inner", (i, ev)) % p for i, ev in enumerate(proof["inner_rounds"])]
    last2 = sc.verify(proof["inner_rounds"], ry, joint, 2, p)
    if last2 is None or len(ry) != num_vars.bit_length():          # log2(2 num_vars) = bit_length(num_vars) for a power of two
        return False, None, None
    eA, eB, eC = matrices_eval(mats_rows, n_w, num_vars, rx, ry, p)
    tail = [u % p] + [x % p for x in X]
    tail = tail + [0] * (num_vars - len(tail))
    eval_X = sc.mle_eval(tail, ry[1:], p)
    eval_Z = ((1 - ry[0]) * proof["eval_W"] + ry[0] * eval_X) % p
    if last2 != (eA + r * eB + r * r * eC) % p * eval_Z % p:
        return False, None, None
    return True, rx, ry
