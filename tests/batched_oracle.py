"""
ORACLE (test infrastructure, NOT product code) -- the end of `compress` in one evaluation claim: Arecibo's batch_eval_reduce and
SuperNova's spartan::batched::BatchedRelaxedR1CSSNARK (reference src/proof/supernova.rs:110,293-317), both restated from the public crate
(Arecibo is not under the reference checkout), built on the sum-check and Spartan oracles of oracle/sumcheck.py and oracle/spartan.py.
The transcript is a stand-in: an explicit challenge function, as everywhere in the oracle.

Parity: UNPINNED against Arecibo's proof bytes; pinned by construction -- the verifiers below accept what the GPU prover
(lurk-beta_b200/spartan.py: batch_eval_reduce, BatchedRelaxedR1CSProver) produces, its transcripts equal the pure-Python provers' for the
same challenges, and tampered instances or claims are rejected (tests/test_oracle_spartan_batched.py, tests/test_gpu_spartan_batched.py).
"""
from oracle import sumcheck as sc
from oracle.spartan import col_map, matrices_eval


# ------------------------------------------------------------------------------------------------ batch_eval_reduce
# Arecibo's batch_eval_reduce with PolyEvalInstance / PolyEvalWitness::batch_diff_size (spartan/mod.rs of the public crate, restated):
# claims P_i(x_i) = e_i, m = max n_i.  challenge(0, [e_i]) -> rho; the batched quadratic sum-check over (P_i, eq(x_i)) with claims e_i and
# coefficients rho^i, challenge(1 + j, round j) -> r_j; challenge(m + 1, [L_i]) -> gamma with L_i = P_i(r[m - n_i:]).  The joint claim is
# about sum_i gamma^i P_i with P_i zero-padded at the top to 2^m elements: its value at r is sum_i gamma^i prod_{j < m - n_i} (1 - r_j) L_i.
def eq_at(x, r, p):
    """eq(x, r) = prod_j (x_j r_j + (1 - x_j)(1 - r_j))"""
    out = 1
    for a, b in zip(x, r):
        out = out * (a * b + (1 - a) * (1 - b)) % p
    return out


def _joint_eval(nv, r, left, weights, p):
    m = len(r)
    total = 0
    for n_i, L, w in zip(nv, left, weights):
        scale = w
        for j in range(m - n_i):
            scale = scale * (1 - r[j]) % p
        total += scale * L
    return total % p


def batch_eval_reduce(polys, points, evals, challenge, p):
    """polys: the P_i (lists of 2^n_i ints), points: the x_i, evals: the e_i; challenge(round, values) -> int.
    Returns dict(rounds, r, claims_left, weights, joint_eval, joint)."""
    nv = [len(x) for x in points]
    m = max(nv)
    rho = challenge(0, list(evals)) % p
    insts = [[list(P), sc.eq_evals(x, p)] for P, x in zip(polys, points)]
    rounds, r, fin, _ = sc.prove_batch(insts, "quad", list(evals), [pow(rho, i, p) for i in range(len(polys))],
                                    lambda rnd, ev: challenge(rnd + 1, ev), p)
    left = [f[0] for f in fin]
    gamma = challenge(m + 1, left) % p
    weights = [pow(gamma, i, p) for i in range(len(polys))]
    joint = [0] * (1 << m)
    for P, w in zip(polys, weights):
        for k, v in enumerate(P):
            joint[k] = (joint[k] + w * v) % p
    return dict(rounds=rounds, r=r, claims_left=left, weights=weights, joint_eval=_joint_eval(nv, r, left, weights, p), joint=joint)


def batch_eval_verify(rounds, points, evals, claims_left, challenge, p):
    """The verifier of batch_eval_reduce: the sum-check starts from sum_i rho^i 2^(m - n_i) e_i and must end in
    sum_i rho^i eq(x_i, r[m - n_i:]) L_i.  Returns (r, joint_eval, weights), or None when a check fails."""
    nv = [len(x) for x in points]
    m = max(nv)
    if len(rounds) != m or len(claims_left) != len(points) or len(evals) != len(points):
        return None
    rho = challenge(0, list(evals)) % p
    coeffs = [pow(rho, i, p) for i in range(len(points))]
    r = [challenge(j + 1, list(ev)) % p for j, ev in enumerate(rounds)]
    last = sc.verify(rounds, r, sum(c * (1 << (m - n)) * e for c, n, e in zip(coeffs, nv, evals)) % p, 2, p)
    if last is None or last != sum(c * eq_at(x, r[m - len(x):], p) * L for c, x, L in zip(coeffs, points, claims_left)) % p:
        return None
    gamma = challenge(m + 1, list(claims_left)) % p
    weights = [pow(gamma, i, p) for i in range(len(points))]
    return r, _joint_eval(nv, r, claims_left, weights, p), weights


# ------------------------------------------------------------------------------------------------ BatchedRelaxedR1CSSNARK
# SuperNova's `compress` (reference src/proof/supernova.rs:110,293-317) proves the running instances of every circuit index with Arecibo's
# spartan::batched::BatchedRelaxedR1CSSNARK (restated from the public crate).  Instance i: rows padded to 2^s_i, z of length
# 2 num_vars_i = 2^(t_i + 1).  Challenge labels (shared with lurk-beta_b200/spartan.py: BatchedRelaxedR1CSProver):
#   "tau" (N)            -> tau; instance i's table is eq(tau, tau^2, tau^4, .., tau^(2^(s_i - 1))) (PowPolynomial::evals_with_powers)
#   "outer_r" (N)        -> outer_r; the cubic batched sum-check of eq_i (Az_i Bz_i - u_i Cz_i - E_i), claims 0, coefficients outer_r^i
#   "outer" (round, evals) -> r_x;  rx_i = r_x[s_max - s_i:]
#   "inner_r" (claims)   -> r, claims = ((Az, Bz, Cz, E)(rx_i) per instance); joint_i = Az + r Bz + r^2 Cz, coefficients (r^3)^i
#   "inner" (round, evals) -> r_y;  ry_i = r_y[max - (t_i + 1):]
#   "batch_eval" (round, values) -> the challenges of batch_eval_reduce over [W_0 .. W_{N-1}, E_0 .. E_{N-1}] at [ry_i[1:] .., rx_i ..]
def _pow_taus(tau, s, p):
    out = [tau % p]
    while len(out) < s:
        out.append(out[-1] * out[-1] % p)
    return out[:s]


def _labelled(challenge, label):
    return lambda rnd, ev: challenge(label, (rnd, list(ev)))


def prove_batched(insts, challenge, p):
    """Pure-Python prover for small sizes.  insts: [dict(R = rows of A, B, C as (col, value) lists, n_w, nv = num_vars, s = log2 of the
    padded rows, rows, W, E, u, X)] (ints).  Returns the proof dict the GPU prover returns (joint as a list)."""
    N = len(insts)
    tau = challenge("tau", N) % p
    outer, Cz, Ep, zs = [], [], [], []
    for I in insts:
        nv, s, n_w = I["nv"], I["s"], I["n_w"]
        z = list(I["W"]) + [0] * (nv - n_w) + [I["u"] % p] + [x % p for x in I["X"]] + [0] * (nv - 1 - len(I["X"]))

        def mv(rowsl):
            return [sum(v * z[col_map(c, n_w, nv)] for c, v in r) % p for r in rowsl] + [0] * ((1 << s) - I["rows"])
        Az, Bz, cz = [mv(r) for r in I["R"]]
        e = list(I["E"]) + [0] * ((1 << s) - I["rows"])
        outer.append([sc.eq_evals(_pow_taus(tau, s, p), p), Az, Bz, [(I["u"] * c + d) % p for c, d in zip(cz, e)]])
        Cz.append(cz)
        Ep.append(e)
        zs.append(z)
    outer_r = challenge("outer_r", N) % p
    o_rounds, r_x, fin, _ = sc.prove_batch(outer, "cubic", [0] * N, [pow(outer_r, i, p) for i in range(N)], _labelled(challenge, "outer"), p)
    rx = [r_x[len(r_x) - I["s"]:] for I in insts]
    claims = []
    for i in range(N):
        eqx = sc.eq_evals(rx[i], p)
        claims.append((fin[i][1], fin[i][2], sc.inner_product(Cz[i], eqx, p), sc.inner_product(Ep[i], eqx, p)))
    r = challenge("inner_r", tuple(claims)) % p
    inner, joint = [], []
    for I, x, c, z in zip(insts, rx, claims, zs):
        eqx = sc.eq_evals(x, p)
        abc = [0] * (2 * I["nv"])
        for k, rowsl in enumerate(I["R"]):
            for row_i, row in enumerate(rowsl):
                for col, v in row:
                    j = col_map(col, I["n_w"], I["nv"])
                    abc[j] = (abc[j] + pow(r, k, p) * eqx[row_i] * v) % p
        inner.append([abc, z])
        joint.append((c[0] + r * c[1] + r * r * c[2]) % p)
    r3 = pow(r, 3, p)
    i_rounds, r_y, _, _ = sc.prove_batch(inner, "quad", joint, [pow(r3, i, p) for i in range(N)], _labelled(challenge, "inner"), p)
    ry = [r_y[len(r_y) - I["nv"].bit_length():] for I in insts]
    Wp = [list(I["W"]) + [0] * (I["nv"] - I["n_w"]) for I in insts]
    eval_W = [sc.mle_eval(w, y[1:], p) for w, y in zip(Wp, ry)]
    red = batch_eval_reduce(Wp + Ep, [y[1:] for y in ry] + rx, eval_W + [c[3] for c in claims], _labelled(challenge, "batch_eval"), p)
    return dict(outer_rounds=o_rounds, inner_rounds=i_rounds, claims=claims, eval_W=eval_W, reduce_rounds=red["rounds"],
                claims_left=red["claims_left"], rx=rx, ry=ry, r=red["r"], weights=red["weights"], joint_eval=red["joint_eval"], joint=red["joint"])


def verify_batched(insts, proof, challenge, p):
    """insts: [dict(R, n_w, nv, s, u, X)]; proof: dict(outer_rounds, inner_rounds, claims, eval_W, reduce_rounds, claims_left).
    Checks both batched sum-checks (the matrices' MLEs evaluated here at (rx_i, ry_i)) and hands the W / E claims to batch_eval_verify.
    Returns (ok, r, joint_eval, weights): the joint polynomial's opening at r remains to be checked against sum_i weights_i C_i."""
    fail = (False, None, None, None)
    N = len(insts)
    if len(proof["claims"]) != N or len(proof["eval_W"]) != N:
        return fail
    S = [I["s"] for I in insts]
    T = [I["nv"].bit_length() for I in insts]
    tau = challenge("tau", N) % p
    outer_r = challenge("outer_r", N) % p
    r_x = [challenge("outer", (i, list(ev))) % p for i, ev in enumerate(proof["outer_rounds"])]
    last = sc.verify(proof["outer_rounds"], r_x, 0, 3, p)
    if last is None or len(r_x) != max(S):
        return fail
    rx = [r_x[len(r_x) - s:] for s in S]
    want = 0
    for i, (I, (cA, cB, cC, cE)) in enumerate(zip(insts, proof["claims"])):
        want += pow(outer_r, i, p) * eq_at(_pow_taus(tau, I["s"], p), rx[i], p) * (cA * cB - I["u"] * cC - cE)
    if last != want % p:
        return fail
    r = challenge("inner_r", tuple(tuple(c) for c in proof["claims"])) % p
    r3 = pow(r, 3, p)
    joint = [(c[0] + r * c[1] + r * r * c[2]) % p for c in proof["claims"]]
    r_y = [challenge("inner", (i, list(ev))) % p for i, ev in enumerate(proof["inner_rounds"])]
    mt = max(T)
    last2 = sc.verify(proof["inner_rounds"], r_y, sum(pow(r3, i, p) * (1 << (mt - t)) * j for i, (t, j) in enumerate(zip(T, joint))) % p, 2, p)
    if last2 is None or len(r_y) != mt:
        return fail
    ry = [r_y[len(r_y) - t:] for t in T]
    want = 0
    for i, I in enumerate(insts):
        eA, eB, eC = matrices_eval(I["R"], I["n_w"], I["nv"], rx[i], ry[i], p)
        tail = [I["u"] % p] + [x % p for x in I["X"]]
        eval_X = sc.mle_eval(tail + [0] * (I["nv"] - len(tail)), ry[i][1:], p)
        eval_Z = ((1 - ry[i][0]) * proof["eval_W"][i] + ry[i][0] * eval_X) % p
        want += pow(r3, i, p) * (eA + r * eB + r * r * eC) % p * eval_Z
    if last2 != want % p:
        return fail
    red = batch_eval_verify(proof["reduce_rounds"], [y[1:] for y in ry] + rx, list(proof["eval_W"]) + [c[3] for c in proof["claims"]],
                               proof["claims_left"], _labelled(challenge, "batch_eval"), p)
    if red is None:
        return fail
    return (True,) + red
