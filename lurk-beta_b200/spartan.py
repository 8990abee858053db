"""Host-side mirror of the Arecibo interfaces behind `compress` (reference src/proof/nova.rs:341-356 -> CompressedSNARK::prove
-> spartan::snark::RelaxedR1CSSNARK::prove): SumcheckProof::prove_quad / prove_cubic_with_additive_term, EqPolynomial::evals,
MultilinearPolynomial::evaluate and provider::ipa_pc::InnerProductArgument::prove, all on device-resident vectors through the C ABI
(include/lurk_b200.h, N4).  The transcript is the caller's: `challenge(round, message_bytes) -> int`."""
import ctypes as C

import numpy as np

from . import _capi

QUAD, CUBIC = _capi.SUMCHECK_QUAD, _capi.SUMCHECK_CUBIC


def _callback(challenge, errors):
    def cb(user, rnd, msg, msg_len, out):
        try:
            r = int(challenge(rnd, bytes(msg[i] for i in range(msg_len))))
            for i, byte in enumerate(r.to_bytes(32, "little")):
                out[i] = byte
            return 0
        except Exception as e:          # never unwind through the C frames
            errors.append(e)
            return 1
    return _capi.CHALLENGE_FN(cb)


def _ints(buf):
    return [int.from_bytes(buf[i:i + 32].tobytes(), "little") for i in range(0, buf.size, 32)]


def _fe(x):
    return np.frombuffer(int(x).to_bytes(32, "little"), dtype=np.uint8).copy()


def sumcheck_prove(field_id, kind, poly_ptrs, num_rounds, claim, challenge, stream=0):
    """poly_ptrs: device pointers of the 2 (QUAD) or 4 (CUBIC) polynomials, 2^num_rounds Montgomery elements each (consumed).
    claim: int.  challenge(round, message) -> int (canonical).  Returns (round_evals [[int]], challenges [int], final_evals [int])."""
    k, deg1 = (2, 3) if kind == QUAD else (4, 4)
    ptrs = (C.c_void_p * k)(*[C.c_void_p(p) for p in poly_ptrs])
    rounds = np.zeros(max(1, num_rounds) * deg1 * 32, dtype=np.uint8)
    chal = np.zeros(max(1, num_rounds) * 32, dtype=np.uint8)
    fin = np.zeros(k * 32, dtype=np.uint8)
    errors = []
    cb = _callback(challenge, errors)
    rc = _capi.lib().lurk_sumcheck_prove_dev(field_id, kind, ptrs, num_rounds, _capi.np_ptr(_fe(claim)), cb, None, _capi.np_ptr(rounds),
                                             _capi.np_ptr(chal), _capi.np_ptr(fin), _capi.FMT_CANONICAL, C.c_void_p(stream))
    if errors:
        raise errors[0]
    _capi.check(rc)
    ev = _ints(rounds)
    return [ev[i * deg1:(i + 1) * deg1] for i in range(num_rounds)], _ints(chal)[:num_rounds], _ints(fin)


def sumcheck_prove_batch(field_id, kind, instances, claims, coeffs, challenge, stream=0):
    """SumcheckProof::prove_*_batch.  instances: [(poly_ptrs, num_rounds)], claims / coeffs: ints.
    Returns (round_evals, challenges, final_evals per instance)."""
    k, deg1 = (2, 3) if kind == QUAD else (4, 4)
    n = len(instances)
    flat = [p for ptrs, _ in instances for p in ptrs]
    ptrs = (C.c_void_p * (n * k))(*[C.c_void_p(p) for p in flat])
    nr = (C.c_int * n)(*[r for _, r in instances])
    mx = max(r for _, r in instances)
    rounds = np.zeros(max(1, mx) * deg1 * 32, dtype=np.uint8)
    chal = np.zeros(max(1, mx) * 32, dtype=np.uint8)
    fin = np.zeros(n * k * 32, dtype=np.uint8)
    cl = np.concatenate([_fe(c) for c in claims])
    co = np.concatenate([_fe(c) for c in coeffs])
    errors = []
    cb = _callback(challenge, errors)
    rc = _capi.lib().lurk_sumcheck_prove_batch_dev(field_id, kind, n, ptrs, nr, _capi.np_ptr(cl), _capi.np_ptr(co), cb, None, _capi.np_ptr(rounds),
                                                   _capi.np_ptr(chal), _capi.np_ptr(fin), _capi.FMT_CANONICAL, C.c_void_p(stream))
    if errors:
        raise errors[0]
    _capi.check(rc)
    ev, fi = _ints(rounds), _ints(fin)
    return [ev[i * deg1:(i + 1) * deg1] for i in range(mx)], _ints(chal)[:mx], [fi[i * k:(i + 1) * k] for i in range(n)]


def eq_evals(field_id, tau, d_out_ptr, out_fmt=_capi.FMT_MONTGOMERY, stream=0):
    """EqPolynomial::new(tau).evals() into device memory (2^len(tau) elements in out_fmt); tau: ints"""
    R = 1 << 256
    if out_fmt == _capi.FMT_MONTGOMERY:
        p = int.from_bytes(field_modulus(field_id), "little")
        tau = [t * R % p for t in tau]
    buf = np.frombuffer(b"".join(int(t).to_bytes(32, "little") for t in tau) or bytes(32), dtype=np.uint8).copy()
    _capi.check(_capi.lib().lurk_eq_evals_dev(field_id, _capi.np_ptr(buf), len(tau), C.c_void_p(d_out_ptr), out_fmt, C.c_void_p(stream)))


def field_modulus(field_id):
    out = np.zeros(32, dtype=np.uint8)
    _capi.check(_capi.lib().lurk_field_modulus(field_id, _capi.np_ptr(out)))
    return out.tobytes()


def inner_product(field_id, d_a_ptr, d_b_ptr, n, stream=0):
    out = np.zeros(32, dtype=np.uint8)
    _capi.check(_capi.lib().lurk_inner_product_dev(field_id, C.c_void_p(d_a_ptr), C.c_void_p(d_b_ptr), n, _capi.np_ptr(out),
                                                   _capi.FMT_CANONICAL, C.c_void_p(stream)))
    return int.from_bytes(out.tobytes(), "little")


def ipa_fold_scalars(field_id, d_a_ptr, n, x, y, stream=0):
    _capi.check(_capi.lib().lurk_ipa_fold_scalars_dev(field_id, C.c_void_p(d_a_ptr), n, _capi.np_ptr(_fe(x)), _capi.np_ptr(_fe(y)),
                                                      _capi.FMT_CANONICAL, C.c_void_p(stream)))


def ipa_fold_bases(curve_id, d_bases_ptr, n, x, y, stream=0):
    _capi.check(_capi.lib().lurk_ipa_fold_bases_dev(curve_id, C.c_void_p(d_bases_ptr), n, _capi.np_ptr(_fe(x)), _capi.np_ptr(_fe(y)),
                                                    _capi.FMT_CANONICAL, C.c_void_p(stream)))


def ipa_prove(curve_id, ck, ck_c, d_a_ptr, d_b_ptr, log_n, challenge, stream=0):
    """InnerProductArgument::prove's rounds under the key of CommitmentKey `ck` (not consumed).  ck_c: (x, y) canonical ints.
    Returns (L points, R points, a_final, b_final); points are (x, y) tuples or None for the identity."""
    gc = np.concatenate([_fe(ck_c[0]), _fe(ck_c[1])])
    Ls = np.zeros(max(1, log_n) * 96, dtype=np.uint8)
    Rs = np.zeros(max(1, log_n) * 96, dtype=np.uint8)
    af, bf = np.zeros(32, dtype=np.uint8), np.zeros(32, dtype=np.uint8)
    errors = []
    cb = _callback(challenge, errors)
    rc = _capi.lib().lurk_ipa_prove_dev(curve_id, ck._ctx, _capi.np_ptr(gc), C.c_void_p(d_a_ptr), C.c_void_p(d_b_ptr), log_n, cb,
                                        None, _capi.np_ptr(Ls), _capi.np_ptr(Rs), _capi.np_ptr(af), _capi.np_ptr(bf), _capi.FMT_CANONICAL,
                                        C.c_void_p(stream))
    if errors:
        raise errors[0]
    _capi.check(rc)

    def pts(buf):
        out = []
        for i in range(log_n):
            b = buf[96 * i:96 * i + 96].tobytes()
            z = int.from_bytes(b[64:], "little")
            out.append((int.from_bytes(b[:32], "little"), int.from_bytes(b[32:64], "little")) if z else None)
        return out
    return pts(Ls), pts(Rs), int.from_bytes(af.tobytes(), "little"), int.from_bytes(bf.tobytes(), "little")


def _fes(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals) or bytes(32), dtype=np.uint8).copy()


def _point_bytes(P):
    """(x, y) or None (the identity) -> x | y | z, 96 bytes canonical"""
    return _fes([0, 0, 0]) if P is None else _fes([P[0], P[1], 1])


def ipa_verify(curve_id, ck, ck_c, comm, c, d_b_ptr, log_n, Ls, Rs, a_final, challenge, stream=0):
    """InnerProductArgument::verify of <a, b> = c with comm = commit(a), from ipa_prove's transcript under the key of CommitmentKey `ck` (not
    consumed).  ck_c: (x, y); comm, Ls, Rs: (x, y) tuples or None; d_b_ptr: 2^log_n Montgomery elements on the device (not modified);
    challenge(round, L | R bytes) -> int as for ipa_prove.  Returns (accepted, ck_hat point or None, b_hat)."""
    assert len(Ls) == log_n and len(Rs) == log_n
    gc = _fes([ck_c[0], ck_c[1]])
    Lb = np.concatenate([_point_bytes(P) for P in Ls]) if log_n else np.zeros(96, dtype=np.uint8)
    Rb = np.concatenate([_point_bytes(P) for P in Rs]) if log_n else np.zeros(96, dtype=np.uint8)
    hat, bh = np.zeros(96, dtype=np.uint8), np.zeros(32, dtype=np.uint8)
    acc = C.c_int(-1)
    errors = []
    cb = _callback(challenge, errors)
    rc = _capi.lib().lurk_ipa_verify_dev(curve_id, ck._ctx, _capi.np_ptr(gc), _capi.np_ptr(_point_bytes(comm)), _capi.np_ptr(_fe(c)), C.c_void_p(d_b_ptr),
                                         log_n, _capi.np_ptr(Lb), _capi.np_ptr(Rb), _capi.np_ptr(_fe(a_final)), cb, None, C.byref(acc), _capi.np_ptr(hat),
                                         _capi.np_ptr(bh), _capi.FMT_CANONICAL, C.c_void_p(stream))
    if errors:
        raise errors[0]
    _capi.check(rc)
    h = _ints(hat)
    return bool(acc.value), ((h[0], h[1]) if h[2] else None), int.from_bytes(bh.tobytes(), "little")


def hyperkzg_prove(curve_id, ck, d_poly_ptr, point, challenge, stream=0):
    """provider::hyperkzg::EvaluationEngine::prove.  ck: a CommitmentKey on the KZG key; point: ints.  challenge(round, message) -> int
    with round 0 = commitments, 1 = evaluations, 2 = witness commitments.  Returns (com points, v [3][l] ints, w points)."""
    l = len(point)
    pt = np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in point), dtype=np.uint8).copy()
    com = np.zeros(max(1, l - 1) * 96, dtype=np.uint8)
    w = np.zeros(3 * 96, dtype=np.uint8)
    v = np.zeros(3 * l * 32, dtype=np.uint8)
    errors = []
    cb = _callback(challenge, errors)
    rc = _capi.lib().lurk_hyperkzg_prove_dev(curve_id, ck._ctx, C.c_void_p(d_poly_ptr), _capi.np_ptr(pt), l, cb, None, _capi.np_ptr(com),
                                             _capi.np_ptr(w), _capi.np_ptr(v), _capi.FMT_CANONICAL, C.c_void_p(stream))
    if errors:
        raise errors[0]
    _capi.check(rc)

    def pts(buf, k):
        out = []
        for i in range(k):
            b = buf[96 * i:96 * i + 96].tobytes()
            out.append((int.from_bytes(b[:32], "little"), int.from_bytes(b[32:64], "little")) if int.from_bytes(b[64:], "little") else None)
        return out
    vi = _ints(v)
    return pts(com, l - 1), [vi[t * l:(t + 1) * l] for t in range(3)], pts(w, 3)


def batch_eval_reduce(field_id, claims, challenge, d_joint_ptr=None, stream=0):
    """Arecibo's batch_eval_reduce: the claims P_i(x_i) = e_i become one claim about sum_i gamma^i P_i (zero-padded to 2^m) at r.
    claims: [(d_ptr, num_vars, point ints, eval int)], P_i Montgomery on the device (not modified).  challenge(round, message) -> int with
    round 0 = the evaluations (-> rho), 1..m = the sum-check rounds, m + 1 = the L_i (-> gamma).  d_joint_ptr: 2^m elements of device
    memory for the joint polynomial (None: allocated here).  Returns (round_evals, r, claims_left, weights, joint_eval, joint tensor or None)."""
    import torch
    n = len(claims)
    nv = [int(c[1]) for c in claims]
    m = max(nv) if nv else 0
    joint = None
    if d_joint_ptr is None:
        joint = torch.empty((1 << m) * 32, dtype=torch.uint8, device="cuda")
        d_joint_ptr = joint.data_ptr()
    ptrs = (C.c_void_p * max(n, 1))(*[C.c_void_p(c[0]) for c in claims])
    nvs = (C.c_int * max(n, 1))(*nv)
    pts = np.frombuffer(b"".join(int(x).to_bytes(32, "little") for c in claims for x in c[2]) or bytes(32), dtype=np.uint8).copy()
    ev = np.frombuffer(b"".join(int(c[3]).to_bytes(32, "little") for c in claims) or bytes(32), dtype=np.uint8).copy()
    rounds = np.zeros(max(1, m) * 3 * 32, dtype=np.uint8)
    r = np.zeros(max(1, m) * 32, dtype=np.uint8)
    left, w, je = np.zeros(max(1, n) * 32, dtype=np.uint8), np.zeros(max(1, n) * 32, dtype=np.uint8), np.zeros(32, dtype=np.uint8)
    errors = []
    cb = _callback(challenge, errors)
    rc = _capi.lib().lurk_batch_eval_reduce_dev(field_id, n, ptrs, nvs, _capi.np_ptr(pts), _capi.np_ptr(ev), cb, None, _capi.np_ptr(rounds),
                                                _capi.np_ptr(r), _capi.np_ptr(left), _capi.np_ptr(w), _capi.np_ptr(je), C.c_void_p(d_joint_ptr),
                                                _capi.FMT_CANONICAL, C.c_void_p(stream))
    if errors:
        raise errors[0]
    _capi.check(rc)
    ri = _ints(rounds)
    return ([ri[3 * j:3 * j + 3] for j in range(m)], _ints(r)[:m], _ints(left)[:n], _ints(w)[:n], int.from_bytes(je.tobytes(), "little"), joint)



# ------------------------------------------------------------------------------------------------ RelaxedR1CSSNARK::prove, the GPU half
class DeviceCSR:
    """a CSR matrix resident on the GPU (row_ptr u64, col u32, val Montgomery field elements)"""

    def __init__(self, field_id, rows, row_ptr, col, val_canonical):
        import torch
        self.rows = rows
        self.rp = torch.from_numpy(np.ascontiguousarray(row_ptr, dtype=np.uint64).view(np.int64)).cuda()
        self.col = torch.from_numpy(np.ascontiguousarray(col, dtype=np.uint32).view(np.int32)).cuda()
        self.val = torch.from_numpy(np.ascontiguousarray(val_canonical, dtype=np.uint8).reshape(-1)).cuda()
        if self.val.numel():
            _capi.check(_capi.lib().lurk_convert_dev(field_id, C.c_void_p(self.val.data_ptr()), self.val.numel() // 32, _capi.FMT_MONTGOMERY,
                                                     C.c_void_p(self.val.data_ptr()), None))

    def mv(self, field_id, d_z_ptr, d_y_ptr):
        _capi.check(_capi.lib().lurk_spmv_csr_dev(field_id, C.c_void_p(self.rp.data_ptr()), C.c_void_p(self.col.data_ptr()), C.c_void_p(self.val.data_ptr()),
                                                  self.rows, C.c_void_p(d_z_ptr), C.c_void_p(d_y_ptr), None))


def padded_and_transposed(mats, n_w, num_vars, rows_pad):
    """host-side set-up (once per circuit shape): columns re-based onto the padded z = (W | 0.. | u | X | 0..) of length 2 num_vars, and the
    transposes (for compute_eval_table_sparse: sum_row eq(rx)[row] M[row][col]) as CSR over 2 num_vars rows.  mats: [(row_ptr, col, val bytes)]"""
    fwd, tr = [], []
    for rp, col, val in mats:
        rp = np.asarray(rp, dtype=np.uint64)
        col = np.asarray(col, dtype=np.int64)
        colm = np.where(col < n_w, col, num_vars + (col - n_w))
        val = np.ascontiguousarray(val, dtype=np.uint8).reshape(-1, 32)
        nrows = len(rp) - 1
        fwd.append((nrows, rp, colm.astype(np.uint32), val.reshape(-1)))
        row_of = np.repeat(np.arange(nrows, dtype=np.int64), np.diff(rp.astype(np.int64)))
        order = np.argsort(colm, kind="stable")
        trp = np.concatenate([[0], np.cumsum(np.bincount(colm, minlength=2 * num_vars))]).astype(np.uint64)
        tr.append((2 * num_vars, trp, row_of[order].astype(np.uint32), val[order].reshape(-1)))
    return fwd, tr


class RelaxedR1CSProver:
    """Control flow of Arecibo's spartan::snark::RelaxedR1CSSNARK::prove (reached from `compress`, reference src/proof/nova.rs:341-356) over the
    C-ABI primitives, every vector device-resident: multiply_vec (SpMV x3), EqPolynomial::evals, the outer (cubic) and inner (quadratic)
    sum-checks, compute_eval_table_sparse (transposed SpMV x3 + AXPY x2) and the evaluation claims.  The Fiat-Shamir transcript is a
    callable `challenge(label, data) -> int`; the polynomial-commitment openings (hyperkzg_prove / ipa_prove) are separate calls."""

    def __init__(self, field_id, mats, n_w, n_x):
        self.field = field_id
        self.p = int.from_bytes(field_modulus(field_id), "little")
        self.n_w, self.n_x = n_w, n_x
        self.rows = len(mats[0][0]) - 1
        self.log_rows = max(1, (self.rows - 1).bit_length())
        self.num_vars = 1 << max(1, (max(n_w, n_x + 1) - 1).bit_length())
        fwd, tr = padded_and_transposed(mats, n_w, self.num_vars, 1 << self.log_rows)
        self.M = [DeviceCSR(field_id, *m) for m in fwd]
        self.MT = [DeviceCSR(field_id, *m) for m in tr]

    def _mont(self, x):
        return _fe(int(x) * (1 << 256) % self.p)

    def _axpy(self, a, b, r, out):
        _capi.check(_capi.lib().lurk_axpy_dev(self.field, C.c_void_p(a.data_ptr()), C.c_void_p(b.data_ptr()), _capi.np_ptr(self._mont(r)), a.numel() // 32,
                                              C.c_void_p(out.data_ptr()), None))

    def pad_z(self, d_W, u, X):
        """(W | 0.. | u | X | 0..), Montgomery, 2 num_vars elements; d_W: device tensor of n_w Montgomery elements"""
        import torch
        z = torch.zeros(2 * self.num_vars * 32, dtype=torch.uint8, device="cuda")
        z[:self.n_w * 32] = d_W[:self.n_w * 32]
        tail = np.concatenate([self._mont(u)] + [self._mont(x) for x in X])
        z[self.num_vars * 32:self.num_vars * 32 + tail.size] = torch.from_numpy(tail).cuda()
        return z

    def prove(self, d_z, d_E, u, challenge, timings=None):
        """d_z: padded z (pad_z); d_E: device tensor of `rows` Montgomery elements.  Returns the transcript the verifier needs plus the points
        (rx, ry) at which E and W have to be opened."""
        import time
        import torch
        f, p, s, nv = self.field, self.p, self.log_rows, self.num_vars
        n_rows_pad = 1 << s
        t = time.perf_counter

        def mark(name, t0):
            if timings is not None:
                torch.cuda.synchronize()
                timings[name] = timings.get(name, 0.0) + (t() - t0) * 1e3

        t0 = t()
        Az, Bz, Cz = (torch.zeros(n_rows_pad * 32, dtype=torch.uint8, device="cuda") for _ in range(3))
        for M, y in zip(self.M, (Az, Bz, Cz)):
            M.mv(f, d_z.data_ptr(), y.data_ptr())
        E = torch.zeros(n_rows_pad * 32, dtype=torch.uint8, device="cuda")
        E[:self.rows * 32] = d_E[:self.rows * 32]
        uCzE = torch.empty_like(E)
        self._axpy(E, Cz, u, uCzE)
        mark("multiply_vec + u Cz + E", t0)
        t0 = t()
        tau = [challenge("tau", i) % p for i in range(s)]
        eq_tau = torch.empty(n_rows_pad * 32, dtype=torch.uint8, device="cuda")
        eq_evals(f, tau, eq_tau.data_ptr())
        mark("eq(tau)", t0)
        t0 = t()
        work = [eq_tau, Az.clone(), Bz.clone(), uCzE]
        outer_rounds, rx, fin = sumcheck_prove(f, CUBIC, [w.data_ptr() for w in work], s, 0,
                                               lambda rnd, msg: challenge("outer", (rnd, _ints(np.frombuffer(msg, dtype=np.uint8)))) % p)
        mark("outer sum-check", t0)
        t0 = t()
        eq_rx = torch.empty(n_rows_pad * 32, dtype=torch.uint8, device="cuda")
        eq_evals(f, rx, eq_rx.data_ptr())
        claims = (fin[1], fin[2], inner_product(f, Cz.data_ptr(), eq_rx.data_ptr(), n_rows_pad), inner_product(f, E.data_ptr(), eq_rx.data_ptr(), n_rows_pad))
        mark("claims at rx", t0)
        t0 = t()
        r = challenge("inner_r", claims) % p
        ys = [torch.empty(2 * nv * 32, dtype=torch.uint8, device="cuda") for _ in range(3)]
        for M, y in zip(self.MT, ys):
            M.mv(f, eq_rx.data_ptr(), y.data_ptr())
        abc = torch.empty_like(ys[0])
        self._axpy(ys[0], ys[1], r, abc)
        self._axpy(abc, ys[2], r * r % p, abc)
        mark("eval table (transposed SpMV)", t0)
        t0 = t()
        joint = (claims[0] + r * claims[1] + r * r * claims[2]) % p
        zc = d_z.clone()
        inner_rounds, ry, fin2 = sumcheck_prove(f, QUAD, [abc.data_ptr(), zc.data_ptr()], nv.bit_length(), joint,
                                                lambda rnd, msg: challenge("inner", (rnd, _ints(np.frombuffer(msg, dtype=np.uint8)))) % p)
        mark("inner sum-check", t0)
        t0 = t()
        eq_ry = torch.empty(nv * 32, dtype=torch.uint8, device="cuda")
        eq_evals(f, ry[1:], eq_ry.data_ptr())
        eval_W = inner_product(f, d_z.data_ptr(), eq_ry.data_ptr(), nv)
        mark("eval W", t0)
        return dict(outer_rounds=outer_rounds, inner_rounds=inner_rounds, claims=claims, eval_W=eval_W, rx=rx, ry=ry, E_padded=E)


# ------------------------------------------------------------------------------------------------ BatchedRelaxedR1CSSNARK::prove, the GPU half
class BatchedRelaxedR1CSProver:
    """Control flow of Arecibo's spartan::batched::BatchedRelaxedR1CSSNARK::prove -- SuperNova's `compress` over the running instances of
    every circuit index (reference src/proof/supernova.rs:110,293-317) -- over the C-ABI primitives, every vector device-resident.  Each
    circuit keeps one RelaxedR1CSProver for its device matrices, transposes and pad_z.  Instance i has 2^s_i rows and 2^(t_i + 1) entries
    of z; the batched sum-checks let the smaller instances join late.  The challenge labels are those of the test oracle (tests/batched_oracle.py):
      "tau" (N) -> tau, instance i's table eq(tau, tau^2, tau^4, .., tau^(2^(s_i - 1))) (PowPolynomial::evals_with_powers);
      "outer_r" (N) -> the outer coefficients outer_r^i;  "outer" (round, s(0..3)) -> r_x;
      "inner_r" (the claims (Az, Bz, Cz, E)(rx_i) per instance) -> r, coefficients (r^3)^i;  "inner" (round, s(0..2)) -> r_y;
      "batch_eval" (round, message) -> the challenges of batch_eval_reduce over [W_0 .. W_{N-1}, E_0 .. E_{N-1}].
    The opening of the joint polynomial (hyperkzg_prove / ipa_prove) is a separate call."""

    def __init__(self, field_id, circuits):
        """circuits: [(mats, n_w, n_x)] per circuit index, mats as RelaxedR1CSProver takes them"""
        self.field = field_id
        self.p = int.from_bytes(field_modulus(field_id), "little")
        self.provers = [RelaxedR1CSProver(field_id, mats, n_w, n_x) for mats, n_w, n_x in circuits]

    def pad_z(self, i, d_W, u, X):
        return self.provers[i].pad_z(d_W, u, X)

    def prove(self, instances, challenge, timings=None):
        """instances: [(d_z, d_E, u)] per circuit (d_z from pad_z, d_E of `rows` Montgomery elements).  Returns the transcript (outer_rounds,
        inner_rounds, claims, eval_W, reduce_rounds, claims_left), the per-instance points rx / ry, and the reduction's r, weights, joint_eval
        and joint polynomial (device tensor, 2^m Montgomery elements) together with the padded E vectors."""
        import time
        import torch
        f, p, N = self.field, self.p, len(self.provers)
        assert len(instances) == N
        S = [pr.log_rows for pr in self.provers]
        T = [pr.num_vars.bit_length() for pr in self.provers]            # log2 of the padded z = t_i + 1
        t = time.perf_counter

        def mark(name, t0):
            if timings is not None:
                torch.cuda.synchronize()
                timings[name] = timings.get(name, 0.0) + (t() - t0) * 1e3

        def cb(label):
            return lambda rnd, msg: challenge(label, (rnd, _ints(np.frombuffer(msg, dtype=np.uint8)))) % p

        def vec(n):
            return torch.zeros(n * 32, dtype=torch.uint8, device="cuda")

        t0 = t()
        tau = challenge("tau", N) % p
        work, Cz, E = [], [], []
        for pr, s, (d_z, d_E, u) in zip(self.provers, S, instances):
            Az, Bz, cz = vec(1 << s), vec(1 << s), vec(1 << s)
            for M, y in zip(pr.M, (Az, Bz, cz)):
                M.mv(f, d_z.data_ptr(), y.data_ptr())
            e = vec(1 << s)
            e[:pr.rows * 32] = d_E[:pr.rows * 32]
            uCzE = torch.empty_like(e)
            pr._axpy(e, cz, u, uCzE)
            powers = [tau]
            while len(powers) < s:
                powers.append(powers[-1] * powers[-1] % p)
            eq_tau = torch.empty_like(e)
            eq_evals(f, powers, eq_tau.data_ptr())
            work.append([eq_tau, Az, Bz, uCzE])
            Cz.append(cz)
            E.append(e)
        mark("multiply_vec + u Cz + E + eq(tau)", t0)
        t0 = t()
        outer_r = challenge("outer_r", N) % p
        outer_rounds, r_x, fin = sumcheck_prove_batch(f, CUBIC, [([w.data_ptr() for w in ws], s) for ws, s in zip(work, S)], [0] * N,
                                                      [pow(outer_r, i, p) for i in range(N)], cb("outer"))
        del work
        mark("outer sum-check (batched)", t0)
        t0 = t()
        rx = [r_x[len(r_x) - s:] for s in S]
        claims, eq_rx = [], []
        for i, s in enumerate(S):
            q = vec(1 << s)
            eq_evals(f, rx[i], q.data_ptr())
            eq_rx.append(q)
            claims.append((fin[i][1], fin[i][2], inner_product(f, Cz[i].data_ptr(), q.data_ptr(), 1 << s), inner_product(f, E[i].data_ptr(), q.data_ptr(), 1 << s)))
        mark("claims at rx", t0)
        t0 = t()
        r = challenge("inner_r", tuple(claims)) % p
        abc, joint = [], []
        for pr, q, c in zip(self.provers, eq_rx, claims):
            ys = [vec(2 * pr.num_vars) for _ in range(3)]
            for M, y in zip(pr.MT, ys):
                M.mv(f, q.data_ptr(), y.data_ptr())
            a = torch.empty_like(ys[0])
            pr._axpy(ys[0], ys[1], r, a)
            pr._axpy(a, ys[2], r * r % p, a)
            abc.append(a)
            joint.append((c[0] + r * c[1] + r * r * c[2]) % p)
        mark("eval tables (transposed SpMV)", t0)
        t0 = t()
        r3 = pow(r, 3, p)
        zc = [inst[0].clone() for inst in instances]
        inner_rounds, r_y, _ = sumcheck_prove_batch(f, QUAD, [([a.data_ptr(), z.data_ptr()], ti) for a, z, ti in zip(abc, zc, T)], joint,
                                                    [pow(r3, i, p) for i in range(N)], cb("inner"))
        del zc, abc
        mark("inner sum-check (batched)", t0)
        t0 = t()
        ry = [r_y[len(r_y) - ti:] for ti in T]
        eval_W = []
        for pr, (d_z, _, _), y in zip(self.provers, instances, ry):
            q = vec(pr.num_vars)
            eq_evals(f, y[1:], q.data_ptr())
            eval_W.append(inner_product(f, d_z.data_ptr(), q.data_ptr(), pr.num_vars))
        mark("eval W", t0)
        t0 = t()
        be = [(inst[0].data_ptr(), ti - 1, y[1:], ev) for inst, ti, y, ev in zip(instances, T, ry, eval_W)]
        be += [(e.data_ptr(), s, x, c[3]) for e, s, x, c in zip(E, S, rx, claims)]
        red_rounds, r_red, left, weights, joint_eval, d_joint = batch_eval_reduce(f, be, cb("batch_eval"))
        mark("batch_eval_reduce", t0)
        return dict(outer_rounds=outer_rounds, inner_rounds=inner_rounds, claims=claims, eval_W=eval_W, reduce_rounds=red_rounds,
                    claims_left=left, rx=rx, ry=ry, r=r_red, weights=weights, joint_eval=joint_eval, joint=d_joint, E_padded=E)


# ------------------------------------------------------------------------------------------------ the Spartan prover context
_SPARTAN_LABELS = {_capi.SPARTAN_OUTER: "outer", _capi.SPARTAN_INNER: "inner", _capi.SPARTAN_BATCH_EVAL: "batch_eval"}


def _spartan_label(phase, rnd, msg, n, batched):
    """(label, data) of one call of the phase-tagged transcript for challenge(label, data); msg: the message bytes"""
    vals = _ints(np.frombuffer(msg, dtype=np.uint8)) if msg else []
    if phase == _capi.SPARTAN_TAU:
        return "tau", n if batched else rnd
    if phase == _capi.SPARTAN_OUTER_R:
        return "outer_r", n
    if phase == _capi.SPARTAN_CLAIMS:
        claims = tuple(tuple(vals[4 * i:4 * i + 4]) for i in range(n))
        return "inner_r", claims if batched else claims[0]
    return _SPARTAN_LABELS[phase], (rnd, vals)


def _spartan_callback(challenge, p, n, batched, errors):
    """the phase-tagged transcript of lurk_spartan_prove_*_dev mapped onto the labels and data RelaxedR1CSProver, BatchedRelaxedR1CSProver and
    tests/batched_oracle.py use, so that one challenge(label, data) function drives every path"""
    def cb(user, phase, rnd, msg, msg_len, out):
        try:
            x = challenge(*_spartan_label(phase, rnd, C.string_at(msg, msg_len) if msg_len else b"", n, batched))
            for i, byte in enumerate((int(x) % p).to_bytes(32, "little")):
                out[i] = byte
            return 0
        except Exception as e:          # never unwind through the C frames
            errors.append(e)
            return 1
    return _capi.SPARTAN_CHALLENGE_FN(cb)


class SpartanContext:
    """lurk_spartan_ctx: one circuit shape's matrices on the device (and their merged transpose, built there), proving RelaxedR1CSSNARK
    from a running instance (W, u, X), E in one C-ABI call.  mats: [(row_ptr, col, val bytes canonical)] over z = (W, u, X), as
    RelaxedR1CSProver takes them.  verifier_only=True (or SpartanContext.verifier) keeps the matrices alone, without the prover's
    transpose: it verifies, evaluates the matrices and checks recursive proofs (recursive.recursive_verify) as a full context does, and
    the library refuses to prove with it."""

    def __init__(self, field_id, mats, n_w, n_x, verifier_only=False):
        self.field, self.n_w, self.n_x, self.verifier_only = field_id, n_w, n_x, verifier_only
        self.p = int.from_bytes(field_modulus(field_id), "little")
        self.rows = len(mats[0][0]) - 1
        keep = []
        for rp, col, val in mats:
            keep += [np.ascontiguousarray(rp, dtype=np.uint64), np.ascontiguousarray(col, dtype=np.uint32),
                     np.ascontiguousarray(val, dtype=np.uint8).reshape(-1)]
        arr = lambda k: (C.c_void_p * 3)(*[keep[3 * m + k].ctypes.data for m in range(3)])
        ctx = C.c_void_p()
        self._ctx = None
        create = _capi.lib().lurk_spartan_ctx_create_verifier if verifier_only else _capi.lib().lurk_spartan_ctx_create
        _capi.check(create(field_id, n_w, n_x, self.rows, arr(0), arr(1), arr(2), _capi.FMT_CANONICAL, C.byref(ctx)))
        self._ctx = ctx
        lr, lv, jl = C.c_int(), C.c_int(), C.c_size_t()
        _capi.check(_capi.lib().lurk_spartan_ctx_info(ctx, None, C.byref(lr), C.byref(lv), C.byref(jl)))
        self.log_rows, self.log_vars, self.joint_len = lr.value, lv.value, jl.value
        self.num_vars = 1 << self.log_vars

    @classmethod
    def verifier(cls, field_id, mats, n_w, n_x):
        """a verifier-only context (lurk_spartan_ctx_create_verifier)"""
        return cls(field_id, mats, n_w, n_x, verifier_only=True)

    def close(self):
        if self._ctx:
            _capi.lib().lurk_spartan_ctx_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def prove(self, d_z_ptr, d_E_ptr, challenge, d_joint_ptr=None, stream=0):
        """RelaxedR1CSSNARK::prove + batch_eval_reduce([W, E]).  d_z_ptr: (W, u, X) Montgomery (LURK_FOLD_BUF_Z1's layout), d_E_ptr: `rows`
        Montgomery elements; neither is modified.  challenge(label, data) -> int.  Returns the transcript (RelaxedR1CSProver's keys plus
        reduce_rounds, claims_left, r, weights, joint_eval) and `joint` (the device tensor allocated here when d_joint_ptr is None)."""
        return _spartan_prove([self], [(d_z_ptr, d_E_ptr)], challenge, d_joint_ptr, stream, batched=False)

    def eval_table(self, d_eq_ptr, r, d_out_ptr, stream=0):
        """compute_eval_table_sparse alone: d_out[j] = sum_row eq[row] (A + r B + r^2 C)[row][j] over 2 num_vars columns"""
        _capi.check(_capi.lib().lurk_spartan_eval_table_dev(self._ctx, C.c_void_p(d_eq_ptr), _capi.np_ptr(_fe(r)), C.c_void_p(d_out_ptr),
                                                            _capi.FMT_CANONICAL, C.c_void_p(stream)))

    def matrix_evals(self, rx, ry, stream=0):
        """(A(rx, ry), B(rx, ry), C(rx, ry)): rx of log_rows ints, ry of log_vars + 1 ints over the padded z"""
        assert len(rx) == self.log_rows and len(ry) == self.log_vars + 1
        out = np.zeros(96, dtype=np.uint8)
        _capi.check(_capi.lib().lurk_spartan_matrix_evals_dev(self._ctx, _capi.np_ptr(_fes(rx)), _capi.np_ptr(_fes(ry)), _capi.np_ptr(out),
                                                              _capi.FMT_CANONICAL, C.c_void_p(stream)))
        return tuple(_ints(out))

    def verify(self, proof, u, X, challenge, compressed=False, stream=0):
        """RelaxedR1CSSNARK::verify + batch_eval_reduce's verifier through lurk_spartan_verify.  proof: what prove returns (round polynomials as
        evaluations), or with compressed=True every round as its coefficients without the linear one.  Returns (accepted, derived) with derived =
        dict(rx, ry, r, weights, joint_eval) of an accepted proof, else None."""
        return _spartan_verify([self], [(u, X)], proof, challenge, compressed, stream, batched=False)


def spartan_prove_batch(ctxs, instances, challenge, d_joint_ptr=None, stream=0):
    """BatchedRelaxedR1CSSNARK::prove through lurk_spartan_prove_batch_dev.  ctxs: SpartanContext per circuit, instances: [(d_z_ptr, d_E_ptr)].
    Returns what BatchedRelaxedR1CSProver.prove returns (without E_padded)."""
    return _spartan_prove(ctxs, instances, challenge, d_joint_ptr, stream, batched=True)


def spartan_verify_batch(ctxs, insts, proof, challenge, compressed=False, stream=0):
    """BatchedRelaxedR1CSSNARK::verify through lurk_spartan_verify_batch.  insts: [(u, X)] per context; proof as spartan_prove_batch returns
    it.  Returns (accepted, derived) as SpartanContext.verify."""
    return _spartan_verify(ctxs, insts, proof, challenge, compressed, stream, batched=True)


def _spartan_verify(ctxs, insts, proof, challenge, compressed, stream, batched):
    n, p = len(ctxs), ctxs[0].p
    S = [c.log_rows for c in ctxs]
    T = [c.log_vars + 1 for c in ctxs]
    mS, mT = max(S), max(T)
    m = max(mS, mT - 1)
    claims = proof["claims"] if batched else [proof["claims"]]
    eval_W = proof["eval_W"] if batched else [proof["eval_W"]]
    per = 0 if compressed else 1                  # a compressed round drops the linear coefficient
    shapes = (("outer_rounds", mS, 3 + per), ("inner_rounds", mT, 2 + per), ("reduce_rounds", m, 2 + per))
    for key, rounds, width in shapes:
        if len(proof[key]) != rounds or any(len(rnd) != width for rnd in proof[key]):
            raise ValueError(f"{key}: {rounds} rounds of {width} values expected")
    if len(claims) != n or any(len(c) != 4 for c in claims) or len(eval_W) != n or len(proof["claims_left"]) != 2 * n:
        raise ValueError("claims, eval_W or claims_left of the wrong length")
    bufs = {key: _fes(x for rnd in proof[key] for x in rnd) for key, _, _ in shapes}
    bufs.update(claims=_fes(x for c in claims for x in c), eval_W=_fes(eval_W), claims_left=_fes(proof["claims_left"]))
    bufs.update({k: np.zeros(max(1, v) * 32, dtype=np.uint8) for k, v in dict(r_x=mS, r_y=mT, r=m, weights=2 * n, joint_eval=1).items()})
    rec = _capi.SpartanProof(**{k: b.ctypes.data for k, b in bufs.items()})
    us = _fes([u for u, _ in insts])
    xs = [_fes(X) for _, X in insts]
    acc = C.c_int(-1)
    errors = []
    cb = _spartan_callback(challenge, p, n, batched, errors)
    fmt_r = _capi.SPARTAN_ROUNDS_COMPRESSED if compressed else _capi.SPARTAN_ROUNDS_EVALS
    lib = _capi.lib()
    if batched:
        cs = (C.c_void_p * n)(*[c._ctx for c in ctxs])
        xp = (C.c_void_p * n)(*[x.ctypes.data for x in xs])
        rc = lib.lurk_spartan_verify_batch(n, cs, _capi.np_ptr(us), xp, C.byref(rec), fmt_r, cb, None, C.byref(acc), _capi.FMT_CANONICAL, C.c_void_p(stream))
    else:
        rc = lib.lurk_spartan_verify(ctxs[0]._ctx, _capi.np_ptr(us), _capi.np_ptr(xs[0]), C.byref(rec), fmt_r, cb, None, C.byref(acc), _capi.FMT_CANONICAL,
                                     C.c_void_p(stream))
    if errors:
        raise errors[0]
    _capi.check(rc)
    if not acc.value:
        return False, None
    v = {k: _ints(bufs[k]) for k in ("r_x", "r_y", "r", "weights", "joint_eval")}
    r_x, r_y = v["r_x"][:mS], v["r_y"][:mT]
    out = dict(r=v["r"][:m], weights=v["weights"][:2 * n], joint_eval=v["joint_eval"][0])
    if batched:
        out.update(rx=[r_x[mS - s:] for s in S], ry=[r_y[mT - t:] for t in T])
    else:
        out.update(rx=r_x, ry=r_y)
    return True, out


def _spartan_prove(ctxs, instances, challenge, d_joint_ptr, stream, batched):
    import torch
    n, p = len(ctxs), ctxs[0].p
    S = [c.log_rows for c in ctxs]
    T = [c.log_vars + 1 for c in ctxs]
    mS, mT = max(S), max(T)
    m = max(mS, mT - 1)
    joint = None
    if d_joint_ptr is None:
        joint = torch.empty((1 << m) * 32, dtype=torch.uint8, device="cuda")
        d_joint_ptr = joint.data_ptr()
    bufs = dict(outer_rounds=mS * 4, r_x=mS, claims=4 * n, inner_rounds=mT * 3, r_y=mT, eval_W=n, reduce_rounds=m * 3, r=m, claims_left=2 * n,
                weights=2 * n, joint_eval=1)
    bufs = {k: np.zeros(max(1, v) * 32, dtype=np.uint8) for k, v in bufs.items()}
    rec = _capi.SpartanProof(**{k: b.ctypes.data for k, b in bufs.items()})
    errors = []
    cb = _spartan_callback(challenge, p, n, batched, errors)
    lib = _capi.lib()
    if batched:
        cs = (C.c_void_p * n)(*[c._ctx for c in ctxs])
        zs = (C.c_void_p * n)(*[C.c_void_p(z) for z, _ in instances])
        es = (C.c_void_p * n)(*[C.c_void_p(e) for _, e in instances])
        rc = lib.lurk_spartan_prove_batch_dev(n, cs, zs, es, cb, None, C.byref(rec), C.c_void_p(d_joint_ptr), _capi.FMT_CANONICAL, C.c_void_p(stream))
    else:
        rc = lib.lurk_spartan_prove_dev(ctxs[0]._ctx, C.c_void_p(instances[0][0]), C.c_void_p(instances[0][1]), cb, None, C.byref(rec),
                                        C.c_void_p(d_joint_ptr), _capi.FMT_CANONICAL, C.c_void_p(stream))
    if errors:
        raise errors[0]
    _capi.check(rc)
    v = {k: _ints(b) for k, b in bufs.items()}
    r_x, r_y = v["r_x"][:mS], v["r_y"][:mT]
    out = dict(outer_rounds=[v["outer_rounds"][4 * j:4 * j + 4] for j in range(mS)], inner_rounds=[v["inner_rounds"][3 * j:3 * j + 3] for j in range(mT)],
               reduce_rounds=[v["reduce_rounds"][3 * j:3 * j + 3] for j in range(m)], r=v["r"][:m], claims_left=v["claims_left"][:2 * n],
               weights=v["weights"][:2 * n], joint_eval=v["joint_eval"][0], joint=joint)
    claims = [tuple(v["claims"][4 * i:4 * i + 4]) for i in range(n)]
    if batched:
        out.update(claims=claims, eval_W=v["eval_W"][:n], rx=[r_x[mS - s:] for s in S], ry=[r_y[mT - t:] for t in T])
    else:
        out.update(claims=claims[0], eval_W=v["eval_W"][0], rx=r_x, ry=r_y)
    return out
