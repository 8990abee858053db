"""CompressedSNARK::prove (reference src/proof/nova.rs:341-356, supernova.rs:293-317) through the compress context of the C ABI
(lurk_compress_ctx_*, lurk_compress_prove_dev; include/lurk_b200.h): for the primary and the secondary circuit, RelaxedR1CSSNARK::prove (or
SuperNova's BatchedRelaxedR1CSSNARK::prove), batch_eval_reduce, the joint commitment and the opening of the joint polynomial -- HyperKZG or
the inner-product argument -- in one call, the two circuits proved at once on library-owned threads and streams.  CompressedSNARK::verify
(nova.rs:358-373, supernova.rs:304-317) through lurk_compress_verify: the same transcript, the pairing of HyperKZG left to a callback.

The transcript is the caller's: challenge(circuit, label, data) -> int, circuit 0 = primary, 1 = secondary.  The Spartan phases use the labels
and data of spartan.SpartanContext ("tau", "outer_r", "outer", "inner_r", "inner", "batch_eval"); the opening's calls are ("pcs", (round,
message bytes)) -- HyperKZG: rounds 0..2 with the messages of spartan.hyperkzg_prove; IPA: round 0 = comm | joint_eval (-> the scale r of
ck_c), rounds 1..m = L | R."""
import ctypes as C

import numpy as np

from . import _capi
from .spartan import _fes, _ints, _spartan_label

_KINDS = {"hyperkzg": _capi.PCS_HYPERKZG, "ipa": _capi.PCS_IPA}


def _point(P):
    """(x, y) or None (the identity) -> the 96-byte x | y | z, canonical"""
    return _fes([0, 0, 0]) if P is None else _fes([P[0], P[1], 1])


def _points(buf, k):
    out = []
    for i in range(k):
        b = buf[96 * i:96 * i + 96].tobytes()
        out.append((int.from_bytes(b[:32], "little"), int.from_bytes(b[32:64], "little")) if int.from_bytes(b[64:], "little") else None)
    return out


def _transcript(challenge, circuits, native, errors):
    """(lurk_compress_challenge_fn, user) for challenge(circuit, label, data), or native's; circuits: [(Spartan contexts, batched)] of the
    primary and the secondary.  Exceptions of `challenge` go to `errors` and abort the call."""
    if native:
        return (native[0] if isinstance(native[0], _capi.COMPRESS_CHALLENGE_FN) else _capi.COMPRESS_CHALLENGE_FN(native[0])), native[1]
    ps = [ctxs[0].p for ctxs, _ in circuits]

    def cb(user, circuit, phase, rnd, msg, msg_len, out):
        try:
            ctxs, bat = circuits[circuit]
            data = C.string_at(msg, msg_len) if msg_len else b""
            if phase == _capi.SPARTAN_PCS:
                x = challenge(circuit, "pcs", (rnd, data))
            else:
                x = challenge(circuit, *_spartan_label(phase, rnd, data, len(ctxs), bat))
            for i, byte in enumerate((int(x) % ps[circuit]).to_bytes(32, "little")):
                out[i] = byte
            return 0
        except Exception as e:          # never unwind through the C frames
            errors.append(e)
            return 1
    return _capi.COMPRESS_CHALLENGE_FN(cb), None


class CompressContext:
    """lurk_compress_ctx: the Spartan contexts of both circuits and their evaluation engines, with the scratch of the openings kept between
    proofs.  primary: a SpartanContext (Nova) or a list of them (SuperNova's circuits, distinct); secondary: a SpartanContext.  pcs_primary /
    pcs_secondary: ("hyperkzg", CommitmentKey on the KZG key) or ("ipa", CommitmentKey, ck_c as an (x, y) of canonical ints, unscaled).
    The contexts and keys are borrowed and must outlive this one."""

    def __init__(self, primary, secondary, pcs_primary, pcs_secondary):
        self._ctx = None
        self.primary = list(primary) if isinstance(primary, (list, tuple)) else [primary]
        self.secondary = secondary
        self._keep = [self.primary, secondary, pcs_primary, pcs_secondary]
        self.kinds = [pcs_primary[0], pcs_secondary[0]]
        pcs = []
        for spec in (pcs_primary, pcs_secondary):
            gc = _fes([spec[2][0], spec[2][1]]) if spec[0] == "ipa" else None
            self._keep.append(gc)
            pcs.append(_capi.CompressPcs(_KINDS[spec[0]], spec[1]._ctx, gc.ctypes.data if gc is not None else None))
        arr = (C.c_void_p * len(self.primary))(*[c._ctx for c in self.primary])
        ctx = C.c_void_p()
        _capi.check(_capi.lib().lurk_compress_ctx_create(len(self.primary), arr, secondary._ctx, C.byref(pcs[0]), C.byref(pcs[1]), _capi.FMT_CANONICAL,
                                                         C.byref(ctx)))
        self._ctx = ctx

    def info(self):
        """device bytes held (0 before the first proof) and the joint-polynomial lengths"""
        b, jp, js = C.c_size_t(), C.c_size_t(), C.c_size_t()
        _capi.check(_capi.lib().lurk_compress_ctx_info(self._ctx, C.byref(b), C.byref(jp), C.byref(js)))
        return dict(device_bytes=b.value, joint_len_primary=jp.value, joint_len_secondary=js.value)

    def close(self):
        if self._ctx:
            _capi.lib().lurk_compress_ctx_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def prove(self, primary, secondary, challenge, batched=None, sequential=False, stream=0, native=None):
        """primary: [(d_z_ptr, d_E_ptr, comm_W, comm_E)] per primary context (d_z / d_E laid out as LURK_FOLD_BUF_Z1 / E1, not modified;
        commitments (x, y) or None); secondary: one such tuple.  batched: BatchedRelaxedR1CSSNARK for the primary (default: more than one
        primary context).  native: (a _capi.COMPRESS_CHALLENGE_FN or the address of a C function of that type, user pointer) to call
        instead of `challenge`.  Returns [primary proof, secondary proof], each the dict spartan.SpartanContext.prove returns
        (without `joint`) plus `comm` and the opening: com, v, w (HyperKZG) or L, R, a_final, b_final (IPA)."""
        n = len(self.primary)
        assert len(primary) == n
        batched = n > 1 if batched is None else batched
        circuits = [(self.primary, batched, primary), ([self.secondary], False, [secondary])]
        rec = _capi.CompressProof()
        bufs = []
        for k, (ctxs, _, _) in enumerate(circuits):
            nk = len(ctxs)
            S, T = [c.log_rows for c in ctxs], [c.log_vars + 1 for c in ctxs]
            m = max(max(S), max(T) - 1)
            sizes = dict(outer_rounds=max(S) * 4, r_x=max(S), claims=4 * nk, inner_rounds=max(T) * 3, r_y=max(T), eval_W=nk, reduce_rounds=m * 3, r=m,
                         claims_left=2 * nk, weights=2 * nk, joint_eval=1)
            b = {key: np.zeros(max(1, v) * 32, dtype=np.uint8) for key, v in sizes.items()}
            opening = dict(comm=3, com=3 * max(1, m - 1), w=9, v=3 * m) if self.kinds[k] == "hyperkzg" else dict(comm=3, L=3 * m, R=3 * m, a_final=1,
                                                                                                               b_final=1)
            o = {key: np.zeros(v * 32, dtype=np.uint8) for key, v in opening.items()}
            cp = rec.primary if k == 0 else rec.secondary
            cp.snark = _capi.SpartanProof(**{key: v.ctypes.data for key, v in b.items()})
            for key, v in o.items():
                setattr(cp, key, v.ctypes.data)
            bufs.append((b, o, S, T, m))
        ptr_arr = lambda vals: (C.c_void_p * n)(*[C.c_void_p(v) for v in vals])
        pts = [_point(x[2]) for x in primary] + [_point(x[3]) for x in primary] + [_point(secondary[2]), _point(secondary[3])]
        cw = (C.c_void_p * n)(*[p.ctypes.data for p in pts[:n]])
        ce = (C.c_void_p * n)(*[p.ctypes.data for p in pts[n:2 * n]])
        errors = []
        fn, user = _transcript(challenge, [(ctxs, bat) for ctxs, bat, _ in circuits], native, errors)
        flags = (_capi.COMPRESS_SEQUENTIAL if sequential else 0) | (_capi.COMPRESS_BATCHED if batched else 0)
        rc = _capi.lib().lurk_compress_prove_dev(self._ctx, n, ptr_arr([x[0] for x in primary]), ptr_arr([x[1] for x in primary]), cw, ce,
                                                 C.c_void_p(secondary[0]), C.c_void_p(secondary[1]), C.c_void_p(pts[2 * n].ctypes.data),
                                                 C.c_void_p(pts[2 * n + 1].ctypes.data), fn, user, flags, C.byref(rec), _capi.FMT_CANONICAL, C.c_void_p(stream))
        if errors:
            raise errors[0]
        _capi.check(rc)
        return [self._result(k, bufs[k], len(circuits[k][0]), circuits[k][1]) for k in range(2)]

    def _result(self, k, bufs, nk, batched):
        b, o, S, T, m = bufs
        mS, mT = max(S), max(T)
        v = {key: _ints(x) for key, x in b.items()}
        r_x, r_y = v["r_x"][:mS], v["r_y"][:mT]
        out = dict(outer_rounds=[v["outer_rounds"][4 * j:4 * j + 4] for j in range(mS)], inner_rounds=[v["inner_rounds"][3 * j:3 * j + 3] for j in range(mT)],
                   reduce_rounds=[v["reduce_rounds"][3 * j:3 * j + 3] for j in range(m)], r=v["r"][:m], claims_left=v["claims_left"][:2 * nk],
                   weights=v["weights"][:2 * nk], joint_eval=v["joint_eval"][0], comm=_points(o["comm"], 1)[0])
        claims = [tuple(v["claims"][4 * i:4 * i + 4]) for i in range(nk)]
        if batched:
            out.update(claims=claims, eval_W=v["eval_W"][:nk], rx=[r_x[mS - s:] for s in S], ry=[r_y[mT - t:] for t in T])
        else:
            out.update(claims=claims[0], eval_W=v["eval_W"][0], rx=r_x, ry=r_y)
        if self.kinds[k] == "hyperkzg":
            vi = _ints(o["v"])
            out.update(com=_points(o["com"], m - 1), w=_points(o["w"], 3), v=[vi[t * m:(t + 1) * m] for t in range(3)])
        else:
            out.update(L=_points(o["L"], m), R=_points(o["R"], m), a_final=_ints(o["a_final"])[0], b_final=_ints(o["b_final"])[0])
        return out


def compress_prove(ctx, primary, secondary, challenge, **kw):
    """CompressContext.prove as a function"""
    return ctx.prove(primary, secondary, challenge, **kw)



def _flat(rounds):
    return _fes([x for rnd in rounds for x in rnd])


def _point_list(pts):
    return np.concatenate([_point(P) for P in pts]) if pts else np.zeros(96, dtype=np.uint8)


def compress_verify(primary, secondary, pcs_primary, pcs_secondary, instances, instance2, proof, challenge, pairing=None, batched=None,
                    sequential=False, compressed=False, stream=0, native=None, native_pairing=None):
    """CompressedSNARK::verify through lurk_compress_verify.  primary: a SpartanContext (Nova) or a list of them (SuperNova), secondary: a
    SpartanContext; full or verifier-only.  pcs_primary / pcs_secondary: ("hyperkzg", g) with g the KZG key's first base as (x, y), or ("ipa",
    CommitmentKey, ck_c as (x, y), unscaled).  instances: [(u, X, comm_W, comm_E)] per primary context; instance2: the secondary's (u, X,
    comm_W, comm_E) of f_U_secondary, the last fold already made.  proof: [primary, secondary] as compress_prove returns them (with
    compressed=True their round polynomials as CompressedUniPoly: every coefficient but the linear one).  challenge(circuit, label, data) ->
    int as for compress_prove; pairing(circuit, P, Q) -> bool, P and Q as (x, y) or None, answers e(P, H) == e(Q, beta H).  native /
    native_pairing: (a C function or its address, user pointer) and a C function or its address, called instead of `challenge` / `pairing`.
    Returns (accepted, [(snark_ok, eval_ok, opening_ok) of the primary, of the secondary]), -1 for a check not reached."""
    ctxs = list(primary) if isinstance(primary, (list, tuple)) else [primary]
    n = len(ctxs)
    assert len(instances) == n
    batched = n > 1 if batched is None else batched
    circuits = [(ctxs, batched), ([secondary], False)]
    kinds = [pcs_primary[0], pcs_secondary[0]]
    keep, rec, vk = [], _capi.CompressProof(), []
    for k, (pr, spec) in enumerate(zip(proof, (pcs_primary, pcs_secondary))):
        bat = circuits[k][1]
        claims = pr["claims"] if bat else [pr["claims"]]
        eval_W = pr["eval_W"] if bat else [pr["eval_W"]]
        b = dict(outer_rounds=_flat(pr["outer_rounds"]), claims=_flat(claims), inner_rounds=_flat(pr["inner_rounds"]), eval_W=_fes(eval_W),
                 reduce_rounds=_flat(pr["reduce_rounds"]), claims_left=_fes(pr["claims_left"]))
        if spec[0] == "hyperkzg":
            o = dict(com=_point_list(pr["com"]), v=_flat(pr["v"]), w=_point_list(pr["w"]))
            g = _fes([spec[1][0], spec[1][1]])
            vk.append(_capi.CompressVkPcs(_capi.PCS_HYPERKZG, None, None, g.ctypes.data))
        else:
            o = dict(L=_point_list(pr["L"]), R=_point_list(pr["R"]), a_final=_fes([pr["a_final"]]))
            g = _fes([spec[2][0], spec[2][1]])
            vk.append(_capi.CompressVkPcs(_capi.PCS_IPA, spec[1]._ctx, g.ctypes.data, None))
        keep += [b, o, g]
        cp = rec.primary if k == 0 else rec.secondary
        cp.snark = _capi.SpartanProof(**{key: v.ctypes.data for key, v in b.items()})
        for key, v in o.items():
            setattr(cp, key, v.ctypes.data)
    us = _fes([x[0] for x in instances])
    xs = [_fes(x[1]) for x in instances] + [_fes(instance2[1])]
    pts = [_point(x[2]) for x in instances] + [_point(x[3]) for x in instances] + [_point(instance2[2]), _point(instance2[3])]
    u2 = _fes([instance2[0]])
    arr = lambda vals: (C.c_void_p * n)(*[C.c_void_p(v) for v in vals])
    errors = []
    fn, user = _transcript(challenge, circuits, native, errors)

    def pcb(user, circuit, P, Q, holds):
        try:
            pq = _points(np.ctypeslib.as_array(P, (96,)), 1) + _points(np.ctypeslib.as_array(Q, (96,)), 1)
            holds[0] = 1 if pairing(circuit, *pq) else 0
            return 0
        except Exception as e:          # never unwind through the C frames
            errors.append(e)
            return 1
    if native_pairing:
        pfn = native_pairing if isinstance(native_pairing, _capi.PAIRING_CHECK_FN) else _capi.PAIRING_CHECK_FN(native_pairing)
    else:
        pfn = _capi.PAIRING_CHECK_FN(pcb) if pairing else _capi.PAIRING_CHECK_FN()
    flags = (_capi.COMPRESS_SEQUENTIAL if sequential else 0) | (_capi.COMPRESS_BATCHED if batched else 0)
    verdicts, acc = (_capi.CompressVerdict * 2)(), C.c_int(-1)
    rc = _capi.lib().lurk_compress_verify(n, arr([c._ctx.value for c in ctxs]), secondary._ctx, C.byref(vk[0]), C.byref(vk[1]), C.c_void_p(us.ctypes.data),
                                          arr([x.ctypes.data for x in xs[:n]]), arr([p.ctypes.data for p in pts[:n]]),
                                          arr([p.ctypes.data for p in pts[n:2 * n]]), C.c_void_p(u2.ctypes.data), C.c_void_p(xs[n].ctypes.data),
                                          C.c_void_p(pts[2 * n].ctypes.data), C.c_void_p(pts[2 * n + 1].ctypes.data), C.byref(rec),
                                          _capi.SPARTAN_ROUNDS_COMPRESSED if compressed else _capi.SPARTAN_ROUNDS_EVALS, fn, pfn, user, flags, verdicts,
                                          C.byref(acc), _capi.FMT_CANONICAL, C.c_void_p(stream))
    if errors:
        raise errors[0]
    _capi.check(rc)
    return bool(acc.value), [(v.snark_ok, v.eval_ok, v.opening_ok) for v in verdicts]


def point_combination_batch(curve, groups, fmt=_capi.FMT_CANONICAL, stream=0):
    """sum_j s_j P_j for each group, all groups in one lurk_point_combination_batch call on the GPU (ordered on `stream`; returns when
    done).  groups: [(points, scalars)] with 1 .. POINT_COMBINATION_MAX_TERMS terms each -- points as k x 96 bytes x | y | z of the
    header's form and scalars as k x 32 bytes, both in `fmt` (uint8 arrays), or, in FMT_CANONICAL, as lists of (x, y) / None and of
    ints.  Returns an (n_groups, 96) uint8 array: per group the bytes lurk_point_combination writes (decode canonical ones with
    points_of)."""
    counts, pts, scs = [], [], []
    for points, scalars in groups:
        if not isinstance(points, np.ndarray) or not isinstance(scalars, np.ndarray):
            assert fmt == _capi.FMT_CANONICAL, "lists of points and scalars are canonical integers"
        p = np.ascontiguousarray(points, dtype=np.uint8).reshape(-1) if isinstance(points, np.ndarray) else list(points)
        s = np.ascontiguousarray(scalars, dtype=np.uint8).reshape(-1) if isinstance(scalars, np.ndarray) else list(scalars)
        p = _point_list(p) if isinstance(p, list) and p else p          # an empty list stays empty, and is refused below
        s = _fes(s) if isinstance(s, list) and s else s
        k = len(p) // 96
        if k == 0 or len(p) != 96 * k or len(s) != 32 * k:
            raise ValueError(f"a group needs k >= 1 points of 96 bytes and k scalars of 32 bytes, got {len(p)} and {len(s)} bytes")
        counts.append(k)
        pts.append(p)
        scs.append(s)
    if not counts:
        raise ValueError("at least one group")
    c = np.array(counts, dtype=np.uint32)
    p, s = np.concatenate(pts), np.concatenate(scs)
    out = np.zeros((len(counts), 96), dtype=np.uint8)
    _capi.check(_capi.lib().lurk_point_combination_batch(curve, len(counts), _capi.np_ptr(c), _capi.np_ptr(p), _capi.np_ptr(s), fmt,
                                                          _capi.np_ptr(out), C.c_void_p(stream)))
    return out


def points_of(out):
    """canonical 96-byte points (as point_combination_batch returns them) -> [(x, y) or None]"""
    b = np.ascontiguousarray(out, dtype=np.uint8).reshape(-1)
    return _points(b, len(b) // 96)
