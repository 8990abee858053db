"""The satisfiability checks of RecursiveSNARK::verify (Proof::verify on a Recursive proof, reference src/proof/nova.rs:358-373,
supernova.rs:304-317) through lurk_recursive_verify / lurk_recursive_verify_dev (include/lurk_b200.h): R1CSShape::is_sat_relaxed on every
running instance and is_sat on the secondary's last fresh instance -- the R1CS rows and the recomputed commitments -- in one call.
The RO hash checks stay with the caller."""
import ctypes as C

import numpy as np

from . import _capi
from .spartan import field_modulus


def _point(P, curve_id, fmt):
    """(x, y) of canonical ints or None (the identity) -> the 96-byte x | y | 1 (0 | 0 | 0 for the identity) in `fmt`"""
    if P is None:
        return np.zeros(96, dtype=np.uint8)
    vals = [P[0], P[1], 1]
    if fmt == _capi.FMT_MONTGOMERY:
        p = int.from_bytes(field_modulus(curve_id ^ 1), "little")      # the base field of curve k is field k ^ 1
        vals = [v * (1 << 256) % p for v in vals]
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint8).copy()


def recursive_verify(instances, fmt=_capi.FMT_CANONICAL, device=True, stream=0):
    """instances: dicts with shape (a SpartanContext, full or verifier-only), ck (a CommitmentKey on the curve of the shape's field), z,
    E (None for a strict instance), comm_W and comm_E ((x, y) of canonical ints, None = the identity; comm_E unused for a strict instance).
    device=True: z and E are device pointers to Montgomery elements (LURK_FOLD_BUF_Z1 / _E1 / _W2 of a fold context) and `fmt` only says
    how the commitments are passed; device=False: z and E are host byte arrays in `fmt`.  One call per proof: Nova [r_U_primary,
    r_U_secondary, l_u_secondary], SuperNova the running primaries then the secondary's two.  Returns (accepted, verdicts), a verdict being
    dict(bad_rows, first_bad_row (None when every row holds), u_ok, comm_W_ok, comm_E_ok)."""
    n = len(instances)
    arr = (_capi.RecursiveInstance * max(1, n))()
    keep = []
    for i, x in enumerate(instances):
        strict = x.get("E") is None
        cw = _point(x["comm_W"], x["ck"].curve_id, fmt)
        ce = None if strict else _point(x.get("comm_E"), x["ck"].curve_id, fmt)
        vec = []
        for v in (x["z"], None if strict else x["E"]):
            if v is None or device:
                vec.append(v)
            else:
                a = np.ascontiguousarray(v, dtype=np.uint8).reshape(-1)
                keep.append(a)
                vec.append(a.ctypes.data)
        keep += [cw, ce]
        arr[i] = _capi.RecursiveInstance(x["shape"]._ctx, x["ck"]._ctx, vec[0], vec[1], cw.ctypes.data, None if ce is None else ce.ctypes.data)
    out = (_capi.RecursiveVerdict * max(1, n))()
    acc = C.c_int()
    call = _capi.lib().lurk_recursive_verify_dev if device else _capi.lib().lurk_recursive_verify
    _capi.check(call(n, arr, out, C.byref(acc), fmt, C.c_void_p(stream)))
    verdicts = [dict(bad_rows=v.bad_rows, first_bad_row=None if v.first_bad_row == 2**64 - 1 else v.first_bad_row, u_ok=bool(v.u_ok),
                     comm_W_ok=bool(v.comm_W_ok), comm_E_ok=bool(v.comm_E_ok)) for v in out[:n]]
    return bool(acc.value), verdicts
