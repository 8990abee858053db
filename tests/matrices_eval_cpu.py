"""Test infrastructure, NOT product code: ctypes front end of tests/csrc/matrices_eval_cpu.c, the OpenMP port of oracle/spartan.py:
matrices_eval (the full-size checker of sp_matrix_eval_kernel and its CPU baseline).  Compiled with gcc into a temporary directory on first
use, so nothing is written into the tree."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="matrices_eval_cpu_"), "libmatrices_eval_cpu.so")
        subprocess.check_call(["/usr/bin/gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-shared", "-Wall", "-Werror",
                               os.path.join(_HERE, "csrc", "matrices_eval_cpu.c"), "-o", out])
        _LIB = C.CDLL(out)
        _LIB.matrices_eval_cpu.restype = C.c_int
        _LIB.matrices_eval_cpu.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                           C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        _LIB.matrices_eval_cpu_threads.restype = C.c_int
    return _LIB


def threads():
    return lib().matrices_eval_cpu_threads()


def _fes(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals) or bytes(32), dtype=np.uint8).copy()


def matrices_eval(p, mats, n_w, num_vars, rx, ry, nthreads=0):
    """(A, B, C)(rx, ry) as ints.  mats: [(row_ptr, col, val bytes canonical)] over z = (W, u, X), as SpartanContext takes them."""
    keep = []
    for rp, col, val in mats:
        keep += [np.ascontiguousarray(rp, dtype=np.uint64), np.ascontiguousarray(col, dtype=np.uint32),
                 np.ascontiguousarray(val, dtype=np.uint8).reshape(-1)]
    arr = lambda k: (C.c_void_p * 3)(*[keep[3 * m + k].ctypes.data for m in range(3)])
    rows = len(keep[0]) - 1
    bp, bx, by = _fes([p]), _fes(rx), _fes(ry)
    out = np.zeros(96, dtype=np.uint8)
    rc = lib().matrices_eval_cpu(bp.ctypes.data, rows, n_w, num_vars, arr(0), arr(1), arr(2), bx.ctypes.data, len(rx), by.ctypes.data, len(ry),
                                 out.ctypes.data, nthreads)
    if rc != 0:
        raise ValueError(f"matrices_eval_cpu failed ({rc})")
    return tuple(int.from_bytes(out[32 * m:32 * m + 32].tobytes(), "little") for m in range(3))
