"""The Spartan prover context (lurk_spartan_ctx_*, lurk_spartan_prove_*_dev in include/lurk_b200.h, N4) on the CPU: every malformed
argument is refused with LURK_ERR_ARG and a message before any device work, a well-formed call without a GPU fails with
LURK_ERR_NOGPU (there is no CPU fallback), and the header drives the library from plain C99 (tests/csrc/spartan_client.c)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def tiny_matrices():
    """A = B = C = identity on the first two columns of z = (W0, W1, u, X0, X1): two rows"""
    rp = np.array([0, 1, 2], dtype=np.uint64)
    col = np.array([0, 1], dtype=np.uint32)
    val = np.zeros(64, dtype=np.uint8)
    val[0] = val[32] = 1
    return [(rp, col, val)] * 3


def create(L, field=0, n_w=2, n_x=2, rows=2, mats=None, fmt=0, null=None):
    E = L._capi
    mats = tiny_matrices() if mats is None else mats
    arr = lambda k: (C.c_void_p * 3)(*[0 if null == (k, m) else mats[m][k].ctypes.data for m in range(3)])
    ctx = C.c_void_p()
    rc = E.lib().lurk_spartan_ctx_create(field, n_w, n_x, rows, arr(0), arr(1), arr(2), fmt, C.byref(ctx))
    return rc, ctx


@pytest.mark.parametrize("bad", [dict(field=9), dict(fmt=3), dict(rows=0), dict(rows=1 << 30), dict(n_w=1 << 31), dict(null=(0, 1)), dict(null=(1, 2)),
                                 dict(null=(2, 0)), dict(n_w=0, n_x=0)],
                         ids=["unknown-field", "bad-format", "no-rows", "2^30-rows", "huge-W", "null-row_ptr", "null-col", "null-val",
                              "column-out-of-range"])
def test_create_refuses_bad_arguments(L, bad):
    rc, ctx = create(L, **bad)
    assert rc == L._capi.ERR_ARG and not ctx.value
    assert len(L._capi.lib().lurk_last_error()) > 0


def test_create_refuses_a_decreasing_row_ptr_and_a_null_out(L):
    mats = tiny_matrices()
    bad = (np.array([0, 2, 1], dtype=np.uint64), mats[0][1], mats[0][2])
    assert create(L, mats=[bad, mats[1], mats[2]])[0] == L._capi.ERR_ARG
    assert b"row_ptr" in L._capi.lib().lurk_last_error()
    arr = (C.c_void_p * 3)(*[m[0].ctypes.data for m in mats])
    assert L._capi.lib().lurk_spartan_ctx_create(0, 2, 2, 2, arr, arr, arr, 0, None) == L._capi.ERR_ARG


def prove(L, n=1, ctx=True, z=True, e=True, cb=True, out=True, joint=True, fmt=0, arrays=True, batched=True):
    """a prover call with one argument broken at a time; the context is a stand-in pointer (never dereferenced on the refusal paths
    exercised here: they come before any use of the context)"""
    E = L._capi
    buf = np.zeros(4096, dtype=np.uint8)
    fn = E.SPARTAN_CHALLENGE_FN(lambda *a: 0) if cb else E.SPARTAN_CHALLENGE_FN()
    rec = E.SpartanProof()
    k = max(n, 1)
    ptr = lambda ok: C.c_void_p(buf.ctypes.data if ok else 0)
    if batched:
        cs = (C.c_void_p * k)(*[ptr(ctx)] * k) if arrays else None
        zs = (C.c_void_p * k)(*[ptr(z)] * k)
        es = (C.c_void_p * k)(*[ptr(e)] * k)
        return E.lib().lurk_spartan_prove_batch_dev(n, cs, zs, es, fn, None, C.byref(rec) if out else None, ptr(joint), fmt, None)
    return E.lib().lurk_spartan_prove_dev(ptr(ctx), ptr(z), ptr(e), fn, None, C.byref(rec) if out else None, ptr(joint), fmt, None)


@pytest.mark.parametrize("batched", [False, True], ids=["plain", "batched"])
@pytest.mark.parametrize("bad,message", [(dict(z=False), b"d_z"), (dict(e=False), b"d_E"), (dict(cb=False), b"callback"), (dict(out=False), b"proof record"),
                                         (dict(joint=False), b"d_joint"), (dict(fmt=2), b"format")],
                         ids=["null-z", "null-E", "null-callback", "null-out", "null-joint", "bad-format"])
def test_prove_refuses_bad_arguments(L, batched, bad, message):
    assert prove(L, batched=batched, **bad) == L._capi.ERR_ARG
    assert message in L._capi.lib().lurk_last_error()


@pytest.mark.parametrize("bad,message", [(dict(n=0), b"instances"), (dict(n=31), b"instances"), (dict(arrays=False), b"instance array"),
                                         (dict(ctx=False), b"context")],
                         ids=["no-instance", "31-instances", "null-contexts", "null-context"])
def test_batched_prove_refuses_bad_counts_and_contexts(L, bad, message):
    assert prove(L, **bad) == L._capi.ERR_ARG
    assert message in L._capi.lib().lurk_last_error()


def test_plain_prove_refuses_a_null_context_and_info_needs_one(L):
    assert prove(L, ctx=False, batched=False) == L._capi.ERR_ARG
    assert b"context" in L._capi.lib().lurk_last_error()
    assert L._capi.lib().lurk_spartan_ctx_info(None, None, None, None, None) == L._capi.ERR_ARG
    r = np.zeros(32, dtype=np.uint8)
    assert L._capi.lib().lurk_spartan_eval_table_dev(None, None, L._capi.np_ptr(r), None, 0, None) == L._capi.ERR_ARG
    L._capi.lib().lurk_spartan_ctx_destroy(None)          # a no-op, like free(NULL)


def test_valid_create_without_gpu_fails_loudly(L):
    if L._capi.lib().lurk_device_count() > 0:
        pytest.skip("GPU present")
    rc, ctx = create(L)
    assert rc == L._capi.ERR_NOGPU and not ctx.value
    assert b"GPU" in L._capi.lib().lurk_last_error() or len(L._capi.lib().lurk_last_error()) > 0


def build_client(tmp_path):
    exe = str(tmp_path / "spartan_client")
    libdir = os.path.join(ROOT, "lurk-beta_b200")
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "csrc", "spartan_client.c"), "-o", exe, "-L", libdir, "-llurk_b200", "-Wl,-rpath," + libdir])
    return exe


def test_plain_c_client_fails_loudly_without_gpu(L, tmp_path):
    """tests/csrc/spartan_client.c, built as strict C99: the refusals hold, and without a CUDA device the context cannot be created"""
    if L._capi.lib().lurk_device_count() > 0:
        pytest.skip("GPU present (tests/test_gpu_spartan_ctx.py runs the client there)")
    out = subprocess.run([build_client(tmp_path)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    assert "spartan_client ok (no GPU: compute entry points fail loudly)" in out.stdout
