"""The recursive verifier (lurk_recursive_verify, lurk_recursive_verify_dev) and the verifier-only Spartan context
(lurk_spartan_ctx_create_verifier) on the CPU: the symbols are exported, every malformed argument is refused with LURK_ERR_ARG and a
message before any CUDA call, and a well-formed call without a GPU fails with LURK_ERR_NOGPU (there is no CPU fallback)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("lurk_recursive_verify", "lurk_recursive_verify_dev", "lurk_spartan_ctx_create_verifier")


def no_gpu(L):
    if L._capi.lib().lurk_device_count() > 0:
        pytest.skip("GPU present (tests/test_gpu_recursive_verify.py covers the device paths)")


def test_symbols_are_exported(L):
    lib = C.CDLL(L._capi.LIB_PATH)
    for s in SYMBOLS:
        assert hasattr(lib, s), s
        assert s in L._capi.PROTOTYPES, s


def verify(L, dev=True, n=3, inst=True, out=True, acc=True, fmt=0, drop=None, strict_with_comm_E=False, relaxed_without_comm_E=False):
    """stand-in pointers everywhere: the shapes and keys are only read after the GPU check"""
    E = L._capi
    buf = np.zeros(4096, dtype=np.uint8)
    p = lambda k: buf.ctypes.data + 64 * k
    k = max(n, 1)
    arr = (E.RecursiveInstance * k)(*[E.RecursiveInstance(p(0), p(1), p(2), p(3), p(4), p(5)) for _ in range(k)])
    arr[k - 1].E, arr[k - 1].comm_E = None, None                  # a strict instance last, as l_u_secondary
    if drop:
        setattr(arr[0], drop, None)
    if strict_with_comm_E:
        arr[k - 1].comm_E = p(5)
    if relaxed_without_comm_E:
        arr[0].comm_E = None
    verdicts = (E.RecursiveVerdict * k)()
    a = C.c_int(7)
    fn = E.lib().lurk_recursive_verify_dev if dev else E.lib().lurk_recursive_verify
    return fn(n, arr if inst else None, verdicts if out else None, C.byref(a) if acc else None, fmt, None)


CASES = [(dict(n=0), b"instances"), (dict(n=33), b"instances"), (dict(inst=False), b"instance array"), (dict(out=False), b"verdict"),
         (dict(acc=False), b"accepted"), (dict(fmt=2), b"format"), (dict(drop="shape"), b"shape"), (dict(drop="ck"), b"key"),
         (dict(drop="z"), b"null z"), (dict(drop="comm_W"), b"comm_W"), (dict(drop="E"), b"go together"),
         (dict(strict_with_comm_E=True), b"go together"), (dict(relaxed_without_comm_E=True), b"go together")]
IDS = ["no-instance", "33-instances", "null-instances", "null-verdicts", "null-accepted", "bad-format", "null-shape", "null-key", "null-z",
       "null-comm_W", "E-without-comm_E", "strict-with-comm_E", "relaxed-without-comm_E"]


@pytest.mark.parametrize("dev", [True, False], ids=["dev", "host"])
@pytest.mark.parametrize("bad,message", CASES, ids=IDS)
def test_verify_refuses_bad_arguments(L, dev, bad, message):
    assert verify(L, dev=dev, **bad) == L._capi.ERR_ARG
    assert message in L._capi.lib().lurk_last_error()


def test_verify_fails_loudly_without_gpu(L):
    no_gpu(L)
    for dev in (True, False):
        for n in (1, 3, 32):
            assert verify(L, dev=dev, n=n) == L._capi.ERR_NOGPU
    assert b"GPU" in L._capi.lib().lurk_last_error() or b"CUDA" in L._capi.lib().lurk_last_error()


def create_verifier(L, out=True, mats=True, field=0, fmt=0, rows=2, bad_col=False, decreasing=False):
    rp = np.array([0, 1, 2] if not decreasing else [0, 2, 1], dtype=np.uint64)
    col = np.array([0, 9 if bad_col else 1], dtype=np.uint32)
    val = np.zeros(64, dtype=np.uint8)
    val[0] = val[32] = 1
    arr = lambda a: (C.c_void_p * 3)(*[a.ctypes.data] * 3)
    ctx = C.c_void_p()
    rc = L._capi.lib().lurk_spartan_ctx_create_verifier(field, 2, 1, rows, arr(rp) if mats else None, arr(col), arr(val), fmt,
                                                         C.byref(ctx) if out else None)
    return rc, ctx


@pytest.mark.parametrize("bad,message", [(dict(out=False), b"null out"), (dict(mats=False), b"null matrix"), (dict(field=9), b"field"),
                                         (dict(fmt=3), b"format"), (dict(rows=0), b"n_rows"), (dict(bad_col=True), b"out of range"),
                                         (dict(decreasing=True), b"decreases")],
                         ids=["null-out", "null-matrices", "unknown-field", "bad-format", "no-rows", "column-out-of-range", "row_ptr-decreases"])
def test_create_verifier_refuses_bad_arguments(L, bad, message):
    rc, ctx = create_verifier(L, **bad)
    assert rc == L._capi.ERR_ARG and not ctx.value
    assert message in L._capi.lib().lurk_last_error()


def test_create_verifier_fails_loudly_without_gpu(L):
    no_gpu(L)
    rc, ctx = create_verifier(L)
    assert rc == L._capi.ERR_NOGPU and not ctx.value


def test_plain_c_client_fails_loudly_without_gpu(L, tmp_path):
    """tests/csrc/recursive_client.c, built as strict C99: the refusals hold, and without a CUDA device nothing can be created"""
    no_gpu(L)
    exe, libdir = str(tmp_path / "recursive_client"), os.path.join(ROOT, "lurk-beta_b200")
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "csrc", "recursive_client.c"), "-o", exe, "-L", libdir, "-llurk_b200", "-Wl,-rpath," + libdir])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    assert "recursive_client ok (no GPU: compute entry points fail loudly)" in out.stdout
