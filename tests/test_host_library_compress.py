"""The compress context (lurk_compress_ctx_*, lurk_compress_prove_dev in include/lurk_b200.h, N4) on the CPU: the symbols are exported, every
malformed argument is refused with LURK_ERR_ARG and a message before any CUDA call, a well-formed call without a GPU fails with
LURK_ERR_NOGPU (there is no CPU fallback), and the header drives the library from plain C99 (tests/csrc/compress_client.c)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("lurk_compress_ctx_create", "lurk_compress_ctx_destroy", "lurk_compress_ctx_info", "lurk_compress_prove_dev")


def no_gpu(L):
    if L._capi.lib().lurk_device_count() > 0:
        pytest.skip("GPU present (tests/test_gpu_compress.py covers the device paths)")


def test_symbols_are_exported(L):
    lib = C.CDLL(L._capi.LIB_PATH)
    for s in SYMBOLS:
        assert hasattr(lib, s), s
        assert s in L._capi.PROTOTYPES, s


def create(L, n=1, primary=True, secondary=True, kinds=(0, 1), cks=(True, True), ck_c=True, fmt=0, out=True, same_ctx=False, same_key=False):
    E = L._capi
    buf = np.zeros(4096, dtype=np.uint8)
    k = max(n, 1)
    ptrs = [buf.ctypes.data + 64 * i for i in range(k)]
    if same_ctx and k > 1:
        ptrs[1] = ptrs[0]
    arr = (C.c_void_p * k)(*ptrs) if primary else None
    sec = C.c_void_p(ptrs[0] if same_ctx and k == 1 else buf.ctypes.data + 2048) if secondary else None
    key = [buf.ctypes.data + 3000, buf.ctypes.data + (3000 if same_key else 3100)]
    pcs = [E.CompressPcs(kinds[i], key[i] if cks[i] else None, buf.ctypes.data + 3500 if ck_c else None) for i in range(2)]
    ctx = C.c_void_p()
    rc = E.lib().lurk_compress_ctx_create(n, arr, sec, C.byref(pcs[0]), C.byref(pcs[1]), fmt, C.byref(ctx) if out else None)
    return rc, ctx


@pytest.mark.parametrize("bad,message", [(dict(n=0), b"primary contexts"), (dict(n=31), b"primary contexts"), (dict(primary=False), b"null"),
                                         (dict(secondary=False), b"null"), (dict(kinds=(0, 5)), b"evaluation engine"), (dict(cks=(False, True)), b"key"),
                                         (dict(ck_c=False), b"ck_c"), (dict(fmt=2), b"format"), (dict(n=2, same_ctx=True), b"same context"),
                                         (dict(same_ctx=True), b"also the secondary"), (dict(same_key=True), b"same context"), (dict(out=False), b"null out")],
                         ids=["no-primary", "31-primaries", "null-primaries", "null-secondary", "unknown-engine", "null-key", "ipa-without-ck_c",
                              "bad-format", "duplicated-primary", "primary-is-secondary", "one-key-for-both", "null-out"])
def test_create_refuses_bad_arguments(L, bad, message):
    rc, ctx = create(L, **bad)
    assert rc == L._capi.ERR_ARG and not ctx.value
    assert message in L._capi.lib().lurk_last_error()


def prove(L, ctx=True, n=1, arrays=True, z2=True, cb=True, flags=0, fmt=0):
    E = L._capi
    buf = np.zeros(4096, dtype=np.uint8)
    p = C.c_void_p(buf.ctypes.data)
    k = max(n, 1)
    arr = (C.c_void_p * k)(*[buf.ctypes.data] * k) if arrays else None
    fn = E.COMPRESS_CHALLENGE_FN(lambda *a: 0) if cb else E.COMPRESS_CHALLENGE_FN()
    rec = E.CompressProof()
    return E.lib().lurk_compress_prove_dev(p if ctx else None, n, arr, arr, arr, arr, p if z2 else None, p, p, p, fn, None, flags, C.byref(rec), fmt, None)


@pytest.mark.parametrize("bad,message", [(dict(ctx=False), b"context"), (dict(cb=False), b"callback"), (dict(fmt=7), b"format"), (dict(flags=8), b"flags"),
                                         (dict(n=0, flags=2), b"primary instances"), (dict(n=31, flags=2), b"primary instances"),
                                         (dict(n=2), b"one instance"), (dict(arrays=False), b"instance array"), (dict(z2=False), b"secondary")],
                         ids=["null-context", "null-callback", "bad-format", "unknown-flag", "no-instance", "31-instances", "plain-with-two",
                              "null-arrays", "null-secondary"])
def test_prove_refuses_bad_arguments(L, bad, message):
    assert prove(L, **bad) == L._capi.ERR_ARG
    assert message in L._capi.lib().lurk_last_error()


def test_info_and_destroy_without_a_context(L):
    assert L._capi.lib().lurk_compress_ctx_info(None, None, None, None) == L._capi.ERR_ARG
    L._capi.lib().lurk_compress_ctx_destroy(None)          # a no-op, like free(NULL)


def test_well_formed_calls_fail_loudly_without_gpu(L):
    """the contexts are only read after the GPU check, so stand-in pointers reach it: LURK_ERR_NOGPU, never a CPU fallback"""
    no_gpu(L)
    rc, ctx = create(L)
    assert rc == L._capi.ERR_NOGPU and not ctx.value
    assert prove(L) == L._capi.ERR_NOGPU
    assert prove(L, n=3, flags=L._capi.COMPRESS_BATCHED | L._capi.COMPRESS_SEQUENTIAL) == L._capi.ERR_NOGPU
    assert b"GPU" in L._capi.lib().lurk_last_error() or b"CUDA" in L._capi.lib().lurk_last_error()


def test_plain_c_client_fails_loudly_without_gpu(L, tmp_path):
    """tests/csrc/compress_client.c, built as strict C99: the refusals hold, and without a CUDA device nothing can be created"""
    no_gpu(L)
    exe, libdir = str(tmp_path / "compress_client"), os.path.join(ROOT, "lurk-beta_b200")
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "csrc", "compress_client.c"), "-o", exe, "-L", libdir, "-llurk_b200", "-Wl,-rpath," + libdir])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    assert "compress_client ok (no GPU: compute entry points fail loudly)" in out.stdout
