"""The compressed verifier (lurk_compress_verify, include/lurk_b200.h, N4) on the CPU: the symbols are exported, every malformed argument is
refused with LURK_ERR_ARG and a message before any callback or CUDA call, a well-formed call without a GPU fails with LURK_ERR_NOGPU (there is
no CPU fallback), lurk_point_combination works on the host alone, and the header drives the library from plain C99
(tests/csrc/compress_verify_client.c)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("lurk_compress_verify", "lurk_point_combination")


def no_gpu(L):
    if L._capi.lib().lurk_device_count() > 0:
        pytest.skip("GPU present (tests/test_gpu_compress_verify.py covers the device paths)")


def test_symbols_are_exported(L):
    lib = C.CDLL(L._capi.LIB_PATH)
    for s in SYMBOLS:
        assert hasattr(lib, s), s
        assert s in L._capi.PROTOTYPES, s


def verify(L, n=1, primary=True, secondary=True, kinds=(0, 1), keys=(True, True), g=True, ck_c=True, pairing=True, cb=True, proof=True,
           out=True, flags=0, fmt=0, rounds_fmt=0, same_ctx=False, same_key=False, u=True):
    """lurk_compress_verify on fake pointers that no check before the GPU check dereferences; returns (rc, callback calls, verdicts)"""
    E = L._capi
    buf = np.zeros(8192, dtype=np.uint8)
    k = max(n, 1)
    ptrs = [buf.ctypes.data + 64 * i for i in range(k)]
    if same_ctx and k > 1:
        ptrs[1] = ptrs[0]
    arr = (C.c_void_p * k)(*ptrs) if primary else None
    sec = C.c_void_p(ptrs[0] if same_ctx and k == 1 else buf.ctypes.data + 2048) if secondary else None
    key = [buf.ctypes.data + 3000, buf.ctypes.data + (3000 if same_key else 3100)]
    pcs = [E.CompressVkPcs(kinds[i], key[i] if keys[i] else None, buf.ctypes.data + 3500 if ck_c else None, buf.ctypes.data + 3600 if g else None)
           for i in range(2)]
    data = (C.c_void_p * k)(*[buf.ctypes.data + 4096] * k)
    calls = []

    def chal(user, circuit, phase, rnd, msg, n, o):
        calls.append(("challenge", circuit))
        return 0

    def pair(user, circuit, P, Q, holds):
        calls.append(("pairing", circuit))
        return 0
    fn = E.COMPRESS_CHALLENGE_FN(chal) if cb else E.COMPRESS_CHALLENGE_FN()
    pfn = E.PAIRING_CHECK_FN(pair) if pairing else E.PAIRING_CHECK_FN()
    rec = E.CompressProof()
    verdicts, acc = (E.CompressVerdict * 2)(), C.c_int(-2)
    p = C.c_void_p(buf.ctypes.data + 5000)
    rc = E.lib().lurk_compress_verify(n, arr, sec, C.byref(pcs[0]), C.byref(pcs[1]), p if u else None, data, data, data, p, p, p, p,
                                      C.byref(rec) if proof else None, rounds_fmt, fn, pfn, None, flags, verdicts if out else None, C.byref(acc), fmt, None)
    return rc, calls, [(v.snark_ok, v.eval_ok, v.opening_ok) for v in verdicts], acc.value


@pytest.mark.parametrize("bad,message", [
    (dict(n=0), b"primary contexts"), (dict(n=31, flags=2), b"primary contexts"), (dict(n=2), b"one instance"), (dict(flags=4), b"flags"),
    (dict(primary=False), b"null"), (dict(secondary=False), b"null"), (dict(kinds=(0, 5)), b"evaluation engine"),
    (dict(keys=(True, False)), b"IPA needs"), (dict(ck_c=False), b"IPA needs"), (dict(g=False), b"HyperKZG needs g"),
    (dict(pairing=False), b"pairing callback"), (dict(cb=False), b"challenge callback"), (dict(proof=False), b"null proof"), (dict(u=False), b"null"),
    (dict(fmt=2), b"format"), (dict(rounds_fmt=3), b"rounds_fmt"), (dict(n=2, flags=2, same_ctx=True), b"same context"),
    (dict(same_ctx=True), b"also the secondary"), (dict(kinds=(1, 1), same_key=True), b"same context")],
    ids=["no-primary", "31-primaries", "two-plain-primaries", "unknown-flag", "null-primaries", "null-secondary", "unknown-engine", "ipa-null-key",
         "ipa-without-ck_c", "hyperkzg-without-g", "hyperkzg-without-pairing", "null-challenge", "null-proof", "null-u", "bad-format",
         "bad-rounds-format", "duplicated-primary", "primary-is-secondary", "one-key-for-both"])
def test_refuses_bad_arguments_before_any_callback(L, bad, message):
    rc, calls, verdicts, acc = verify(L, **bad)
    assert rc == L._capi.ERR_ARG and calls == [] and acc == 0
    assert verdicts == [(-1, -1, -1)] * 2
    assert message in L._capi.lib().lurk_last_error()


def test_null_verdicts_are_refused(L):
    rc, calls, _, _ = verify(L, out=False)
    assert rc == L._capi.ERR_ARG and calls == [] and b"verdict" in L._capi.lib().lurk_last_error()


def test_without_a_gpu_a_well_formed_call_fails_loudly(L):
    no_gpu(L)
    rc, calls, verdicts, acc = verify(L)
    assert rc == L._capi.ERR_NOGPU and calls == [] and acc == 0 and verdicts == [(-1, -1, -1)] * 2


def test_point_combination_on_the_host(L):
    """sum_k s_k P_k against the oracle's affine arithmetic, on every curve, in both formats of the scalars' and points' bytes"""
    from oracle import spec
    from util import pack
    E = L._capi
    for curve in range(4):
        C_ = spec.CURVES[curve]
        pb, q = spec.FIELD_MODULUS[C_["base"]], spec.FIELD_MODULUS[C_["scalar"]]
        pts = [spec.ec_mul(3 + 5 * i, C_["gen"], pb) for i in range(5)] + [None]
        sc = [(7 ** (i + 20)) % q for i in range(6)]
        want = None
        for s, P in zip(sc, pts):
            want = spec.ec_add(want, spec.ec_mul(s, P, pb), pb)
        buf = pack([c for P in pts for c in ((0, 0, 0) if P is None else (P[0], P[1], 1))])
        out = np.zeros(96, dtype=np.uint8)
        assert E.lib().lurk_point_combination(curve, E.np_ptr(buf), E.np_ptr(pack(sc)), 6, E.FMT_CANONICAL, E.np_ptr(out)) == E.OK
        v = [int.from_bytes(out[32 * i:32 * i + 32].tobytes(), "little") for i in range(3)]
        assert (v[0], v[1]) == want and v[2] == 1
        off = pack([1, 1, 1])
        assert E.lib().lurk_point_combination(curve, E.np_ptr(off), E.np_ptr(pack([1])), 1, E.FMT_CANONICAL, E.np_ptr(out)) == E.ERR_RANGE
    assert E.lib().lurk_point_combination(7, None, None, 0, E.FMT_CANONICAL, E.np_ptr(out)) == E.ERR_ARG


def test_plain_c_client_builds_and_refuses_without_a_gpu(L, tmp_path):
    """tests/csrc/compress_verify_client.c, built as strict C99: the refusals hold, and without a CUDA device nothing can be created"""
    no_gpu(L)
    exe, libdir = str(tmp_path / "compress_verify_client"), os.path.join(ROOT, "lurk-beta_b200")
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "csrc", "compress_verify_client.c"), "-o", exe, "-L", libdir, "-llurk_b200", "-Wl,-rpath," + libdir])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    assert "compress_verify_client ok (no GPU: compute entry points fail loudly)" in out.stdout
