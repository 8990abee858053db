"""The verifier entry points (lurk_spartan_matrix_evals_dev, lurk_spartan_verify, lurk_spartan_verify_batch, lurk_ipa_verify_dev in
include/lurk_b200.h, N4) on the CPU: every malformed argument is refused with LURK_ERR_ARG and a message before any device work, and a
well-formed call without a GPU fails with LURK_ERR_NOGPU."""
import ctypes as C

import numpy as np
import pytest


def verify(L, n=1, ctx=True, ctxs=True, shared=False, u=True, X=True, proof=True, field=None, cb=True, accepted=True, fmt=0, rounds_fmt=0,
           batched=True):
    """a verifier call with one argument broken at a time; contexts are zero-filled stand-ins (only their sizes and field are read on the
    refusal paths: field 0, n_x = 0)"""
    E = L._capi
    keep = [np.zeros(4096, dtype=np.uint8) for _ in range(max(n, 1) + 2)]
    buf = keep[-1]
    ptr = lambda ok, b=buf: C.c_void_p(b.ctypes.data if ok else 0)
    fn = E.SPARTAN_CHALLENGE_FN(lambda *a: 0) if cb else E.SPARTAN_CHALLENGE_FN()
    names = ("outer_rounds", "r_x", "claims", "inner_rounds", "r_y", "eval_W", "reduce_rounds", "r", "claims_left", "weights", "joint_eval")
    rec = E.SpartanProof(**{k: (0 if k == field else buf.ctypes.data) for k in names})
    acc = C.c_int(7)
    k = max(n, 1)
    stand_ins = [ptr(True, keep[0] if shared else keep[i]) for i in range(k)]
    if not ctx:
        stand_ins[-1] = C.c_void_p(0)
    if batched:
        cs = (C.c_void_p * k)(*stand_ins) if ctxs else None
        xs = (C.c_void_p * k)(*[ptr(X)] * k) if X else None
        return E.lib().lurk_spartan_verify_batch(n, cs, ptr(u), xs, C.byref(rec) if proof else None, rounds_fmt, fn, None,
                                                 C.byref(acc) if accepted else None, fmt, None)
    return E.lib().lurk_spartan_verify(stand_ins[0], ptr(u), ptr(X), C.byref(rec) if proof else None, rounds_fmt, fn, None,
                                       C.byref(acc) if accepted else None, fmt, None)


@pytest.mark.parametrize("batched", [False, True], ids=["plain", "batched"])
@pytest.mark.parametrize("bad,message", [(dict(u=False), b"u"), (dict(cb=False), b"callback"), (dict(proof=False), b"proof record"),
                                         (dict(accepted=False), b"accepted"), (dict(fmt=2), b"format"), (dict(rounds_fmt=2), b"rounds_fmt"),
                                         (dict(field="outer_rounds"), b"proof field"), (dict(field="claims"), b"proof field"),
                                         (dict(field="inner_rounds"), b"proof field"), (dict(field="eval_W"), b"proof field"),
                                         (dict(field="reduce_rounds"), b"proof field"), (dict(field="claims_left"), b"proof field"),
                                         (dict(ctx=False), b"context")],
                         ids=["null-u", "null-callback", "null-proof", "null-accepted", "bad-format", "unknown-rounds_fmt", "null-outer_rounds",
                              "null-claims", "null-inner_rounds", "null-eval_W", "null-reduce_rounds", "null-claims_left", "null-context"])
def test_verify_refuses_bad_arguments(L, batched, bad, message):
    assert verify(L, batched=batched, **bad) == L._capi.ERR_ARG
    assert message in L._capi.lib().lurk_last_error()


@pytest.mark.parametrize("bad,message", [(dict(n=0), b"instances"), (dict(n=31), b"instances"), (dict(ctxs=False), b"instance array"),
                                         (dict(X=False), b"instance array"), (dict(n=3, shared=True), b"share a context")],
                         ids=["no-instance", "31-instances", "null-contexts", "null-X-array", "shared-context"])
def test_batched_verify_refuses_bad_counts_and_contexts(L, bad, message):
    assert verify(L, **bad) == L._capi.ERR_ARG
    assert message in L._capi.lib().lurk_last_error()


def test_derived_fields_may_be_null_and_a_well_formed_call_needs_a_gpu(L):
    """r_x, r_y, r, weights and joint_eval are outputs: NULL is not a refusal; without a device the call fails with LURK_ERR_NOGPU"""
    if L._capi.lib().lurk_device_count() > 0:
        pytest.skip("GPU present")
    for derived in ("r_x", "r_y", "r", "weights", "joint_eval"):
        assert verify(L, field=derived) == L._capi.ERR_NOGPU
        assert verify(L, field=derived, batched=False) == L._capi.ERR_NOGPU


def test_matrix_evals_refuses_bad_arguments(L):
    E = L._capi
    buf = np.zeros(4096, dtype=np.uint8)
    p = C.c_void_p(buf.ctypes.data)
    for args in [(None, p, p, p, 0), (p, None, p, p, 0), (p, p, None, p, 0), (p, p, p, None, 0), (p, p, p, p, 2)]:
        assert E.lib().lurk_spartan_matrix_evals_dev(*args, None) == E.ERR_ARG
    if E.lib().lurk_device_count() == 0:
        assert E.lib().lurk_spartan_matrix_evals_dev(p, p, p, p, 0, None) == E.ERR_NOGPU


def ipa_verify(L, curve=0, ck=True, gc=True, comm=True, c=True, b=True, log_n=2, LR=True, a=True, cb=True, accepted=True, fmt=0):
    E = L._capi
    buf = np.zeros(4096, dtype=np.uint8)
    ptr = lambda ok: C.c_void_p(buf.ctypes.data if ok else 0)
    fn = E.CHALLENGE_FN(lambda *a: 0) if cb else E.CHALLENGE_FN()
    acc = C.c_int(7)
    return E.lib().lurk_ipa_verify_dev(curve, ptr(ck), ptr(gc), ptr(comm), ptr(c), ptr(b), log_n, ptr(LR), ptr(LR), ptr(a), fn, None,
                                       C.byref(acc) if accepted else None, None, None, fmt, None)


@pytest.mark.parametrize("bad", [dict(ck=False), dict(gc=False), dict(comm=False), dict(c=False), dict(b=False), dict(a=False), dict(cb=False),
                                 dict(accepted=False), dict(log_n=-1), dict(log_n=31), dict(LR=False), dict(fmt=5)],
                         ids=["null-key", "null-ck_c", "null-comm", "null-c", "null-b", "null-a_final", "null-callback", "null-accepted",
                              "log_n-negative", "log_n-31", "null-L-R", "bad-format"])
def test_ipa_verify_refuses_bad_arguments(L, bad):
    assert ipa_verify(L, **bad) == L._capi.ERR_ARG
    assert len(L._capi.lib().lurk_last_error()) > 0


def test_ipa_verify_needs_a_gpu(L):
    if L._capi.lib().lurk_device_count() > 0:
        pytest.skip("GPU present")
    assert ipa_verify(L) == L._capi.ERR_NOGPU
    assert ipa_verify(L, log_n=0, LR=False) == L._capi.ERR_NOGPU
