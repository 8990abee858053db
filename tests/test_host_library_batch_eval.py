"""lurk_batch_eval_reduce_dev (include/lurk_b200.h, N4) on the CPU: every malformed argument is refused with LURK_ERR_ARG before any
device work, and a well-formed call without a GPU fails with LURK_ERR_NOGPU and a message (there is no CPU fallback)."""
import ctypes as C

import numpy as np
import pytest


def call(L, n=2, polys=True, nv=(3, 2), points=True, evals=True, cb=True, joint=True, fmt=0):
    E = L._capi
    buf = np.zeros(1 << 12, dtype=np.uint8)
    other = np.zeros(1 << 12, dtype=np.uint8)
    nvs = list(nv) + [0] * max(0, n - len(nv))
    ptrs = (C.c_void_p * max(n, 1))(*[C.c_void_p(buf.ctypes.data if polys else 0)] * max(n, 1))
    nva = (C.c_int * max(n, 1))(*(nvs[:max(n, 1)]))
    pts = np.zeros(32 * max(1, sum(max(0, v) for v in nvs)), dtype=np.uint8)
    ev = np.zeros(32 * max(n, 1), dtype=np.uint8)
    fn = E.CHALLENGE_FN(lambda user, rnd, msg, k, out: 0)
    joint_ptr = joint if not isinstance(joint, bool) else (other.ctypes.data if joint else 0)
    return L._capi.lib().lurk_batch_eval_reduce_dev(0, n, ptrs, nva, E.np_ptr(pts) if points else None, E.np_ptr(ev) if evals else None,
                                                    fn if cb else E.CHALLENGE_FN(), None, None, None, None, None, None, C.c_void_p(joint_ptr),
                                                    fmt, None)


@pytest.mark.parametrize("bad", [dict(n=0), dict(n=61), dict(nv=(3, -1)), dict(nv=(41, 2)), dict(polys=False), dict(points=False),
                                 dict(evals=False), dict(cb=False), dict(joint=False), dict(fmt=7)],
                         ids=["no-claim", "61-claims", "negative-vars", "41-vars", "null-poly", "null-points", "null-evals",
                              "null-callback", "null-joint", "bad-format"])
def test_bad_arguments_are_refused(L, bad):
    assert call(L, **bad) == L._capi.ERR_ARG
    assert len(L._capi.lib().lurk_last_error()) > 0


def test_points_may_be_null_without_variables_and_joint_must_not_overlap(L):
    E = L._capi
    if L._capi.lib().lurk_device_count() == 0:
        assert call(L, nv=(0, 0), points=False) == E.ERR_NOGPU
    # the joint polynomial written over an input polynomial
    buf = np.zeros(1 << 12, dtype=np.uint8)
    ptrs = (C.c_void_p * 1)(C.c_void_p(buf.ctypes.data))
    nva = (C.c_int * 1)(3)
    z = np.zeros(32 * 3, dtype=np.uint8)
    fn = E.CHALLENGE_FN(lambda user, rnd, msg, k, out: 0)
    rc = E.lib().lurk_batch_eval_reduce_dev(0, 1, ptrs, nva, E.np_ptr(z), E.np_ptr(z), fn, None, None, None, None, None, None,
                                            C.c_void_p(buf.ctypes.data + 64), 0, None)
    assert rc == E.ERR_ARG and b"overlap" in E.lib().lurk_last_error()


def test_valid_call_without_gpu_fails_loudly(L):
    if L._capi.lib().lurk_device_count() > 0:
        pytest.skip("GPU present")
    assert call(L) == L._capi.ERR_NOGPU
    assert len(L._capi.lib().lurk_last_error()) > 0
