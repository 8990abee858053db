"""lurk_point_combination_batch (include/lurk_b200.h) on the CPU: the symbol is exported, every malformed argument is refused with
LURK_ERR_ARG and a message on any machine, and without a GPU a well-formed call fails with LURK_ERR_NOGPU -- there is no CPU fallback;
lurk_point_combination is the host's entry point."""
import ctypes as C

import numpy as np
import pytest

from util import pack


def no_gpu(L):
    if L._capi.lib().lurk_device_count() > 0:
        pytest.skip("GPU present (tests/test_gpu_point_combination.py covers the device path)")


def test_symbol_is_exported(L):
    lib = C.CDLL(L._capi.LIB_PATH)
    assert hasattr(lib, "lurk_point_combination_batch")
    assert "lurk_point_combination_batch" in L._capi.PROTOTYPES
    assert L._capi.POINT_COMBINATION_MAX_TERMS == 4096


def call(L, curve=0, n_groups=None, counts=(1, 2), points=True, scalars=True, out=True, fmt=0):
    """a valid call unless told otherwise: group 0 = [G], group 1 = [G, identity], scalars 5, 7, 9"""
    E = L._capi
    pts = pack([1, 2, 1] + [1, 2, 1] + [0, 0, 0])
    sc = pack([5, 7, 9])
    c = np.array(counts, dtype=np.uint32)
    o = np.zeros(96 * 2, dtype=np.uint8)
    rc = E.lib().lurk_point_combination_batch(curve, len(counts) if n_groups is None else n_groups, E.np_ptr(c), E.np_ptr(pts) if points else None,
                                              E.np_ptr(sc) if scalars else None, fmt, E.np_ptr(o) if out else None, None)
    return rc, E.lib().lurk_last_error(), o


@pytest.mark.parametrize("bad,message", [
    (dict(points=False), b"null"), (dict(scalars=False), b"null"), (dict(out=False), b"null"), (dict(n_groups=0), b"at least one group"),
    (dict(n_groups=-3), b"at least one group"), (dict(fmt=2), b"bad format"), (dict(curve=4), b"unknown curve"), (dict(curve=-1), b"unknown curve"),
    (dict(counts=(1, 0)), b"group 1 has 0 terms"), (dict(counts=(4097, 1)), b"group 0 has 4097 terms")],
    ids=["null-points", "null-scalars", "null-out", "no-groups", "negative-groups", "bad-format", "curve-4", "curve-minus-1", "zero-count",
         "over-the-limit"])
def test_refuses_bad_arguments(L, bad, message):
    rc, msg, o = call(L, **bad)
    assert rc == L._capi.ERR_ARG and message in msg
    assert not o.any()


def test_without_a_gpu_a_well_formed_call_fails_loudly(L):
    no_gpu(L)
    rc, msg, o = call(L)
    assert rc == L._capi.ERR_NOGPU and not o.any()
    with pytest.raises(L._capi.LurkError) as e:
        L.point_combination_batch(0, [([(1, 2)], [5])])
    assert e.value.code == L._capi.ERR_NOGPU


def test_binding_refuses_malformed_groups_before_the_library(L):
    with pytest.raises(ValueError):
        L.point_combination_batch(0, [])
    with pytest.raises(ValueError):
        L.point_combination_batch(0, [([], [])])
    with pytest.raises(ValueError):
        L.point_combination_batch(0, [(np.zeros(96, dtype=np.uint8), np.zeros(64, dtype=np.uint8))])
