"""CPU checks of the SHA-256 coprocessor's C ABI (lurk_sha256_witness_*, lurk_fold_ctx_add_sha256_batch): block lengths
from the host-built schedule, refusals that come before any launch, and LURK_ERR_NOGPU without a device."""
import ctypes as C

import numpy as np
import pytest


def _lib(L):
    return L._capi.lib()


def test_block_length_refusals(L):
    lib = _lib(L)
    assert lib.lurk_sha256_witness_block(0, 0) == 0
    assert lib.lurk_sha256_witness_block(0, -1) == 0
    assert lib.lurk_sha256_witness_block(9, 1) == 0
    assert lib.lurk_sha256_witness_block(0, 33) == 0 and lib.lurk_sha256_witness_block(0, 32) > 0
    with pytest.raises(ValueError):
        L.witness_block(0, 0)


def test_argument_errors_come_first(L):
    lib = _lib(L)
    buf = np.zeros(64 * 4, dtype=np.uint8)
    out = np.zeros(32, dtype=np.uint8)
    p, o = L._capi.np_ptr(buf), L._capi.np_ptr(out)
    offs = (C.c_uint64 * 1)(0)
    ARG = L._capi.ERR_ARG
    assert lib.lurk_sha256_witness_batch(0, 0, p, 1, o, 0) == ARG              # n < 1
    assert lib.lurk_sha256_witness_batch(5, 1, p, 1, o, 0) == ARG              # unknown field
    assert lib.lurk_sha256_witness_batch(0, 1, p, 1, o, 2) == ARG              # unknown format
    assert lib.lurk_sha256_witness_batch(0, 1, None, 1, o, 0) == ARG
    assert lib.lurk_sha256_witness_batch(0, 1, p, 1, None, 0) == ARG
    assert lib.lurk_sha256_witness_batch_dev(0, 1, None, 1, o, 0, None) == ARG
    assert lib.lurk_sha256_witness_batch_dev(0, 0, p, 1, o, 0, None) == ARG
    assert lib.lurk_sha256_witness_scatter_dev(0, 1, p, 1, None, o, 0, None) == ARG   # null offsets
    assert lib.lurk_sha256_witness_scatter_dev(0, 1, p, 1, offs, None, 0, None) == ARG
    assert lib.lurk_sha256_witness_scatter_dev(3, 40, p, 1, offs, o, 0, None) == ARG
    assert lib.lurk_fold_ctx_add_sha256_batch(None, 1, 1, offs) == ARG


def test_no_cpu_fallback(L):
    lib = _lib(L)
    if lib.lurk_device_count() > 0:
        pytest.skip("GPU present")
    buf = np.zeros(64, dtype=np.uint8)
    with pytest.raises(L.LurkError) as e:
        L.sha256_witness_batch(0, 1, buf)
    assert e.value.code == L._capi.ERR_NOGPU
    out = np.zeros(32, dtype=np.uint8)
    offs = (C.c_uint64 * 1)(0)
    NOGPU = L._capi.ERR_NOGPU
    assert lib.lurk_sha256_witness_batch_dev(0, 1, L._capi.np_ptr(buf), 1, L._capi.np_ptr(out), 0, None) == NOGPU
    assert lib.lurk_sha256_witness_scatter_dev(0, 1, L._capi.np_ptr(buf), 1, offs, L._capi.np_ptr(out), 0, None) == NOGPU


def test_native_compute_sha256(L):
    co = L.Sha256Coprocessor(1)
    assert co.arity() == 1 and co.witness_block(0) == L.witness_block(0, 1)
    with pytest.raises(ValueError):
        co.compute_sha256(0, [(1, 2), (3, 4)])
    with pytest.raises(ValueError):
        L.Sha256Coprocessor(0)
