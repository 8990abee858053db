"""CPU checks of the trie store's device-resident forms (lurk_trie_ctx_apply_dev / lurk_trie_ctx_register_dev): the
symbols, the header under strict C99, the refusals the host can make, in their order and before LURK_ERR_NOGPU, the
Python argument checks of DeviceTrie.apply_dev / register_dev, and the Rust declarations."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.abspath(__file__)).rsplit(os.sep, 1)[0]
SYMBOLS = ("lurk_trie_ctx_apply_dev", "lurk_trie_ctx_register_dev")
FAKE = 0x1000    # a non-NULL device address: every call here is refused before anything is read


def _ctx(L, height=2, capacity=8, field=0):
    ctx = C.c_void_p()
    assert L._capi.lib().lurk_trie_ctx_create(field, height, capacity, C.byref(ctx)) == 0, L._capi.lib().lurk_last_error()
    return ctx


def _err(L):
    return L._capi.lib().lurk_last_error().decode()


def test_symbols(L):
    lib = L._capi.lib()
    for name in SYMBOLS:
        assert hasattr(lib, name), name
        assert name in L._capi.PROTOTYPES, name


def test_header_is_strict_c99(tmp_path):
    src = tmp_path / "t.c"
    src.write_text('#include "lurk_b200.h"\n'
                   "int main(void) {\n"
                   "    int (*apply)(lurk_trie_ctx *, size_t, const int32_t *, const int64_t *, const void *, const void *, const void *, int,\n"
                   "                 void *, void *, void *, void *) = lurk_trie_ctx_apply_dev;\n"
                   "    int (*reg)(lurk_trie_ctx *, const void *, size_t, void *, int, void *) = lurk_trie_ctx_register_dev;\n"
                   "    (void)apply; (void)reg;\n"
                   "    return 0;\n"
                   "}\n")
    subprocess.check_call(["gcc", "-std=c99", "-pedantic", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(src), "-o",
                           str(tmp_path / "t.o")])


def test_apply_dev_host_refusals_in_order(L):
    """null ctx, bad fmt, NULL kinds / prev / keys with n > 0, n >= 2^31: LURK_ERR_ARG in that order, each before the
    next is looked at; a NULL roots or values pointer is not refused here (whether it is read depends on the batch)"""
    lib = L._capi.lib()
    ARG = L._capi.ERR_ARG
    ctx = _ctx(L)
    apply = lambda c, n, k, p, r, key, v, fmt: lib.lurk_trie_ctx_apply_dev(c, n, k, p, r, key, v, fmt, None, None, None, None)
    assert apply(None, 1 << 31, None, None, None, None, None, 7) == ARG and "null trie context" in _err(L)
    assert apply(ctx, 1 << 31, None, None, None, None, None, 7) == ARG and "format 7" in _err(L)
    for k, p, key in ((None, FAKE, FAKE), (FAKE, None, FAKE), (FAKE, FAKE, None)):
        assert apply(ctx, 1 << 31, k, p, None, key, None, 0) == ARG and "null kinds, prev or keys" in _err(L)
    assert apply(ctx, 1 << 31, FAKE, FAKE, None, FAKE, None, 0) == ARG and "2^31" in _err(L)
    assert apply(ctx, 0, None, None, None, None, None, 0) != ARG, _err(L)      # an empty batch needs no arrays
    lib.lurk_trie_ctx_destroy(ctx)


def test_register_dev_host_refusals_in_order(L):
    lib = L._capi.lib()
    ARG = L._capi.ERR_ARG
    ctx = _ctx(L, height=2, capacity=8)     # 2 empty roots: 6 more nodes fit
    assert lib.lurk_trie_ctx_register_dev(None, None, 7, None, 7, None) == ARG and "null trie context" in _err(L)
    assert lib.lurk_trie_ctx_register_dev(ctx, None, 7, None, 7, None) == ARG and "format 7" in _err(L)
    assert lib.lurk_trie_ctx_register_dev(ctx, None, 7, None, 0, None) == ARG and "null preimages" in _err(L)
    assert lib.lurk_trie_ctx_register_dev(ctx, FAKE, 7, None, 1, None) == ARG and "capacity 8" in _err(L)
    assert lib.lurk_trie_ctx_register_dev(ctx, None, 0, None, 0, None) != ARG, _err(L)
    lib.lurk_trie_ctx_destroy(ctx)


def test_no_gpu_comes_after_the_host_refusals(L):
    lib = L._capi.lib()
    if lib.lurk_device_count() > 0:
        pytest.skip("GPU present")
    NOGPU = L._capi.ERR_NOGPU
    ctx = _ctx(L)
    assert lib.lurk_trie_ctx_apply_dev(ctx, 3, FAKE, FAKE, None, FAKE, None, 1, None, None, None, None) == NOGPU
    assert lib.lurk_trie_ctx_apply_dev(ctx, 0, None, None, None, None, None, 0, None, None, None, None) == NOGPU
    assert lib.lurk_trie_ctx_register_dev(ctx, FAKE, 6, FAKE, 0, None) == NOGPU
    n = C.c_uint64()
    assert lib.lurk_trie_ctx_info(ctx, C.byref(n), None) == 0 and n.value == 2
    lib.lurk_trie_ctx_destroy(ctx)


def test_python_refuses_bad_tensors(L):
    """wrong dtype, shape, contiguity or device raises ValueError naming the argument, before the library is called"""
    torch = pytest.importorskip("torch")
    lib = L._capi.lib()
    if lib.lurk_device_count() > 0:
        pytest.skip("GPU present: the device case is covered by the GPU tests")
    dt = L.DeviceTrie(0, 2, 64)
    n = 3
    good = dict(kinds=torch.zeros(n, dtype=torch.int32), prev=torch.full((n,), -1, dtype=torch.int64),
                roots=torch.zeros((n, 32), dtype=torch.uint8), keys=torch.zeros((n, 32), dtype=torch.uint8),
                values=torch.zeros((n, 32), dtype=torch.uint8))
    cases = [("kinds", dict(kinds=torch.zeros(n, dtype=torch.int64))),
             ("prev", dict(prev=torch.zeros(n, dtype=torch.int32))),
             ("prev", dict(prev=torch.zeros(n + 1, dtype=torch.int64))),
             ("keys", dict(keys=torch.zeros((n, 31), dtype=torch.uint8))),
             ("keys", dict(keys=[0] * n)),
             ("roots", dict(roots=torch.zeros((n, 64), dtype=torch.uint8)[:, ::2])),
             ("values", dict(values=torch.zeros((n, 32), dtype=torch.int8))),
             ("kinds", dict())]    # every argument right but on the CPU: the first one checked is named
    for word, bad in cases:
        args = dict(good)
        args.update(bad)
        with pytest.raises(ValueError, match=word):
            dt.apply_dev(**args)
    for word, bad in (("preimages", torch.zeros((2, 8, 32), dtype=torch.int32)), ("preimages", torch.zeros((2, 7, 32), dtype=torch.uint8)),
                      ("preimages", torch.zeros((2, 8, 64), dtype=torch.uint8)[:, :, ::2]), ("preimages", torch.zeros((2, 8, 32), dtype=torch.uint8))):
        with pytest.raises(ValueError, match=word):
            dt.register_dev(bad)
    dt.close()


def test_rust_binding_declares_both_calls():
    header = open(os.path.join(ROOT, "include", "lurk_b200.h")).read()
    rust = open(os.path.join(ROOT, "integration", "rust", "ffi.rs")).read()
    for name in SYMBOLS:
        h = re.search(name + r"\(([^;]*)\);", header)
        r = re.search(r"pub fn " + name + r"\(([^;]*)\)( -> c_int)?;", rust)
        assert h and r, name
        assert len(h.group(1).split(",")) == len(r.group(1).split(",")), name
