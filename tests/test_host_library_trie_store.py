"""CPU checks of the device trie store's C ABI (lurk_trie_ctx_*): the symbols, the header under strict C99, every
argument refusal of lurk_trie_ctx_apply naming its operation before LURK_ERR_NOGPU, and LURK_ERR_NOGPU without a device.
A context is created without a GPU too (it holds no store until one is present), so the refusals are checked here."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("lurk_trie_ctx_create", "lurk_trie_ctx_destroy", "lurk_trie_ctx_empty_root", "lurk_trie_ctx_info", "lurk_trie_ctx_register",
           "lurk_trie_ctx_apply")


def _ctx(L, height=2, capacity=64, field=0):
    ctx = C.c_void_p()
    rc = L._capi.lib().lurk_trie_ctx_create(field, height, capacity, C.byref(ctx))
    assert rc == 0, L._capi.lib().lurk_last_error()
    return ctx


def _apply(L, ctx, ops, fmt=0):
    """ops: (kind, prev, root, key, value) -> return code"""
    from util import pack
    n = len(ops)
    kinds = np.array([o[0] for o in ops], dtype=np.int32)
    prev = np.array([o[1] for o in ops], dtype=np.int64)
    roots, keys, vals = (pack([o[k] for o in ops]) for k in (2, 3, 4))
    res = np.zeros(32 * n, dtype=np.uint8)
    ptr = L._capi.np_ptr
    return L._capi.lib().lurk_trie_ctx_apply(ctx, n, ptr(kinds), ptr(prev), ptr(roots), ptr(keys), ptr(vals), fmt, ptr(res), None, None, None)


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
                   "    lurk_trie_ctx *ctx = 0;\n"
                   "    uint64_t n = 0, cap = 0;\n"
                   "    int (*create)(int, int, uint64_t, lurk_trie_ctx **) = lurk_trie_ctx_create;\n"
                   "    int (*reg)(lurk_trie_ctx *, const uint8_t *, size_t, uint8_t *, int) = lurk_trie_ctx_register;\n"
                   "    int (*apply)(lurk_trie_ctx *, size_t, const int *, const int64_t *, const uint8_t *, const uint8_t *, const uint8_t *, int,\n"
                   "                 uint8_t *, void *, void *, void *) = lurk_trie_ctx_apply;\n"
                   "    int (*root)(lurk_trie_ctx *, uint8_t *, int) = lurk_trie_ctx_empty_root;\n"
                   "    void (*destroy)(lurk_trie_ctx *) = lurk_trie_ctx_destroy;\n"
                   "    (void)create; (void)reg; (void)apply; (void)root; (void)destroy;\n"
                   "    return lurk_trie_ctx_info(ctx, &n, &cap) == LURK_ERR_ARG ? 0 : 1;\n"
                   "}\n")
    subprocess.check_call(["gcc", "-std=c99", "-pedantic", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(src), "-o",
                           str(tmp_path / "t.o")])


def test_create_refusals(L):
    lib = L._capi.lib()
    ARG = L._capi.ERR_ARG
    ctx = C.c_void_p()
    for field, H, cap in ((0, 0, 64), (0, 86, 1000), (0, -1, 64), (4, 2, 64), (-1, 2, 64), (0, 3, 2), (0, 2, 1 << 31)):
        assert lib.lurk_trie_ctx_create(field, H, cap, C.byref(ctx)) == ARG, (field, H, cap)
        assert not ctx.value
    assert lib.lurk_trie_ctx_create(0, 86, 1000, C.byref(ctx)) == ARG and "height 86" in _err(L)
    assert lib.lurk_trie_ctx_create(0, 2, 64, None) == ARG
    assert lib.lurk_trie_ctx_info(None, None, None) == ARG
    assert lib.lurk_trie_ctx_apply(None, 0, None, None, None, None, None, 0, None, None, None, None) == ARG
    assert lib.lurk_trie_ctx_register(None, None, 0, None, 0) == ARG


@pytest.mark.parametrize("field", [0, 1, 2, 3])
def test_apply_refusals_name_the_operation(L, field):
    """each refusal comes before any device work (so also before LURK_ERR_NOGPU) and names the operation"""
    from oracle import spec
    p = spec.FIELD_MODULUS[field]
    lib = L._capi.lib()
    ctx = _ctx(L, height=2, capacity=2 + 2 * 3, field=field)
    ARG = L._capi.ERR_ARG
    LOOK, INS = L.TRIE_LOOKUP, L.TRIE_INSERT
    cases = [
        ([(LOOK, -1, 0, 1, 0), (2, -1, 0, 1, 0)], 1, "kind"),                       # bad kind
        ([(LOOK, -1, 0, 1, 0), (INS, -1, 0, 1, 5), (INS, 2, 0, 1, 5)], 2, "prev"),  # prev >= i
        ([(INS, -1, 0, 1, 5), (INS, -2, 0, 1, 5)], 1, "prev"),                      # prev < -1
        ([(LOOK, -1, 0, 1, 0), (INS, 0, 0, 1, 5)], 1, "lookup"),                    # prev names a lookup
        ([(INS, -1, 0, 1, 5), (INS, 0, 0, 2, 5), (INS, 0, 0, 3, 5)], 2, "fork"),    # fork inside the batch
        ([(INS, -1, 0, 1, 5), (LOOK, 0, 0, 1, 0), (INS, -1, p, 1, 5)], 2, "root"),  # root >= p
        ([(INS, -1, 0, 1, 5), (LOOK, -1, 0, p + 3, 0)], 1, "key"),                  # key >= p
        ([(LOOK, -1, 0, 1, 0), (INS, -1, 0, 1, p)], 1, "value"),                    # value >= p
    ]
    for ops, bad, word in cases:
        assert _apply(L, ctx, ops) == ARG, (ops, _err(L))
        msg = _err(L)
        assert f"operation {bad}" in msg and word in msg, (ops, msg)
    # a root >= p is not read where prev names an insert, and a lookup's value is never read
    ok = [(INS, -1, 0, 1, 5), (INS, 0, p + 1, 2, 6), (LOOK, 1, p, 2, p)]
    assert _apply(L, ctx, ok) != ARG, _err(L)
    # capacity: 2 empty roots + H x inserts must fit
    assert _apply(L, ctx, [(INS, -1, 0, k, 1) for k in range(3)]) != ARG, _err(L)
    assert _apply(L, ctx, [(INS, -1, 0, k, 1) for k in range(4)]) == ARG and "capacity" in _err(L)
    assert _apply(L, ctx, [(LOOK, -1, 0, 1, 0)], fmt=2) == ARG
    n, cap = C.c_uint64(), C.c_uint64()
    assert lib.lurk_trie_ctx_info(ctx, C.byref(n), C.byref(cap)) == 0 and cap.value == 8
    if lib.lurk_device_count() == 0:
        assert n.value == 2
    lib.lurk_trie_ctx_destroy(ctx)


def test_no_cpu_fallback(L):
    lib = L._capi.lib()
    if lib.lurk_device_count() > 0:
        pytest.skip("GPU present")
    NOGPU = L._capi.ERR_NOGPU
    ctx = _ctx(L)
    assert _apply(L, ctx, [(L.TRIE_INSERT, -1, 0, 1, 5), (L.TRIE_LOOKUP, 0, 0, 1, 0)]) == NOGPU
    out = np.zeros(32 * 8, dtype=np.uint8)
    assert lib.lurk_trie_ctx_empty_root(ctx, L._capi.np_ptr(out), 0) == NOGPU
    assert lib.lurk_trie_ctx_register(ctx, L._capi.np_ptr(out), 1, None, 0) == NOGPU
    lib.lurk_trie_ctx_destroy(ctx)
    with pytest.raises(L.LurkError) as e:
        L.DeviceTrie(0, 2, 64).empty_root()
    assert e.value.code == NOGPU


def test_capacity_refusal_names_the_first_insert_that_does_not_fit(L):
    """capacity 8 at H = 2 holds the 2 empty roots and 3 inserts' nodes: the 4th insert (operation 4 here) is named"""
    ctx = _ctx(L, height=2, capacity=8)
    LOOK, INS = L.TRIE_LOOKUP, L.TRIE_INSERT
    ops = [(INS, -1, 0, 0, 1), (LOOK, 0, 0, 0, 0), (INS, 0, 0, 1, 1), (INS, 2, 0, 2, 1), (INS, 3, 0, 3, 1), (INS, 4, 0, 4, 1)]
    assert _apply(L, ctx, ops) == L._capi.ERR_ARG
    assert "operation 4:" in _err(L) and "capacity" in _err(L), _err(L)
    L._capi.lib().lurk_trie_ctx_destroy(ctx)


def test_roots_and_values_may_be_null_when_never_read(L):
    lib = L._capi.lib()
    ctx = _ctx(L, height=2)
    from util import pack
    ptr = L._capi.np_ptr
    LOOK, INS = L.TRIE_LOOKUP, L.TRIE_INSERT

    def call(kinds, prev, roots, values):
        keys = pack([1] * len(kinds))
        k = np.array(kinds, dtype=np.int32)
        pv = np.array(prev, dtype=np.int64)
        r = ptr(pack([0] * len(kinds))) if roots else None
        v = ptr(pack([5] * len(kinds))) if values else None
        return lib.lurk_trie_ctx_apply(ctx, len(kinds), ptr(k), ptr(pv), r, ptr(keys), v, 0, None, None, None, None)

    ARG = L._capi.ERR_ARG
    assert call([LOOK, LOOK], [-1, -1], True, False) != ARG, _err(L)          # lookups only: values unread
    assert call([INS, LOOK], [-1, 0], True, False) == ARG and "operation 0:" in _err(L) and "values" in _err(L)
    assert call([INS, INS], [-1, 0], False, True) == ARG and "operation 0:" in _err(L) and "roots" in _err(L)
    assert call([LOOK, INS, LOOK], [-1, -1, 1], True, False) == ARG and "operation 1:" in _err(L)
    assert lib.lurk_trie_ctx_apply(ctx, 1, None, None, None, None, None, 0, None, None, None, None) == ARG
    lib.lurk_trie_ctx_destroy(ctx)


def test_write_trie_batch_refuses_unreduced_elements_before_converting(L):
    """write_trie_batch converts to Montgomery on the host, which would reduce an element >= p: it refuses them first"""
    from oracle import spec
    p = spec.FIELD_MODULUS[0]

    class NoStore:
        field_id, height = 0, 2

    for ops, word in (([(L.TRIE_INSERT, -1, 0, p, 1)], "key"), ([(L.TRIE_INSERT, -1, p + 2, 1, 1)], "root"),
                      ([(L.TRIE_INSERT, -1, 0, 1, p)], "value"), ([(L.TRIE_LOOKUP, -1, 0, 1 << 255, 0)], "key")):
        with pytest.raises(ValueError, match=f"operation 0: the {word}"):
            L.write_trie_batch(NoStore(), None, 0, 0, ops)


def test_rust_binding_declares_the_trie_context():
    """integration/rust/ffi.rs declares the opaque context and every lurk_trie_ctx_* entry point with the header's
    parameter count"""
    import re
    header = open(os.path.join(ROOT, "include", "lurk_b200.h")).read()
    rust = open(os.path.join(ROOT, "integration", "rust", "ffi.rs")).read()
    assert re.search(r"#\[repr\(C\)\]\s*pub struct lurk_trie_ctx \{ _private: \[u8; 0\] \}", rust)
    for name in SYMBOLS:
        h = re.search(name + r"\(([^;]*)\);", header)
        r = re.search(r"pub fn " + name + r"\(([^;]*)\)( -> c_int)?;", rust)
        assert h and r, name
        assert len(h.group(1).split(",")) == len(r.group(1).split(",")), name
