"""CPU checks of the trie coprocessor's C ABI (lurk_trie_witness_*, lurk_fold_ctx_add_trie_batch): block lengths,
refusals that come before any launch, LURK_ERR_NOGPU without a device, the header under strict C99, and the proofs
and input packing of trie.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = {0: 354, 1: 364, 2: 298, 3: 301}


def _lib(L):
    return L._capi.lib()


def test_symbols_and_block_lengths(L):
    lib = _lib(L)
    for name in ("lurk_trie_witness_block", "lurk_trie_witness_batch", "lurk_trie_witness_batch_dev", "lurk_trie_witness_scatter_dev",
                 "lurk_fold_ctx_add_trie_batch"):
        assert hasattr(lib, name), name
    for field, d in D.items():
        for H in (1, 2, 3, 85):
            assert lib.lurk_trie_witness_block(field, L.TRIE_LOOKUP, H) == d + 403 * H
            assert lib.lurk_trie_witness_block(field, L.TRIE_INSERT, H) == d + 799 * H
            assert L.trie_witness_block(field, L.TRIE_INSERT, H) == d + 799 * H
    assert lib.lurk_trie_witness_block(0, 0, 85) == 34609 and lib.lurk_trie_witness_block(0, 1, 85) == 68269
    for field, op, H in ((0, 2, 1), (0, -1, 1), (0, 0, 0), (0, 1, 86), (0, 0, -3), (4, 0, 1), (-1, 1, 1)):
        assert lib.lurk_trie_witness_block(field, op, H) == 0, (field, op, H)
    with pytest.raises(ValueError):
        L.trie_witness_block(0, 0, 86)


def test_argument_errors_come_first(L):
    lib = _lib(L)
    buf = np.zeros(32 * 19, dtype=np.uint8)
    out = np.zeros(32, dtype=np.uint8)
    p, o = L._capi.np_ptr(buf), L._capi.np_ptr(out)
    offs = (C.c_uint64 * 1)(0)
    ARG = L._capi.ERR_ARG
    assert lib.lurk_trie_witness_batch(0, 2, 1, p, 1, o, 0) == ARG              # bad op
    assert lib.lurk_trie_witness_batch(0, 0, 0, p, 1, o, 0) == ARG              # bad height
    assert lib.lurk_trie_witness_batch(0, 0, 86, p, 1, o, 0) == ARG
    assert lib.lurk_trie_witness_batch(7, 0, 1, p, 1, o, 0) == ARG              # bad field
    assert lib.lurk_trie_witness_batch(0, 0, 1, p, 1, o, 2) == ARG              # bad format
    assert lib.lurk_trie_witness_batch(0, 0, 1, None, 1, o, 0) == ARG
    assert lib.lurk_trie_witness_batch(0, 0, 1, p, 1, None, 0) == ARG
    assert lib.lurk_trie_witness_batch_dev(0, 1, 1, None, 1, o, 0, None) == ARG
    assert lib.lurk_trie_witness_batch_dev(0, 1, 0, p, 1, o, 0, None) == ARG
    assert lib.lurk_trie_witness_scatter_dev(0, 0, 1, p, 1, None, o, 0, None) == ARG   # null offsets
    assert lib.lurk_trie_witness_scatter_dev(0, 0, 1, p, 1, offs, None, 0, None) == ARG
    assert lib.lurk_trie_witness_scatter_dev(3, 3, 1, p, 1, offs, o, 0, None) == ARG
    assert lib.lurk_fold_ctx_add_trie_batch(None, 0, 1, 1, offs) == ARG
    with pytest.raises(ValueError):
        L.trie_witness_batch(0, L.TRIE_LOOKUP, 1, np.zeros(32 * 9, dtype=np.uint8))   # not a whole call


def test_no_cpu_fallback(L):
    lib = _lib(L)
    if lib.lurk_device_count() > 0:
        pytest.skip("GPU present")
    buf = np.zeros(32 * 10, dtype=np.uint8)
    with pytest.raises(L.LurkError) as e:
        L.trie_witness_batch(0, L.TRIE_LOOKUP, 1, buf)
    assert e.value.code == L._capi.ERR_NOGPU
    out = np.zeros(32, dtype=np.uint8)
    offs = (C.c_uint64 * 1)(0)
    NOGPU = L._capi.ERR_NOGPU
    assert lib.lurk_trie_witness_batch_dev(0, 0, 1, L._capi.np_ptr(buf), 1, L._capi.np_ptr(out), 0, None) == NOGPU
    assert lib.lurk_trie_witness_scatter_dev(0, 1, 1, L._capi.np_ptr(buf), 1, offs, L._capi.np_ptr(out), 0, None) == NOGPU


def test_header_is_strict_c99(tmp_path):
    src = tmp_path / "t.c"
    src.write_text('#include "lurk_b200.h"\n'
                   "int main(void) {\n"
                   "    int (*batch)(int, int, int, const uint8_t *, size_t, uint8_t *, int) = lurk_trie_witness_batch;\n"
                   "    int (*dev)(int, int, int, const void *, size_t, void *, int, void *) = lurk_trie_witness_batch_dev;\n"
                   "    int (*scatter)(int, int, int, const void *, size_t, const uint64_t *, void *, int, void *) = lurk_trie_witness_scatter_dev;\n"
                   "    int (*fold)(lurk_fold_ctx *, int, int, size_t, const uint64_t *) = lurk_fold_ctx_add_trie_batch;\n"
                   "    (void)batch; (void)dev; (void)scatter; (void)fold;\n"
                   "    return (int)lurk_trie_witness_block(0, LURK_TRIE_LOOKUP, LURK_TRIE_MAX_HEIGHT) + LURK_TRIE_INSERT;\n"
                   "}\n")
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-c", str(src), "-o", str(tmp_path / "t.o")])


def test_proofs_and_packing(L):
    """prove_lookup / prove_insert over a tiny trie with an injected hash: the reference's semantics without a GPU"""
    class Cache:
        field_id = 0

        def compute_hash(self, pre):
            return (sum((i + 1) * x for i, x in enumerate(pre)) * 7 + 1) % (1 << 200)

    t = L.Trie(Cache(), 8, 3)
    proof = t.prove_lookup(0o123)
    assert len(proof.preimage_path) == 3 and proof.preimage_path[0] == (t.empty_roots[1],) * 8
    root0 = t.root
    ins, inserted = t.prove_insert(0o123, 99)
    assert inserted and t.root != root0 and t.lookup(0o123) == 99
    assert ins.old_proof == proof
    assert ins.new_proof.preimage_path[2][3] == 99 and ins.new_proof == t.prove_lookup(0o123)
    x = L.lookup_inputs(root0, 0o123, proof)
    assert len(x) == 2 + 8 * 3 and x[:2] == [root0, 0o123]
    y = L.insert_inputs(root0, 0o123, 99, ins)
    assert len(y) == 3 + 16 * 3 and y[27:] == [v for pre in ins.new_proof.preimage_path for v in pre]

