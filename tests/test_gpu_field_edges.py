"""csrc/field.cuh as ptxas compiled it for sm_90a, operation by operation, at the carry and reduction edges the limb model
(tests/field_model.py) constructs.

The device keeps its carries in the condition-code register across separate asm statements; the harness
tests/csrc/field_dev_test.cu (built by the library's Makefile into csrc/build/libfield_dev_test.so) runs every operation on arrays of
raw operands, and the constructed cases are checked against Python integers (the dot products against the model, which also
predicts reduce<3>'s results past its bound).  2^22 random products per field are checked against the same source built for the
host with the carry flag emulated.  Then the same edge operands go through the library's own entry points, where the code is
inlined into the real kernels: lurk_axpy_dev, lurk_cross_term_dev, lurk_spmv_csr_dev, lurk_convert_dev, lurk_ipa_fold_scalars_dev."""
import ctypes
import os

import numpy as np
import pytest

import field_model as fm
from test_field_model import build_host_harness, check_constructed, run_harness

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV_LIB = os.path.join(ROOT, "lurk-beta_b200", "csrc", "build", "libfield_dev_test.so")
BULK = 1 << 22


@pytest.fixture(scope="module")
def devlib(L):
    assert os.path.exists(DEV_LIB), "the operation harness is built by the library's Makefile (build())"
    L._capi.lib()                      # the library first: the harness links its own static CUDA runtime
    return ctypes.CDLL(DEV_LIB)


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    return build_host_harness(tmp_path_factory.mktemp("fdt"), emulate=True)


@pytest.fixture(scope="module", params=fm.FIELDS)
def constructed(request):
    F = fm.Field(request.param)
    cases = fm.constructed_cases(F)
    return F, cases, fm.model_events(F, cases)


def test_operations_on_constructed_cases(devlib, constructed):
    """every operation, inversion and conversion on the constructed operands; WideAcc k = 1..15 through reduce<3> and reduce<4>"""
    F, cases, (_, dots) = constructed
    check_constructed(devlib, F, cases, dots)
    # both inversions as x * x^-1 = 1 (Montgomery one) besides pow
    xs = [t for t in cases["inv"] if t[0]]
    for op in ("inv", "inv_vartime"):
        inv = run_harness(devlib, F.fid, op, xs)
        assert run_harness(devlib, F.fid, "mul", [(x, y) for (x,), y in zip(xs, inv)]) == [F.mont(1)] * len(xs), op
    # the canonical <-> Montgomery round trip
    canon = [t[0] for t in cases["from_canonical"]]
    mont = run_harness(devlib, F.fid, "from_canonical", [(x,) for x in canon])
    assert run_harness(devlib, F.fid, "to_canonical", [(x,) for x in mont]) == canon


@pytest.mark.parametrize("k", [1, 2, 7, 8, 9, 15, 16, 17])
def test_csr_row_dot_at_group_boundaries(devlib, k):
    """csr_row_dot (spmv3.cuh, the fold's and Spartan's R1CS rows): the one-product shortcut and the groups of 8 products, on rows at the
    reduction bound (all p - 1, and the constructed dot operands of each round) and near-top / word-pattern rows"""
    for fid in fm.FIELDS:
        F = fm.Field(fid)
        rng = np.random.default_rng(k)
        rows = [[F.p - 1] * (2 * k), [0] * (2 * k)]
        for g in (min(k, 8), k % 8):
            for rnd in range(1, 4):
                d = fm.dot_at_round(F, g, rnd, rng, tries=100) if g else None
                if d is not None:
                    rows.append(d[0] + [F.p - 1] * (k - g) + d[1] + [F.p - 1] * (k - g))
        rows += [fm.near_top(F, rng, 2 * k) for _ in range(64)] + [fm.word_patterns(F, rng, 2 * k) for _ in range(64)]
        rows = [tuple(r) for r in rows]
        assert run_harness(devlib, fid, "csr_row", rows, k) == [fm.expected(F, "dot4", r) for r in rows], (fid, k)


@pytest.mark.parametrize("field", fm.FIELDS)
def test_random_operations_against_the_emulated_host_build(devlib, hostlib, field):
    """2^22 random products, sums and differences, 2^19 of every one-operand operation, fewer inversions and dot products:
    the device bit for bit equal to the host build with the carry flag emulated"""
    F = fm.Field(field)
    rng = np.random.default_rng(1000 + field)

    def both(op, n, width, k=0):
        buf = fm.random_words(F, rng, n * width)
        if op in ("final_sub", "is_reduced"):
            buf = rng.integers(0, 1 << 32, size=(n, 8), dtype=np.uint64).astype(np.uint32)
        outs = []
        for lib in (devlib, hostlib):
            out = np.zeros((n, 8), dtype=np.uint32)
            assert lib.fdt_run(field, fm.OP[op], k, ctypes.c_size_t(n), buf.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p)) == 0
            outs.append(out)
        bad = np.flatnonzero((outs[0] != outs[1]).any(axis=1))
        assert bad.size == 0, (op, k, bad[:4], buf.reshape(n, -1)[bad[0]].tolist())
        return buf, outs[0]

    for op in ("mul", "add", "sub"):
        buf, out = both(op, BULK, 2)
        if op == "mul":      # spot-check the host build itself against integers
            a = fm.from_words(buf.reshape(-1, 2, 8)[:2000, 0].astype(np.uint64))
            b = fm.from_words(buf.reshape(-1, 2, 8)[:2000, 1].astype(np.uint64))
            assert fm.from_words(out[:2000].astype(np.uint64)) == [x * y * F.rinv % F.p for x, y in zip(a, b)]
    for op in ("sqr", "neg", "dbl", "pow5", "from_canonical", "to_canonical", "final_sub", "is_reduced"):
        both(op, BULK // 8, 1)
    both("inv_vartime", 1 << 14, 1)
    both("inv", 1 << 11, 1)
    for op in ("mul_sub_mul", "ipa_fold"):
        both(op, 1 << 17, 4)
    for k in (2, 8, 9, 11, 15):
        both("dot" if k <= fm.REDUCE3_MAX_K[field] else "dot4", 1 << 15, 2 * k, k)


# ------------------------------------------------------------------------------------------------------------------- real kernels
def _dev(words):
    import torch
    return torch.from_numpy(np.ascontiguousarray(fm.pack_cases([(v,) for v in words]))).cuda()


def _host(t):
    return fm.from_words(t.cpu().numpy().view("<u4").astype(np.uint64))


def _edge_operands(F, rng, n):
    vals = fm.edge_values(F) + [fm.near_top(F, rng, 1)[0] for _ in range(32)] + fm.word_patterns(F, rng, 64)
    return [vals[i] for i in rng.integers(0, len(vals), size=n)]


@pytest.mark.parametrize("field", fm.FIELDS)
def test_edge_operands_inside_the_library_kernels(L, field):
    """the constructed operands through the entry points whose operands the caller controls (Montgomery form in and out)"""
    import torch
    lib, F = L._capi.lib(), fm.Field(field)
    p, ri = F.p, F.rinv
    rng = np.random.default_rng(field)
    pairs = fm.chosen_products(F, rng)
    m = len(pairs)
    a, b = [x for x, _ in pairs], [y for _, y in pairs]
    c, d = _edge_operands(F, rng, m), _edge_operands(F, rng, m)
    da, db, dc, dd = _dev(a), _dev(b), _dev(c), _dev(d)
    out = torch.empty_like(da)
    # out = a + r b
    for r in fm.edge_values(F)[::3] + [p - 1]:
        L._capi.check(lib.lurk_axpy_dev(field, da.data_ptr(), db.data_ptr(), L._capi.np_ptr(fm.pack_cases([(r,)])), m, out.data_ptr(), None))
        assert _host(out) == [(x + r * y * ri) % p for x, y in zip(a, b)], hex(r)
    # T = az1 bz2 + az2 bz1 - u1 cz2 - u2 cz1 with (az1, bz2) the chosen-product pairs
    for u1, u2 in ((p - 1, p - 1), (0, p - 1), (F.mont(1), 1), (fm.near_top(F, rng, 1)[0], p - 2)):
        L._capi.check(lib.lurk_cross_term_dev(field, da.data_ptr(), dc.data_ptr(), dd.data_ptr(), dd.data_ptr(), db.data_ptr(), dc.data_ptr(),
                                              L._capi.np_ptr(fm.pack_cases([(u1,)])), L._capi.np_ptr(fm.pack_cases([(u2,)])), m, out.data_ptr(), None))
        want = [(x * y + w * z - u1 * z2 - u2 * w2) * ri % p for x, y, w, z, z2, w2 in zip(a, b, d, c, c, d)]
        assert _host(out) == want, (hex(u1), hex(u2))
    # format conversion both ways, in place and out of place
    canon = [x % p for x in a]
    dcan = _dev(canon)
    L._capi.check(lib.lurk_convert_dev(field, dcan.data_ptr(), m, L.FMT_MONTGOMERY, out.data_ptr(), None))
    assert _host(out) == [x * fm.R % p for x in canon]
    L._capi.check(lib.lurk_convert_dev(field, out.data_ptr(), m, L.FMT_CANONICAL, out.data_ptr(), None))
    assert _host(out) == canon
    # IPA scalar fold: a'[i] = x a[i] + y a[i + n/2]
    n = 1 << (m.bit_length() - 1)
    for x, y in ((p - 1, p - 1), (F.mont(1), p - 1), (fm.near_top(F, rng, 1)[0], 0)):
        buf = _dev(a[:n // 2] + b[:n // 2])
        L._capi.check(lib.lurk_ipa_fold_scalars_dev(field, buf.data_ptr(), n, L._capi.np_ptr(fm.pack_cases([(x,)])),
                                                    L._capi.np_ptr(fm.pack_cases([(y,)])), L.FMT_MONTGOMERY, None))
        assert _host(buf)[:n // 2] == [(x * lo + y * hi) * ri % p for lo, hi in zip(a[:n // 2], b[:n // 2])]
    # y = M z: rows of 1, 2, 7, 8, 9, 15, 16 and 17 non-zeros, coefficients and z at the constructed values
    lens = [1, 2, 7, 8, 9, 15, 16, 17] * 24
    nnz = sum(lens)
    z = a + b
    val = [v for i in range(nnz) for v in ([p - 1, a[i % m], b[i % m]][i % 3],)]
    col = rng.integers(0, len(z), size=nnz).astype(np.uint32)
    col[: nnz // 4] = np.arange(nnz // 4) % m        # column i of (a, b) against its chosen partner as the value
    val[: nnz // 4] = [b[i % m] for i in range(nnz // 4)]
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    d_rp, d_col = torch.from_numpy(rp).cuda(), torch.from_numpy(col).cuda()
    d_val, d_z = _dev(val), _dev(z)
    y = torch.empty(len(lens) * 32, dtype=torch.uint8, device="cuda")
    L._capi.check(lib.lurk_spmv_csr_dev(field, d_rp.data_ptr(), d_col.data_ptr(), d_val.data_ptr(), len(lens), d_z.data_ptr(), y.data_ptr(), None))
    want = [sum(val[k] * z[int(col[k])] for k in range(int(rp[i]), int(rp[i + 1]))) * ri % p for i in range(len(lens))]
    assert _host(y) == want
