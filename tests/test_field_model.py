"""The limb model of csrc/field.cuh (tests/field_model.py) against Python integers, the coverage of its operand builders, and the
operation harness tests/csrc/field_dev_test.cu built for the host (carry flag emulated, and the host's 64-bit product) on the same
constructed cases.  tests/test_gpu_field_edges.py runs the harness built for sm_90a on them."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import field_model as fm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

COMMON = {"merge_carry", "cmad_n_carry", "final_sub", "sub_borrow", "round1", "round2", "round3",
          "ce0", "ce1", "ce2", "ce3", "co0", "co1", "co2", "co3",
          "inv_zero", "inv_no_loop", "inv_exit_u", "inv_exit_w", "inv_halve_odd"}
REACHABLE = {0: COMMON | {"mod0_carry"}, 1: COMMON | {"mod0_carry"}, 2: COMMON | {"round4"}, 3: COMMON | {"round4"}}
# events the model never shows, and why
NEVER = {
    "mod1_carry": "the carry out of cmad_mod<1>, which mad_row_redc drops: the running sum stays below 2p < 2^256 + 2^224 at every row",
    "addc_overflow": "a carry out of an addc without carry-out (odd[7], r[7], t[16], the pending counters) would be lost: bounded like mod1_carry",
    "ce4": "column 16 of WideAcc's even half is reached only by hi(a[7] b[7]) + 1 per product; a[7], b[7] < 2^30 keep 15 products below 2^32",
    "unreduced": "redc17 leaves a value >= p only when k exceeds the ROUNDS bound of WideAcc::reduce's comment",
}
NEVER_ON = {
    "mod0_carry": ({2, 3}, "Pasta's modulus words 4..6 are zero, so the m*p row carries out of even[7] only when columns 4..7 of the even half are "
                           "all ones; no constructed, word-pattern or random operand gets there"),
    "round4": ({0, 1}, "BN254: 15 products give at most (15 p / 2^256 + 1) p < 3.84 p before the subtractions"),
}


@pytest.fixture(scope="module", params=fm.FIELDS)
def constructed(request):
    F = fm.Field(request.param)
    cases = fm.constructed_cases(F)
    return F, cases, fm.model_events(F, cases)


def test_model_equals_integers(constructed):
    F, cases, (_, dots) = constructed
    for op, fn in (("mul", fm.mul), ("add", fm.add), ("sub", fm.sub)):
        args = cases[op]
        out, _ = fn(F, fm.to_words([t[0] for t in args]), fm.to_words([t[1] for t in args]))
        assert fm.from_words(out) == [fm.expected(F, op, t) for t in args], op
    raw = [t[0] for t in cases["final_sub"]]
    out, reduced, _ = fm.final_sub(F, fm.to_words(raw))
    assert fm.from_words(out) == [fm.expected(F, "final_sub", (v,)) for v in raw]
    assert list(reduced) == [bool(fm.expected(F, "is_reduced", (v,))) for v in raw]
    for (x,) in cases["inv_vartime"]:
        assert fm.inv_vartime(F, x)[0] == fm.expected(F, "inv", (x,)), x
    for (k, rounds), (vals, ev) in dots.items():
        want = [fm.expected(F, "dot4", r) for r in cases[("dot", k)]]
        if rounds == 4 or k <= fm.REDUCE3_MAX_K[F.fid]:
            assert vals == want and not ev["unreduced"].any(), (k, rounds)
        else:
            # past the bound reduce<3> is wrong exactly where the model says the value is still >= p
            assert [v % F.p for v in vals] == want
            assert [v != w for v, w in zip(vals, want)] == list(ev["unreduced"])


def test_model_reaches_every_event(constructed):
    """the constructed operands reach every event of REACHABLE; the others are never seen over them plus 10^5 random and 10^5
    word-pattern products and 10^5 near-top dot operands"""
    F, cases, (seen, dots) = constructed
    never = set(NEVER) | {e for e, (fields, _) in NEVER_ON.items() if F.fid in fields}
    assert seen == REACHABLE[F.fid], (sorted(REACHABLE[F.fid] - seen), sorted(seen - REACHABLE[F.fid]))
    assert not seen & never
    rng = np.random.default_rng(100 + F.fid)
    extra = set()
    for gen in (fm.random_below, fm.word_patterns):
        _, ev = fm.mul(F, fm.to_words(gen(F, rng, 100000)), fm.to_words(gen(F, rng, 100000)))
        extra |= {e for e, m in ev.items() if m.any()}
    for k in (9, 15):
        n = 100000 // (2 * k)
        A = np.stack([fm.random_words(F, rng, n).astype(np.uint64) for _ in range(k)], axis=1)
        A[:n // 2] = np.stack([fm.to_words(fm.near_top(F, rng, n // 2)) for _ in range(k)], axis=1)
        B = np.stack([fm.to_words(fm.near_top(F, rng, n)) for _ in range(k)], axis=1)
        _, ev, _ = fm.dot(F, A, B, 4)
        extra |= {e for e, m in ev.items() if m.any()}
    assert not extra & never, sorted(extra & never)


def test_reasons_for_the_unreachable_rounds():
    """the bounds behind NEVER_ON["round4"] and ce4, and why Pasta's 2nd subtraction at k = 4 has no operands (dot_at_round finds none):
    with a = p - alpha, b = p - beta the value before the subtractions reaches 2p only if sum (alpha + beta) < 4 d + 1 and
    sum alpha beta = p (d = p - 2^254), and sum alpha beta <= (sum (alpha + beta))^2 / 4 < 4 d^2 + 2 d + 1 < p"""
    for fid in (0, 1):
        p = fm.Field(fid).p
        assert 15 * (p - 1) ** 2 + (fm.R - 1) * p < 4 * p * fm.R
    for fid in fm.FIELDS:
        top = fm.Field(fid).mod[7]
        assert 15 * ((top * top >> 32) + 1) < 1 << 32
    for fid in (2, 3):
        F = fm.Field(fid)
        d = F.p - (1 << 254)
        assert (4 * d + 1) ** 2 // 4 < F.p
        assert fm.dot_at_round(F, 4, 2, np.random.default_rng(0), tries=500) is None
        assert fm.dot_at_round(F, 8, 3, np.random.default_rng(0)) is not None
        assert fm.dot_at_round(F, 12, 4, np.random.default_rng(0)) is not None


def build_host_harness(out_dir, emulate):
    out = os.path.join(str(out_dir), "libfdt_%s.so" % ("emulated" if emulate else "host"))
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas"]
                          + (["-DLURK_HOST_EMULATE_CC"] if emulate else []) +
                          ["-I", os.path.join(ROOT, "lurk-beta_b200", "csrc"), "-x", "c++",
                           os.path.join(ROOT, "tests", "csrc", "field_dev_test.cu"), "-o", out])
    return ctypes.CDLL(out)


def run_harness(lib, fid, op, args, k=0):
    buf = fm.pack_cases(args)
    out = np.zeros(32 * len(args), dtype=np.uint8)
    rc = lib.fdt_run(fid, fm.OP[op], k, ctypes.c_size_t(len(args)), buf.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p))
    assert rc == 0, (op, rc)
    return fm.from_words(out.view("<u4").astype(np.uint64))


def check_constructed(lib, F, cases, dots):
    """every operation of the harness on the constructed cases: Python integers, and the model for the dot products"""
    for op in fm.OPS[:fm.OP["dot"]]:
        args = cases[op]
        assert run_harness(lib, F.fid, op, args) == [fm.expected(F, op, t) for t in args], op
    for k in range(1, 16):
        rows = cases[("dot", k)]
        for rounds, op in ((3, "dot"), (4, "dot4")):
            assert run_harness(lib, F.fid, op, rows, k) == dots[(k, rounds)][0], (op, k)


@pytest.mark.parametrize("emulate", [True, False], ids=["emulated_gpu_limbs", "host_fast_path"])
def test_host_harness_on_constructed_cases(tmp_path_factory, constructed, emulate):
    F, cases, (_, dots) = constructed
    check_constructed(build_host_harness(tmp_path_factory.mktemp("fdt"), emulate), F, cases, dots)
