"""The MSM (csrc/msm_impl.cuh) checked exactly on keys of known discrete logarithm, and driven through every branch of the group law.

If base i is [k_i]G then commit(s) = [sum s_i k_i mod q]G: one Python scalar multiplication gives the exact result at any size and on
any curve.  Two kinds of key:
  * tiled keys: a handful of points [k]G (k = 0, +-1, 2 .. 8) laid out by an index array, so that sums collide on purpose;
  * powers-of-tau keys beta^i g: distinct points, expected [f(beta)]g by Horner.

Random keys never make two bucket sums collide, so the kernels' group-law branches (P + P doubles, P + (-P) is the identity, an
identity operand is passed through) are reached only by inputs built for it.  The degenerate patterns below are built for it, and a
plan model restates make_plan and the signed digits in Python and replays the accumulation, merge and bucket reduction on the
discrete logs, recording which branch every addition takes.  Inside a bucket the order of the sorted entries is decided by the sort's
atomics, so the model replays a bucket's additions only where that order cannot change them: every entry the same point, or (under
the warp-aggregated sort) every contributing warp laying down the same sequence.  Each test asserts that the designed collisions do
happen in the model, so a later plan change cannot quietly stop a test from reaching its branch, and test_model_reaches_every_branch
asserts that together they reach every named branch of every kernel.
"""
import functools
from collections import Counter

import numpy as np
import pytest

from oracle import kzg
from util import ints, pack, random_elements

pytestmark = pytest.mark.gpu
CURVES = [0, 1, 2, 3]

# csrc/msm_impl.cuh
MSM_LONG_PARTIALS, MSM_MERGE_LONG_THREADS, BITSUM_THREADS = 16, 256, 256
MSM_SORT_SMEM_MAX = 128 << 10


# ------------------------------------------------------------------------------------------------------------------------- plan model
@functools.lru_cache(maxsize=None)
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


class Plan:
    """make_plan(n, bits, fixed_c) with the SM count of the device, and whether a read-back commitment takes the table (msm_launch)"""

    def __init__(self, n, bits, fixed_c=0, sms=None):
        lg = n.bit_length() - 1
        self.n, self.bits = n, bits
        self.c = fixed_c or min(20, max(4, lg - 5))
        self.nwin = bits // self.c + 1
        self.fixed = fixed_c != 0
        self.nb = 1 << (self.c - 1)
        self.rwin = 1 if self.fixed else self.nwin
        self.K = min(8, self.nb)
        self.G = self.nb // self.K
        self.nq = 1
        while (1 << (self.nq - 1)) < self.G:
            self.nq += 1
        self.SL = min(32, max(1, self.G // 2048))
        self.slice = self.G // self.SL
        cap, want = n * self.nwin, (sms or sm_count()) * 1024
        self.seg = min(32, max(8, -(-cap // want)))
        # a table is used only when its shared bucket set is well filled
        self.table_pays = not self.fixed or n * self.nwin >= 8 << (self.c - 1)

    def smem_sort(self, legacy):
        return self.fixed and self.nb * 4 <= MSM_SORT_SMEM_MAX and not legacy

    def __repr__(self):
        return "Plan(c=%d nwin=%d K=%d G=%d nq=%d SL=%d seg=%d)" % (self.c, self.nwin, self.K, self.G, self.nq, self.SL, self.seg)


def signed_digits(s, c, nwin):
    """(window, magnitude, negative) of every non-zero signed c-bit digit, as msm_count_kernel cuts them"""
    out, carry, half = [], 0, 1 << (c - 1)
    for w in range(nwin):
        raw = ((s >> (w * c)) & ((1 << c) - 1)) + carry
        neg = raw > half
        mag = (1 << c) - raw if neg else raw
        carry = int(neg)
        if mag:
            out.append((w, mag, neg))
    return out


class Group:
    """point additions on discrete logs mod q: each records which branch of XYZZ::add / add_affine it takes"""

    def __init__(self, q):
        self.q, self.seen = q, set()

    def add(self, stage, a, b):
        if b == 0:
            self.seen.add((stage, "id_rhs"))
            return a
        if a == 0:
            self.seen.add((stage, "id_lhs"))
            return b
        if a == b:
            self.seen.add((stage, "dbl"))
            return 2 * a % self.q
        if (a + b) % self.q == 0:
            self.seen.add((stage, "inf"))
            return 0
        return (a + b) % self.q


def model(plan, key_dlog, kidx, sval, sidx, q, warp_sort):
    """Replay one commitment on discrete logs.  Returns (result, branches seen, facts about the buckets)."""
    grp, facts = Group(q), set()
    n = len(kidx)
    m = len(sval)
    digits = [signed_digits(s, plan.c, plan.nwin) for s in sval]
    # warps of the scatter kernel: 32 consecutive scalars; identical warps lay down identical sequences
    combo = np.full(-(-n // 32) * 32, -1, dtype=np.int64)
    combo[:n] = kidx.astype(np.int64) * m + sidx
    rows, row_count = np.unique(combo.reshape(-1, 32), axis=0, return_counts=True)
    contrib = {}                                 # bucket -> [(row, window, chunk of discrete logs in lane order)]
    for r, row in enumerate(rows):
        chunks = {}
        for cmb in row:
            if cmb < 0:
                continue
            k = key_dlog[cmb // m]
            for w, mag, neg in digits[cmb % m]:
                e = k << (plan.c * w) if plan.fixed else k
                e = (-e if neg else e) % q
                key = (0 if plan.fixed else w * plan.nb) + mag - 1
                chunks.setdefault((key, w), []).append(e)
        for (key, w), ch in chunks.items():
            contrib.setdefault(key, []).append((r, w, ch))
    counts = {key: sum(len(ch) * int(row_count[r]) for r, w, ch in lst) for key, lst in contrib.items()}
    offsets, run = {}, 0
    for key in sorted(counts):
        offsets[key] = run
        run += counts[key]
    seg = plan.seg
    B = {}
    for key, lst in contrib.items():
        lo, hi = offsets[key], offsets[key] + counts[key]
        entries = Counter()
        for r, w, ch in lst:
            for e in ch:
                entries[e] += int(row_count[r])
        total = sum(e * c for e, c in entries.items()) % q
        if total == 0 and any(entries):
            facts.add(("bucket", "inf"))         # a non-empty bucket whose sum is the identity
        if 0 in entries:
            grp.seen.add(("accumulate", "id_rhs"))   # an identity entry is skipped wherever it lands
        if len(entries) == 1 or hi - lo == 2:    # the additions do not depend on the order
            seq = sorted(entries.elements())
            period = 1 if len(entries) == 1 else 2
            at = lambda t, seq=seq: seq[t % len(seq)]
        elif warp_sort and len(lst) == 1:        # every contributing warp lays down the same sequence
            seq = lst[0][2]
            period = len(seq)
            at = lambda t, seq=seq: seq[t % len(seq)]
        else:
            B[key] = total                       # the order inside the bucket is the atomics': only its sum is known
            continue
        facts.add(("bucket", "exact"))
        # pieces of the bucket cut at segment boundaries: the first is the bucket's own slot, the others partials
        memo, pieces, a = {}, [], lo
        while a < hi:
            b = min(hi, (a // seg + 1) * seg)
            mk = (a - lo) % period, b - a
            if mk not in memo:
                acc = 0
                for t in range(a - lo, b - lo):
                    acc = grp.add("accumulate", acc, at(t))
                memo[mk] = acc
            pieces.append(memo[mk])
            a = b
        acc, parts = pieces[0], pieces[1:]
        if len(parts) <= MSM_LONG_PARTIALS:
            for p in parts:
                acc = grp.add("merge", acc, p)
        else:
            facts.add(("bucket", "long"))
            sm = []
            for tid in range(MSM_MERGE_LONG_THREADS):
                x = acc if tid == 0 else 0
                for j in range(tid, len(parts), MSM_MERGE_LONG_THREADS):
                    x = grp.add("merge_long", x, parts[j])
                sm.append(x)
            acc = _tree(grp, "merge_long", sm)
        assert acc == total
        B[key] = acc
    # bucket reduction: msm_chunk_kernel, msm_bitsum_kernel, msm_slice_sum_kernel
    tri, runs = {}, {}
    for g in sorted({key // plan.K for key in B if B[key]}):
        r_, t_ = 0, 0
        for b in range(plan.K - 1, -1, -1):
            r_ = grp.add("chunk", r_, B.get(g * plan.K + b, 0))
            t_ = grp.add("chunk", t_, r_)
        tri[g], runs[g] = t_, r_
    wins = []
    for w in range(plan.rwin):
        for qq in range(plan.nq):
            sl_sums = [_bitsum(grp, plan, tri, runs, w, qq, sl) for sl in range(plan.SL)]
            if plan.SL > 1:
                lanes = sl_sums + [0] * (32 - plan.SL)
                for d in (16, 8, 4, 2, 1):
                    if d < plan.SL:
                        lanes = [grp.add("slice", lanes[l], lanes[l ^ d]) for l in range(32)]
                wins.append(lanes[0])
            else:
                wins.append(sl_sums[0])
    logk = plan.K.bit_length() - 1
    if plan.fixed:                               # msm_horner_kernel: doublings per lane, then a butterfly
        lanes = [0] * 32
        for l in range(plan.nq):
            lanes[l] = wins[l] << (logk + l - 1) if l else wins[0]
        lanes = [x % q for x in lanes]
        for d in (16, 8, 4, 2, 1):
            lanes = [grp.add("horner", lanes[l], lanes[l ^ d]) for l in range(32)]
        result = lanes[0]
    else:                                        # msm_finish on the host
        result = 0
        for w in range(plan.nwin - 1, -1, -1):
            a = 0
            for k in range(plan.nq - 1, 0, -1):
                a = grp.add("host", 2 * a % q, wins[w * plan.nq + k])
            a = grp.add("host", (a << logk) % q, wins[w * plan.nq])
            result = grp.add("host", (result << plan.c) % q, a)
    if plan.fixed and any(key_dlog[k] == 0 for k in set(kidx.tolist())):
        grp.seen.add(("precompute", "id"))       # an identity base: its table rows stay the identity
    return result, grp.seen | facts


def _tree(grp, stage, sm):
    stride = len(sm) // 2
    while stride:
        for t in range(stride):
            sm[t] = grp.add(stage, sm[t], sm[t + stride])
        stride //= 2
    return sm[0]


def _bitsum(grp, plan, tri, runs, w, qq, sl):
    """block (sl, qq, w) of msm_bitsum_kernel: strided sums per thread, then the shared-memory tree"""
    base = w * plan.G + sl * plan.slice
    items = []                                   # (thread, order, value)
    src = tri if qq == 0 else runs
    lo, hi = base, base + plan.slice
    for g in (g for g in src if lo <= g < hi):
        local = g - base
        if qq == 0:
            items.append((local % BITSUM_THREADS, local, src[g]))
        else:
            k = qq - 1
            if plan.slice > 1 << k:
                if (local >> k) & 1:
                    j = ((local >> (k + 1)) << k) | (local & ((1 << k) - 1))
                    items.append((j % BITSUM_THREADS, j, src[g]))
            elif ((sl * plan.slice) >> k) & 1:
                items.append((local % BITSUM_THREADS, local, src[g]))
    if not items:
        return 0
    sm = [0] * BITSUM_THREADS
    for tid, _, v in sorted(items):
        sm[tid] = grp.add("bitsum", sm[tid], v)
    return _tree(grp, "bitsum", sm)


# ------------------------------------------------------------------------------------------------------------ degenerate patterns
# tiled keys index this table of discrete logs; -1 stands for q - 1
KEY_DLOGS = [0, 1, -1, 2, 3, 4, 5, 6, 7, 8]
ID, G1, NEG = 0, 1, 2


def _mult(k):
    return KEY_DLOGS.index(k)


def _aligned(n, period, warps=True):
    """length of the prefix whose scalars are used: whole periods, and whole warps once there is more than one warp, so that every warp
    of the scatter lays down the same sequence (the tail's scalars are zero)"""
    step = int(np.lcm(period, 32)) if warps and n > 32 else period
    return n - n % step


def _spread(plan, digits):
    """the same digits in every slice of the bucket reduction (fixed-base: one bucket set), so that the slice sums are equal"""
    sk = plan.slice * plan.K
    return [d + j * sk for j in range(plan.SL if plan.fixed else 1) for d in digits]


def pat_equal(n, plan):
    """every base G: each run is [m]G, a long bucket's partials are all equal; digits 1 and 2 equally often make two equal buckets
    in one chunk, digits K + 1 and K + 2 an equal chunk beside it (the bit sums' tree adds two equal points), repeated in every slice"""
    vals = [0] + _spread(plan, [1, 2] + ([plan.K + 1, plan.K + 2] if plan.G >= 2 else []))
    L = _aligned(n, len(vals) - 1)
    i = np.arange(n)
    return np.full(n, G1), vals, np.where(i < L, 1 + i % (len(vals) - 1), 0)


def pat_alternating(n, plan):
    """G, -G, G, ... (powers of tau with beta = q - 1) and one digit: the bucket sums to the identity; a warp's runs cancel every
    second entry.  Warp 0 instead holds a bucket of exactly {G, -G} and one of exactly {G, G}"""
    i = np.arange(n)
    sidx = np.where(i < _aligned(n, 2), 1, 0)
    sidx[:32] = 0
    sidx[:2] = 2
    sidx[2:5:2] = 3
    return np.where(i % 2 == 0, G1, NEG), [0, 1, 3, 5], sidx[:n]


def pat_blocks(n, plan):
    """a block of G, then a block of -G, each as long as a segment: whole partials cancel inside the merge"""
    i = np.arange(n)
    return np.where((i // plan.seg) % 2 == 0, G1, NEG), [0, 1], np.where(i < _aligned(n, 2 * plan.seg), 1, 0)


def pat_sparse(n, plan):
    """G and the identity alternating: the accumulation skips identity entries, the table keeps identity rows"""
    i = np.arange(n)
    return np.where(i % 2 == 0, G1, ID), [0, 1], np.where(i < _aligned(n, 2), 1, 0)


def pat_multiples(n, plan):
    """[8]G with digit 1, [4]G with digit 2 (twice as often), [2]G with 4, G with 8: four different buckets of one chunk with equal
    sums (different points), repeated in every slice"""
    block = [(8, 1)] + [(4, 2)] * 2 + [(2, 4)] * 4 + [(1, 8)] * 8
    per = len(block)
    vals = [0] + _spread(plan, [1, 2, 4, 8])
    kd, sd = [], []
    for j in range(plan.SL if plan.fixed else 1):
        for k, d in block:
            kd.append(_mult(k))
            sd.append(1 + 4 * j + [1, 2, 4, 8].index(d))
    period = len(kd)
    i = np.arange(n)
    L = _aligned(n, period, warps=False)         # every bucket holds one point: the order does not matter
    return np.array(kd)[i % period], vals, np.where(i < L, np.array(sd)[i % period], 0)


def pat_weights(n, plan):
    """the final weighted sums: digit 2K alone makes T = K S_0 (bucket K - 1 of chunk 1 carries weight K in T and K in S_0), so the
    last level of msm_horner_kernel's butterfly and the host's Horner over one bucket set add equal points.  Windowed, digit 1 in
    window 1 once and digit 2^(c-1) in window 0 twice give R_1 2^c = R_0 (the larger windowed sizes), equal operands in the host's
    Horner over the windows"""
    i = np.arange(n)
    if plan.fixed or n < 4096:
        vals, per = [0, 2 * plan.K], [1]
    else:
        vals, per = [0, 1 << plan.c, 1 << (plan.c - 1)], [1, 2, 2, 0]
    per = np.array(per)
    L = _aligned(n, len(per))
    return np.full(n, G1), vals, np.where(i < L, per[i % len(per)], 0)


PATTERNS = {"equal": pat_equal, "alternating": pat_alternating, "blocks": pat_blocks, "sparse": pat_sparse, "multiples": pat_multiples,
            "weights": pat_weights}


def designed(pattern, plan, seen, n_used, warp_sort):
    """the collisions each pattern is built to make, where its plan allows them"""
    want = set()
    merge = "merge_long" if ("bucket", "long") in seen else "merge"
    if pattern == "equal":
        want.add(("chunk", "dbl"))
        if n_used >= 4:
            want.add(("accumulate", "dbl"))
        if n_used >= 8 * plan.seg * plan.SL:     # digit 1's bucket starts a segment and has a whole partial
            want.add((merge, "dbl"))
        if plan.G >= 2:
            want.add(("bitsum", "dbl"))
        if plan.SL > 1:
            want.add(("slice", "dbl"))
    elif pattern == "weights":
        if plan.fixed:
            want.add(("horner", "dbl"))
        elif plan.G >= 2:
            want.add(("host", "dbl"))
    elif pattern == "alternating":
        want.add(("accumulate", "inf"))
        if plan.n >= 5:
            want.add(("accumulate", "dbl"))
        if plan.n >= 64:
            want.add(("bucket", "inf"))
    elif pattern == "blocks":
        if n_used >= 2 * plan.seg:
            want.add(("bucket", "inf"))
            if warp_sort and 32 % (2 * plan.seg) == 0:
                want.add((merge, "inf"))
    elif pattern == "sparse":
        want.add(("accumulate", "id_rhs"))
        if plan.fixed:
            want.add(("precompute", "id"))
    elif pattern == "multiples":
        if n_used >= 15:
            want.add(("chunk", "dbl"))
        if plan.SL > 1:
            want.add(("slice", "dbl"))
    return want


# ------------------------------------------------------------------------------------------------------------------ keys and checks
@functools.lru_cache(maxsize=None)
def _point_table(curve):
    from oracle import spec
    Cv = spec.CURVES[curve]
    pb, q = spec.FIELD_MODULUS[Cv["base"]], spec.FIELD_MODULUS[Cv["scalar"]]
    pts = [spec.ec_mul(k % q, Cv["gen"], pb) for k in KEY_DLOGS]
    return np.stack([pack(p if p else (0, 0)) for p in pts])


def curve_consts(spec, curve):
    Cv = spec.CURVES[curve]
    return spec.FIELD_MODULUS[Cv["base"]], spec.FIELD_MODULUS[Cv["scalar"]], spec.FIELD_NUM_BITS[Cv["scalar"]], Cv["gen"]


def point_record(spec, curve, k, g=None):
    """[k]g as the library returns it: canonical x | y | 1, the identity all zeros"""
    pb, q, _, gen = curve_consts(spec, curve)
    P = spec.ec_mul(k % q, g or gen, pb)
    return np.zeros(96, dtype=np.uint8) if P is None else pack([P[0], P[1], 1])


class Case:
    """one degenerate input on one curve: key (host bytes), scalars (host bytes), expected point, and the plan model's verdict"""

    def __init__(self, spec, curve, pattern, n, fixed_c=0, warp_sort=True, device=True):
        pb, q, bits, _ = curve_consts(spec, curve)
        self.plan = Plan(n, bits, fixed_c)
        kidx, sval, sidx = PATTERNS[pattern](n, self.plan)
        dl = [k % q for k in KEY_DLOGS]
        combo, cnt = np.unique(kidx.astype(np.int64) * len(sval) + sidx, return_counts=True)
        self.dlog = sum(dl[c // len(sval)] * sval[c % len(sval)] * int(k) for c, k in zip(combo, cnt)) % q
        self.n_used = int(np.count_nonzero(sidx))
        self.model_result, self.seen = model(self.plan, dl, kidx, sval, sidx, q, warp_sort)
        self.designed = designed(pattern, self.plan, self.seen, self.n_used, warp_sort)
        if device:
            self.bases = _point_table(curve)[kidx].reshape(-1)
            self.scalars = pack(sval).reshape(-1, 32)[sidx].reshape(-1)
            self.want = point_record(spec, curve, self.dlog)

    def check_model(self):
        assert self.model_result == self.dlog, self.plan
        missing = self.designed - self.seen
        assert not missing, (missing, self.plan)


WINDOWED_SIZES = [2, 33, 1025, 1 << 14, (1 << 16) + 1]
FIXED_N = 1 << 19                   # the table pays at every window below: n * nwin >= 8 * 2^(c - 1)
FIXED_WINDOWS = [10, 13, 16, 17, 20]


@pytest.mark.parametrize("pattern", list(PATTERNS))
@pytest.mark.parametrize("n", WINDOWED_SIZES)
@pytest.mark.parametrize("curve", CURVES)
def test_windowed_degenerate(L, spec, curve, n, pattern):
    case = Case(spec, curve, pattern, n)
    case.check_model()
    assert np.array_equal(L.CommitmentKey(curve, case.bases).commit(case.scalars), case.want), (pattern, n, case.plan)


@pytest.mark.parametrize("pattern", list(PATTERNS))
@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("c", FIXED_WINDOWS)
def test_fixed_base_degenerate(L, spec, monkeypatch, c, curve, pattern):
    """the fixed-base table at every window the sort treats differently: c = 16, the largest shared-memory histogram; c = 17, global
    atomics with SL = 4; c = 20, SL = 32; and, wherever the shared-memory sort is the default, LURK_MSM_SORT=legacy too"""
    ck = None
    try:
        for legacy in (False, True):
            plan = Plan(FIXED_N, 254, c)
            case = Case(spec, curve, pattern, FIXED_N, c, warp_sort=not plan.smem_sort(legacy))
            assert case.plan.table_pays and case.plan.c == c
            case.check_model()
            ck = ck or L.CommitmentKey(curve, case.bases).precompute(c)
            if legacy:
                monkeypatch.setenv("LURK_MSM_SORT", "legacy")
            else:
                monkeypatch.delenv("LURK_MSM_SORT", raising=False)
            assert np.array_equal(ck.commit(case.scalars), case.want), (pattern, c, legacy, case.plan)
            if not plan.smem_sort(False):
                break                              # the global-atomics sort is already the default
    finally:
        if ck:
            ck.close()


@pytest.mark.parametrize("curve", CURVES)
def test_launch_device_and_finish(L, spec, curve):
    import torch
    case = Case(spec, curve, "multiples", 1025)
    ck = L.CommitmentKey(curve, case.bases)
    d = torch.from_numpy(case.scalars).cuda()
    ck.launch_device(d.data_ptr(), 1025, fmt=L.FMT_CANONICAL, stream=torch.cuda.current_stream().cuda_stream)
    assert np.array_equal(ck.finish(), case.want)


def test_model_reaches_every_branch(spec):
    """together the patterns reach, in the model, every group-law branch of every kernel that adds points"""
    seen = set()
    for curve in (0, 2):
        for pattern in PATTERNS:
            for n in WINDOWED_SIZES:
                seen |= Case(spec, curve, pattern, n, device=False).seen
            for c in FIXED_WINDOWS:
                for ws in (False, True):
                    seen |= Case(spec, curve, pattern, FIXED_N, c, warp_sort=ws, device=False).seen
    want = {("accumulate", b) for b in ("dbl", "inf", "id_rhs")}
    want |= {(s, b) for s in ("merge", "merge_long") for b in ("dbl", "inf")}
    want |= {("chunk", "dbl"), ("bitsum", "dbl"), ("slice", "dbl"), ("horner", "dbl"), ("host", "dbl"), ("precompute", "id")}
    want |= {("bucket", "inf"), ("bucket", "long")}
    assert not want - seen, sorted(want - seen)


# --------------------------------------------------------------------------------------------------------------- distinct-point keys
def horner(coeffs, beta, q):
    acc = 0
    for s in reversed(coeffs):
        acc = (acc * beta + s) % q
    return acc


def _beta(spec, curve, seed):
    return ints(random_elements(spec.CURVES[curve]["scalar"], 1, seed=seed))[0]


@pytest.mark.parametrize("curve", CURVES)
def test_powers_of_tau_key_windowed_and_fixed(L, spec, curve):
    """a small powers-of-tau key, plain and with a table: [f(beta)]g, f the scalar vector"""
    pb, q, bits, gen = curve_consts(spec, curve)
    g = spec.ec_mul(987654321, gen, pb)
    beta, n = _beta(spec, curve, 7 + curve), 5000
    ck = L.CommitmentKey.powers_of_tau(curve, g, beta, n)
    sc = random_elements(spec.CURVES[curve]["scalar"], n, seed=curve, shape="witness")
    want = point_record(spec, curve, horner(ints(sc), beta, q), g)
    assert np.array_equal(ck.commit(sc), want)
    ck.precompute(10)
    assert np.array_equal(ck.commit(sc), want)


# ------------------------------------------------------------------------------------------------------------- exact at full size
def test_full_size_bn254_powers_of_tau_c20_and_c16(L, spec):
    """the fold's key: 2^21 BN254 points with the c = 20 table (32 slices): 911 900 witness-shaped scalars and 2^21 uniform ones; the
    same key with a c = 16 table: 1 114 100 scalars, 34 % of them non-zero (the shape of commit(T))"""
    curve, n_key = 0, 1 << 21
    pb, q, bits, gen = curve_consts(spec, curve)
    beta = _beta(spec, curve, 2121)
    k20 = L.CommitmentKey.powers_of_tau(curve, gen, beta, n_key)
    k16 = L.CommitmentKey.from_device(curve, k20._bases.data_ptr(), n_key)
    k20.precompute()
    k16.precompute(16)
    assert Plan(911_900, bits, 20).table_pays and Plan(1_114_100, bits, 16).table_pays
    for sc in (random_elements(0, 911_900, seed=51, shape="witness"), random_elements(0, n_key, seed=52)):
        assert np.array_equal(k20.commit(sc), point_record(spec, curve, horner(ints(sc), beta, q))), len(sc)
    sc = random_elements(0, 1_114_100, seed=53).reshape(-1, 32)
    sc[np.random.default_rng(54).random(len(sc)) >= 0.34] = 0
    sc = sc.reshape(-1)
    assert np.array_equal(k16.commit(sc), point_record(spec, curve, horner(ints(sc), beta, q)))
    k16.close()


def test_full_size_all_equal_bases_c20(L, spec):
    """2^21 copies of G (powers of tau with beta = 1), c = 20: commit(s) = [sum s_i]G"""
    curve, n = 0, 1 << 21
    pb, q, bits, gen = curve_consts(spec, curve)
    ck = L.CommitmentKey.powers_of_tau(curve, gen, 1, n).precompute()
    sc = random_elements(0, n, seed=61, shape="witness")
    assert np.array_equal(ck.commit(sc), point_record(spec, curve, sum(ints(sc))))


def test_full_size_pallas_2_24_windowed(L, spec):
    """2^24 Pallas powers of tau, windowed (c = 19, SL = 16): the shape of the full-size Pallas commitment"""
    curve, n = 2, 1 << 24
    pb, q, bits, gen = curve_consts(spec, curve)
    p = Plan(n, bits)
    assert (p.c, p.SL) == (19, 16)
    beta = _beta(spec, curve, 2424)
    ck = L.CommitmentKey.powers_of_tau(curve, gen, beta, n)
    sc = random_elements(spec.CURVES[curve]["scalar"], n, seed=31, shape="witness")
    assert np.array_equal(ck.commit(sc), point_record(spec, curve, horner(ints(sc), beta, q)))
