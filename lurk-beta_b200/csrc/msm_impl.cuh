// K4: Pedersen commitment = Pippenger multi-scalar multiplication on sm_90a.
//
// Replaces Arecibo's CommitmentEngineTrait::commit -> DlogGroup::vartime_multiscalar_mul (third-party crate, called
// from RecursiveSNARK::prove_step; reference call sites src/proof/nova.rs:287,292, src/proof/supernova.rs:231-244).
// The commitment key is fixed per (rc, Lang) (src/proof/nova.rs:196-216), so it is uploaded once into a context and
// kept in HBM in Montgomery affine form (64 B / point); every call streams 32 B scalars.
//
// Pipeline (all on one stream, no host synchronisation before the final 2 KB read-back; launch and finish are
// separate entry points so that independent commitments overlap):
//   1. digits+histogram: one thread per scalar; signed c-bit windows (buckets 1..2^(c-1), sign folded into the point);
//      warp-aggregated atomics (__match_any_sync) so the 0/1-heavy witness vectors (SURVEY.md H6) do not serialise on
//      one counter.
//   2. exclusive scan of the (windows x 2^(c-1)) bucket counts.
//   3. scatter: point index | sign written at its bucket's next slot (counting sort; order inside a bucket is free
//      because point addition commutes -- the affine result is canonical).
//   4. bucket accumulation, the hot kernel: the sorted list is cut into fixed-length segments, one per thread,
//      independent of the bucket sizes (perfect balance for any scalar distribution).  A thread gathers its bases
//      with 128-bit loads (next point prefetched during the current addition), adds them in XYZZ coordinates
//      (8M+2S mixed addition, no inversions) and flushes a bucket sum whenever the bucket id changes.  The first run
//      of a segment may continue a bucket started by the previous thread: it goes to a (key, point) partial list
//      which is reduced by the same rule in a few geometrically shrinking passes.
//   5. per-window running-sum reduction (chunks of buckets in parallel, then one CTA per window).
//   6. host: Horner combine of the <= 64 window sums and one inversion to affine.
// Integer-ALU bound: ~10 Montgomery products per (scalar, window); algorithmic traffic 96 B per term.
#pragma once
#include "common.cuh"

#include <algorithm>
#include <atomic>
#include <mutex>
#include <thread>

namespace lurk {

static constexpr uint32_t KEY_NONE = 0xffffffffu;

struct MsmPlan {
    int c = 0;             // window bits
    int nwin = 0;          // windows
    uint32_t nb = 0;       // buckets per bucket set = 2^(c-1)
    uint32_t total_buckets = 0;
    uint32_t seg = 0;      // sorted entries per level-1 thread
    uint32_t t1 = 0;       // level-1 threads = partial slots
    // fixed-base mode (window multiples of every base precomputed): all windows share ONE bucket set of 2^(c-1) buckets;
    // entries address table[w * key_n + i]
    bool fixed = false;
    // bucket reduction (see msm_chunk_kernel): rwin bucket sets of nb buckets, chunks of K, G = nb / K chunks per set,
    // nq = 1 + log2 G sums per set, each cut into SL slices of `slice` chunks
    uint32_t rwin = 0, K = 0, G = 0, nq = 0, SL = 0, slice = 0;
};
static constexpr uint32_t MSM_MAX_RESULT_POINTS = 512;    // rwin * nq <= 64 * 1 .. 13 * 17: read back per commitment

// Window width of the fixed-base mode: 2^(c-1) buckets for ~n * 254 / c entries.  c = 20 from half a million bases up (the
// step circuit's witness, 911 900 terms, and a 2^21-point key get the same 13 windows); smaller keys keep >= 20 entries per
// bucket so that the bucket reduction (2 additions per bucket) stays a small fraction of the accumulation.
inline int fixed_base_window(size_t key_n) {
    int lg = 0;
    while (((size_t)1 << (lg + 1)) <= key_n) lg++;
    return std::min(20, std::max(10, lg + 1));
}

inline MsmPlan make_plan(size_t n, int scalar_bits, int fixed_c = 0) {
    MsmPlan p;
    int lg = 0;
    while (((size_t)1 << (lg + 1)) <= n) lg++;
    p.c = fixed_c ? fixed_c : std::min(20, std::max(4, lg - 5));
    p.nwin = scalar_bits / p.c + 1;
    p.fixed = fixed_c != 0;
    p.nb = 1u << (p.c - 1);
    p.rwin = p.fixed ? 1u : (uint32_t)p.nwin;
    p.total_buckets = p.nb * p.rwin;
    p.K = std::min<uint32_t>(8, p.nb);
    p.G = p.nb / p.K;
    p.nq = 1;
    while ((1u << (p.nq - 1)) < p.G) p.nq++;
    p.SL = std::min<uint32_t>(32, std::max<uint32_t>(1, p.G / 2048));
    p.slice = p.G / p.SL;
    size_t cap = n * (size_t)p.nwin;
    size_t want_threads = (size_t)sm_count() * 1024;
    size_t seg = (cap + want_threads - 1) / want_threads;
    static const size_t seg_cap = [] { const char *e = getenv("LURK_MSM_SEG"); return e ? (size_t)atoi(e) : (size_t)32; }();   // tuning aid
    p.seg = (uint32_t)std::min<size_t>(seg_cap, std::max<size_t>(8, seg));
    p.t1 = (uint32_t)((cap + p.seg - 1) / p.seg);
    if (p.t1 == 0) p.t1 = 1;
    return p;
}

// ----------------------------------------------------------------------------- kernels
// unsigned c-bit window starting at `bit` of a 256-bit little-endian integer
__device__ __forceinline__ uint32_t window_bits(const uint32_t k[8], int bit, int c) {
    int word = bit >> 5, sh = bit & 31;
    if (word >= 8) return 0;
    uint32_t lo = k[word] >> sh;
    if (sh + c > 32 && word + 1 < 8) lo |= k[word + 1] << (32 - sh);
    return lo & ((1u << c) - 1);
}

template <class Fs>
__global__ void __launch_bounds__(256) msm_count_kernel(const Fs *__restrict__ scalars, const Fs *__restrict__ sub, size_t n, int fmt, int c, int nwin,
                                                        uint32_t key_stride, uint32_t *__restrict__ counts) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < n;
    // all lanes walk the windows together so the warp-aggregation below sees converged lanes
    Fs k = Fs::zero();
    if (live) {
        k = load_fe<Fs>(scalars + i);
        if (sub) k = k - load_fe<Fs>(sub + i);       // commit(s) = commit(s - d) + commit(d): see lurk_msm_ctx::d_sub
        if (fmt == LURK_FMT_MONTGOMERY) k = k.to_canonical();
    }
    uint32_t carry = 0;
    const uint32_t half = 1u << (c - 1);
    const uint32_t lane = threadIdx.x & 31;
    for (int w = 0; w < nwin; w++) {
        uint32_t raw = window_bits(k.v, w * c, c) + carry;
        uint32_t neg = raw > half;
        uint32_t mag = neg ? (1u << c) - raw : raw;
        carry = neg;
        uint32_t key = (live && mag) ? (uint32_t)w * key_stride + (mag - 1) : KEY_NONE;
        uint32_t peers = __match_any_sync(0xffffffffu, key);
        if (key != KEY_NONE && lane == (uint32_t)(__ffs(peers) - 1)) atomicAdd(counts + key, (uint32_t)__popc(peers));
    }
}

// ---- exclusive scan of the bucket counts: offsets[0..len], offsets[len] = total.
// Three small launches: per-CTA sums of 4096 counts, one CTA scanning the <= 2048 CTA sums, per-CTA scan with carry-in.
static constexpr uint32_t SCAN_TILE = 4096;

__device__ __forceinline__ uint32_t block_exclusive_scan_1024(uint32_t sum, uint32_t *total) {
    __shared__ uint32_t warp_sums[32];
    __shared__ uint32_t carry_s;
    const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    uint32_t incl = sum;
    for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= (uint32_t)d) incl += t; }
    if (lane == 31) warp_sums[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        uint32_t ws = warp_sums[lane], wi = ws;
        for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, wi, d); if (lane >= (uint32_t)d) wi += t; }
        warp_sums[lane] = wi - ws;
        if (lane == 31) carry_s = wi;
    }
    __syncthreads();
    if (total) *total = carry_s;
    return warp_sums[wid] + incl - sum;
}

static __global__ void __launch_bounds__(1024) msm_scan_tile_sums_kernel(const uint32_t *__restrict__ counts, uint32_t len, uint32_t *__restrict__ tile_sums) {
    const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * 4;
    uint32_t sum = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) if (base + k < len) sum += counts[base + k];
    uint32_t total;
    block_exclusive_scan_1024(sum, &total);
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}
// one CTA: tile_offsets[0..ntiles] from tile_sums (ntiles <= 4096)
static __global__ void __launch_bounds__(1024) msm_scan_tiles_kernel(const uint32_t *__restrict__ tile_sums, uint32_t ntiles, uint32_t *__restrict__ tile_offsets) {
    const uint32_t base = threadIdx.x * 4;
    uint32_t v[4], sum = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) { v[k] = base + k < ntiles ? tile_sums[base + k] : 0; sum += v[k]; }
    uint32_t total;
    uint32_t run = block_exclusive_scan_1024(sum, &total);
#pragma unroll
    for (int k = 0; k < 4; k++) { if (base + k < ntiles) tile_offsets[base + k] = run; run += v[k]; }
    if (threadIdx.x == 0) tile_offsets[ntiles] = total;
}
static __global__ void __launch_bounds__(1024) msm_scan_apply_kernel(const uint32_t *__restrict__ counts, uint32_t len, const uint32_t *__restrict__ tile_offsets,
                                                              uint32_t ntiles, uint32_t *__restrict__ offsets) {
    const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * 4;
    uint32_t v[4], sum = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) { v[k] = base + k < len ? counts[base + k] : 0; sum += v[k]; }
    uint32_t run = tile_offsets[blockIdx.x] + block_exclusive_scan_1024(sum, nullptr);
#pragma unroll
    for (int k = 0; k < 4; k++) { if (base + k < len) offsets[base + k] = run; run += v[k]; }
    if (blockIdx.x == 0 && threadIdx.x == 0) offsets[len] = tile_offsets[ntiles];
}

template <class Fs>
__global__ void __launch_bounds__(256) msm_scatter_kernel(const Fs *__restrict__ scalars, const Fs *__restrict__ sub, size_t n, int fmt, int c, int nwin,
                                                          uint32_t key_stride, uint32_t base_stride, const uint32_t *__restrict__ offsets,
                                                          uint32_t *__restrict__ cursor, uint32_t *__restrict__ sorted) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < n;
    Fs k = Fs::zero();
    if (live) {
        k = load_fe<Fs>(scalars + i);
        if (sub) k = k - load_fe<Fs>(sub + i);
        if (fmt == LURK_FMT_MONTGOMERY) k = k.to_canonical();
    }
    uint32_t carry = 0;
    const uint32_t half = 1u << (c - 1);
    const uint32_t lane = threadIdx.x & 31;
    for (int w = 0; w < nwin; w++) {
        uint32_t raw = window_bits(k.v, w * c, c) + carry;
        uint32_t neg = raw > half;
        uint32_t mag = neg ? (1u << c) - raw : raw;
        carry = neg;
        uint32_t key = (live && mag) ? (uint32_t)w * key_stride + (mag - 1) : KEY_NONE;
        uint32_t peers = __match_any_sync(0xffffffffu, key);
        uint32_t leader = (uint32_t)(__ffs(peers) - 1);
        uint32_t base = 0;
        if (key != KEY_NONE && lane == leader) base = atomicAdd(cursor + key, (uint32_t)__popc(peers));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (key != KEY_NONE) {
            uint32_t rank = __popc(peers & ((1u << lane) - 1));
            sorted[offsets[key] + base + rank] = ((uint32_t)i + (uint32_t)w * base_stride) | (neg << 31);
        }
    }
}

template <class Fb>
__device__ __forceinline__ Affine<Fb> load_affine(const Affine<Fb> *p) {
    Affine<Fb> a;
    a.x = load_fe<Fb>(&p->x);
    a.y = load_fe<Fb>(&p->y);
    return a;
}
template <class Fb>
__device__ __forceinline__ XYZZ<Fb> load_xyzz(const XYZZ<Fb> *p) {
    XYZZ<Fb> a;
    a.x = load_fe<Fb>(&p->x); a.y = load_fe<Fb>(&p->y); a.zz = load_fe<Fb>(&p->zz); a.zzz = load_fe<Fb>(&p->zzz);
    return a;
}
template <class Fb>
__device__ __forceinline__ void store_xyzz(XYZZ<Fb> *p, const XYZZ<Fb> &a) {
    store_fe(&p->x, a.x); store_fe(&p->y, a.y); store_fe(&p->zz, a.zz); store_fe(&p->zzz, a.zzz);
}

// level 1: fixed-length segments of the sorted list
// MINB = resident CTAs per SM the register allocation is held to: 4 (126 registers, no spills) is best while the key is
// L2 resident; the fixed-base table (1.7 GB, DRAM gathers) gains ~5 % from 5 CTAs (96 registers, ~150 B of spills).
// DIRECT: the list is already a list of affine points (the output of the pair rounds below): entry `pos` is bases[pos], no sign
template <class Fb, int MINB, bool DIRECT = false>
__global__ void __launch_bounds__(128, MINB) msm_accumulate_kernel(const uint32_t *__restrict__ offsets, uint32_t nbuckets,
                                                             const uint32_t *__restrict__ sorted, const Affine<Fb> *__restrict__ bases,
                                                             XYZZ<Fb> *__restrict__ bucket_acc, uint32_t *__restrict__ pkey,
                                                             XYZZ<Fb> *__restrict__ ppt, uint32_t seg, uint32_t nthreads) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nthreads) return;
    const uint32_t total = offsets[nbuckets];
    const uint64_t start64 = (uint64_t)t * seg;
    if (start64 >= total) { pkey[t] = KEY_NONE; return; }
    const uint32_t start = (uint32_t)start64;
    const uint32_t end = (uint32_t)min((uint64_t)total, start64 + seg);
    // bucket containing `start`: largest key with offsets[key] <= start
    uint32_t lo = 0, hi = nbuckets;
    while (hi - lo > 1) {
        uint32_t mid = (lo + hi) >> 1;
        if (offsets[mid] <= start) lo = mid; else hi = mid;
    }
    uint32_t key = lo;
    uint32_t run_end = min(offsets[key + 1], end);
    bool first_run = true;
    uint32_t e_next = DIRECT ? start : sorted[start];
    Affine<Fb> p_next = load_affine(bases + (e_next & 0x7fffffffu));
    XYZZ<Fb> acc = XYZZ<Fb>::identity();
    // ONE flat loop over the segment: every lane performs exactly one addition per iteration, so lanes whose bucket
    // boundaries fall at different positions stay converged (a nested per-run loop makes each lane wait for the
    // longest run in the warp -- measured ~2x on the IMAD pipe).  Flushing a finished run is a short predicated tail.
    for (uint32_t pos = start; pos < end;) {
        const uint32_t e = e_next;
        const Affine<Fb> p = p_next;
        pos++;
        if (pos < end) {   // prefetch the next entry while this addition runs
            e_next = DIRECT ? pos : sorted[pos];
            p_next = load_affine(bases + (e_next & 0x7fffffffu));
        }
        acc.add_affine(p, (e >> 31) != 0);
        if (pos == run_end) {
            if (first_run) { pkey[t] = key; store_xyzz(ppt + t, acc); first_run = false; }
            else store_xyzz(bucket_acc + key, acc);   // this run starts exactly at the bucket start: sole initialiser
            acc = XYZZ<Fb>::identity();
            if (pos < end) {
                key++;
                while (offsets[key + 1] <= pos) key++;   // skip empty buckets
                run_end = min(offsets[key + 1], end);
            }
        }
    }
}

// ---- pair rounds: batched-affine additions in front of the XYZZ accumulation ------------------------------------------------
// A mixed XYZZ addition costs 10 field products; an AFFINE addition costs 3 (lambda = dy / dx; x3 = lambda^2 - x1 - x2;
// y3 = lambda (x1 - x3) - y1) plus one inversion -- and inversions batch: Montgomery's trick turns the inversions of a whole CTA
// warp (32 threads x PAIR_B additions) into ONE inversion (binary GCD, on the ALU pipe, by one lane) + 3 products per addition + a
// dozen products per thread for the cross-lane prefix / suffix products.  ~7 products per addition instead of 10.
// Independent additions come from the sorted list itself: inside every bucket's run, entries 2j and 2j + 1 are added pairwise (an odd
// tail is copied), which halves every run: out run k has ceil(m_k / 2) affine points.  One or two such rounds (half resp. three
// quarters of all additions) run before the fixed-length-segment XYZZ accumulation takes the rest.
static constexpr int PAIR_B = 16;        // output points per thread and batch
// default number of pair rounds for long / short average runs: 0 = off (one round makes the fold step slower as implemented,
// 4.94 vs 4.34 ms on an H100 at 400 W: the per-batch inversion stalls its CTA) -- LURK_MSM_PAIR_ROUNDS overrides
static constexpr int MSM_PAIR_ROUNDS_LONG = 0, MSM_PAIR_ROUNDS_SHORT = 0;

static __global__ void __launch_bounds__(256) msm_halve_kernel(const uint32_t *__restrict__ offs_in, uint32_t nbuckets, uint32_t *__restrict__ counts_out) {
    for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k <= nbuckets; k += gridDim.x * blockDim.x)
        counts_out[k] = k < nbuckets ? (offs_in[k + 1] - offs_in[k] + 1u) >> 1 : 0u;
}

// the two inputs of output slot q of bucket k and how they combine
template <class Fb>
struct PairIn {
    Affine<Fb> p1, p2;
    int kind;            // 0 copy p1, 1 chord addition, 2 doubling of p1, 3 result is the identity
};
template <class Fb, bool FIRST>
__device__ __forceinline__ Affine<Fb> pair_load(const uint32_t *__restrict__ sorted, const Affine<Fb> *__restrict__ pts, uint32_t pos) {
    if (!FIRST) return load_affine(pts + pos);
    const uint32_t e = sorted[pos];
    Affine<Fb> p = load_affine(pts + (e & 0x7fffffffu));
    if (e >> 31) p.y = p.y.neg();
    return p;
}
template <class Fb, bool FIRST>
__device__ __forceinline__ PairIn<Fb> pair_fetch(const uint32_t *__restrict__ sorted, const Affine<Fb> *__restrict__ pts, uint32_t in, uint32_t run_end) {
    PairIn<Fb> r;
    r.p1 = pair_load<Fb, FIRST>(sorted, pts, in);
    r.kind = 0;
    r.p2 = r.p1;
    if (in + 1 < run_end) {
        r.p2 = pair_load<Fb, FIRST>(sorted, pts, in + 1);
        if (r.p1.is_identity()) { r.p1 = r.p2; }                       // 0 + Q: copy Q
        else if (r.p2.is_identity()) {}                                  // P + 0: copy P
        else if (r.p1.x == r.p2.x) r.kind = (r.p1.y == r.p2.y && !r.p1.y.is_zero()) ? 2 : 3;
        else r.kind = 1;
    }
    return r;
}
template <class Fb>
__device__ __forceinline__ Fb pair_denominator(const PairIn<Fb> &in) {
    if (in.kind == 1) return in.p2.x - in.p1.x;
    if (in.kind == 2) return in.p1.y.dbl();
    return Fb::one();
}

// 1 / v for every lane of a warp with ONE field inversion (v != 0 everywhere): inclusive prefix and suffix products by shuffles,
// lane 31 inverts the total (binary GCD: shifts and adds on the ALU pipe, the multiplier stays free for the other warps of the SM)
template <class Fb>
__device__ __forceinline__ Fb warp_batch_inverse(const Fb &v) {
    const int lane = threadIdx.x & 31;
    Fb pre = v, suf = v;
#pragma unroll 1
    for (int d = 1; d < 32; d <<= 1) {
        Fb a, b;
#pragma unroll
        for (int i = 0; i < 8; i++) { a.v[i] = __shfl_up_sync(0xffffffffu, pre.v[i], d); b.v[i] = __shfl_down_sync(0xffffffffu, suf.v[i], d); }
        if (lane >= d) pre = pre * a;
        if (lane + d < 32) suf = suf * b;
    }
    Fb inv = Fb::zero();
    if (lane == 31) inv = pre.inv_vartime();
    Fb ep, es, r;                                  // exclusive prefix / suffix, inverse of the warp total
#pragma unroll
    for (int i = 0; i < 8; i++) {
        ep.v[i] = __shfl_up_sync(0xffffffffu, pre.v[i], 1);
        es.v[i] = __shfl_down_sync(0xffffffffu, suf.v[i], 1);
        r.v[i] = __shfl_sync(0xffffffffu, inv.v[i], 31);
    }
    if (lane > 0) r = r * ep;
    if (lane < 31) r = r * es;
    return r;
}

// One pair round.  offs_in / offs_out: bucket offsets of the input / output lists (offs_out = scan of ceil(m / 2)).
// Thread t produces output slots [t * PAIR_B, (t + 1) * PAIR_B); a warp shares one inversion per batch of 32 x PAIR_B additions.
template <class Fb, bool FIRST>
__global__ void __launch_bounds__(128) msm_pair_kernel(const uint32_t *__restrict__ offs_in, const uint32_t *__restrict__ offs_out, uint32_t nbuckets,
                                                       const uint32_t *__restrict__ sorted, const Affine<Fb> *__restrict__ pts_in,
                                                       Affine<Fb> *__restrict__ pts_out) {
    const uint32_t total = offs_out[nbuckets];
    const uint64_t gtid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if ((gtid & ~31ull) * PAIR_B >= total) return;                              // the whole warp is past the end
    const uint64_t start64 = gtid * PAIR_B;
    const bool active = start64 < total;
    const uint32_t start = active ? (uint32_t)start64 : 0, end = active ? (uint32_t)min((uint64_t)total, start64 + PAIR_B) : 0;
    uint32_t k = 0;
    if (active) {
        uint32_t lo = 0, hi = nbuckets;
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (offs_out[mid] <= start) lo = mid; else hi = mid; }
        k = lo;
    }
    Fb pref[PAIR_B];                                 // running products of the denominators (thread-private, L1-resident)
    Fb run = Fb::one();
    for (uint32_t q = start; q < end; q++) {
        while (offs_out[k + 1] <= q) k++;
        const uint32_t in = offs_in[k] + 2 * (q - offs_out[k]);
        const PairIn<Fb> pi = pair_fetch<Fb, FIRST>(sorted, pts_in, in, offs_in[k + 1]);
        run = run * pair_denominator(pi);
        pref[q - start] = run;
    }
    Fb inv = warp_batch_inverse(run);              // 1 / (product of this thread's denominators)
    // backwards: peel one denominator at a time
    for (uint32_t q = end; q-- > start;) {
        while (offs_out[k] > q) k--;
        const uint32_t in = offs_in[k] + 2 * (q - offs_out[k]);
        const PairIn<Fb> pi = pair_fetch<Fb, FIRST>(sorted, pts_in, in, offs_in[k + 1]);
        const uint32_t j = q - start;
        const Fb den = pair_denominator(pi);
        const Fb inv_d = j ? inv * pref[j - 1] : inv;     // 1 / den
        inv = inv * den;
        Affine<Fb> o = pi.p1;
        if (pi.kind == 3) { o.x = Fb::zero(); o.y = Fb::zero(); }
        else if (pi.kind) {
            Fb num;
            if (pi.kind == 1) num = pi.p2.y - pi.p1.y;
            else { const Fb xx = pi.p1.x.sqr(); num = xx.dbl() + xx; }
            const Fb lam = num * inv_d;
            const Fb x3 = lam.sqr() - pi.p1.x - pi.p2.x;
            o.y = lam * (pi.p1.x - x3) - pi.p1.y;
            o.x = x3;
        }
        store_fe(&pts_out[q].x, o.x);
        store_fe(&pts_out[q].y, o.y);
    }
}

// levels >= 2: the same rule on (key, point) lists; keys are non-decreasing, KEY_NONE only as a tail
template <class Fb>
__global__ void __launch_bounds__(128) msm_partial_kernel(const uint32_t *__restrict__ keys_in, const XYZZ<Fb> *__restrict__ pts_in,
                                                          uint32_t count, XYZZ<Fb> *__restrict__ bucket_acc, uint32_t *__restrict__ keys_out,
                                                          XYZZ<Fb> *__restrict__ pts_out, uint32_t seg, int last_level) {
    const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t s64 = (uint64_t)u * seg;
    if (s64 >= count) return;
    const uint32_t s = (uint32_t)s64, e = (uint32_t)min((uint64_t)count, s64 + seg);
    uint32_t cur = KEY_NONE;
    bool first_run = true, wrote_out = false;
    XYZZ<Fb> acc = XYZZ<Fb>::identity();
    for (uint32_t i = s; i <= e; i++) {
        const uint32_t k = i < e ? keys_in[i] : KEY_NONE;   // one extra step flushes the last run
        if (k == cur && k != KEY_NONE) { acc.add(load_xyzz(pts_in + i)); continue; }
        if (cur != KEY_NONE) {
            if (first_run && !last_level) { keys_out[u] = cur; store_xyzz(pts_out + u, acc); wrote_out = true; }
            else { XYZZ<Fb> b = load_xyzz(bucket_acc + cur); b.add(acc); store_xyzz(bucket_acc + cur, b); }
            first_run = false;
        }
        if (k == KEY_NONE) break;
        cur = k;
        acc = load_xyzz(pts_in + i);
    }
    if (!wrote_out && !last_level) keys_out[u] = KEY_NONE;
}

template <class Fb>
__device__ __forceinline__ XYZZ<Fb> shfl_up_xyzz(const XYZZ<Fb> &p, int d) {
    XYZZ<Fb> r;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        r.x.v[i] = __shfl_up_sync(0xffffffffu, p.x.v[i], d);
        r.y.v[i] = __shfl_up_sync(0xffffffffu, p.y.v[i], d);
        r.zz.v[i] = __shfl_up_sync(0xffffffffu, p.zz.v[i], d);
        r.zzz.v[i] = __shfl_up_sync(0xffffffffu, p.zzz.v[i], d);
    }
    return r;
}

// Later levels are latency-bound (few entries): one warp takes 32 consecutive (key, point) entries and combines equal
// keys with a segmented Hillis-Steele scan over shuffles -- 5 dependent additions per 32x shrink instead of 32.
template <class Fb>
__global__ void __launch_bounds__(128) msm_partial_warp_kernel(const uint32_t *__restrict__ keys_in, const XYZZ<Fb> *__restrict__ pts_in,
                                                               uint32_t count, XYZZ<Fb> *__restrict__ bucket_acc, uint32_t *__restrict__ keys_out,
                                                               XYZZ<Fb> *__restrict__ pts_out, int last_level) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if ((uint64_t)gw * 32 >= count) return;   // whole warp out of range
    const uint32_t i = gw * 32 + lane;
    const uint32_t key = i < count ? keys_in[i] : KEY_NONE;
    XYZZ<Fb> pt = XYZZ<Fb>::identity();
    if (key != KEY_NONE) pt = load_xyzz(pts_in + i);
#pragma unroll 1
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t k2 = __shfl_up_sync(0xffffffffu, key, d);
        const XYZZ<Fb> p2 = shfl_up_xyzz(pt, d);
        if (lane >= (uint32_t)d && k2 == key && key != KEY_NONE) pt.add(p2);
    }
    const uint32_t first_key = __shfl_sync(0xffffffffu, key, 0);
    const uint32_t next_key = __shfl_down_sync(0xffffffffu, key, 1);
    const bool run_end = key != KEY_NONE && (lane == 31 || next_key != key);
    if (run_end) {
        if (key == first_key && !last_level) { keys_out[gw] = key; store_xyzz(pts_out + gw, pt); }
        else { XYZZ<Fb> b = load_xyzz(bucket_acc + key); b.add(pt); store_xyzz(bucket_acc + key, b); }
    }
    if (first_key == KEY_NONE && lane == 0 && !last_level) keys_out[gw] = KEY_NONE;
}

// ---- bucket reduction: R_w = sum_b (b + 1) B_{w,b} per window, in three short, wide kernels.
// With chunks of K buckets (g = chunk index, G = buckets per window / K):
//     R_w = sum_g tri_g + K * sum_g g * run_g,   tri_g = sum_j (j + 1) B_{gK + j},   run_g = sum_j B_{gK + j}
// and the weighted sum over chunks is taken bit by bit: sum_g g run_g = sum_k 2^k S_k, S_k = sum of run_g over the g with
// bit k set.  Every S_k (and the plain sum of the tri_g) is an ordinary tree reduction, so nothing on this path is longer
// than 2K + a few dozen dependent point additions and no scalar multiplication is needed; the final Horner over the
// (1 + log2 G) sums per window runs on the host in msm_finish.

// level 0: one thread per chunk of K buckets
template <class Fb>
__global__ void __launch_bounds__(128) msm_chunk_kernel(const XYZZ<Fb> *__restrict__ bucket_acc, uint32_t K, uint32_t nchunks_total,
                                                        XYZZ<Fb> *__restrict__ tri_out, XYZZ<Fb> *__restrict__ run_out) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= nchunks_total) return;
    const XYZZ<Fb> *B = bucket_acc + (size_t)g * K;
    XYZZ<Fb> run = XYZZ<Fb>::identity(), tri = XYZZ<Fb>::identity();
    for (int b = (int)K - 1; b >= 0; b--) {
        run.add(load_xyzz(B + b));
        tri.add(run);
    }
    store_xyzz(tri_out + g, tri);
    store_xyzz(run_out + g, run);
}

// level 1: block (sl, q, w) sums, over slice sl of window w's G chunks, the tri_g (q = 0) or the run_g with bit q-1 of g
// set (q >= 1).  out[((w * nq) + q) * SL + sl].  Slices are aligned powers of two, so "bit k set" is enumerated directly.
template <class Fb>
__global__ void __launch_bounds__(256) msm_bitsum_kernel(const XYZZ<Fb> *__restrict__ tri, const XYZZ<Fb> *__restrict__ run, uint32_t G,
                                                         uint32_t slice, XYZZ<Fb> *__restrict__ out) {
    __shared__ XYZZ<Fb> sm[256];
    const uint32_t sl = blockIdx.x, q = blockIdx.y, w = blockIdx.z, tid = threadIdx.x;
    const uint32_t SL = gridDim.x, nq = gridDim.y;
    const size_t base = (size_t)w * G + (size_t)sl * slice;
    XYZZ<Fb> acc = XYZZ<Fb>::identity();
    if (q == 0) {
        for (uint32_t i = tid; i < slice; i += blockDim.x) acc.add(load_xyzz(tri + base + i));
    } else {
        const uint32_t k = q - 1;
        if (slice > (1u << k)) {
            const uint32_t low = (1u << k) - 1;
            for (uint32_t j = tid; j < slice / 2; j += blockDim.x) {
                const uint32_t local = ((j >> k) << (k + 1)) | (1u << k) | (j & low);
                acc.add(load_xyzz(run + base + local));
            }
        } else if (((sl * slice) >> k) & 1u) {       // bit k is constant over this slice
            for (uint32_t i = tid; i < slice; i += blockDim.x) acc.add(load_xyzz(run + base + i));
        }
    }
    sm[tid] = acc;
    __syncthreads();
    for (uint32_t stride = blockDim.x / 2; stride > 0; stride >>= 1) {
        if (tid < stride) { XYZZ<Fb> a = sm[tid]; a.add(sm[tid + stride]); sm[tid] = a; }
        __syncthreads();
    }
    if (tid == 0) store_xyzz(out + ((size_t)w * nq + q) * SL + sl, sm[0]);
}

template <class Fb>
__device__ __forceinline__ XYZZ<Fb> shfl_xor_xyzz(const XYZZ<Fb> &p, int d) {
    XYZZ<Fb> r;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        r.x.v[i] = __shfl_xor_sync(0xffffffffu, p.x.v[i], d);
        r.y.v[i] = __shfl_xor_sync(0xffffffffu, p.y.v[i], d);
        r.zz.v[i] = __shfl_xor_sync(0xffffffffu, p.zz.v[i], d);
        r.zzz.v[i] = __shfl_xor_sync(0xffffffffu, p.zzz.v[i], d);
    }
    return r;
}

// level 2 (only when a window was cut into SL > 1 slices): one warp per (w, q) adds the SL <= 32 slice sums
template <class Fb>
__global__ void __launch_bounds__(128) msm_slice_sum_kernel(const XYZZ<Fb> *__restrict__ in, uint32_t SL, uint32_t count,
                                                            XYZZ<Fb> *__restrict__ out) {
    const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (gw >= count) return;                           // whole warps exit together
    XYZZ<Fb> pt = XYZZ<Fb>::identity();
    if (lane < SL) pt = load_xyzz(in + (size_t)gw * SL + lane);
#pragma unroll 1
    for (int d = 16; d > 0; d >>= 1) {
        const XYZZ<Fb> p2 = shfl_xor_xyzz(pt, d);
        if ((uint32_t)d < SL) pt.add(p2);             // uniform per warp: lanes >= SL hold the identity anyway
    }
    if (lane == 0) store_xyzz(out + gw, pt);
}

// level 3 (fixed-base mode: one bucket set): R = T + K * sum_k 2^k S_k on the device, one warp.  Lane 0 holds T, lane q >= 1
// holds S_(q-1) and doubles it log2(K) + q - 1 times; a butterfly of 5 additions sums the lanes.  Longest chain:
// log2(K) + nq - 2 doublings + 5 additions (21 + 5 for a 2^21-point key) instead of the 36 sequential operations of a
// Horner walk -- this kernel sits on the fold's critical chain.  The result stays on the device (XYZZ, 128 bytes) for the
// fold context's challenge kernel; lurk_msm_ctx_finish reads it back and normalises it on the host.
template <class Fb>
__global__ void __launch_bounds__(32) msm_horner_kernel(const XYZZ<Fb> *__restrict__ wins, uint32_t nq, uint32_t K, const Affine<Fb> *__restrict__ offset,
                                                        XYZZ<Fb> *__restrict__ out) {
    const uint32_t lane = threadIdx.x;
    XYZZ<Fb> pt = XYZZ<Fb>::identity();
    if (lane < nq) pt = load_xyzz(wins + lane);
    uint32_t logk = 0;
    while ((1u << logk) < K) logk++;
    const uint32_t mine = (lane >= 1 && lane < nq) ? logk + lane - 1 : 0;
    const uint32_t longest = nq >= 2 ? logk + nq - 2 : 0;
#pragma unroll 1
    for (uint32_t d = 0; d < longest; d++)
        if (d < mine) pt = pt.dbl();
#pragma unroll 1
    for (int d = 16; d > 0; d >>= 1) {
        const XYZZ<Fb> p2 = shfl_xor_xyzz(pt, d);
        pt.add(p2);
    }
    if (lane == 0) {
        if (offset) pt.add_affine(load_affine(offset));      // + commit(d), see lurk_msm_ctx::d_sub
        store_xyzz(out, pt);
    }
}

// Fixed-base table: table[w * n + i] = 2^(c w) * bases[i], affine.  One thread per base walks the windows with c
// doublings each (XYZZ), then normalises its nwin points with one inversion (Montgomery's trick on the ZZZ coordinates).
static constexpr int MSM_MAX_TABLE_WINDOWS = 26;
template <class Fb>
__global__ void __launch_bounds__(128) msm_precompute_kernel(const Affine<Fb> *__restrict__ bases, size_t n, int c, int nwin,
                                                             Affine<Fb> *__restrict__ table) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Affine<Fb> p0 = load_affine(bases + i);
    XYZZ<Fb> pts[MSM_MAX_TABLE_WINDOWS];
    Fb pref[MSM_MAX_TABLE_WINDOWS];
    XYZZ<Fb> cur = XYZZ<Fb>::from_affine(p0);
    Fb run = Fb::one();
    for (int w = 0; w < nwin; w++) {
        if (w) for (int d = 0; d < c; d++) cur = cur.dbl();
        pts[w] = cur;
        pref[w] = run;
        if (!cur.is_identity()) run = run * cur.zzz;
    }
    Fb inv = run.inv();
    for (int w = nwin - 1; w >= 0; w--) {
        Affine<Fb> a;
        a.x = Fb::zero();
        a.y = Fb::zero();
        if (!pts[w].is_identity()) {
            const Fb zi = inv * pref[w];            // 1 / ZZZ_w
            inv = inv * pts[w].zzz;
            const Fb zz_inv = (zi * pts[w].zz).sqr();
            a.x = pts[w].x * zz_inv;
            a.y = pts[w].y * zi;
        }
        store_fe(&table[(size_t)w * n + i].x, a.x);
        store_fe(&table[(size_t)w * n + i].y, a.y);
    }
}

// counts affine points (Montgomery coordinates) that are neither the identity encoding (0, 0) nor on y^2 = x^3 + b:
// the analogue of the on-curve check the reference's point deserialisation performs before a key is used
template <class Fb>
__global__ void __launch_bounds__(256) msm_on_curve_kernel(const Affine<Fb> *__restrict__ bases, size_t n, Fb b, int *bad) {
    int local = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const Affine<Fb> p = load_affine(bases + i);
        if (p.is_identity()) continue;
        const Fb lhs = p.y.sqr(), rhs = p.x.sqr() * p.x + b;
        local += lhs == rhs ? 0 : 1;
    }
    local = __reduce_add_sync(0xffffffffu, local);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(bad, local);
}

// affine bases: canonical -> Montgomery in place
template <class Fb>
__global__ void __launch_bounds__(256) msm_bases_to_mont_kernel(Fb *coords, size_t count) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (size_t)gridDim.x * blockDim.x)
        store_fe(coords + i, Fb::from_canonical(load_fe<Fb>(coords + i)));
}

// ----------------------------------------------------------------------------- context
struct MsmScratch {
    DevBuf counts, offsets, tiles, sorted, buckets, pkey[2], ppt[2], chunks, chunk_sums, slices, wins, result, scalars, pair_offs[2], pair_pts[2];
    void *h_wins = nullptr;   // pinned
    void *h_stage[2] = {nullptr, nullptr};          // pinned staging for host-buffer scalars
    cudaEvent_t stage_done[2] = {nullptr, nullptr};
    cudaStream_t stage_stream = nullptr;            // private non-blocking stream of the host-buffer entry point
    ~MsmScratch() {
        if (h_wins) cudaFreeHost(h_wins);
        if (stage_stream) cudaStreamDestroy(stage_stream);
        for (int k = 0; k < 2; k++) { if (h_stage[k]) cudaFreeHost(h_stage[k]); if (stage_done[k]) cudaEventDestroy(stage_done[k]); }
    }
};

}  // namespace lurk

using namespace lurk;

struct lurk_msm_ctx {
    int curve_id = 0;
    int device = 0;
    size_t n = 0;
    void *d_bases = nullptr;
    bool owns_bases = false;
    void *d_table = nullptr;      // fixed-base table (nwin x n affine), optional
    bool owns_table = false;
    int fixed_c = 0;
    std::mutex mu;
    MsmScratch scratch;
    // optional device timing of the dominant kernel (bucket accumulation), on the launching stream
    bool profile = false;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    float last_accumulate_ms = 0.f;
    unsigned last_launches = 0;
    // launch / finish split
    bool pending = false;
    int pending_fmt = 0, pending_c = 0, pending_nwin = 0;
    bool pending_fixed = false;
    uint32_t pending_nq = 0, pending_K = 0;
    cudaEvent_t done = nullptr;
    // optional SM partitioning (set by the fold context): the one-warp finishing kernel (msm_horner_kernel) is enqueued on
    // `tiny_stream` -- a stream of a small green-context partition reserved for the single-CTA kernels of the fold chain, so
    // that they do not share an SM's multiplier pipe with thousands of bucket-accumulation warps.  Without read-back the
    // result is then ready on `tiny_stream`, not on the caller's stream.
    cudaStream_t tiny_stream = nullptr;
    // Optional constant part of the scalar vector (set by the fold context; device-resident results only): when most of a
    // vector repeats a fixed vector d from call to call -- the dummy slot witnesses of a Lurk step (src/lem/multiframe.rs:553-577:
    // unused slots share one cached witness) -- the context commits to s - d, whose entries vanish wherever s repeats d and
    // are skipped by the bucket sort, and msm_horner_kernel adds the precomputed point commit(d).  d_sub: key-length vector in
    // the scalar field (Montgomery); d_offset: one affine point.
    const void *d_sub = nullptr;
    const void *d_offset = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
};

namespace lurk {

template <class Fb>
void point_to_bytes(const XYZZ<Fb> &p, int fmt, uint8_t out[96]) {
    memset(out, 0, 96);
    if (p.is_identity()) return;
    Affine<Fb> a = p.to_affine();
    Fb one = Fb::one();
    if (fmt == LURK_FMT_CANONICAL) { a.x = a.x.to_canonical(); a.y = a.y.to_canonical(); one = one.to_canonical(); }
    memcpy(out, a.x.v, 32); memcpy(out + 32, a.y.v, 32); memcpy(out + 64, one.v, 32);
}

// a context's buffers live on the device that was current when it was created
inline int ctx_check_device(const lurk_msm_ctx *ctx) {
    int dev = -1;
    LURK_CUDA_TRY(cudaGetDevice(&dev));
    if (dev != ctx->device) { set_error("context belongs to device %d but device %d is current", ctx->device, dev); return LURK_ERR_ARG; }
    return LURK_OK;
}

// enqueue the whole pipeline on stream s, ending with the async read-back of the window sums
template <class C>
int msm_launch(lurk_msm_ctx *ctx, const void *d_scalars, size_t n, int fmt, cudaStream_t s, bool readback) {
    using Fb = typename C::Base;
    using Fs = typename C::Scalar;
    using Pt = XYZZ<Fb>;
    if (ctx->pending) { set_error("a launch is already pending on this context (call lurk_msm_ctx_finish)"); return LURK_ERR_ARG; }
    LURK_TRY(ctx_check_device(ctx));
    if (!ctx->done) LURK_CUDA_TRY(cudaEventCreateWithFlags(&ctx->done, cudaEventDisableTiming));
    ctx->pending_fmt = fmt;
    ctx->pending_nwin = 0;
    MsmScratch &S = ctx->scratch;
    if (S.result.bytes < sizeof(Pt)) LURK_TRY(S.result.alloc(sizeof(Pt)));
    if (n == 0) {
        if (readback) ctx->pending = true;
        else LURK_CUDA_TRY(cudaMemsetAsync(S.result.p, 0, sizeof(Pt), s));     // all-zero XYZZ = identity
        return LURK_OK;
    }
    // The fixed-base table pays when the shared bucket set is well filled; a SHORT scalar vector under a big key (the fold chain of a
    // HyperKZG opening: n/2, n/4, ... terms under a 2^21-point key) would spend its time reducing 2^(c-1) nearly empty buckets, so it
    // takes the plain windowed path on the same bases instead (results are identical).  Device-resident results keep the table.
    const bool table_pays = !readback || n * (size_t)(Fs::Params::NBITS / std::max(ctx->fixed_c, 1) + 1) >= ((size_t)8 << (std::max(ctx->fixed_c, 1) - 1));
    const bool fixed = ctx->d_table != nullptr && table_pays;
    if (!readback && !fixed) { set_error("device-resident results need the fixed-base table (lurk_msm_ctx_precompute)"); return LURK_ERR_ARG; }
    MsmPlan P = make_plan(n, Fs::Params::NBITS, fixed ? ctx->fixed_c : 0);
    // sorted-entry offsets are 32-bit: one launch handles < 2^32 (scalar, window) pairs; larger keys are sharded
    if ((uint64_t)n * (uint64_t)P.nwin >= (1ull << 32)) { set_error("%zu scalars exceed one launch (shard the commitment key)", n); return LURK_ERR_ARG; }
    const uint32_t TB = P.total_buckets;
    const uint32_t ntiles = (TB + SCAN_TILE - 1) / SCAN_TILE;
    // pair rounds (batched-affine additions in front of the XYZZ accumulation): only when the runs are long enough to pair
    const size_t cap = n * (size_t)P.nwin;
    int rounds = 0;
    {
        static const int forced = [] { const char *e = getenv("LURK_MSM_PAIR_ROUNDS"); return e ? atoi(e) : -1; }();   // tuning aid
        const size_t avg = cap / TB;
        if (forced >= 0) rounds = forced;
        else if (n >= 8192) rounds = avg >= 12 ? MSM_PAIR_ROUNDS_LONG : (avg >= 5 ? MSM_PAIR_ROUNDS_SHORT : 0);
        if (rounds > 4) rounds = 4;
    }
    size_t cap_final = cap;
    for (int r = 0; r < rounds; r++) cap_final = cap_final / 2 + TB + 1;       // sum of ceil(m_k / 2) <= cap / 2 + buckets
    const uint32_t t1 = rounds ? (uint32_t)((cap_final + P.seg - 1) / P.seg) : P.t1;
    const uint32_t t1_alloc = std::max(t1, P.t1);
    {
        // scratch grows monotonically; a context is normally run at one size (the circuit's witness length)
        auto ensure = [](DevBuf &b, size_t bytes) { return b.bytes >= bytes ? LURK_OK : b.alloc(bytes); };
        LURK_TRY(ensure(S.counts, ((size_t)TB + 1) * 2 * sizeof(uint32_t)));   // counts | cursor
        LURK_TRY(ensure(S.offsets, ((size_t)TB + 1) * sizeof(uint32_t)));
        LURK_TRY(ensure(S.tiles, ((size_t)ntiles + 1) * 2 * sizeof(uint32_t)));  // tile sums | tile offsets
        LURK_TRY(ensure(S.sorted, n * (size_t)P.nwin * sizeof(uint32_t)));
        LURK_TRY(ensure(S.buckets, (size_t)TB * sizeof(Pt)));
        LURK_TRY(ensure(S.pkey[0], (size_t)t1_alloc * sizeof(uint32_t)));
        LURK_TRY(ensure(S.ppt[0], (size_t)t1_alloc * sizeof(Pt)));
        size_t t2 = ((size_t)t1_alloc + 7) / 8;
        LURK_TRY(ensure(S.pkey[1], t2 * sizeof(uint32_t)));
        LURK_TRY(ensure(S.ppt[1], t2 * sizeof(Pt)));
        const size_t nchunks_all = (size_t)P.rwin * P.G;
        LURK_TRY(ensure(S.chunks, nchunks_all * sizeof(Pt)));          // tri_g
        LURK_TRY(ensure(S.chunk_sums, nchunks_all * sizeof(Pt)));      // run_g
        LURK_TRY(ensure(S.slices, (size_t)P.rwin * P.nq * P.SL * sizeof(Pt)));
        LURK_TRY(ensure(S.wins, MSM_MAX_RESULT_POINTS * sizeof(Pt)));
        if (!S.h_wins) LURK_CUDA_TRY(cudaMallocHost(&S.h_wins, MSM_MAX_RESULT_POINTS * sizeof(Pt)));
    }
    if (ntiles > 4096) { set_error("bucket table too large for the scan"); return LURK_ERR_ARG; }
    uint32_t *counts = S.counts.as<uint32_t>();
    uint32_t *cursor = counts + (TB + 1);
    uint32_t *offsets = S.offsets.as<uint32_t>();
    uint32_t *tile_sums = S.tiles.as<uint32_t>(), *tile_offsets = tile_sums + (ntiles + 1);
    uint32_t *sorted = S.sorted.as<uint32_t>();
    Pt *buckets = S.buckets.as<Pt>();

    LURK_CUDA_TRY(cudaMemsetAsync(counts, 0, ((size_t)TB + 1) * 2 * sizeof(uint32_t), s));
    LURK_CUDA_TRY(cudaMemsetAsync(buckets, 0, (size_t)TB * sizeof(Pt), s));   // all-zero = identity
    const unsigned gs = (unsigned)((n + 255) / 256);
    unsigned launches = 0;
    const uint32_t key_stride = fixed ? 0u : P.nb;                 // fixed-base: all windows share one bucket set
    const uint32_t base_stride = fixed ? (uint32_t)ctx->n : 0u;     // ... and address table[w * n + i]
    const Affine<Fb> *bases = (const Affine<Fb> *)(fixed ? ctx->d_table : ctx->d_bases);
    const Fs *sub = (!readback && fmt == LURK_FMT_MONTGOMERY) ? (const Fs *)ctx->d_sub : nullptr;
    msm_count_kernel<Fs><<<gs, 256, 0, s>>>((const Fs *)d_scalars, sub, n, fmt, P.c, P.nwin, key_stride, counts);
    msm_scan_tile_sums_kernel<<<ntiles, 1024, 0, s>>>(counts, TB, tile_sums);
    msm_scan_tiles_kernel<<<1, 1024, 0, s>>>(tile_sums, ntiles, tile_offsets);
    msm_scan_apply_kernel<<<ntiles, 1024, 0, s>>>(counts, TB, tile_offsets, ntiles, offsets);
    msm_scatter_kernel<Fs><<<gs, 256, 0, s>>>((const Fs *)d_scalars, sub, n, fmt, P.c, P.nwin, key_stride, base_stride, offsets, cursor, sorted);
    if (ctx->profile) LURK_CUDA_TRY(cudaEventRecord(ctx->ev0, s));
    // ---- pair rounds
    const uint32_t *acc_offs = offsets;
    const Affine<Fb> *acc_pts = bases;
    size_t cap_r = cap;
    for (int r = 0; r < rounds; r++) {
        cap_r = cap_r / 2 + TB + 1;                                        // sum of ceil(m_k / 2) <= cap / 2 + buckets
        DevBuf &ob = S.pair_offs[r & 1], &pb = S.pair_pts[r & 1];
        if (ob.bytes < ((size_t)TB + 1) * sizeof(uint32_t)) LURK_TRY(ob.alloc(((size_t)TB + 1) * sizeof(uint32_t)));
        if (pb.bytes < cap_r * sizeof(Affine<Fb>)) LURK_TRY(pb.alloc(cap_r * sizeof(Affine<Fb>)));
        uint32_t *o2 = ob.as<uint32_t>();
        msm_halve_kernel<<<(TB + 256) / 256, 256, 0, s>>>(acc_offs, TB, counts);          // `counts` is free after the scatter
        msm_scan_tile_sums_kernel<<<ntiles, 1024, 0, s>>>(counts, TB, tile_sums);
        msm_scan_tiles_kernel<<<1, 1024, 0, s>>>(tile_sums, ntiles, tile_offsets);
        msm_scan_apply_kernel<<<ntiles, 1024, 0, s>>>(counts, TB, tile_offsets, ntiles, o2);
        const size_t pthreads = (cap_r + PAIR_B - 1) / PAIR_B;
        const unsigned pgrid = (unsigned)((pthreads + 127) / 128);
        if (r == 0) msm_pair_kernel<Fb, true><<<pgrid, 128, 0, s>>>(acc_offs, o2, TB, sorted, acc_pts, pb.as<Affine<Fb>>());
        else msm_pair_kernel<Fb, false><<<pgrid, 128, 0, s>>>(acc_offs, o2, TB, sorted, acc_pts, pb.as<Affine<Fb>>());
        launches += 5;
        acc_offs = o2;
        acc_pts = pb.as<Affine<Fb>>();
    }
    if (rounds)
        msm_accumulate_kernel<Fb, 5, true><<<(t1 + 127) / 128, 128, 0, s>>>(acc_offs, TB, sorted, acc_pts, buckets, S.pkey[0].as<uint32_t>(),
                                                                              S.ppt[0].as<Pt>(), P.seg, t1);
    else if (fixed)
        msm_accumulate_kernel<Fb, 5><<<(P.t1 + 127) / 128, 128, 0, s>>>(offsets, TB, sorted, bases, buckets, S.pkey[0].as<uint32_t>(),
                                                                         S.ppt[0].as<Pt>(), P.seg, P.t1);
    else
        msm_accumulate_kernel<Fb, 4><<<(P.t1 + 127) / 128, 128, 0, s>>>(offsets, TB, sorted, bases, buckets, S.pkey[0].as<uint32_t>(),
                                                                         S.ppt[0].as<Pt>(), P.seg, P.t1);
    if (ctx->profile) LURK_CUDA_TRY(cudaEventRecord(ctx->ev1, s));
    launches += 6;
    // shrinking passes over the partial list: one throughput-shaped pass (8 entries per thread), then warp-cooperative
    // passes (32x per pass, 5 dependent additions each) until a single warp finishes
    uint32_t count = t1;
    int cur = 0;
    if (count > 32) {
        const uint32_t seg2 = 8, threads = (count + seg2 - 1) / seg2;
        msm_partial_kernel<Fb><<<(threads + 127) / 128, 128, 0, s>>>(S.pkey[cur].as<uint32_t>(), S.ppt[cur].as<Pt>(), count, buckets,
                                                                    S.pkey[cur ^ 1].as<uint32_t>(), S.ppt[cur ^ 1].as<Pt>(), seg2, 0);
        launches++;
        count = threads;
        cur ^= 1;
    }
    for (;;) {
        const uint32_t warps = (count + 31) / 32;
        const int last = warps == 1;
        msm_partial_warp_kernel<Fb><<<(warps * 32 + 127) / 128, 128, 0, s>>>(S.pkey[cur].as<uint32_t>(), S.ppt[cur].as<Pt>(), count, buckets,
                                                                            S.pkey[cur ^ 1].as<uint32_t>(), S.ppt[cur ^ 1].as<Pt>(), last);
        launches++;
        if (last) break;
        count = warps;
        cur ^= 1;
    }
    // bucket reduction: chunk sums, per-bit tree sums, (slice sums); the host finishes with a Horner over nq points per set
    const uint32_t nchunks = P.rwin * P.G, nres = P.rwin * P.nq;
    if (nres > MSM_MAX_RESULT_POINTS) { set_error("internal: %u result points", nres); return LURK_ERR_ARG; }
    msm_chunk_kernel<Fb><<<(nchunks + 127) / 128, 128, 0, s>>>(buckets, P.K, nchunks, S.chunks.as<Pt>(), S.chunk_sums.as<Pt>());
    msm_bitsum_kernel<Fb><<<dim3(P.SL, P.nq, P.rwin), 256, 0, s>>>(S.chunks.as<Pt>(), S.chunk_sums.as<Pt>(), P.G, P.slice,
                                                                  P.SL > 1 ? S.slices.as<Pt>() : S.wins.as<Pt>());
    launches += 2;
    if (P.SL > 1) {
        msm_slice_sum_kernel<Fb><<<(nres * 32 + 127) / 128, 128, 0, s>>>(S.slices.as<Pt>(), P.SL, nres, S.wins.as<Pt>());
        launches++;
    }
    if (fixed) {   // one bucket set: finish the weighted sum on the device (result stays resident for chained consumers)
        cudaStream_t st = ctx->tiny_stream ? ctx->tiny_stream : s;
        if (st != s) {
            LURK_CUDA_TRY(cudaEventRecord(ctx->ev_fork, s));
            LURK_CUDA_TRY(cudaStreamWaitEvent(st, ctx->ev_fork, 0));
        }
        msm_horner_kernel<Fb><<<1, 32, 0, st>>>(S.wins.as<Pt>(), P.nq, P.K, sub ? (const Affine<Fb> *)ctx->d_offset : nullptr, S.result.as<Pt>());
        launches++;
        if (st != s && readback) {
            LURK_CUDA_TRY(cudaEventRecord(ctx->ev_join, st));
            LURK_CUDA_TRY(cudaStreamWaitEvent(s, ctx->ev_join, 0));
        }
    }
    ctx->last_launches = launches;
    LURK_CUDA_TRY(cudaGetLastError());
    if (!readback) return LURK_OK;
    if (fixed) LURK_CUDA_TRY(cudaMemcpyAsync(S.h_wins, S.result.p, sizeof(Pt), cudaMemcpyDeviceToHost, s));
    else LURK_CUDA_TRY(cudaMemcpyAsync(S.h_wins, S.wins.p, (size_t)nres * sizeof(Pt), cudaMemcpyDeviceToHost, s));
    LURK_CUDA_TRY(cudaEventRecord(ctx->done, s));
    ctx->pending = true;
    ctx->pending_c = P.c;
    ctx->pending_nwin = P.nwin;
    ctx->pending_fixed = fixed;
    ctx->pending_nq = P.nq;
    ctx->pending_K = P.K;
    return LURK_OK;
}

// wait for the read-back, Horner over the windows on the host, one inversion to affine
template <class C>
int msm_finish(lurk_msm_ctx *ctx, uint8_t out[96]) {
    using Fb = typename C::Base;
    using Pt = XYZZ<Fb>;
    if (!ctx->pending) { set_error("no launch pending on this context"); return LURK_ERR_ARG; }
    ctx->pending = false;
    if (ctx->pending_nwin == 0) { memset(out, 0, 96); return LURK_OK; }
    LURK_CUDA_TRY(cudaEventSynchronize(ctx->done));
    if (ctx->profile) cudaEventElapsedTime(&ctx->last_accumulate_ms, ctx->ev0, ctx->ev1);
    const Pt *h = reinterpret_cast<const Pt *>(ctx->scratch.h_wins);
    const uint32_t nq = ctx->pending_nq;
    // bucket set r: R_r = T + K * sum_k 2^k S_k with (T, S_0, .., S_{nq-2}) = h[r * nq ..]  (see msm_chunk_kernel)
    auto bucket_set = [&](uint32_t r) {
        const Pt *q = h + (size_t)r * nq;
        Pt a = Pt::identity();
        for (uint32_t k = nq - 1; k >= 1; k--) { a = a.dbl(); a.add(q[k]); }
        for (uint32_t m = ctx->pending_K; m > 1; m >>= 1) a = a.dbl();
        a.add(q[0]);
        return a;
    };
    Pt acc = Pt::identity();
    if (ctx->pending_fixed) {
        acc = h[0];                                // msm_horner_kernel: the table already carries the 2^(c w) factors
    } else {
        for (int i = ctx->pending_nwin - 1; i >= 0; i--) {
            for (int d = 0; d < ctx->pending_c; d++) acc = acc.dbl();
            acc.add(bucket_set((uint32_t)i));
        }
    }
    point_to_bytes(acc, ctx->pending_fmt, out);
    return LURK_OK;
}

template <class C>
int msm_run(lurk_msm_ctx *ctx, const void *d_scalars, size_t n, int fmt, uint8_t out[96], cudaStream_t s) {
    LURK_TRY(msm_launch<C>(ctx, d_scalars, n, fmt, s, true));
    return msm_finish<C>(ctx, out);
}

template <class C>
int ctx_upload(lurk_msm_ctx *ctx, const uint8_t *bases, size_t n, int fmt) {
    using Fb = typename C::Base;
    LURK_CUDA_TRY(cudaMalloc(&ctx->d_bases, n * 64));
    ctx->owns_bases = true;
    LURK_CUDA_TRY(cudaMemcpy(ctx->d_bases, bases, n * 64, cudaMemcpyHostToDevice));
    int bad = 0;
    LURK_TRY(check_reduced_dev<Fb>(ctx->d_bases, n * 2, 0, &bad));
    if (bad) { set_error("%d base coordinate(s) are not reduced below the field modulus", bad); return LURK_ERR_RANGE; }
    if (fmt == LURK_FMT_CANONICAL) {
        msm_bases_to_mont_kernel<Fb><<<sm_count() * 8, 256>>>((Fb *)ctx->d_bases, n * 2);
        LURK_CUDA_TRY(cudaGetLastError());
        LURK_CUDA_TRY(cudaDeviceSynchronize());
    }
    // curve membership: b = y_G^2 - x_G^3 from the generator
    const Affine<Fb> g = curve_generator<C>();
    const Fb b = g.y.sqr() - g.x.sqr() * g.x;
    DevBuf d_bad;
    LURK_TRY(d_bad.alloc(sizeof(int)));
    LURK_CUDA_TRY(cudaMemset(d_bad.p, 0, sizeof(int)));
    msm_on_curve_kernel<Fb><<<sm_count() * 8, 256>>>((const Affine<Fb> *)ctx->d_bases, n, b, d_bad.as<int>());
    LURK_CUDA_TRY(cudaGetLastError());
    LURK_CUDA_TRY(cudaMemcpy(&bad, d_bad.p, sizeof(int), cudaMemcpyDeviceToHost));
    if (bad) { set_error("%d base point(s) are not on the curve", bad); return LURK_ERR_RANGE; }
    return LURK_OK;
}

// builds the fixed-base table of a context (see lurk_msm_ctx_precompute)
template <class C>
int msm_precompute(lurk_msm_ctx *ctx, int c_override) {
    using Fb = typename C::Base;
    LURK_TRY(ctx_check_device(ctx));
    const int c = c_override ? c_override : fixed_base_window(ctx->n);
    if (c < 4 || c > 22) { set_error("window width %d out of range", c); return LURK_ERR_ARG; }
    const int nwin = C::Scalar::Params::NBITS / c + 1;
    if (nwin > MSM_MAX_TABLE_WINDOWS || (uint64_t)nwin * ctx->n >= (1ull << 31)) { set_error("commitment key too large for a fixed-base table"); return LURK_ERR_ARG; }
    void *t = nullptr;
    LURK_CUDA_TRY(cudaMalloc(&t, (size_t)nwin * ctx->n * sizeof(Affine<Fb>)));
    msm_precompute_kernel<Fb><<<(unsigned)((ctx->n + 127) / 128), 128>>>((const Affine<Fb> *)ctx->d_bases, ctx->n, c, nwin, (Affine<Fb> *)t);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { cudaFree(t); set_error("fixed-base precomputation failed: %s", cudaGetErrorString(e)); return LURK_ERR_CUDA; }
    ctx->d_table = t;
    ctx->owns_table = true;
    ctx->fixed_c = c;
    return LURK_OK;
}

// everything that launches kernels, instantiated once per curve in msm_inst.cu
#define LURK_MSM_INSTANTIATE(C)                                                                    \
    template int msm_launch<C>(lurk_msm_ctx *, const void *, size_t, int, cudaStream_t, bool);    \
    template int msm_finish<C>(lurk_msm_ctx *, uint8_t *);                                         \
    template int msm_run<C>(lurk_msm_ctx *, const void *, size_t, int, uint8_t *, cudaStream_t);  \
    template int ctx_upload<C>(lurk_msm_ctx *, const uint8_t *, size_t, int);                      \
    template int msm_precompute<C>(lurk_msm_ctx *, int);
#define LURK_MSM_EXTERN(C)                                                                                \
    extern template int msm_launch<C>(lurk_msm_ctx *, const void *, size_t, int, cudaStream_t, bool);    \
    extern template int msm_finish<C>(lurk_msm_ctx *, uint8_t *);                                         \
    extern template int msm_run<C>(lurk_msm_ctx *, const void *, size_t, int, uint8_t *, cudaStream_t);  \
    extern template int ctx_upload<C>(lurk_msm_ctx *, const uint8_t *, size_t, int);                      \
    extern template int msm_precompute<C>(lurk_msm_ctx *, int);

}  // namespace lurk
