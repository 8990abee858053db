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
//      Fixed-base mode with c <= 16 keeps the histogram in shared memory, one private copy per CTA, and replaces step 3 by two
//      coalesced passes (by bucket range, then by bucket): msm_hist_smem_kernel .. msm_range_sort_kernel below.
//   2. exclusive scan of the (windows x 2^(c-1)) bucket counts.
//   3. scatter: point index | sign written at its bucket's next slot (counting sort; order inside a bucket is free
//      because point addition commutes -- the affine result is canonical).
//   4. bucket accumulation, the hot kernel: the sorted list is cut into fixed-length segments, one per thread,
//      independent of the bucket sizes (perfect balance for any scalar distribution).  A thread gathers its bases
//      with 128-bit loads (next point prefetched during the current addition), adds them in XYZZ coordinates
//      (8M+2S mixed addition, no inversions) and flushes a bucket sum whenever the bucket id changes.  The first run
//      of a segment may continue a bucket started by the previous thread: it is stored as that thread's partial sum.
//   5. merge: bucket b adds the partials of the threads whose segment starts strictly inside it -- a contiguous range of
//      thread indices found from the offsets alone (one thread per bucket; one CTA per listed long bucket).
//   6. per-window running-sum reduction (chunks of buckets in parallel, then one CTA per window).
//   7. host: Horner combine of the <= 64 window sums and one inversion to affine.
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
static constexpr uint32_t MSM_MAX_SEG = 32;                // longest segment of the sorted list one level-1 thread accumulates

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
    p.seg = (uint32_t)std::min<size_t>(MSM_MAX_SEG, std::max<size_t>(8, seg));
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
// Level-1 threads of the bucket accumulation whose segment [t * seg, ..) starts strictly inside bucket [lo, hi): each leaves
// one partial sum of the bucket, ppt[first .. first + count).  The thread holding `lo` writes the bucket itself.
struct BucketPartials { uint32_t first, count; };
__host__ __device__ __forceinline__ BucketPartials bucket_partials(uint32_t lo, uint32_t hi, uint32_t seg) {
    BucketPartials r{lo / seg + 1, 0};
    if (hi >= lo + 2) {
        const uint32_t last = (hi - 1) / seg;
        if (last >= r.first) r.count = last - r.first + 1;
    }
    return r;
}
// buckets with more partials than this are merged by a whole CTA (msm_merge_long_kernel); the others by one thread each
static constexpr uint32_t MSM_LONG_PARTIALS = 16;

// long_list: appends every bucket with more than MSM_LONG_PARTIALS partials for segments of `seg` entries; long_list[-1] is its
// length, zeroed before the launch
static __global__ void __launch_bounds__(1024) msm_scan_apply_kernel(const uint32_t *__restrict__ counts, uint32_t len, const uint32_t *__restrict__ tile_offsets,
                                                              uint32_t ntiles, uint32_t *__restrict__ offsets, uint32_t seg, uint32_t *long_list) {
    const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * 4;
    uint32_t v[4], sum = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) { v[k] = base + k < len ? counts[base + k] : 0; sum += v[k]; }
    uint32_t run = tile_offsets[blockIdx.x] + block_exclusive_scan_1024(sum, nullptr);
#pragma unroll
    for (int k = 0; k < 4; k++) {
        if (base + k < len) {
            offsets[base + k] = run;
            if (bucket_partials(run, run + v[k], seg).count > MSM_LONG_PARTIALS) long_list[atomicAdd(long_list - 1, 1u)] = base + k;
        }
        run += v[k];
    }
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

// ---- the same counting sort in two coalesced levels (fixed-base mode, c <= 16) ----------------------------------------------------
// All windows of the fixed-base mode share ONE bucket set, so the whole histogram is nb * 4 bytes: 128 KB at c = 16, inside the
// 227 KB a CTA may have on sm_90.  A persistent grid of G CTAs (one per SM) gives each CTA a contiguous range of scalars and a
// private histogram; the digits of a full-width scalar are spread over 2^15 buckets, where the warp aggregation of the kernels
// above merges nothing.  Here a zero scalar (two thirds of the fold's vectors) costs one load and no window walk.
// Writing each digit straight to its bucket's slot is one scattered 4-byte store per digit (a CTA holds ~1.4 digits per bucket at
// c = 16, too few to stage); instead the buckets are grouped into ranges of MSM_RANGE_BUCKETS consecutive buckets and the digits
// move in two coalesced passes, first to their range, then inside it to their bucket:
//   msm_hist_smem_kernel     cnt[g][b] = digits of CTA g's scalars in bucket b; rng[g][j] = the same per range j
//   msm_hist_columns_kernel  counts[b] = column total of cnt, tile sums of counts for the scan; rng[g][j] -> exclusive prefix over g
//   (the scan kernels above turn counts into offsets)
//   msm_partition_kernel     CTA g re-walks its scalars a tile at a time, groups the tile's digits by range in shared memory and
//                            appends each group to the CTA's slice of the range's span [offsets[first bucket], offsets[last + 1])
//                            as 8-byte entries (sorted word, bucket): runs of dozens of entries instead of single words
//   msm_range_sort_kernel    fixed-size slices of every range's span: a counting sort by bucket in shared memory, then each bucket's
//                            run is written out contiguously at a place taken from a per-bucket cursor (one global atomic per bucket
//                            and slice, so a hot bucket spread over many slices -- a 0/1-heavy witness -- still spreads over all SMs)
static constexpr uint32_t MSM_SORT_THREADS = 1024;
static constexpr size_t MSM_SORT_SMEM_MAX = (size_t)128 << 10;
static constexpr uint32_t MSM_RANGE_BITS = 7, MSM_RANGE_BUCKETS = 1u << MSM_RANGE_BITS;   // 256 ranges at c = 16
static constexpr uint32_t MSM_MAX_RANGES = (1u << 15) / MSM_RANGE_BUCKETS;
static constexpr uint32_t MSM_PART_DIGITS = 32768;      // digits a partition tile stages (6 B each: 192 KB)
static constexpr uint32_t MSM_PART_SCALARS = 2 * MSM_SORT_THREADS;
static constexpr uint32_t MSM_RSORT_PER_THREAD = 8, MSM_RSORT_SLICE = MSM_RSORT_PER_THREAD * MSM_SORT_THREADS;

__host__ __device__ __forceinline__ uint32_t msm_ranges(uint32_t nb) { return (nb + MSM_RANGE_BUCKETS - 1) / MSM_RANGE_BUCKETS; }
// scalars per partition tile: every digit of the tile fits the staging buffer
inline uint32_t msm_part_scalars(int nwin) { return std::min<uint32_t>(MSM_PART_SCALARS, MSM_PART_DIGITS / (uint32_t)nwin); }

// scalar i as the sort sees it (minus the constant part, canonical); false when it is zero and contributes no digit
template <class Fs>
__device__ __forceinline__ void prefetch_scalar(const Fs *__restrict__ scalars, const Fs *__restrict__ sub, size_t i) {
    // the sort kernels run one 1024-thread CTA per SM with a serial chain per thread: ask L2 for the next scalar early
    asm volatile("prefetch.global.L2 [%0];" ::"l"(scalars + i));
    if (sub) asm volatile("prefetch.global.L2 [%0];" ::"l"(sub + i));
}
template <class Fs>
__device__ __forceinline__ bool sort_scalar(const Fs *__restrict__ scalars, const Fs *__restrict__ sub, size_t i, int fmt, Fs &k) {
    k = load_fe<Fs>(scalars + i);
    if (sub) k = k - load_fe<Fs>(sub + i);
    if (k.is_zero()) return false;               // zero is zero in either form
    if (fmt == LURK_FMT_MONTGOMERY) k = k.to_canonical();
    return true;
}

// f(w, bucket, negative) for every non-zero signed digit of k.  The fold tables' shape (c = 16, 16 windows) is unrolled at compile
// time, so the window indices are constants and the scalar's limbs stay in registers instead of a stack frame indexed per window.
template <int C, int NWIN, class Fs, class F>
__device__ __forceinline__ void walk_digits_unrolled(const Fs &k, F f) {
    uint32_t carry = 0;
#pragma unroll
    for (int w = 0; w < NWIN; w++) {
        const uint32_t raw = window_bits(k.v, w * C, C) + carry;
        carry = raw > (1u << (C - 1));
        const uint32_t mag = carry ? (1u << C) - raw : raw;
        if (mag) f((uint32_t)w, mag - 1, carry);
    }
}
template <class Fs, class F>
__device__ __forceinline__ void walk_digits(const Fs &k, int c, int nwin, F f) {
    if (c == 16 && nwin == 16) { walk_digits_unrolled<16, 16>(k, f); return; }
    uint32_t kv[8];                                  // a copy for the per-window indexing, so that k itself stays in registers
#pragma unroll
    for (int i = 0; i < 8; i++) kv[i] = k.v[i];
    const uint32_t half = 1u << (c - 1);
    uint32_t carry = 0;
    for (int w = 0; w < nwin; w++) {
        const uint32_t raw = window_bits(kv, w * c, c) + carry;
        carry = raw > half;
        const uint32_t mag = carry ? (1u << c) - raw : raw;
        if (mag) f((uint32_t)w, mag - 1, carry);
    }
}

// zero: `nzero` words the later kernels accumulate into (the scan's tile sums, the long-bucket count), cleared by CTA 0
template <class Fs>
__global__ void __launch_bounds__(MSM_SORT_THREADS) msm_hist_smem_kernel(const Fs *__restrict__ scalars, const Fs *__restrict__ sub, size_t n, int fmt, int c,
                                                                         int nwin, uint32_t nb, uint32_t *__restrict__ cnt, uint32_t *__restrict__ rng,
                                                                         uint32_t *__restrict__ zero, uint32_t nzero) {
    extern __shared__ uint32_t sort_smem[];
    if (blockIdx.x == 0)
        for (uint32_t t = threadIdx.x; t < nzero; t += MSM_SORT_THREADS) zero[t] = 0;
    for (uint32_t b = threadIdx.x; b < nb; b += MSM_SORT_THREADS) sort_smem[b] = 0;
    __syncthreads();
    const size_t lo = (size_t)blockIdx.x * n / gridDim.x, hi = (size_t)(blockIdx.x + 1) * n / gridDim.x;
    for (size_t i = lo + threadIdx.x; i < hi; i += MSM_SORT_THREADS) {
        if (i + MSM_SORT_THREADS < hi) prefetch_scalar(scalars, sub, i + MSM_SORT_THREADS);
        Fs k;
        if (!sort_scalar(scalars, sub, i, fmt, k)) continue;
        walk_digits(k, c, nwin, [&](uint32_t, uint32_t b, uint32_t) { atomicAdd(sort_smem + b, 1u); });
    }
    __syncthreads();
    uint32_t *row = cnt + (size_t)blockIdx.x * nb;
    for (uint32_t b = threadIdx.x; b < nb; b += MSM_SORT_THREADS) row[b] = sort_smem[b];
    // one warp per range
    const uint32_t R = msm_ranges(nb), lane = threadIdx.x & 31;
    for (uint32_t j = threadIdx.x >> 5; j < R; j += MSM_SORT_THREADS / 32) {
        uint32_t v = 0;
        for (uint32_t b = j * MSM_RANGE_BUCKETS + lane; b < min(nb, (j + 1) * MSM_RANGE_BUCKETS); b += 32) v += sort_smem[b];
        v = __reduce_add_sync(0xffffffffu, v);
        if (lane == 0) rng[(size_t)blockIdx.x * R + j] = v;
    }
}

// One thread per bucket: counts[b] = sum over the G rows, cursor[b] = 0 (msm_range_sort_kernel's), and each warp adds its buckets to
// their scan tile's sum (tile_sums zeroed by msm_hist_smem_kernel) -- the first of the three scan launches, fused.  Warp j < R also
// turns column j of rng into its exclusive prefix over the CTAs.
static __global__ void __launch_bounds__(256) msm_hist_columns_kernel(const uint32_t *__restrict__ cnt, uint32_t *__restrict__ rng, uint32_t G, uint32_t nb,
                                                                      uint32_t *__restrict__ counts, uint32_t *__restrict__ cursor,
                                                                      uint32_t *__restrict__ tile_sums) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31;
    uint32_t run = 0;
    if (b < nb) {
        for (uint32_t g0 = 0; g0 < G; g0 += 8) {     // eight independent loads in flight per thread
            uint32_t v[8];
#pragma unroll
            for (uint32_t j = 0; j < 8; j++) v[j] = g0 + j < G ? cnt[(size_t)(g0 + j) * nb + b] : 0u;
#pragma unroll
            for (uint32_t j = 0; j < 8; j++) run += v[j];
        }
        counts[b] = run;
        cursor[b] = 0;
    }
    const uint32_t wsum = __reduce_add_sync(0xffffffffu, run);
    if (lane == 0 && wsum) atomicAdd(tile_sums + b / SCAN_TILE, wsum);     // a warp's 32 buckets lie in one tile
    const uint32_t j = b >> 5, R = msm_ranges(nb);
    if (j >= R) return;
    uint32_t carry = 0;
    for (uint32_t g0 = 0; g0 < G; g0 += 32) {
        const uint32_t g = g0 + lane;
        const uint32_t v = g < G ? rng[(size_t)g * R + j] : 0u;
        uint32_t incl = v;
        for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= (uint32_t)d) incl += t; }
        if (g < G) rng[(size_t)g * R + j] = carry + incl - v;
        carry += __shfl_sync(0xffffffffu, incl, 31);
    }
}

// CTA g: the scalars of msm_hist_smem_kernel's CTA g, `ts` at a time (two per thread; ts * nwin <= the staging buffer).  Per tile:
// count the digits per range, scan, stage them grouped by range (sorted word + bucket, 6 B), then append each range's group to
// the CTA's cursor in that range's span.  Consecutive threads write consecutive entries of one group: the stores coalesce.
template <class Fs>
__global__ void __launch_bounds__(MSM_SORT_THREADS) msm_partition_kernel(const Fs *__restrict__ scalars, const Fs *__restrict__ sub, size_t n, int fmt, int c,
                                                                         int nwin, uint32_t nb, uint32_t ts, uint32_t base_stride,
                                                                         const uint32_t *__restrict__ offsets, const uint32_t *__restrict__ rng,
                                                                         uint2 *__restrict__ parts) {
    extern __shared__ uint32_t part_smem[];
    uint32_t *wbuf = part_smem;                                           // ts * nwin sorted words
    uint16_t *bbuf = reinterpret_cast<uint16_t *>(part_smem + (size_t)ts * nwin);   // ... and their buckets
    __shared__ uint32_t rcnt[MSM_MAX_RANGES], rstart[MSM_MAX_RANGES], rfill[MSM_MAX_RANGES], rcur[MSM_MAX_RANGES];
    const uint32_t tid = threadIdx.x, R = msm_ranges(nb);
    if (tid < R) rcur[tid] = offsets[tid * MSM_RANGE_BUCKETS] + rng[(size_t)blockIdx.x * R + tid];
    const size_t lo = (size_t)blockIdx.x * n / gridDim.x, hi = (size_t)(blockIdx.x + 1) * n / gridDim.x;
    for (size_t t0 = lo; t0 < hi; t0 += ts) {
        if (tid < R) rcnt[tid] = 0;
        __syncthreads();
        Fs k[2];
        bool live[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const uint32_t t = tid + h * MSM_SORT_THREADS;
            if (t < ts && t0 + ts + t < hi) prefetch_scalar(scalars, sub, t0 + ts + t);      // the next tile's
            live[h] = t < ts && t0 + t < hi && sort_scalar(scalars, sub, t0 + t, fmt, k[h]);
            if (live[h]) walk_digits(k[h], c, nwin, [&](uint32_t, uint32_t b, uint32_t) { atomicAdd(rcnt + (b >> MSM_RANGE_BITS), 1u); });
        }
        __syncthreads();
        uint32_t total;
        const uint32_t ex = block_exclusive_scan_1024(tid < R ? rcnt[tid] : 0u, &total);
        if (tid < R) { rstart[tid] = ex; rfill[tid] = ex; }
        __syncthreads();
#pragma unroll
        for (int h = 0; h < 2; h++) {
            if (!live[h]) continue;
            const uint32_t i = (uint32_t)(t0 + tid + h * MSM_SORT_THREADS);
            walk_digits(k[h], c, nwin, [&](uint32_t w, uint32_t b, uint32_t neg) {
                const uint32_t p = atomicAdd(rfill + (b >> MSM_RANGE_BITS), 1u);
                wbuf[p] = (i + w * base_stride) | (neg << 31);
                bbuf[p] = (uint16_t)b;
            });
        }
        __syncthreads();
        for (uint32_t p = tid; p < total; p += MSM_SORT_THREADS) {
            const uint32_t b = bbuf[p], j = b >> MSM_RANGE_BITS;
            parts[rcur[j] + p - rstart[j]] = make_uint2(wbuf[p], b);
        }
        __syncthreads();
        if (tid < R) rcur[tid] += rcnt[tid];
    }
}

// Persistent grid over the slices of MSM_RSORT_SLICE entries of every range's span (a range's last slice may be shorter).  A slice:
// counting sort by bucket in shared memory (ranks from shared atomics, kept in registers), one global atomic per non-empty bucket
// to claim that many places in the bucket, and a linear pass that writes each bucket's run contiguously.
static constexpr int MSM_RSORT_CTAS_PER_SM = 2;     // one CTA's barriers overlap the other's loads
static __global__ void __launch_bounds__(MSM_SORT_THREADS, MSM_RSORT_CTAS_PER_SM) msm_range_sort_kernel(const uint32_t *__restrict__ offsets, uint32_t nb,
                                                                              const uint2 *__restrict__ parts, uint32_t *__restrict__ cursor,
                                                                              uint32_t *__restrict__ sorted) {
    __shared__ uint32_t sp[MSM_MAX_RANGES + 1];
    __shared__ uint32_t hist[MSM_RANGE_BUCKETS], start[MSM_RANGE_BUCKETS], base[MSM_RANGE_BUCKETS];
    __shared__ uint32_t obuf[MSM_RSORT_SLICE];
    __shared__ uint8_t obkt[MSM_RSORT_SLICE];
    const uint32_t tid = threadIdx.x, R = msm_ranges(nb);
    {   // slices per range -> their exclusive prefix sp[0..R]
        uint32_t s = 0;
        if (tid < R) s = (offsets[min(nb, (tid + 1) * MSM_RANGE_BUCKETS)] - offsets[tid * MSM_RANGE_BUCKETS] + MSM_RSORT_SLICE - 1) / MSM_RSORT_SLICE;
        uint32_t total;
        const uint32_t ex = block_exclusive_scan_1024(s, &total);
        if (tid < R) sp[tid] = ex;
        if (tid == 0) sp[R] = total;
        __syncthreads();
    }
    for (uint32_t u = blockIdx.x; u < sp[R]; u += gridDim.x) {
        uint32_t j0 = 0, j1 = R;                  // the range: largest j with sp[j] <= u
        while (j1 - j0 > 1) { const uint32_t m = (j0 + j1) >> 1; if (sp[m] <= u) j0 = m; else j1 = m; }
        const uint32_t r0 = j0 * MSM_RANGE_BUCKETS, rb = min(MSM_RANGE_BUCKETS, nb - r0);
        const uint32_t lo = offsets[r0] + (u - sp[j0]) * MSM_RSORT_SLICE, hi = min(lo + MSM_RSORT_SLICE, offsets[r0 + rb]);
        if (tid < MSM_RANGE_BUCKETS) hist[tid] = 0;
        __syncthreads();
        uint32_t word[MSM_RSORT_PER_THREAD], key[MSM_RSORT_PER_THREAD];   // key = bucket in range | rank in bucket << 8
#pragma unroll
        for (uint32_t e = 0; e < MSM_RSORT_PER_THREAD; e++) {
            const uint32_t p = lo + e * MSM_SORT_THREADS + tid;
            key[e] = ~0u;                         // past the slice
            if (p < hi) {
                const uint2 v = parts[p];
                const uint32_t lb = v.y - r0;
                word[e] = v.x;
                key[e] = lb | atomicAdd(hist + lb, 1u) << 8;
            }
        }
        __syncthreads();
        if (tid < 32) {   // exclusive scan of the <= 128 bucket counts, four per lane
            uint32_t v[MSM_RANGE_BUCKETS / 32], sum = 0;
#pragma unroll
            for (uint32_t q = 0; q < MSM_RANGE_BUCKETS / 32; q++) { v[q] = hist[tid * (MSM_RANGE_BUCKETS / 32) + q]; sum += v[q]; }
            uint32_t incl = sum;
            for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d); if (tid >= (uint32_t)d) incl += t; }
            uint32_t run = incl - sum;
#pragma unroll
            for (uint32_t q = 0; q < MSM_RANGE_BUCKETS / 32; q++) { start[tid * (MSM_RANGE_BUCKETS / 32) + q] = run; run += v[q]; }
        }
        if (tid < rb && hist[tid]) base[tid] = offsets[r0 + tid] + atomicAdd(cursor + r0 + tid, hist[tid]);
        __syncthreads();
#pragma unroll
        for (uint32_t e = 0; e < MSM_RSORT_PER_THREAD; e++) {
            if (key[e] != ~0u) {
                const uint32_t lb = key[e] & 0xffu, q = start[lb] + (key[e] >> 8);
                obuf[q] = word[e];
                obkt[q] = (uint8_t)lb;
            }
        }
        __syncthreads();
        for (uint32_t q = tid; q < hi - lo; q += MSM_SORT_THREADS) {
            const uint32_t lb = obkt[q];
            sorted[base[lb] + q - start[lb]] = obuf[q];
        }
        __syncthreads();                          // hist, start, base and the buffers are reused by the next slice
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
template <class Fb, int MINB>
__global__ void __launch_bounds__(128, MINB) msm_accumulate_kernel(const uint32_t *__restrict__ offsets, uint32_t nbuckets,
                                                             const uint32_t *__restrict__ sorted, const Affine<Fb> *__restrict__ bases,
                                                             XYZZ<Fb> *__restrict__ bucket_acc, XYZZ<Fb> *__restrict__ ppt, uint32_t seg,
                                                             uint32_t nthreads) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nthreads) return;
    const uint32_t total = offsets[nbuckets];
    const uint64_t start64 = (uint64_t)t * seg;
    if (start64 >= total) return;
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
    // a first run that starts inside its bucket continues another thread's run: it becomes the partial ppt[t], which
    // msm_merge_kernel adds to the bucket (see bucket_partials); every other run starts its bucket and writes it
    bool first_run = offsets[key] != start;
    uint32_t e_next = sorted[start];
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
            e_next = sorted[pos];
            p_next = load_affine(bases + (e_next & 0x7fffffffu));
        }
        acc.add_affine(p, (e >> 31) != 0);
        if (pos == run_end) {
            if (first_run) { store_xyzz(ppt + t, acc); first_run = false; }
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

// ---- merge of the level-1 partials: bucket b receives the partials ppt[first .. first + count) of the threads whose segment
// starts strictly inside it (bucket_partials), a contiguous range, so no keys and no search are needed.  Every bucket is
// written here or by the long-bucket kernel (empty buckets as the identity), so bucket_acc is not cleared before a launch.
// Longest chain: MSM_LONG_PARTIALS additions here, ceil(partials / 256) + 8 in msm_merge_long_kernel -- instead of the
// 8 + 5 per pass of the shrinking (key, point) passes this replaces, which also walked one slot per level-1 thread.
static constexpr uint32_t MSM_MERGE_THREADS = 64, MSM_MERGE_LONG_THREADS = 256;
template <class Fb>
__global__ void __launch_bounds__(MSM_MERGE_THREADS) msm_merge_kernel(const uint32_t *__restrict__ offsets, uint32_t nbuckets, uint32_t seg,
                                                                      const XYZZ<Fb> *__restrict__ ppt, XYZZ<Fb> *__restrict__ bucket_acc) {
    const uint32_t b = blockIdx.x * MSM_MERGE_THREADS + threadIdx.x;
    if (b >= nbuckets) return;
    const uint32_t lo = offsets[b], hi = offsets[b + 1];
    const BucketPartials bp = bucket_partials(lo, hi, seg);
    if (bp.count > MSM_LONG_PARTIALS) return;                    // msm_merge_long_kernel's
    XYZZ<Fb> acc = XYZZ<Fb>::identity();
    if (hi > lo) acc = load_xyzz(bucket_acc + b);
    for (uint32_t i = 0; i < bp.count; i++) acc.add(load_xyzz(ppt + bp.first + i));
    store_xyzz(bucket_acc + b, acc);
}

// the long buckets listed by msm_scan_apply_kernel (0/1-heavy witness vectors, equal scalars, the shared bucket set of
// fixed-base mode): one bucket per CTA at a time, strided sums, then a shared-memory tree
template <class Fb>
__global__ void __launch_bounds__(MSM_MERGE_LONG_THREADS) msm_merge_long_kernel(const uint32_t *__restrict__ offsets, uint32_t seg,
                                                                                const XYZZ<Fb> *__restrict__ ppt, const uint32_t *__restrict__ long_list,
                                                                                XYZZ<Fb> *__restrict__ bucket_acc) {
    __shared__ XYZZ<Fb> sm[MSM_MERGE_LONG_THREADS];
    const uint32_t tid = threadIdx.x, nlong = long_list[-1];
    for (uint32_t i = blockIdx.x; i < nlong; i += gridDim.x) {
        const uint32_t b = long_list[i];
        const BucketPartials bp = bucket_partials(offsets[b], offsets[b + 1], seg);
        XYZZ<Fb> acc = XYZZ<Fb>::identity();
        if (tid == 0) acc = load_xyzz(bucket_acc + b);            // a long bucket is not empty
        for (uint32_t j = tid; j < bp.count; j += MSM_MERGE_LONG_THREADS) acc.add(load_xyzz(ppt + bp.first + j));
        sm[tid] = acc;
        __syncthreads();
        for (uint32_t stride = MSM_MERGE_LONG_THREADS / 2; stride > 0; stride >>= 1) {
            if (tid < stride) { XYZZ<Fb> x = sm[tid]; x.add(sm[tid + stride]); sm[tid] = x; }
            __syncthreads();
        }
        if (tid == 0) store_xyzz(bucket_acc + b, sm[0]);
        __syncthreads();                                          // sm is reused by the next long bucket
    }
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
    DevBuf counts, hist, offsets, tiles, sorted, parts, buckets, ppt, chunks, chunk_sums, slices, wins, result, scalars;
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
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_sort = nullptr;   // ev_sort .. ev0: the digit sort; ev0 .. ev1: the accumulation
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
    // a long bucket holds more than MSM_LONG_PARTIALS segment starts, so there are at most t1 / (MSM_LONG_PARTIALS + 1)
    const uint32_t max_long = P.t1 / (MSM_LONG_PARTIALS + 1) + 1;
    // digit sort: per-CTA shared-memory histograms and two coalesced passes when one bucket set fits a CTA's shared memory (see
    // msm_hist_smem_kernel).
    // LURK_MSM_SORT=legacy forces the global-atomics kernels (tuning aid, read at every launch so that one process can compare both)
    const char *sort_env = getenv("LURK_MSM_SORT");
    const bool smem_sort = fixed && (size_t)P.nb * sizeof(uint32_t) <= MSM_SORT_SMEM_MAX && !(sort_env && !strcmp(sort_env, "legacy"));
    const uint32_t sort_ctas = (uint32_t)std::min<size_t>((size_t)sm_count(), (n + MSM_SORT_THREADS - 1) / MSM_SORT_THREADS);
    {
        // scratch grows monotonically; a context is normally run at one size (the circuit's witness length)
        auto ensure = [](DevBuf &b, size_t bytes) { return b.bytes >= bytes ? LURK_OK : b.alloc(bytes); };
        LURK_TRY(ensure(S.counts, (((size_t)TB + 1) * 2 + 1 + max_long) * sizeof(uint32_t)));   // counts | cursor | long count | long list
        if (smem_sort) {
            LURK_TRY(ensure(S.hist, (size_t)sort_ctas * (P.nb + msm_ranges(P.nb)) * sizeof(uint32_t)));   // cnt[G][nb] | rng[G][R]
            LURK_TRY(ensure(S.parts, n * (size_t)P.nwin * sizeof(uint2)));   // (sorted word, bucket) grouped by bucket range
        }
        LURK_TRY(ensure(S.offsets, ((size_t)TB + 1) * sizeof(uint32_t)));
        LURK_TRY(ensure(S.tiles, ((size_t)ntiles + 1) * 2 * sizeof(uint32_t)));  // tile sums | tile offsets
        LURK_TRY(ensure(S.sorted, n * (size_t)P.nwin * sizeof(uint32_t)));
        LURK_TRY(ensure(S.buckets, (size_t)TB * sizeof(Pt)));
        LURK_TRY(ensure(S.ppt, (size_t)P.t1 * sizeof(Pt)));              // one partial slot per level-1 thread
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
    uint32_t *long_list = cursor + (TB + 1) + 1;                        // long_list[-1] is zeroed with the counts
    Pt *buckets = S.buckets.as<Pt>();       // every bucket is written by the accumulation or the merge: no clearing

    if (ctx->profile) LURK_CUDA_TRY(cudaEventRecord(ctx->ev_sort, s));
    unsigned launches = 0;
    const uint32_t key_stride = fixed ? 0u : P.nb;                 // fixed-base: all windows share one bucket set
    const uint32_t base_stride = fixed ? (uint32_t)ctx->n : 0u;     // ... and address table[w * n + i]
    const Affine<Fb> *bases = (const Affine<Fb> *)(fixed ? ctx->d_table : ctx->d_bases);
    const Fs *sub = (!readback && fmt == LURK_FMT_MONTGOMERY) ? (const Fs *)ctx->d_sub : nullptr;
    if (smem_sort) {
        const size_t smem = (size_t)P.nb * sizeof(uint32_t);
        const uint32_t ts = msm_part_scalars(P.nwin);
        const size_t part_smem = (size_t)ts * P.nwin * (sizeof(uint32_t) + sizeof(uint16_t));
        uint32_t *cnt = S.hist.as<uint32_t>(), *rng = cnt + (size_t)sort_ctas * P.nb;
        uint2 *parts = S.parts.as<uint2>();
        // above the default limit a kernel opts in, per device
        if (smem > ((size_t)48 << 10)) LURK_CUDA_TRY(cudaFuncSetAttribute(msm_hist_smem_kernel<Fs>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        if (part_smem > ((size_t)48 << 10))
            LURK_CUDA_TRY(cudaFuncSetAttribute(msm_partition_kernel<Fs>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)part_smem));
        // every count is written; only the long-list length is cleared, and the scan's tile sums by the histogram kernel's CTA 0
        LURK_CUDA_TRY(cudaMemsetAsync(long_list - 1, 0, sizeof(uint32_t), s));
        msm_hist_smem_kernel<Fs><<<sort_ctas, MSM_SORT_THREADS, smem, s>>>((const Fs *)d_scalars, sub, n, fmt, P.c, P.nwin, P.nb, cnt, rng, tile_sums, ntiles);
        msm_hist_columns_kernel<<<(P.nb + 255) / 256, 256, 0, s>>>(cnt, rng, sort_ctas, P.nb, counts, cursor, tile_sums);
        msm_scan_tiles_kernel<<<1, 1024, 0, s>>>(tile_sums, ntiles, tile_offsets);
        msm_scan_apply_kernel<<<ntiles, 1024, 0, s>>>(counts, TB, tile_offsets, ntiles, offsets, P.seg, long_list);
        msm_partition_kernel<Fs><<<sort_ctas, MSM_SORT_THREADS, part_smem, s>>>((const Fs *)d_scalars, sub, n, fmt, P.c, P.nwin, P.nb, ts, base_stride,
                                                                                 offsets, rng, parts);
        msm_range_sort_kernel<<<MSM_RSORT_CTAS_PER_SM * sm_count(), MSM_SORT_THREADS, 0, s>>>(offsets, P.nb, parts, cursor, sorted);
        launches++;
    } else {
        LURK_CUDA_TRY(cudaMemsetAsync(counts, 0, (((size_t)TB + 1) * 2 + 1) * sizeof(uint32_t), s));
        msm_count_kernel<Fs><<<(unsigned)((n + 255) / 256), 256, 0, s>>>((const Fs *)d_scalars, sub, n, fmt, P.c, P.nwin, key_stride, counts);
        msm_scan_tile_sums_kernel<<<ntiles, 1024, 0, s>>>(counts, TB, tile_sums);
        msm_scan_tiles_kernel<<<1, 1024, 0, s>>>(tile_sums, ntiles, tile_offsets);
        // the offsets the accumulation walks also give the merge its long buckets
        msm_scan_apply_kernel<<<ntiles, 1024, 0, s>>>(counts, TB, tile_offsets, ntiles, offsets, P.seg, long_list);
        msm_scatter_kernel<Fs><<<(unsigned)((n + 255) / 256), 256, 0, s>>>((const Fs *)d_scalars, sub, n, fmt, P.c, P.nwin, key_stride, base_stride, offsets, cursor, sorted);
    }
    if (ctx->profile) LURK_CUDA_TRY(cudaEventRecord(ctx->ev0, s));
    if (fixed)
        msm_accumulate_kernel<Fb, 5><<<(P.t1 + 127) / 128, 128, 0, s>>>(offsets, TB, sorted, bases, buckets, S.ppt.as<Pt>(), P.seg, P.t1);
    else
        msm_accumulate_kernel<Fb, 4><<<(P.t1 + 127) / 128, 128, 0, s>>>(offsets, TB, sorted, bases, buckets, S.ppt.as<Pt>(), P.seg, P.t1);
    if (ctx->profile) LURK_CUDA_TRY(cudaEventRecord(ctx->ev1, s));
    launches += 6;
    // merge of the partials into their buckets: long buckets (one CTA each, a grid of at most two per SM walking the list)
    // and the others (one thread each) are disjoint, so the two launches do not depend on each other
    msm_merge_long_kernel<Fb><<<std::min<uint32_t>(max_long, 2 * sm_count()), MSM_MERGE_LONG_THREADS, 0, s>>>(offsets, P.seg, S.ppt.as<Pt>(),
                                                                                                             long_list, buckets);
    msm_merge_kernel<Fb><<<(TB + MSM_MERGE_THREADS - 1) / MSM_MERGE_THREADS, MSM_MERGE_THREADS, 0, s>>>(offsets, TB, P.seg, S.ppt.as<Pt>(), buckets);
    launches += 2;
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
