// A device-resident node store of the arity-8 Poseidon trie (reference src/coprocessor/trie/mod.rs: Trie with its inverse
// Poseidon cache), and a batch of lookups and inserts applied to it in program order, level by level, each operation's
// LookupProof / InsertProof written in the layout lurk_trie_witness_batch reads.
//
// Store: an open-addressed table (linear probing, 2^k >= 2 x capacity slots of u32 node index + 1) from digest to node,
// and per node its digest and its 8-element preimage, all canonical.  Nodes are only ever added.
//
// One batch (K operations, m inserts; chains and versions as in include/lurk_b200.h):
//   1. walk     one thread per operation walks its chain's base root down its key's path and records the node index at
//               every depth.  A digest missing from the store sets a device flag (the lowest (operation, depth) wins);
//               every later kernel reads the flag and writes nothing once it is set.
//   2. levels   d = H-1 down to 0.  The node at depth d on an operation's path, in the version it sees, is its base
//               node with child c replaced by the depth-(d+1) digest (at d = H-1 the value) of the last visible insert
//               of its chain whose key extends the same prefix by c.  The inserts sorted by (chain, prefix of d+1
//               chunks, index) -- a 64-bit radix sort of (prefix group rank, index) -- answer that with one binary
//               search per (operation, child).  That preimage is the old-path entry; an insert also sets its own child
//               to its new digest from depth d+1, and the m new preimages of the level are hashed (the arity-8 digest
//               launch of poseidon_kernel.cuh) and registered.  Nothing in one level depends on another thread's work
//               in the same level, and no level waits for the host.
//   3. finish   roots, keys, values and results.
// lurk_trie_ctx_apply plans on the host (plan_batch: argument checks, chains, ranks, the inserts sorted by (chain, key
// path) once) and uploads the plan.  lurk_trie_ctx_apply_dev, whose operations are already in device memory, plans on
// the device (plan_dev: validate, pointer jumping over prev, a CUB scan for the ranks, stable CUB radix passes for the
// order) and reads back only a status word before the levels.  Both then run the same levels (run_levels).
#include "common.cuh"
#include "poseidon_api.h"
#include "trie.cuh"

#include <cub/cub.cuh>

#include <algorithm>
#include <cstring>
#include <numeric>

struct lurk_trie_ctx;

namespace lurk {

#define LURK_TRIE_STORE_EXTERN(F)                                                                                             \
    extern template int launch_poseidon<F, false>(int, const void *, size_t, void *, int, int, cudaStream_t, const uint64_t *, \
                                                  const PoseidonGather *);
LURK_TRIE_STORE_EXTERN(Fe<Bn254Fr>)
LURK_TRIE_STORE_EXTERN(Fe<Bn254Fq>)
LURK_TRIE_STORE_EXTERN(Fe<PallasFq>)
LURK_TRIE_STORE_EXTERN(Fe<PallasFp>)

namespace {

constexpr int ARITY = 8, TS_THREADS = 128;
constexpr uint32_t NONE = 0xffffffffu, CLAIM = 0x80000000u;
constexpr unsigned long long NO_ERR = ~0ull;

// one operation as the kernels see it: the key's path (low 3H bits of the canonical key), its chain (the index of the
// chain's first operation), the last insert index it sees (-1: none), prev, its rank among the operations of its kind
struct OpDev {
    uint32_t path[8];
    uint32_t chain;
    int32_t bound, prev;
    uint32_t rank, kind, pad[3];
};

__host__ __device__ __forceinline__ int chunk_at(const uint32_t *path, int height, int d) {
    const int lo = 3 * (height - 1 - d);
    int k = 0;
    for (int t = 0; t < 3; t++) k |= (int)((path[(lo + t) >> 5] >> ((lo + t) & 31)) & 1) << t;
    return k;
}

__device__ __forceinline__ uint32_t slot_of(const uint32_t *v, uint64_t mask) {
    return (uint32_t)(((uint64_t)v[0] ^ ((uint64_t)v[1] << 32) ^ ((uint64_t)v[2] * 0x9E3779B97F4A7C15ull)) & mask);
}

__device__ __forceinline__ bool eq8(const uint32_t *a, const uint32_t *b) {
    bool e = true;
#pragma unroll
    for (int i = 0; i < 8; i++) e &= a[i] == b[i];
    return e;
}

// node index of digest d, NONE when absent (no claims are pending outside registration)
template <class F>
__device__ uint32_t find_node(const uint32_t *__restrict__ table, uint64_t mask, const F *__restrict__ dig, const F &d) {
    for (uint64_t h = slot_of(d.v, mask);; h = (h + 1) & mask) {
        const uint32_t v = table[h];
        if (!v) return NONE;
        const F x = load_fe<F>(dig + (v - 1));
        if (eq8(x.v, d.v)) return v - 1;
    }
}

template <class F>
__device__ __forceinline__ F out_fmt(const F &x, int fmt) { return fmt == LURK_FMT_MONTGOMERY ? F::from_canonical(x) : x; }

template <class F>
__global__ void __launch_bounds__(TS_THREADS) walk_kernel(int n, int height, const OpDev *__restrict__ ops, const F *__restrict__ base,
                                                          const uint32_t *__restrict__ table, uint64_t mask, const F *__restrict__ dig,
                                                          const F *__restrict__ pre, uint32_t *__restrict__ nodes,
                                                          unsigned long long *err) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    F d = load_fe<F>(base + i);
    for (int depth = 0; depth < height; depth++) {
        const uint32_t x = find_node(table, mask, dig, d);
        if (x == NONE) { atomicMin(err, ((unsigned long long)i << 8) | (unsigned)depth); return; }
        nodes[(size_t)depth * n + i] = x;
        if (depth + 1 < height) d = load_fe<F>(pre + (size_t)x * ARITY + chunk_at(ops[i].path, height, depth));
    }
}

__global__ void group_flags_kernel(int m, const int16_t *__restrict__ lcp, int e, uint32_t *__restrict__ flags) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < m) flags[p] = p == 0 || lcp[p] < e;
}

__global__ void sort_keys_kernel(int m, const uint32_t *__restrict__ rank, const uint32_t *__restrict__ order, uint64_t *__restrict__ keys) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < m) keys[p] = ((uint64_t)rank[p] << 32) | order[p];
}

// (chain, path >> s, index) of a against b: -1, 0, 1
__device__ __forceinline__ int cmp_entry(const OpDev &a, uint32_t ja, uint32_t chain, const uint32_t *path, int s, int64_t idx) {
    if (a.chain != chain) return a.chain < chain ? -1 : 1;
    for (int w = 7; w >= (s >> 5); w--) {
        const uint32_t mk = w == (s >> 5) ? (0xffffffffu << (s & 31)) : 0xffffffffu;
        const uint32_t x = a.path[w] & mk, y = path[w] & mk;
        if (x != y) return x < y ? -1 : 1;
    }
    return (int64_t)ja < idx ? -1 : ((int64_t)ja == idx ? 0 : 1);
}

// thread (i, c): child c of operation i's node at depth d
template <class F>
__global__ void __launch_bounds__(TS_THREADS) level_kernel(int n, int height, int d, const OpDev *__restrict__ ops, const uint32_t *__restrict__ nodes,
                                                           const F *__restrict__ pre, const uint64_t *__restrict__ sorted, int m,
                                                           const F *__restrict__ child_dig, const F *__restrict__ vals, F *__restrict__ newpre,
                                                           F *__restrict__ results, uint8_t *lookup_out, uint8_t *insert_out, int fmt,
                                                           const unsigned long long *err) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)n * ARITY || *err != NO_ERR) return;
    const int i = (int)(t >> 3), c = (int)(t & 7);
    const OpDev &o = ops[i];
    const int own = chunk_at(o.path, height, d), lo = 3 * (height - 1 - d);
    F v = load_fe<F>(pre + (size_t)nodes[(size_t)d * n + i] * ARITY + c);
    // the target prefix: the operation's first d chunks, then c
    uint32_t target[8];
#pragma unroll
    for (int w = 0; w < 8; w++) target[w] = o.path[w];
    for (int q = 0; q < 3; q++) {
        const int b = lo + q;
        target[b >> 5] = (target[b >> 5] & ~(1u << (b & 31))) | ((uint32_t)((c >> q) & 1) << (b & 31));
    }
    if (o.bound >= 0) {
        int a = 0, z = m;   // first entry greater than (chain, target, bound)
        while (a < z) {
            const int mid = (a + z) >> 1;
            const uint32_t j = (uint32_t)sorted[mid];
            if (cmp_entry(ops[j], j, o.chain, target, lo, o.bound) <= 0) a = mid + 1;
            else z = mid;
        }
        if (a > 0) {
            const uint32_t j = (uint32_t)sorted[a - 1];
            const OpDev &q = ops[j];
            if (q.chain == o.chain && cmp_entry(q, 0, o.chain, target, lo, 0) == 0)
                v = d == height - 1 ? load_fe<F>(vals + j) : load_fe<F>(child_dig + q.rank);
        }
    }
    const size_t H = (size_t)height;
    if (o.kind == LURK_TRIE_LOOKUP) {
        if (lookup_out) store_fe(lookup_out + ((size_t)o.rank * (2 + 8 * H) + 2 + 8 * (size_t)d + c) * 32, out_fmt(v, fmt));
        if (d == height - 1 && c == own) store_fe(results + i, v);
        return;
    }
    const F nv = c != own ? v : (d == height - 1 ? load_fe<F>(vals + i) : load_fe<F>(child_dig + o.rank));
    store_fe(newpre + (size_t)o.rank * ARITY + c, nv);
    if (insert_out) {
        uint8_t *x = insert_out + (size_t)o.rank * (3 + 16 * H) * 32;
        store_fe(x + (3 + 8 * (size_t)d + c) * 32, out_fmt(v, fmt));
        store_fe(x + (3 + 8 * H + 8 * (size_t)d + c) * 32, out_fmt(nv, fmt));
    }
}

// registration, pass 1: each new digest probes the table; the first of equal new digests claims an empty slot with its
// own index, every other one (and any digest already stored) finds it there and is dropped
template <class F>
__global__ void __launch_bounds__(TS_THREADS) claim_kernel(int m, const F *__restrict__ fresh, uint32_t *table, uint64_t mask,
                                                           const F *__restrict__ dig, uint32_t *__restrict__ claim_at,
                                                           const unsigned long long *err) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= m || *err != NO_ERR) return;
    const F d = load_fe<F>(fresh + k);
    claim_at[k] = NONE;
    for (uint64_t h = slot_of(d.v, mask);; h = (h + 1) & mask) {
        uint32_t v = table[h];
        if (!v) {
            v = atomicCAS(table + h, 0u, CLAIM | (uint32_t)k);
            if (!v) { claim_at[k] = (uint32_t)h; return; }
        }
        const F x = (v & CLAIM) ? load_fe<F>(fresh + (v & ~CLAIM)) : load_fe<F>(dig + (v - 1));
        if (eq8(x.v, d.v)) return;
    }
}

// pass 2: every claim becomes a node
template <class F>
__global__ void __launch_bounds__(TS_THREADS) publish_kernel(int m, const F *__restrict__ fresh, const F *__restrict__ fresh_pre, uint32_t *table,
                                                             F *__restrict__ dig, F *__restrict__ pre, uint32_t *count,
                                                             const uint32_t *__restrict__ claim_at, const unsigned long long *err) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= m || *err != NO_ERR || claim_at[k] == NONE) return;
    const uint32_t x = atomicAdd(count, 1u);
    store_fe(dig + x, load_fe<F>(fresh + k));
    for (int c = 0; c < ARITY; c++) store_fe(pre + (size_t)x * ARITY + c, load_fe<F>(fresh_pre + (size_t)k * ARITY + c));
    table[claim_at[k]] = x + 1;
}

template <class F>
__global__ void __launch_bounds__(TS_THREADS) finish_kernel(int n, int height, const OpDev *__restrict__ ops, const F *__restrict__ base,
                                                            const F *__restrict__ keys, const F *__restrict__ vals, const F *__restrict__ dig0,
                                                            F *__restrict__ results, uint8_t *lookup_out, uint8_t *insert_out, int fmt,
                                                            const unsigned long long *err) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || *err != NO_ERR) return;
    const OpDev &o = ops[i];
    const F root = o.prev < 0 ? load_fe<F>(base + i) : load_fe<F>(dig0 + ops[o.prev].rank);
    const size_t H = (size_t)height;
    uint8_t *x = o.kind == LURK_TRIE_LOOKUP ? (lookup_out ? lookup_out + (size_t)o.rank * (2 + 8 * H) * 32 : nullptr)
                                            : (insert_out ? insert_out + (size_t)o.rank * (3 + 16 * H) * 32 : nullptr);
    if (x) {
        store_fe(x, out_fmt(root, fmt));
        store_fe(x + 32, out_fmt(load_fe<F>(keys + i), fmt));
        if (o.kind == LURK_TRIE_INSERT) store_fe(x + 64, out_fmt(load_fe<F>(vals + i), fmt));
    }
    store_fe(results + i, out_fmt(o.kind == LURK_TRIE_INSERT ? load_fe<F>(dig0 + o.rank) : load_fe<F>(results + i), fmt));
}

__global__ void fill8_kernel(uint8_t *pre, const uint8_t *d) {
    const int i = threadIdx.x;
    if (i < ARITY * 32) pre[i] = d[i & 31];
}

// ---- planning on the device (lurk_trie_ctx_apply_dev): the same OpDev array, bases, canonical keys and values, insert
// order and lcp that plan_batch builds on the host.  Per-operation refusals go into one 64-bit word as (i << 8) | code,
// the lowest operation winning, and the codes of one operation in the order plan_batch checks them.
enum PlanErr : unsigned { PE_KIND = 1, PE_PREV, PE_PREV_LOOKUP, PE_FORK, PE_ROOTS_NULL, PE_VALUES_NULL, PE_ROOT, PE_KEY, PE_VALUE };

struct PlanStatus {
    unsigned long long err;
    uint32_t inserts, cap_first;   // m, and the operation of insert rank `fits` (NONE: there is none)
};

// first[j]: the lowest insert with prev = j.  Once every earlier operation is valid the inserts of a chain form a list,
// so an insert i with prev = j is plan_batch's fork (latest[chain] != j) exactly when first[j] != i.
__global__ void first_continuer_kernel(int n, const int32_t *__restrict__ kinds, const int64_t *__restrict__ prev, uint32_t *first) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t j = prev[i];
    if (kinds[i] == LURK_TRIE_INSERT && j >= 0 && j < i) atomicMin(first + j, (uint32_t)i);
}

// one operation: checks, canonical key / value / root, masked path, bound; link[i] = a valid prev, else i (the chain's
// head after pointer jumping); flags[i] = 1 for an insert
template <class F>
__global__ void __launch_bounds__(TS_THREADS) validate_kernel(int n, int height, const int32_t *__restrict__ kinds, const int64_t *__restrict__ prev,
                                                              const F *__restrict__ roots, const F *__restrict__ keys_in, const F *__restrict__ vals_in,
                                                              int fmt, const uint32_t *__restrict__ first, OpDev *__restrict__ ops, F *__restrict__ base,
                                                              F *__restrict__ keys, F *__restrict__ vals, uint32_t *__restrict__ link,
                                                              uint32_t *__restrict__ flags, PlanStatus *status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int k = kinds[i];
    const int64_t j = prev[i];
    const bool ins = k == LURK_TRIE_INSERT;
    link[i] = j >= 0 && j < i ? (uint32_t)j : (uint32_t)i;
    flags[i] = ins;
    unsigned code = 0;
    F root = F::zero(), key = F::zero(), val = F::zero();
    if (k != LURK_TRIE_LOOKUP && !ins) code = PE_KIND;
    else if (j < -1 || j >= i) code = PE_PREV;
    else if (j >= 0 && kinds[j] != LURK_TRIE_INSERT) code = PE_PREV_LOOKUP;
    else if (ins && j >= 0 && first[j] != (uint32_t)i) code = PE_FORK;
    else if (j < 0 && !roots) code = PE_ROOTS_NULL;
    else if (ins && !vals_in) code = PE_VALUES_NULL;
    else {
        if (j < 0) root = load_fe<F>(roots + i);
        key = load_fe<F>(keys_in + i);
        if (ins) val = load_fe<F>(vals_in + i);
        if (j < 0 && !root.is_reduced()) code = PE_ROOT;
        else if (!key.is_reduced()) code = PE_KEY;
        else if (!val.is_reduced()) code = PE_VALUE;
    }
    if (code) { atomicMin(&status->err, ((unsigned long long)i << 8) | code); return; }
    if (fmt == LURK_FMT_MONTGOMERY) { root = root.to_canonical(); key = key.to_canonical(); val = val.to_canonical(); }
    OpDev o{};
    o.kind = (uint32_t)k;
    o.prev = (int32_t)j;
    o.bound = ins ? i - 1 : (int32_t)j;
    const int bits = 3 * height;   // the path is the key's low 3H bits
#pragma unroll
    for (int w = 0; w < 8; w++) {
        const int lo = 32 * w;
        o.path[w] = lo >= bits ? 0u : (bits - lo < 32 ? key.v[w] & ((1u << (bits - lo)) - 1) : key.v[w]);
    }
    ops[i] = o;   // chain and rank follow in chain_rank_kernel
    store_fe(base + i, root);
    store_fe(keys + i, key);
    store_fe(vals + i, val);
}

// one round of pointer jumping over prev
__global__ void jump_kernel(int n, const uint32_t *__restrict__ in, uint32_t *__restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[in[i]];
}

// chain, base root from the chain's head, rank (incl: inclusive scan of the insert flags); the inserts in index order
// go to order[rank].  Nothing is planned further once an operation is refused.
template <class F>
__global__ void __launch_bounds__(TS_THREADS) chain_rank_kernel(int n, const uint32_t *__restrict__ head, const uint32_t *__restrict__ incl,
                                                                uint64_t fits, OpDev *ops, F *base, uint32_t *__restrict__ order,
                                                                PlanStatus *status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || status->err != NO_ERR) return;
    OpDev &o = ops[i];
    const uint32_t c = head[i];
    o.chain = c;
    if (o.prev >= 0) store_fe(base + i, load_fe<F>(base + c));   // a chain's head has prev = -1 and is not written here
    if (o.kind == LURK_TRIE_INSERT) {
        o.rank = incl[i] - 1;
        order[o.rank] = (uint32_t)i;
        if (o.rank == fits) status->cap_first = (uint32_t)i;
    } else {
        o.rank = (uint32_t)i - incl[i];
    }
    if (i == n - 1) status->inserts = incl[i];
}

// the sort key of one least-significant-first pass: path word w (0..7), then the chain (w = 8)
__global__ void order_key_kernel(int m, const OpDev *__restrict__ ops, const uint32_t *__restrict__ order, int w, uint32_t *__restrict__ key) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    const OpDev &o = ops[order[p]];
    key[p] = w < 8 ? o.path[w] : o.chain;
}

// plan_batch's lcp: common leading chunks of order[p - 1] and order[p], -1 across chains
__global__ void lcp_kernel(int m, int height, const OpDev *__restrict__ ops, const uint32_t *__restrict__ order, int16_t *__restrict__ lcp) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    if (p == 0) { lcp[0] = 0; return; }
    const OpDev &a = ops[order[p - 1]], &b = ops[order[p]];
    if (a.chain != b.chain) { lcp[p] = -1; return; }
    int hi = -1;   // the highest differing bit
    for (int w = 7; w >= 0 && hi < 0; w--) {
        const uint32_t x = a.path[w] ^ b.path[w];
        if (x) hi = 32 * w + 31 - __clz(x);
    }
    lcp[p] = (int16_t)(hi < 0 ? height : height - 1 - hi / 3);
}

// register_dev's input: canonical preimages, and the lowest unreduced element's index in *bad
template <class F>
__global__ void __launch_bounds__(TS_THREADS) canon_check_kernel(size_t n, const F *__restrict__ in, int fmt, F *__restrict__ out,
                                                                 unsigned long long *bad) {
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const F x = load_fe<F>(in + e);
    if (!x.is_reduced()) { atomicMin(bad, (unsigned long long)e); return; }
    store_fe(out + e, fmt == LURK_FMT_MONTGOMERY ? x.to_canonical() : x);
}

unsigned blocks(size_t n) { return (unsigned)((n + TS_THREADS - 1) / TS_THREADS); }

// a 256-byte aligned bump allocator over one device buffer
struct Carve {
    uint8_t *base;
    size_t used = 0;
    template <class T>
    T *take(size_t n) {
        T *p = reinterpret_cast<T *>(base ? base + used : nullptr);
        used += (n * sizeof(T) + 255) & ~(size_t)255;
        return p;
    }
};

template <class F>
bool reduced(const uint8_t *x) {
    for (int w = 7; w >= 0; w--) {
        uint32_t v;
        memcpy(&v, x + 4 * w, 4);
        const uint32_t p = F::Params::MOD(w);
        if (v != p) return v < p;
    }
    return false;
}

template <class F>
void to_canonical_host(const uint8_t *x, int fmt, uint8_t *out) {
    F v;
    memcpy(v.v, x, 32);
    if (fmt == LURK_FMT_MONTGOMERY) v = v.to_canonical();
    memcpy(out, v.v, 32);
}

}  // namespace
}  // namespace lurk

using namespace lurk;

struct lurk_trie_ctx {
    int field_id, height;
    uint64_t capacity, count = 0, mask = 0;
    int device = -1;
    uint8_t empty_root[32] = {};
    DevBuf table, dig, pre, dcount, err, plan, scratch;   // plan: one batch's plan (and its planner's scratch); scratch: its levels
};

namespace lurk {
namespace {

// register m canonical preimages already on the device (d_pre, m x 8) whose digests go to d_fresh; asynchronous
template <class F>
int register_dev(lurk_trie_ctx *ctx, const F *d_pre, F *d_fresh, uint32_t *d_claim, int m, cudaStream_t st) {
    if (!m) return LURK_OK;
    LURK_TRY((launch_poseidon<F, false>(ARITY, d_pre, (size_t)m, d_fresh, LURK_FMT_CANONICAL, LURK_FMT_CANONICAL, st)));
    claim_kernel<F><<<blocks(m), TS_THREADS, 0, st>>>(m, d_fresh, ctx->table.as<uint32_t>(), ctx->mask, ctx->dig.as<F>(), d_claim,
                                                      ctx->err.as<unsigned long long>());
    publish_kernel<F><<<blocks(m), TS_THREADS, 0, st>>>(m, d_fresh, d_pre, ctx->table.as<uint32_t>(), ctx->dig.as<F>(), ctx->pre.as<F>(),
                                                        ctx->dcount.as<uint32_t>(), d_claim, ctx->err.as<unsigned long long>());
    LURK_CUDA_TRY(cudaGetLastError());
    return LURK_OK;
}

int sync_count(lurk_trie_ctx *ctx, cudaStream_t st) {
    uint32_t c = 0;
    LURK_CUDA_TRY(cudaMemcpyAsync(&c, ctx->dcount.p, 4, cudaMemcpyDeviceToHost, st));
    LURK_CUDA_TRY(cudaStreamSynchronize(st));
    ctx->count = c;
    return LURK_OK;
}

int ensure(DevBuf &b, size_t bytes) {
    if (b.bytes >= bytes) return LURK_OK;
    LURK_CUDA_TRY(cudaDeviceSynchronize());   // the old buffer may still be read by an earlier call's stream
    return b.alloc(bytes);
}

template <class F>
int build_store(lurk_trie_ctx *ctx) {
    LURK_CUDA_TRY(cudaGetDevice(&ctx->device));
    uint64_t slots = 1;
    while (slots < 2 * ctx->capacity) slots <<= 1;
    ctx->mask = slots - 1;
    LURK_TRY(ctx->table.alloc(slots * 4));
    LURK_TRY(ctx->dig.alloc(ctx->capacity * 32));
    LURK_TRY(ctx->pre.alloc(ctx->capacity * 32 * ARITY));
    LURK_TRY(ctx->dcount.alloc(4));
    LURK_TRY(ctx->err.alloc(8));
    LURK_CUDA_TRY(cudaMemset(ctx->table.p, 0, ctx->table.bytes));
    LURK_CUDA_TRY(cudaMemset(ctx->dcount.p, 0, 4));
    LURK_CUDA_TRY(cudaMemset(ctx->err.p, 0xff, 8));
    // the H empty roots: level h's preimage is 8 copies of level h - 1's digest, level 0 the empty element 0
    DevBuf b;
    LURK_TRY(b.alloc(32 * ARITY + 32 + 32 + 4));
    uint8_t *p = b.as<uint8_t>(), *d = p + 32 * ARITY, *zero = d + 32;
    LURK_CUDA_TRY(cudaMemset(zero, 0, 32));
    const uint8_t *prev = zero;
    for (int h = 0; h < ctx->height; h++) {
        fill8_kernel<<<1, 256>>>(p, prev);
        LURK_TRY(register_dev<F>(ctx, (const F *)p, (F *)d, (uint32_t *)(zero + 32), 1, 0));
        LURK_CUDA_TRY(cudaMemcpy(zero, d, 32, cudaMemcpyDeviceToDevice));
        prev = zero;
    }
    LURK_CUDA_TRY(cudaMemcpy(ctx->empty_root, zero, 32, cudaMemcpyDeviceToHost));
    return sync_count(ctx, 0);
}

// the host side of one batch: argument checks, chains, ranks and the inserts' (chain, path) order
struct Plan {
    std::vector<OpDev> ops;
    std::vector<uint8_t> base, keys, vals;   // canonical, n x 32
    std::vector<uint32_t> order;             // the inserts sorted by (chain, path, index)
    std::vector<int16_t> lcp;                // common leading chunks of order[p - 1] and order[p]; -1 across chains
    int inserts = 0, lookups = 0;
};

template <class F>
int plan_batch(const lurk_trie_ctx *ctx, size_t n, const int *kinds, const int64_t *prev, const uint8_t *roots, const uint8_t *keys,
               const uint8_t *values, int fmt, Plan &P) {
    const int H = ctx->height;
    P.ops.assign(n, OpDev{});
    P.base.assign(n * 32, 0);
    P.keys.assign(n * 32, 0);
    P.vals.assign(n * 32, 0);
    std::vector<int64_t> latest(n, -1);   // per chain: its last insert so far
    for (size_t i = 0; i < n; i++) {
        OpDev &o = P.ops[i];
        const int k = kinds[i];
        if (k != LURK_TRIE_LOOKUP && k != LURK_TRIE_INSERT) { set_error("trie operation %zu: kind %d is neither LURK_TRIE_LOOKUP nor LURK_TRIE_INSERT", i, k); return LURK_ERR_ARG; }
        const int64_t j = prev[i];
        if (j < -1 || j >= (int64_t)i) { set_error("trie operation %zu: prev %lld is not -1 or an earlier operation", i, (long long)j); return LURK_ERR_ARG; }
        if (j >= 0 && kinds[j] != LURK_TRIE_INSERT) { set_error("trie operation %zu: prev %lld is a lookup, not an insert", i, (long long)j); return LURK_ERR_ARG; }
        o.kind = (uint32_t)k;
        o.prev = (int32_t)j;
        o.chain = j < 0 ? (uint32_t)i : P.ops[j].chain;
        if (k == LURK_TRIE_INSERT) {
            if (j >= 0 && latest[o.chain] != j) {
                set_error("trie operation %zu: insert after insert %lld, which insert %lld already continued (a fork inside a batch)", i, (long long)j,
                          (long long)latest[o.chain]);
                return LURK_ERR_ARG;
            }
            latest[o.chain] = (int64_t)i;
            o.bound = (int32_t)i - 1;
            o.rank = (uint32_t)P.inserts++;
        } else {
            o.bound = (int32_t)j;
            o.rank = (uint32_t)P.lookups++;
        }
        if (j < 0 && !roots) { set_error("trie operation %zu: prev -1 names roots[%zu], but roots is NULL", i, i); return LURK_ERR_ARG; }
        if (k == LURK_TRIE_INSERT && !values) { set_error("trie operation %zu: an insert reads values[%zu], but values is NULL", i, i); return LURK_ERR_ARG; }
        const uint8_t *root = j < 0 ? roots + i * 32 : nullptr;
        if ((root && !reduced<F>(root)) || !reduced<F>(keys + i * 32) || (k == LURK_TRIE_INSERT && !reduced<F>(values + i * 32))) {
            set_error("trie operation %zu: an element (%s) is not reduced below the field modulus", i, root && !reduced<F>(root) ? "root" : (!reduced<F>(keys + i * 32) ? "key" : "value"));
            return LURK_ERR_ARG;
        }
        if (root) to_canonical_host<F>(root, fmt, &P.base[i * 32]);
        else memcpy(&P.base[i * 32], &P.base[(size_t)o.chain * 32], 32);
        to_canonical_host<F>(keys + i * 32, fmt, &P.keys[i * 32]);
        if (k == LURK_TRIE_INSERT) to_canonical_host<F>(values + i * 32, fmt, &P.vals[i * 32]);
        memcpy(o.path, &P.keys[i * 32], 32);
        const int bits = 3 * H;   // the path is the key's low 3H bits
        for (int w = 0; w < 8; w++) {
            const int lo = 32 * w;
            if (lo >= bits) o.path[w] = 0;
            else if (bits - lo < 32) o.path[w] &= (1u << (bits - lo)) - 1;
        }
    }
    if ((uint64_t)P.inserts * H > ctx->capacity - ctx->count) {
        // the first insert whose H new nodes would not fit
        const uint64_t fits = (ctx->capacity - ctx->count) / (uint64_t)H;
        size_t first = 0;
        for (size_t i = 0; i < n; i++)
            if (P.ops[i].kind == LURK_TRIE_INSERT && P.ops[i].rank == fits) { first = i; break; }
        set_error("trie operation %zu: insert %llu of the batch may add nodes past the capacity: %d inserts may add %llu nodes to a "
                  "store of %llu nodes and capacity %llu", first, (unsigned long long)fits, P.inserts, (unsigned long long)P.inserts * H,
                  (unsigned long long)ctx->count, (unsigned long long)ctx->capacity);
        return LURK_ERR_ARG;
    }
    P.order.clear();
    for (size_t i = 0; i < n; i++) if (P.ops[i].kind == LURK_TRIE_INSERT) P.order.push_back((uint32_t)i);
    auto path_less = [](const OpDev &a, const OpDev &b) {
        for (int w = 7; w >= 0; w--) if (a.path[w] != b.path[w]) return a.path[w] < b.path[w];
        return false;
    };
    std::sort(P.order.begin(), P.order.end(), [&](uint32_t x, uint32_t y) {
        const OpDev &a = P.ops[x], &b = P.ops[y];
        if (a.chain != b.chain) return a.chain < b.chain;
        if (path_less(a, b)) return true;
        if (path_less(b, a)) return false;
        return x < y;
    });
    P.lcp.assign(P.order.size(), 0);
    for (size_t p = 1; p < P.order.size(); p++) {
        const OpDev &a = P.ops[P.order[p - 1]], &b = P.ops[P.order[p]];
        if (a.chain != b.chain) { P.lcp[p] = -1; continue; }
        int hi = -1;   // the highest differing bit
        for (int w = 7; w >= 0 && hi < 0; w--) {
            const uint32_t x = a.path[w] ^ b.path[w];
            if (x) hi = 32 * w + 31 - __builtin_clz(x);
        }
        P.lcp[p] = (int16_t)(hi < 0 ? H : H - 1 - hi / 3);
    }
    return LURK_OK;
}

// one batch's plan in device memory: the host planner's upload or the device planner's output.  order and lcp hold the
// m inserts; the rest of the arrays n entries.  The device planner's own scratch follows them.
template <class F>
struct DevPlan {
    OpDev *ops;
    F *base, *keys, *vals;
    uint32_t *order;
    int16_t *lcp;
    uint32_t *first, *link_a, *link_b, *flags, *incl, *key_a, *key_b, *order_b;
    PlanStatus *status;
    void *tmp;
    size_t tmp_bytes = 0;
};

template <class F>
int take_plan(lurk_trie_ctx *ctx, int n, bool planner, cudaStream_t st, DevPlan<F> &D) {
    if (planner) {   // CUB scratch for one scan of n flags and one stable 32-bit key-value sort of up to n inserts
        size_t scan_bytes = 0, sort_bytes = 0;
        cub::DoubleBuffer<uint32_t> k(nullptr, nullptr), v(nullptr, nullptr);
        LURK_CUDA_TRY(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (const uint32_t *)nullptr, (uint32_t *)nullptr, n, st));
        LURK_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, k, v, n, 0, 32, st));
        D.tmp_bytes = std::max(scan_bytes, sort_bytes);
    }
    auto lay = [&](Carve &c) {
        D.ops = c.take<OpDev>(n); D.base = c.take<F>(n); D.keys = c.take<F>(n); D.vals = c.take<F>(n);
        D.order = c.take<uint32_t>(n); D.lcp = c.take<int16_t>(n);
        if (!planner) return;
        D.first = c.take<uint32_t>(n); D.link_a = c.take<uint32_t>(n); D.link_b = c.take<uint32_t>(n); D.flags = c.take<uint32_t>(n);
        D.incl = c.take<uint32_t>(n); D.key_a = c.take<uint32_t>(n); D.key_b = c.take<uint32_t>(n); D.order_b = c.take<uint32_t>(n);
        D.status = c.take<PlanStatus>(1); D.tmp = c.take<uint8_t>(D.tmp_bytes);
    };
    Carve probe{nullptr};
    lay(probe);
    LURK_TRY(ensure(ctx->plan, probe.used));
    Carve c{ctx->plan.as<uint8_t>()};
    lay(c);
    return LURK_OK;
}

// the device planner: n operations in device memory -> D and m, or the refusal plan_batch would give (LURK_ERR_ARG,
// naming the same operation).  One read of the status word, after the ranks; the inserts are ordered only once the
// batch is known to be accepted.
template <class F>
int plan_dev(lurk_trie_ctx *ctx, int n, const int32_t *kinds, const int64_t *prev, const F *roots, const F *keys, const F *values,
             int fmt, cudaStream_t st, DevPlan<F> &D, int &m) {
    const int H = ctx->height;
    LURK_TRY(take_plan<F>(ctx, n, true, st, D));
    LURK_CUDA_TRY(cudaMemsetAsync(D.status, 0xff, sizeof(PlanStatus), st));
    LURK_CUDA_TRY(cudaMemsetAsync(D.first, 0xff, (size_t)n * 4, st));
    first_continuer_kernel<<<blocks(n), TS_THREADS, 0, st>>>(n, kinds, prev, D.first);
    validate_kernel<F><<<blocks(n), TS_THREADS, 0, st>>>(n, H, kinds, prev, roots, keys, values, fmt, D.first, D.ops, D.base, D.keys, D.vals,
                                                         D.link_a, D.flags, D.status);
    LURK_CUDA_TRY(cudaGetLastError());
    uint32_t *head = D.link_a, *spare = D.link_b;
    for (int r = 0; (1ll << r) < n; r++) {   // ceil(log2 n) rounds: every chain is shorter than n
        jump_kernel<<<blocks(n), TS_THREADS, 0, st>>>(n, head, spare);
        std::swap(head, spare);
    }
    size_t tb = D.tmp_bytes;
    LURK_CUDA_TRY(cub::DeviceScan::InclusiveSum(D.tmp, tb, D.flags, D.incl, n, st));
    const uint64_t fits = (ctx->capacity - ctx->count) / (uint64_t)H;
    chain_rank_kernel<F><<<blocks(n), TS_THREADS, 0, st>>>(n, head, D.incl, fits, D.ops, D.base, D.order, D.status);
    LURK_CUDA_TRY(cudaGetLastError());
    PlanStatus s;
    LURK_CUDA_TRY(cudaMemcpyAsync(&s, D.status, sizeof s, cudaMemcpyDeviceToHost, st));
    LURK_CUDA_TRY(cudaStreamSynchronize(st));
    if (s.err != NO_ERR) {
        const size_t i = (size_t)(s.err >> 8);
        int32_t k = 0;
        int64_t j = 0;
        LURK_CUDA_TRY(cudaMemcpy(&k, kinds + i, 4, cudaMemcpyDeviceToHost));
        LURK_CUDA_TRY(cudaMemcpy(&j, prev + i, 8, cudaMemcpyDeviceToHost));
        switch ((unsigned)(s.err & 0xff)) {
        case PE_KIND: set_error("trie operation %zu: kind %d is neither LURK_TRIE_LOOKUP nor LURK_TRIE_INSERT", i, k); break;
        case PE_PREV: set_error("trie operation %zu: prev %lld is not -1 or an earlier operation", i, (long long)j); break;
        case PE_PREV_LOOKUP: set_error("trie operation %zu: prev %lld is a lookup, not an insert", i, (long long)j); break;
        case PE_FORK: {
            uint32_t f = 0;
            LURK_CUDA_TRY(cudaMemcpy(&f, D.first + j, 4, cudaMemcpyDeviceToHost));
            set_error("trie operation %zu: insert after insert %lld, which insert %u already continued (a fork inside a batch)", i, (long long)j, f);
            break;
        }
        case PE_ROOTS_NULL: set_error("trie operation %zu: prev -1 names roots[%zu], but roots is NULL", i, i); break;
        case PE_VALUES_NULL: set_error("trie operation %zu: an insert reads values[%zu], but values is NULL", i, i); break;
        default: {
            const unsigned c = (unsigned)(s.err & 0xff);
            set_error("trie operation %zu: an element (%s) is not reduced below the field modulus", i, c == PE_ROOT ? "root" : (c == PE_KEY ? "key" : "value"));
        }
        }
        return LURK_ERR_ARG;
    }
    m = (int)s.inserts;
    if ((uint64_t)m * H > ctx->capacity - ctx->count) {
        set_error("trie operation %u: insert %llu of the batch may add nodes past the capacity: %d inserts may add %llu nodes to a "
                  "store of %llu nodes and capacity %llu", s.cap_first, (unsigned long long)fits, m, (unsigned long long)m * H,
                  (unsigned long long)ctx->count, (unsigned long long)ctx->capacity);
        return LURK_ERR_ARG;
    }
    if (m > 1) {
        // stable least-significant-first passes: path word 0 .. the key's top word, then the chain -> (chain, path, index)
        const int bits = 3 * H, chain_bits = 32 - __builtin_clz((unsigned)(n - 1));
        cub::DoubleBuffer<uint32_t> key(D.key_a, D.key_b), ord(D.order, D.order_b);
        for (int w = 0; w <= 8; w++) {
            if (w < 8 && 32 * w >= bits) continue;
            order_key_kernel<<<blocks(m), TS_THREADS, 0, st>>>(m, D.ops, ord.Current(), w, key.Current());
            tb = D.tmp_bytes;
            LURK_CUDA_TRY(cub::DeviceRadixSort::SortPairs(D.tmp, tb, key, ord, m, 0, w < 8 ? std::min(32, bits - 32 * w) : chain_bits, st));
        }
        D.order = ord.Current();
    }
    if (m) lcp_kernel<<<blocks(m), TS_THREADS, 0, st>>>(m, H, D.ops, D.order, D.lcp);
    LURK_CUDA_TRY(cudaGetLastError());
    return LURK_OK;
}

// the levels of one planned batch (steps 1-3 above), shared by both forms.  Results go to d_results (device, n elements
// in fmt) when it is given, else to results_out (host, may be NULL).
template <class F>
int run_levels(lurk_trie_ctx *ctx, int n, int m, const DevPlan<F> &D, F *d_results, uint8_t *results_out, void *d_lookup, void *d_insert,
               int fmt, cudaStream_t st) {
    const int H = ctx->height;
    const OpDev *ops = D.ops;
    const F *base = D.base, *keys = D.keys, *vals = D.vals;
    const uint32_t *order = D.order;
    const int16_t *lcp = D.lcp;
    // CUB scratch for one scan and one sort of m keys
    size_t scan_bytes = 0, sort_bytes = 0;
    const int rank_bits = 33 - (m ? __builtin_clz((unsigned)m) : 32);
    if (m) {
        LURK_CUDA_TRY(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (const uint32_t *)nullptr, (uint32_t *)nullptr, m, st));
        LURK_CUDA_TRY(cub::DeviceRadixSort::SortKeys(nullptr, sort_bytes, (const uint64_t *)nullptr, (uint64_t *)nullptr, m, 0, 32 + rank_bits, st));
    }
    Carve cv{nullptr};
    auto lay = [&](Carve &c, F *&res, uint32_t *&nodes, uint32_t *&flags, uint32_t *&rank, uint64_t *&kin, uint64_t *&kout, F *&dig_a,
                   F *&dig_b, F *&newpre, uint32_t *&claim, void *&tmp) {
        res = c.take<F>(n); nodes = c.take<uint32_t>((size_t)n * H); flags = c.take<uint32_t>(m); rank = c.take<uint32_t>(m);
        kin = c.take<uint64_t>(m); kout = c.take<uint64_t>(m); dig_a = c.take<F>(m); dig_b = c.take<F>(m);
        newpre = c.take<F>((size_t)m * ARITY); claim = c.take<uint32_t>(m); tmp = c.take<uint8_t>(std::max(scan_bytes, sort_bytes));
    };
    F *res, *dig_a, *dig_b, *newpre; uint32_t *nodes, *flags, *rank, *claim;
    uint64_t *kin, *kout; void *tmp;
    lay(cv, res, nodes, flags, rank, kin, kout, dig_a, dig_b, newpre, claim, tmp);
    LURK_TRY(ensure(ctx->scratch, cv.used));
    Carve c{ctx->scratch.as<uint8_t>()};
    lay(c, res, nodes, flags, rank, kin, kout, dig_a, dig_b, newpre, claim, tmp);
    if (d_results) res = d_results;   // written only once the walk found every node
    const size_t tmp_bytes = std::max(scan_bytes, sort_bytes);
    auto *err = ctx->err.as<unsigned long long>();
    LURK_CUDA_TRY(cudaMemsetAsync(err, 0xff, 8, st));

    walk_kernel<F><<<blocks(n), TS_THREADS, 0, st>>>(n, H, ops, base, ctx->table.as<uint32_t>(), ctx->mask, ctx->dig.as<F>(), ctx->pre.as<F>(),
                                                     nodes, err);
    LURK_CUDA_TRY(cudaGetLastError());
    F *child = dig_b, *cur = dig_a;   // the digests of the inserts' new nodes at depth d + 1 and d
    for (int d = H - 1; d >= 0; d--) {
        if (m) {
            group_flags_kernel<<<blocks(m), TS_THREADS, 0, st>>>(m, lcp, d + 1, flags);
            LURK_CUDA_TRY(cub::DeviceScan::InclusiveSum(tmp, scan_bytes, flags, rank, m, st));
            sort_keys_kernel<<<blocks(m), TS_THREADS, 0, st>>>(m, rank, order, kin);
            size_t sb = tmp_bytes;
            LURK_CUDA_TRY(cub::DeviceRadixSort::SortKeys(tmp, sb, kin, kout, m, 0, 32 + rank_bits, st));
        }
        level_kernel<F><<<blocks((size_t)n * ARITY), TS_THREADS, 0, st>>>(n, H, d, ops, nodes, ctx->pre.as<F>(), kout, m, child, vals, newpre, res,
                                                                         (uint8_t *)d_lookup, (uint8_t *)d_insert, fmt, err);
        LURK_CUDA_TRY(cudaGetLastError());
        LURK_TRY(register_dev<F>(ctx, newpre, cur, claim, m, st));
        std::swap(child, cur);
    }
    finish_kernel<F><<<blocks(n), TS_THREADS, 0, st>>>(n, H, ops, base, keys, vals, child, res, (uint8_t *)d_lookup, (uint8_t *)d_insert, fmt, err);
    LURK_CUDA_TRY(cudaGetLastError());
    unsigned long long e = NO_ERR;
    LURK_CUDA_TRY(cudaMemcpyAsync(&e, err, 8, cudaMemcpyDeviceToHost, st));
    LURK_TRY(sync_count(ctx, st));
    if (e != NO_ERR) {
        // the first operation whose walk missed a digest: its base root, or the child its parent node selects
        const int i = (int)(e >> 8), depth = (int)(e & 0xff);
        uint8_t miss[32];
        if (depth == 0) LURK_CUDA_TRY(cudaMemcpy(miss, base + i, 32, cudaMemcpyDeviceToHost));
        else {
            uint32_t parent = 0;
            OpDev o;
            LURK_CUDA_TRY(cudaMemcpy(&parent, nodes + (size_t)(depth - 1) * n + i, 4, cudaMemcpyDeviceToHost));
            LURK_CUDA_TRY(cudaMemcpy(&o, ops + i, sizeof o, cudaMemcpyDeviceToHost));
            LURK_CUDA_TRY(cudaMemcpy(miss, ctx->pre.as<F>() + (size_t)parent * ARITY + chunk_at(o.path, H, depth - 1), 32,
                                     cudaMemcpyDeviceToHost));
        }
        char hex[65];
        for (int b = 0; b < 32; b++) snprintf(hex + 2 * b, 3, "%02x", miss[31 - b]);
        set_error("trie operation %d: MissingPreimage(0x%s) at depth %d (%s)", i, hex, depth, depth ? "a node on the key's path" : "its root");
        return LURK_ERR_RANGE;
    }
    if (results_out) LURK_CUDA_TRY(cudaMemcpy(results_out, res, (size_t)n * 32, cudaMemcpyDeviceToHost));
    return LURK_OK;
}

// the host form: upload plan_batch's plan, then the levels
template <class F>
int apply_batch(lurk_trie_ctx *ctx, const Plan &P, uint8_t *results_out, void *d_lookup, void *d_insert, int fmt, cudaStream_t st) {
    const int n = (int)P.ops.size(), m = P.inserts;
    DevPlan<F> D;
    LURK_TRY(take_plan<F>(ctx, n, false, st, D));
    LURK_CUDA_TRY(cudaMemcpyAsync(D.ops, P.ops.data(), (size_t)n * sizeof(OpDev), cudaMemcpyHostToDevice, st));
    LURK_CUDA_TRY(cudaMemcpyAsync(D.base, P.base.data(), (size_t)n * 32, cudaMemcpyHostToDevice, st));
    LURK_CUDA_TRY(cudaMemcpyAsync(D.keys, P.keys.data(), (size_t)n * 32, cudaMemcpyHostToDevice, st));
    LURK_CUDA_TRY(cudaMemcpyAsync(D.vals, P.vals.data(), (size_t)n * 32, cudaMemcpyHostToDevice, st));
    if (m) {
        LURK_CUDA_TRY(cudaMemcpyAsync(D.order, P.order.data(), (size_t)m * 4, cudaMemcpyHostToDevice, st));
        LURK_CUDA_TRY(cudaMemcpyAsync(D.lcp, P.lcp.data(), (size_t)m * 2, cudaMemcpyHostToDevice, st));
    }
    return run_levels<F>(ctx, n, m, D, nullptr, results_out, d_lookup, d_insert, fmt, st);
}

int ctx_ready(lurk_trie_ctx *ctx) {
    LURK_TRY(require_gpu());
    if (ctx->device >= 0) return LURK_OK;
    return dispatch_field(ctx->field_id, [&](auto f) { return build_store<decltype(f)>(ctx); });
}

}  // namespace
}  // namespace lurk

extern "C" {

int lurk_trie_ctx_create(int field_id, int height, uint64_t capacity_nodes, lurk_trie_ctx **out) {
    if (!out) { set_error("null output"); return LURK_ERR_ARG; }
    *out = nullptr;
    if (field_id < LURK_FIELD_BN254_FR || field_id > LURK_FIELD_PALLAS_FP) { set_error("unknown field id %d", field_id); return LURK_ERR_ARG; }
    if (height < 1 || height > LURK_TRIE_MAX_HEIGHT) { set_error("trie height %d: 1..%d", height, LURK_TRIE_MAX_HEIGHT); return LURK_ERR_ARG; }
    if (capacity_nodes < (uint64_t)height || capacity_nodes >= CLAIM) {
        set_error("trie capacity %llu: at least the height's %d empty roots, below 2^31", (unsigned long long)capacity_nodes, height);
        return LURK_ERR_ARG;
    }
    auto *ctx = new lurk_trie_ctx;
    ctx->field_id = field_id;
    ctx->height = height;
    ctx->capacity = capacity_nodes;
    ctx->count = (uint64_t)height;   // the empty roots, registered when the store is built
    if (lurk_device_count() > 0) {
        const int rc = ctx_ready(ctx);
        if (rc != LURK_OK) { delete ctx; return rc; }
    }
    *out = ctx;
    return LURK_OK;
}

void lurk_trie_ctx_destroy(lurk_trie_ctx *ctx) { delete ctx; }

int lurk_trie_ctx_info(const lurk_trie_ctx *ctx, uint64_t *node_count, uint64_t *capacity) {
    if (!ctx) { set_error("null trie context"); return LURK_ERR_ARG; }
    if (node_count) *node_count = ctx->count;
    if (capacity) *capacity = ctx->capacity;
    return LURK_OK;
}

int lurk_trie_ctx_empty_root(lurk_trie_ctx *ctx, uint8_t out[32], int fmt) {
    if (!ctx || !out) { set_error("null trie context or output"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    LURK_TRY(ctx_ready(ctx));
    return dispatch_field(ctx->field_id, [&](auto f) {
        using F = decltype(f);
        F v;
        memcpy(v.v, ctx->empty_root, 32);
        if (fmt == LURK_FMT_MONTGOMERY) v = F::from_canonical(v);
        memcpy(out, v.v, 32);
        return LURK_OK;
    });
}

int lurk_trie_ctx_register(lurk_trie_ctx *ctx, const uint8_t *preimages, size_t n, uint8_t *digests_out, int fmt) {
    if (!ctx) { set_error("null trie context"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    if (n && !preimages) { set_error("null preimages"); return LURK_ERR_ARG; }
    if (n > ctx->capacity - ctx->count) {
        set_error("trie register: %zu nodes into a store of %llu nodes and capacity %llu", n, (unsigned long long)ctx->count,
                  (unsigned long long)ctx->capacity);
        return LURK_ERR_ARG;
    }
    return dispatch_field(ctx->field_id, [&](auto f) {
        using F = decltype(f);
        std::vector<uint8_t> canon(n * ARITY * 32);
        for (size_t e = 0; e < n * ARITY; e++) {
            if (!reduced<F>(preimages + e * 32)) { set_error("trie register: preimage %zu element %zu is not reduced below the field modulus", e / ARITY, e % ARITY); return LURK_ERR_ARG; }
            to_canonical_host<F>(preimages + e * 32, fmt, &canon[e * 32]);
        }
        LURK_TRY(ctx_ready(ctx));
        if (!n) return LURK_OK;
        DevBuf b;
        LURK_TRY(b.alloc(n * (ARITY * 32 + 32 + 4)));
        F *pre = b.as<F>(), *dig = pre + n * ARITY;
        LURK_CUDA_TRY(cudaMemcpy(pre, canon.data(), canon.size(), cudaMemcpyHostToDevice));
        LURK_CUDA_TRY(cudaMemset(ctx->err.p, 0xff, 8));
        LURK_TRY(register_dev<F>(ctx, pre, dig, (uint32_t *)(dig + n), (int)n, 0));
        LURK_TRY(sync_count(ctx, 0));
        if (digests_out) {
            LURK_CUDA_TRY(cudaMemcpy(digests_out, dig, n * 32, cudaMemcpyDeviceToHost));
            if (fmt == LURK_FMT_MONTGOMERY)
                for (size_t k = 0; k < n; k++) {
                    F v;
                    memcpy(v.v, digests_out + k * 32, 32);
                    v = F::from_canonical(v);
                    memcpy(digests_out + k * 32, v.v, 32);
                }
        }
        return LURK_OK;
    });
}

int lurk_trie_ctx_apply(lurk_trie_ctx *ctx, size_t n, const int *kinds, const int64_t *prev, const uint8_t *roots, const uint8_t *keys,
                        const uint8_t *values, int fmt, uint8_t *results_out, void *d_lookup_inputs, void *d_insert_inputs, void *stream) {
    if (!ctx) { set_error("null trie context"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    if (n && (!kinds || !prev || !keys)) { set_error("null kinds, prev or keys"); return LURK_ERR_ARG; }
    if (n >= (size_t)1 << 31) { set_error("trie batch of %zu operations: at most 2^31 - 1", n); return LURK_ERR_ARG; }
    return dispatch_field(ctx->field_id, [&](auto f) {
        using F = decltype(f);
        Plan P;
        LURK_TRY(plan_batch<F>(ctx, n, kinds, prev, roots, keys, values, fmt, P));
        LURK_TRY(ctx_ready(ctx));
        if (!n) return LURK_OK;
        return apply_batch<F>(ctx, P, results_out, d_lookup_inputs, d_insert_inputs, fmt, (cudaStream_t)stream);
    });
}

int lurk_trie_ctx_register_dev(lurk_trie_ctx *ctx, const void *d_preimages, size_t n, void *d_digests_out, int fmt, void *stream) {
    if (!ctx) { set_error("null trie context"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    if (n && !d_preimages) { set_error("null preimages"); return LURK_ERR_ARG; }
    if (n > ctx->capacity - ctx->count) {
        set_error("trie register: %zu nodes into a store of %llu nodes and capacity %llu", n, (unsigned long long)ctx->count,
                  (unsigned long long)ctx->capacity);
        return LURK_ERR_ARG;
    }
    return dispatch_field(ctx->field_id, [&](auto f) {
        using F = decltype(f);
        LURK_TRY(ctx_ready(ctx));
        if (!n) return LURK_OK;
        const cudaStream_t st = (cudaStream_t)stream;
        F *pre, *dig;
        uint32_t *claim;
        unsigned long long *bad;
        auto lay = [&](Carve &c) { pre = c.take<F>(n * ARITY); dig = c.take<F>(n); claim = c.take<uint32_t>(n); bad = c.take<unsigned long long>(1); };
        Carve probe{nullptr};
        lay(probe);
        LURK_TRY(ensure(ctx->plan, probe.used));
        Carve c{ctx->plan.as<uint8_t>()};
        lay(c);
        LURK_CUDA_TRY(cudaMemsetAsync(bad, 0xff, 8, st));
        canon_check_kernel<F><<<blocks(n * ARITY), TS_THREADS, 0, st>>>(n * ARITY, (const F *)d_preimages, fmt, pre, bad);
        LURK_CUDA_TRY(cudaGetLastError());
        unsigned long long e = NO_ERR;
        LURK_CUDA_TRY(cudaMemcpyAsync(&e, bad, 8, cudaMemcpyDeviceToHost, st));
        LURK_CUDA_TRY(cudaStreamSynchronize(st));
        if (e != NO_ERR) {
            set_error("trie register: preimage %llu element %llu is not reduced below the field modulus", e / ARITY, e % ARITY);
            return LURK_ERR_ARG;
        }
        LURK_CUDA_TRY(cudaMemsetAsync(ctx->err.p, 0xff, 8, st));
        LURK_TRY(register_dev<F>(ctx, pre, dig, claim, (int)n, st));
        if (d_digests_out) {
            if (fmt == LURK_FMT_MONTGOMERY) LURK_TRY(convert_dev<F>(dig, n, LURK_FMT_MONTGOMERY, d_digests_out, st));
            else LURK_CUDA_TRY(cudaMemcpyAsync(d_digests_out, dig, n * 32, cudaMemcpyDeviceToDevice, st));
        }
        return sync_count(ctx, st);
    });
}

int lurk_trie_ctx_apply_dev(lurk_trie_ctx *ctx, size_t n, const int32_t *d_kinds, const int64_t *d_prev, const void *d_roots, const void *d_keys,
                            const void *d_values, int fmt, void *d_results, void *d_lookup_inputs, void *d_insert_inputs, void *stream) {
    if (!ctx) { set_error("null trie context"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    if (n && (!d_kinds || !d_prev || !d_keys)) { set_error("null kinds, prev or keys"); return LURK_ERR_ARG; }
    if (n >= (size_t)1 << 31) { set_error("trie batch of %zu operations: at most 2^31 - 1", n); return LURK_ERR_ARG; }
    return dispatch_field(ctx->field_id, [&](auto f) {
        using F = decltype(f);
        LURK_TRY(ctx_ready(ctx));
        if (!n) return LURK_OK;
        const cudaStream_t st = (cudaStream_t)stream;
        DevPlan<F> D;
        int m = 0;
        LURK_TRY(plan_dev<F>(ctx, (int)n, d_kinds, d_prev, (const F *)d_roots, (const F *)d_keys, (const F *)d_values, fmt, st, D, m));
        return run_levels<F>(ctx, (int)n, m, D, (F *)d_results, nullptr, d_lookup_inputs, d_insert_inputs, fmt, st);
    });
}

}  // extern "C"
