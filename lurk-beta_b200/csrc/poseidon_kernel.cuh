// K1 / K3: batch Poseidon digests and slot witnesses on sm_90a.
//
// Replaces (reference): PoseidonCache::hash3/4/6/8 (src/hash.rs:180-203) and the Poseidon body of
// allocate_slot (src/lem/circuit.rs:212-315) for whole batches.  Both run Neptune's optimised round schedule
// (SURVEY.md Appendix A), so the witness kernel emits exactly the values the circuit allocates:
// per S-box x^2, x^4, x^5 + post-key.
//
// Mapping: one thread per sponge, persistent grid-stride loop.  The work is integer-ALU bound (about 2e5
// IMAD.WIDE per arity-8 hash for 288 algorithmic bytes), so the design goal is IMAD-pipe occupancy:
//   * all constants of the (field, arity) instance (compressed round keys, MDS, pre-sparse matrix, the R_P sparse
//     factors; 20-40 KB) are staged ONCE per CTA into shared memory by a single TMA bulk copy
//     (cp.async.bulk + mbarrier) and read with conflict-free broadcast LDS.128;
//   * the sponge state lives in shared memory in a [lane][half][thread] uint4 layout (conflict-free LDS.128 /
//     STS.128), which keeps the round loops rolled (small I-cache footprint) and the register budget for the
//     multiplier;
//   * every MDS / sparse dot product is accumulated lazily in 512+ bits and reduced once (WideAcc).
// Preimages are read and digests / witness blocks written with 128-bit vector accesses.
#pragma once
#include "poseidon_api.h"

#include <map>
#include <memory>

namespace lurk {


// ---- TMA bulk staging helpers (global -> shared, completion on an mbarrier)
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t phase) {
    uint32_t ok;
    do {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(ok)
                     : "r"(smem_u32(bar)), "r"(phase)
                     : "memory");
    } while (!ok);
}

template <class F>
__device__ __forceinline__ F lds_fe(const F *p) {
    const uint4 *q = reinterpret_cast<const uint4 *>(p);
    uint4 lo = q[0], hi = q[1];
    F r;
    r.v[0] = lo.x; r.v[1] = lo.y; r.v[2] = lo.z; r.v[3] = lo.w;
    r.v[4] = hi.x; r.v[5] = hi.y; r.v[6] = hi.z; r.v[7] = hi.w;
    return r;
}

// Per-thread view of the shared-memory sponge state: element i is two uint4 at [i][half][thread].
template <class F>
struct SpongeState {
    uint4 *base;    // already offset by the thread index
    int stride;     // threads per CTA
    __device__ __forceinline__ F ld(int i) const {
        uint4 lo = base[(i * 2 + 0) * stride], hi = base[(i * 2 + 1) * stride];
        F r;
        r.v[0] = lo.x; r.v[1] = lo.y; r.v[2] = lo.z; r.v[3] = lo.w;
        r.v[4] = hi.x; r.v[5] = hi.y; r.v[6] = hi.z; r.v[7] = hi.w;
        return r;
    }
    __device__ __forceinline__ void st(int i, const F &x) const {
        base[(i * 2 + 0) * stride] = make_uint4(x.v[0], x.v[1], x.v[2], x.v[3]);
        base[(i * 2 + 1) * stride] = make_uint4(x.v[4], x.v[5], x.v[6], x.v[7]);
    }
};

// Witness sink: appends field elements to the slot block of this sponge (no-op for digest-only kernels).
template <class F, bool WITNESS>
struct AuxSink {
    F *next;
    int fmt;
    __device__ __forceinline__ void put(const F &v) {
        if (WITNESS) { store_fe(next, fmt == LURK_FMT_MONTGOMERY ? v : v.to_canonical()); next++; }
    }
};

// x <- x^5 (+ key) on every lane, emitting x^2, x^4, x^5+key per lane
template <class F, int T, bool WITNESS>
__device__ __forceinline__ void sbox_all(const SpongeState<F> &S, const F *keys, AuxSink<F, WITNESS> &aux) {
#pragma unroll 1
    for (int i = 0; i < T; i++) {
        F x = S.ld(i);
        F x2 = x.sqr();
        F x4 = x2.sqr();
        F x5 = x4 * x;
        if (keys) x5 = x5 + lds_fe(keys + i);
        aux.put(x2); aux.put(x4); aux.put(x5);
        S.st(i, x5);
    }
}

// state <- state * M for columns [j0, j1); M row-major in shared memory
template <class F, int T>
__device__ __forceinline__ void matvec(const SpongeState<F> &S, const F *M, int j0, int j1) {
    F s[T];
#pragma unroll
    for (int i = 0; i < T; i++) s[i] = S.ld(i);
#pragma unroll 1
    for (int j = j0; j < j1; j++) {
        WideAcc<typename F::Params> acc;
        acc.clear();
#pragma unroll
        for (int i = 0; i < T; i++) acc.mul_acc(s[i], lds_fe(M + i * T + j));
        S.st(j, acc.reduce());
    }
}

// element offsets of sponge h's preimage and witness block (see PoseidonGather)
template <int ARITY>
__device__ __forceinline__ void gather_at(const PoseidonGather &G, size_t h, const uint64_t *__restrict__ offs, size_t &pre, size_t &blk) {
    if (G.per_call == 1) {
        pre = h * G.in_stride + G.in_first;
        blk = (offs ? offs[h] : h * G.out_stride) + G.out0;
        return;
    }
    const size_t c = h / (unsigned)G.per_call;
    const int l = (int)(h - c * (unsigned)G.per_call);
    pre = c * G.in_stride + G.in_first + (size_t)ARITY * l;
    blk = (offs ? offs[c] : c * G.out_stride) + (l < G.split ? G.out0 + G.step0 * l : G.out1 + G.step1 * (l - G.split));
}

template <class F, int ARITY, bool WITNESS>
__global__ void __launch_bounds__(ARITY >= 6 ? 384 : 512)
poseidon_kernel(const F *__restrict__ g_consts, PoseidonLayout L, F tag, const F *__restrict__ pre, size_t n,
                F *__restrict__ out, const uint64_t *__restrict__ offs, PoseidonGather G, int in_fmt, int out_fmt) {
    constexpr int T = ARITY + 1;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ __align__(8) uint64_t mbar;
    F *C = reinterpret_cast<F *>(smem_raw);
    const int tid = threadIdx.x;
    SpongeState<F> S;
    S.base = reinterpret_cast<uint4 *>(smem_raw + (size_t)L.flat_len * sizeof(F)) + tid;
    S.stride = blockDim.x;

    // stage the constants: one elected thread issues a single bulk copy
    if (tid == 0) mbar_init(&mbar, 1);
    __syncthreads();
    if (tid == 0) {
        const uint32_t bytes = (uint32_t)L.flat_len * (uint32_t)sizeof(F);
        mbar_expect_tx(&mbar, bytes);
        bulk_g2s(C, g_consts, bytes, &mbar);
    }
    mbar_wait(&mbar, 0);

    const int half = L.rf / 2;
    for (size_t h = (size_t)blockIdx.x * blockDim.x + tid; h < n; h += (size_t)gridDim.x * blockDim.x) {
        size_t pre_at, blk_at;
        gather_at<ARITY>(G, h, offs, pre_at, blk_at);
        const F *p = pre + pre_at;
        F *wout = WITNESS ? out + blk_at : nullptr;
        AuxSink<F, WITNESS> aux;
        aux.next = wout + ARITY;
        aux.fmt = out_fmt;

        // absorb: domain tag | preimage, plus the round-0 keys
        S.st(0, tag + lds_fe(C));
#pragma unroll 1
        for (int i = 1; i < T; i++) {
            F raw = load_fe<F>(p + (i - 1));
            F m = in_fmt == LURK_FMT_MONTGOMERY ? raw : F::from_canonical(raw);
            if (WITNESS) {
                F o = out_fmt == LURK_FMT_MONTGOMERY ? m : (in_fmt == LURK_FMT_MONTGOMERY ? m.to_canonical() : raw);
                store_fe(wout + (i - 1), o);
            }
            S.st(i, m + lds_fe(C + i));
        }
        const F *key = C + T;

        // R_F full rounds with the R_P partial rounds spliced in after the first half.  One call site each for
        // the S-box sweep and the matrix product keeps the kernel body small (instruction cache).
#pragma unroll 1
        for (int r = 0; r < L.rf; r++) {
            const bool last = r == L.rf - 1;
            sbox_all<F, T, WITNESS>(S, last ? nullptr : key, aux);   // the last round has no post-key
            if (!last) key += T;
            // first-half rounds end with the pre-sparse matrix; the last round only needs the digest lane
            matvec<F, T>(S, C + (r == half - 1 ? L.off_pre : L.off_mds), last ? 1 : 0, last ? 2 : T);
            if (r != half - 1) continue;
            // partial rounds: S-box on lane 0, one sparse matrix each
            F s0 = S.ld(0);
            const F *w = C + L.off_sw;
            const F *v = C + L.off_sv;
#pragma unroll 1
            for (int q = 0; q < L.rp; q++) {
                F x2 = s0.sqr();
                F x4 = x2.sqr();
                s0 = x4 * s0 + lds_fe(key);
                key++;
                aux.put(x2); aux.put(x4); aux.put(s0);
                WideAcc<typename F::Params> acc;
                acc.clear();
                acc.mul_acc(s0, lds_fe(w));
#pragma unroll 1
                for (int j = 1; j < T; j++) {
                    F x = S.ld(j);
                    acc.mul_acc(x, lds_fe(w + j));
                    S.st(j, x + s0 * lds_fe(v + (j - 1)));
                }
                s0 = acc.reduce();
                w += T;
                v += T - 1;
            }
            S.st(0, s0);
        }

        F d = S.ld(1);
        if (out_fmt != LURK_FMT_MONTGOMERY) d = d.to_canonical();
        if (WITNESS) store_fe(aux.next, d);
        else store_fe(out + h, d);
    }
}

// ----------------------------------------------------------------------------- warp-per-sponge (latency shape)
// Small batches (the few thousand slots of one fold, one level of the store DAG) are latency bound with one thread per
// sponge: ~1e5..2e5 dependent multiplier instructions.  Here T = arity + 1 adjacent lanes own one sponge, one state
// element per lane, floor(32 / T) sponges per warp:
//   full round    every lane does its own S-box; lane j gathers the T post-S-box elements with warp shuffles and
//                 computes column j of state * M as one lazy dot product (T word products deep instead of T^2 + 3T);
//   partial round lane 0's S-box, its result broadcast; every lane forms its term of <w, s> and its own update
//                 s_j + x v_(j-1) concurrently; the T terms are summed by a shuffle tree.
// ~4x lower latency than the thread-per-sponge kernel at ~1/3 of its throughput, so it is used only for small n.
template <class F>
__device__ __forceinline__ F shfl_fe(const F &x, int src_lane) {
    F r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = __shfl_sync(0xffffffffu, x.v[i], src_lane);
    return r;
}
template <class F>
__device__ __forceinline__ F shfl_down_fe(const F &x, int d) {
    F r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = __shfl_down_sync(0xffffffffu, x.v[i], d);
    return r;
}

template <class F, int ARITY, bool WITNESS>
__global__ void __launch_bounds__(128)
poseidon_warp_kernel(const F *__restrict__ g_consts, PoseidonLayout L, F tag, const F *__restrict__ pre, size_t n,
                     F *__restrict__ out, const uint64_t *__restrict__ offs, PoseidonGather G, int in_fmt, int out_fmt) {
    constexpr int T = ARITY + 1;
    constexpr int GPW = 32 / T;   // sponges per warp
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ __align__(8) uint64_t mbar;
    F *C = reinterpret_cast<F *>(smem_raw);
    const int tid = threadIdx.x;
    if (tid == 0) mbar_init(&mbar, 1);
    __syncthreads();
    if (tid == 0) {
        const uint32_t bytes = (uint32_t)L.flat_len * (uint32_t)sizeof(F);
        mbar_expect_tx(&mbar, bytes);
        bulk_g2s(C, g_consts, bytes, &mbar);
    }
    mbar_wait(&mbar, 0);

    const int lane = tid & 31;
    const int g = lane / T, i = lane - g * T;         // sponge within the warp, state element
    const int base_lane = g * T;
    const size_t warp = ((size_t)blockIdx.x * blockDim.x + tid) >> 5;
    const size_t h = warp * GPW + g;
    const bool live = g < GPW && h < n;                // idle lanes run the same code on zeros and never store
    const int half = L.rf / 2;

    size_t pre_at = 0, blk_at = 0;
    if (live) gather_at<ARITY>(G, h, offs, pre_at, blk_at);
    F *wout = (WITNESS && live) ? out + blk_at : nullptr;
    const bool mont_out = out_fmt == LURK_FMT_MONTGOMERY;
    // absorb
    F s = tag;
    if (i > 0) {
        F raw = live ? load_fe<F>(pre + pre_at + (i - 1)) : F::zero();
        s = in_fmt == LURK_FMT_MONTGOMERY ? raw : F::from_canonical(raw);
        if (WITNESS && live) store_fe(wout + (i - 1), mont_out ? s : (in_fmt == LURK_FMT_MONTGOMERY ? s.to_canonical() : raw));
    }
    s = s + lds_fe(C + i);
    const F *key = C + T;
    int aux = ARITY;                                   // next free element of the witness block

#pragma unroll 1
    for (int r = 0; r < L.rf; r++) {
        const bool last = r == L.rf - 1;
        {   // S-box on every lane
            F x2 = s.sqr();
            F x4 = x2.sqr();
            s = x4 * s;
            if (!last) s = s + lds_fe(key + i);
            if (WITNESS && live) {
                F *o = wout + aux + 3 * i;
                store_fe(o, mont_out ? x2 : x2.to_canonical());
                store_fe(o + 1, mont_out ? x4 : x4.to_canonical());
                store_fe(o + 2, mont_out ? s : s.to_canonical());
            }
            aux += 3 * T;
            if (!last) key += T;
        }
        {   // column i of state * M
            const F *M = C + (r == half - 1 ? L.off_pre : L.off_mds);
            WideAcc<typename F::Params> acc;
            acc.clear();
#pragma unroll 1
            for (int m = 0; m < T; m++) acc.mul_acc(shfl_fe(s, base_lane + m), lds_fe(M + m * T + i));
            s = acc.reduce();
        }
        if (r != half - 1) continue;
        // partial rounds
        const F *w = C + L.off_sw;
        const F *v = C + L.off_sv;
#pragma unroll 1
        for (int q = 0; q < L.rp; q++) {
            F x2 = s.sqr();                            // only lane 0's S-box is used; the others keep lock step
            F x4 = x2.sqr();
            F x = x4 * s + lds_fe(key);
            key++;
            if (WITNESS && live && i == 0) {
                F *o = wout + aux;
                store_fe(o, mont_out ? x2 : x2.to_canonical());
                store_fe(o + 1, mont_out ? x4 : x4.to_canonical());
                store_fe(o + 2, mont_out ? x : x.to_canonical());
            }
            aux += 3;
            x = shfl_fe(x, base_lane);                 // lane 0's S-box output
            F term = (i == 0 ? x : s) * lds_fe(w + i); // term i of <w, s'>
            F upd = s;
            if (i > 0) upd = s + x * lds_fe(v + (i - 1));
            // sum the T terms into lane 0 of the group
#pragma unroll
            for (int d = 1; d < T; d <<= 1) {
                F t2 = shfl_down_fe(term, d);
                if (i + d < T) term = term + t2;
            }
            s = i == 0 ? term : upd;
            w += T;
            v += T - 1;
        }
    }
    if (live && i == 1) {
        F d = mont_out ? s : s.to_canonical();
        if (WITNESS) store_fe(wout + aux, d);
        else store_fe(out + h, d);
    }
}

// ----------------------------------------------------------------------------- bit decomposition slots
// aux order of bellpepper-core AllocatedNum::to_bits_le_strict (call site src/lem/circuit.rs:241-243) preceded by
// the slot's preimage element: walking the bits of p-1 from the top, a bit under a 1 of p-1 is allocated and
// joins the current run; at the first 0 after a run the run (plus the previous run result) is AND-folded, one
// aux per AND, then the bit is allocated.  Output values are 0/1 field elements.  bitdecomp_aux writes the aux of
// canonical x, the block without its leading value: o[0 .. block - 1).
template <class F>
__device__ void bitdecomp_aux(const F &x, F *o, int out_fmt) {
    using P = typename F::Params;
    const F one = out_fmt == LURK_FMT_MONTGOMERY ? F::one() : F::from_u64(1).to_canonical();
    const F zero = F::zero();
    uint32_t b[8];
    b[0] = P::MOD(0) - 1;   // p is odd: no borrow
#pragma unroll
    for (int i = 1; i < 8; i++) b[i] = P::MOD(i);
    int k = 0;
    bool found = false, have_last = false;
    uint32_t last = 0;
    int run_len = 0;
    for (int i = 255; i >= 0; i--) {
        uint32_t bb = (b[i >> 5] >> (i & 31)) & 1, ab = (x.v[i >> 5] >> (i & 31)) & 1;
        found |= bb != 0;
        if (!found) continue;
        if (bb) {
            store_fe(o + k++, ab ? one : zero);   // AllocatedBit::alloc, joins the current run
            run_len++;
        } else {
            if (run_len) {
                // k-ary AND of the run (top bit first), then of the previous run's result: one aux per AND
                uint32_t cur = 1;
                for (int q = 0; q < run_len; q++) {
                    int pos = i + run_len - q;
                    uint32_t bit = (x.v[pos >> 5] >> (pos & 31)) & 1;
                    cur = q == 0 ? bit : (cur & bit);
                    if (q > 0) store_fe(o + k++, cur ? one : zero);
                }
                if (have_last) { cur &= last; store_fe(o + k++, cur ? one : zero); }
                last = cur;
                have_last = true;
                run_len = 0;
            }
            store_fe(o + k++, ab ? one : zero);   // AllocatedBit::alloc_conditionally
        }
    }
}

template <class F>
__global__ void bitdecomp_kernel(const F *__restrict__ vals, size_t n, F *__restrict__ out, const uint64_t *__restrict__ offs,
                                 int block_elems, int in_fmt, int out_fmt) {
    size_t h = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n) return;
    F raw = load_fe<F>(vals + h);
    F x = in_fmt == LURK_FMT_MONTGOMERY ? raw.to_canonical() : raw;
    F *o = out + (offs ? offs[h] : h * (size_t)block_elems);
    store_fe(o, out_fmt == LURK_FMT_MONTGOMERY ? (in_fmt == LURK_FMT_MONTGOMERY ? raw : F::from_canonical(raw)) : x);
    bitdecomp_aux(x, o + 1, out_fmt);
}

// ----------------------------------------------------------------------------- constant cache + launch
template <class F>
struct PoseidonInstance {
    PoseidonParams<F> params;
    PoseidonLayout layout;
    std::map<int, F *> dev_consts;   // per device
};

template <class F>
PoseidonInstance<F> &instance(int arity) {
    static std::mutex mu;
    static std::map<int, std::unique_ptr<PoseidonInstance<F>>> cache;   // mirrors OnceCell in src/hash.rs:42-46
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(arity);
    if (it == cache.end()) {
        auto inst = std::make_unique<PoseidonInstance<F>>();
        inst->params = make_poseidon_params<F>(arity);
        const auto &p = inst->params;
        PoseidonLayout &L = inst->layout;
        L.rf = p.rf; L.rp = p.rp;
        L.off_mds = (int)p.off_mds(); L.off_pre = (int)p.off_pre(); L.off_sw = (int)p.off_sw(); L.off_sv = (int)p.off_sv();
        L.flat_len = (int)p.flat_len();
        L.block_elems = arity + p.num_aux() + 1;
        it = cache.emplace(arity, std::move(inst)).first;
    }
    return *it->second;
}

template <class F>
int device_consts(PoseidonInstance<F> &inst, const F **out) {
    static std::mutex mu;
    std::lock_guard<std::mutex> g(mu);
    int dev = 0;
    LURK_CUDA_TRY(cudaGetDevice(&dev));
    auto it = inst.dev_consts.find(dev);
    if (it == inst.dev_consts.end()) {
        std::vector<F> flat = inst.params.flat();
        F *d = nullptr;
        LURK_CUDA_TRY(cudaMalloc(&d, flat.size() * sizeof(F)));
        LURK_CUDA_TRY(cudaMemcpy(d, flat.data(), flat.size() * sizeof(F), cudaMemcpyHostToDevice));
        it = inst.dev_consts.emplace(dev, d).first;
    }
    *out = it->second;
    return LURK_OK;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize opt-in, once per (kernel instantiation, device).  A failed attempt is not
// remembered, so a transient error is retried by the next launch; any number of devices.
struct SmemOptIn {
    std::mutex mu;
    std::vector<int> done;
    template <class K>
    int ensure(K kern, size_t bytes) {
        int dev = 0;
        LURK_CUDA_TRY(cudaGetDevice(&dev));
        std::lock_guard<std::mutex> g(mu);
        for (int d : done) if (d == dev) return LURK_OK;
        LURK_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        done.push_back(dev);
        return LURK_OK;
    }
};

template <class F, int ARITY, bool WITNESS>
int launch_one(const F *d_consts, const PoseidonInstance<F> &inst, const void *d_pre, size_t n, void *d_out,
                      const uint64_t *d_offs, const PoseidonGather &G, int in_fmt, int out_fmt, int grid, int block, cudaStream_t s) {
    constexpr int T = ARITY + 1;
    constexpr int BIG = ARITY >= 6 ? 384 : 512;
    auto kern = poseidon_kernel<F, ARITY, WITNESS>;
    static SmemOptIn optin;           // per device: opt in to the large dynamic shared-memory carve-out
    LURK_TRY(optin.ensure(kern, (size_t)inst.layout.flat_len * sizeof(F) + (size_t)T * 2 * BIG * sizeof(uint4)));
    size_t smem = (size_t)inst.layout.flat_len * sizeof(F) + (size_t)T * 2 * block * sizeof(uint4);
    kern<<<grid, block, smem, s>>>(d_consts, inst.layout, inst.params.domain_tag, (const F *)d_pre, n, (F *)d_out, d_offs, G, in_fmt, out_fmt);
    LURK_CUDA_TRY(cudaGetLastError());
    return LURK_OK;
}

template <class F, int ARITY, bool WITNESS>
int launch_arity(const void *d_pre, size_t n, void *d_out, const uint64_t *d_offs, const PoseidonGather *g, int in_fmt, int out_fmt,
                 cudaStream_t s) {
    if (n == 0) return LURK_OK;
    PoseidonInstance<F> &inst = instance<F>(ARITY);
    const PoseidonGather G = g ? *g : PoseidonGather{1, 1, ARITY, 0, (uint64_t)inst.layout.block_elems, 0, 0, 0, 0};
    const F *d_consts = nullptr;
    LURK_TRY(device_consts(inst, &d_consts));
    const int sms = sm_count();
    constexpr int BIG = ARITY >= 6 ? 384 : 512;
    if (n >= (size_t)sms * BIG / 2) {
        // throughput shape: one persistent CTA per SM
        return launch_one<F, ARITY, WITNESS>(d_consts, inst, d_pre, n, d_out, d_offs, G, in_fmt, out_fmt, sms, BIG, s);
    }
    if (n <= 8192) {
        // latency shape (the slot batches of one fold, one level of the store DAG): warp-per-sponge kernel
        constexpr int GPW = 32 / (ARITY + 1);
        const size_t warps = (n + GPW - 1) / GPW;
        const unsigned grid = (unsigned)((warps + 3) / 4);
        auto kern = poseidon_warp_kernel<F, ARITY, WITNESS>;
        const size_t smem = (size_t)inst.layout.flat_len * sizeof(F);
        static SmemOptIn optin;
        LURK_TRY(optin.ensure(kern, smem));
        kern<<<grid, 128, smem, s>>>(d_consts, inst.layout, inst.params.domain_tag, (const F *)d_pre, n, (F *)d_out, d_offs, G, in_fmt, out_fmt);
        LURK_CUDA_TRY(cudaGetLastError());
        return LURK_OK;
    }
    // medium batches: thread-per-sponge; the widest CTA that still gives every SM one (each CTA stages the 20-40 KB of
    // constants once, so one-warp CTAs are used only when there are fewer warps than SMs x 2)
    const int block = n >= (size_t)sms * 128 ? 128 : (n >= (size_t)sms * 64 ? 64 : 32);
    int grid = (int)((n + block - 1) / block);
    return launch_one<F, ARITY, WITNESS>(d_consts, inst, d_pre, n, d_out, d_offs, G, in_fmt, out_fmt, grid, block, s);
}

template <class F, bool WITNESS>
int launch_poseidon(int arity, const void *d_pre, size_t n, void *d_out, int in_fmt, int out_fmt, cudaStream_t s, const uint64_t *d_offs,
                    const PoseidonGather *g) {
    switch (arity) {
        case 3: return launch_arity<F, 3, WITNESS>(d_pre, n, d_out, d_offs, g, in_fmt, out_fmt, s);
        case 4: return launch_arity<F, 4, WITNESS>(d_pre, n, d_out, d_offs, g, in_fmt, out_fmt, s);
        case 6: return launch_arity<F, 6, WITNESS>(d_pre, n, d_out, d_offs, g, in_fmt, out_fmt, s);
        case 8: return launch_arity<F, 8, WITNESS>(d_pre, n, d_out, d_offs, g, in_fmt, out_fmt, s);
    }
    set_error("unsupported Poseidon arity %d (HashArity is 3, 4, 6 or 8; src/hash.rs:11-29)", arity);
    return LURK_ERR_ARG;
}


template <class F>
int poseidon_instance_info(int arity, const PoseidonParams<F> **params, PoseidonLayout *layout) {
    PoseidonInstance<F> &inst = instance<F>(arity);
    if (params) *params = &inst.params;
    if (layout) *layout = inst.layout;
    return LURK_OK;
}
template <class F>
int launch_bitdecomp(const void *d_values, size_t n, void *d_blocks, int blk, int fmt, cudaStream_t s, const uint64_t *d_offs) {
    bitdecomp_kernel<F><<<(unsigned)((n + 127) / 128), 128, 0, s>>>((const F *)d_values, n, (F *)d_blocks, d_offs, blk, fmt, fmt);
    LURK_CUDA_TRY(cudaGetLastError());
    return LURK_OK;
}

}  // namespace lurk
