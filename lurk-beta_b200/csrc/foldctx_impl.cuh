// The GPU half of one Nova / SuperNova running instance: RecursiveSNARK::prove_step's NIFS::prove on device-resident state.
//
// Replaces (reference call sites): `Proof::prove_recursively` src/proof/nova.rs:260-339 / supernova.rs:207-291 -- per
// step `RecursiveSNARK::new` (first) or `.prove_step` (nova.rs:286-293), i.e. Arecibo's (third-party, not in tree)
//     comm_W2 = commit(W2);  T = commit_T(U1, W1, U2, W2);  comm_T = commit(T);
//     r = RO(pp_digest, U2, comm_T) [Poseidon sponge, width 25, 128 challenge bits];
//     W1 += r W2, E1 += r T, u1 += r, X1 += r X2, comm_W1 += r comm_W2, comm_E1 += r comm_T       (SURVEY.md App. B)
// and lurk-beta's witness-thread / fold-thread split (nova.rs:297-326) as two stages on CUDA streams:
//   stage A (chain independent, `depth - 1` steps ahead): inputs H2D, slot witnesses written in place into W2
//           (src/lem/multiframe.rs:520-592), commit(W2), A z2, B z2, C z2;
//   stage B (the sequential chain):  A z1, B z1, C z1 -> cross term T -> commit(T) -> [exchange of the partial commitments
//           over NVLink peer memory when the key is sharded] -> affine normalisation -> RO challenge -> AXPY over
//           z = (W, u, X) and E.  Everything between the launch of commit(T) and the AXPYs runs on the device: no event
//           synchronisation, no D2H copy, no host arithmetic on the chain; the host only enqueues.
//   side stream: comm_W1 / comm_E1 update (two 128-bit scalar multiplications) and the 512-byte result record D2H.
#pragma once
#include "msm_impl.cuh"
#include "poseidon_api.h"

#include <memory>
#include <string>

namespace lurk {

static constexpr int FOLD_MAX_WORLD = 16;
static constexpr int FOLD_MAX_DEPTH = 4;
static constexpr int FOLD_MAX_SPANS = 4;
static constexpr int FOLD_RO_RATE = 24;            // Arecibo's RO: neptune sponge over PoseidonConstants<_, U24>
// Windows of the fold's own tables.  On an H100 (400 W) at fib rc = 100, W = 16 / 17 / 18 and T = 15 / 16 / 17 all land within
// 1 % of each other (4.31-4.37 ms per fold, about the run-to-run spread); a narrower window than the key's c = 20 shortens the
// bucket reduction on the chain.
static constexpr int FOLD_W_WINDOW = 17;           // window of commit(W2 - D) (own table when narrower than the key's)
static constexpr int FOLD_T_WINDOW = 16;           // widest window of the chain-critical commit(T)

// ----------------------------------------------------------------------------- fold kernels (witness field)
struct CsrDev {
    const uint64_t *row_ptr;
    const uint32_t *col;
    const void *val;
};

// y_m = M_m z for the three R1CS matrices in one launch (blockIdx.y = matrix), one row per thread
template <class F>
__global__ void __launch_bounds__(256) spmv3_kernel(CsrDev A, CsrDev B, CsrDev C, size_t rows, const F *__restrict__ z, F *__restrict__ ya,
                                                    F *__restrict__ yb, F *__restrict__ yc) {
    const CsrDev M = blockIdx.y == 0 ? A : (blockIdx.y == 1 ? B : C);
    F *y = blockIdx.y == 0 ? ya : (blockIdx.y == 1 ? yb : yc);
    const F *val = (const F *)M.val;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += (size_t)gridDim.x * blockDim.x) {
        const uint64_t k0 = M.row_ptr[i], k1 = M.row_ptr[i + 1];
        F acc = F::zero();
        if (k1 - k0 == 1) {
            acc = load_fe<F>(val + k0) * load_fe<F>(z + M.col[k0]);
        } else if (k1 > k0) {
            // lazy accumulation: one Montgomery reduction per group of <= 8 products
            for (uint64_t k = k0; k < k1;) {
                WideAcc<typename F::Params> w;
                w.clear();
                const uint64_t ke = k1 - k > 8 ? k + 8 : k1;
                for (; k < ke; k++) w.mul_acc(load_fe<F>(val + k), load_fe<F>(z + M.col[k]));
                acc = acc + w.reduce();
            }
        }
        store_fe(y + i, acc);
    }
}

// T = az1*bz2 + az2*bz1 - u1*cz2 - u2*cz1 with u1, u2 read from the device-resident z vectors
template <class F>
__global__ void __launch_bounds__(256) cross_term_dev_kernel(const F *__restrict__ az1, const F *__restrict__ bz1, const F *__restrict__ cz1,
                                                             const F *__restrict__ az2, const F *__restrict__ bz2, const F *__restrict__ cz2,
                                                             const F *__restrict__ u1p, const F *__restrict__ u2p, size_t n, F *__restrict__ t) {
    const F u1 = load_fe<F>(u1p), u2 = load_fe<F>(u2p);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        WideAcc<typename F::Params> acc;
        acc.clear();
        acc.mul_acc(load_fe<F>(az1 + i), load_fe<F>(bz2 + i));
        acc.mul_acc(load_fe<F>(az2 + i), load_fe<F>(bz1 + i));
        F pos = acc.reduce();
        WideAcc<typename F::Params> neg;
        neg.clear();
        neg.mul_acc(u1, load_fe<F>(cz2 + i));
        neg.mul_acc(u2, load_fe<F>(cz1 + i));
        store_fe(t + i, pos - neg.reduce());
    }
}

// the fold: z1 += r z2 over (W, u, X), E1 += r T and -- A, B, C being linear -- A z1 += r A z2, B z1 += r B z2, C z1 += r C z2
// (which takes the three sparse products of the running instance off the chain), one launch; r from device memory (written
// by the challenge kernel)
template <class F>
struct FoldAxpyArgs {
    F *dst[5];
    const F *src[5];
    size_t end[5];       // cumulative element counts
};
template <class F>
__global__ void __launch_bounds__(256) fold_axpy_kernel(FoldAxpyArgs<F> a, const F *__restrict__ rp) {
    const F r = load_fe<F>(rp);
    const size_t total = a.end[4];
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        int v = 0;
        while (i >= a.end[v]) v++;
        const size_t j = v ? i - a.end[v - 1] : i;
        store_fe(a.dst[v] + j, load_fe<F>(a.dst[v] + j) + r * load_fe<F>(a.src[v] + j));
    }
}

// relaxed R1CS residual: counts rows with az*bz != u*cz + e; with `kept` vectors (the incrementally folded A z, B z, C z) also
// rows where those differ from the freshly computed products
template <class F>
__global__ void __launch_bounds__(256) relaxed_residual_kernel(const F *__restrict__ az, const F *__restrict__ bz, const F *__restrict__ cz,
                                                               const F *__restrict__ e, const F *__restrict__ up, const F *__restrict__ kept_a,
                                                               const F *__restrict__ kept_b, const F *__restrict__ kept_c, size_t n,
                                                               unsigned long long *bad) {
    const F u = load_fe<F>(up);
    unsigned local = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const F a = load_fe<F>(az + i), b = load_fe<F>(bz + i), c = load_fe<F>(cz + i);
        const F lhs = a * b;
        const F rhs = u * c + load_fe<F>(e + i);
        bool ok = lhs == rhs;
        if (kept_a) ok = ok && a == load_fe<F>(kept_a + i) && b == load_fe<F>(kept_b + i) && c == load_fe<F>(kept_c + i);
        local += ok ? 0u : 1u;
    }
    local = __reduce_add_sync(0xffffffffu, local);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(bad, (unsigned long long)local);
}

// strided element-wise conversion (canonical -> Montgomery) of the spans of W2 the host fills
template <class F>
__global__ void __launch_bounds__(256) span_to_mont_kernel(F *base, uint64_t first, uint64_t row_elems, uint64_t stride, uint64_t rows) {
    const uint64_t total = row_elems * rows;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        F *p = base + first + (i / row_elems) * stride + (i % row_elems);
        store_fe(p, F::from_canonical(load_fe<F>(p)));
    }
}

// ----------------------------------------------------------------------------- the challenge kernel (commitment field)
// peer-visible exchange slot: one per (parity, source rank)
template <class Fb>
struct alignas(128) XchgSlot {
    XYZZ<Fb> w, t;
    unsigned long long flag;
    unsigned long long pad[15];
};
template <class Fb>
struct XchgBuf {
    XchgSlot<Fb> slot[2][FOLD_MAX_WORLD];
};

template <class Fb, class Fs>
struct FoldRecord {
    Fb cw_x, cw_y, ct_x, ct_y;       // affine Montgomery, (0, 0) for the identity: comm_W2 and comm_T of the step (whole key)
    Fb hash;                         // the squeezed sponge element (Montgomery)
    Fs r;                            // challenge in the witness field, Montgomery
    Fb uw_x, uw_y, ue_x, ue_y;       // running comm_W / comm_E after the step's fold (side stream)
    uint32_t cw_inf, ct_inf, uw_inf, ue_inf;
    uint32_t status;                 // 0 ok, 1 exchange time-out
    uint32_t pad[3];
    unsigned long long seq;
    unsigned long long pad2;
};

enum { FOLD_RO_CONST = 0, FOLD_RO_W_X = 1, FOLD_RO_W_Y = 2, FOLD_RO_W_INF = 3, FOLD_RO_T_X = 4, FOLD_RO_T_Y = 5, FOLD_RO_T_INF = 6 };
enum { FOLD_MODE_FOLD = 0, FOLD_MODE_COMMIT_ONLY = 1 };

template <class Fb, class Fs>
struct ChallengeArgs {
    const XYZZ<Fb> *part_w, *part_t;       // this rank's partial commitments (MSM results); part_t may be null = identity
    int world, rank;
    unsigned long long *seq;                // device counter, bumped by the kernel: the exchange epoch
    XchgBuf<Fb> *peers[FOLD_MAX_WORLD];     // peers[p] = rank p's exchange buffer as mapped in this process (peers[rank] = own)
    const Fb *ro_consts;                    // width-25 Poseidon constants image [compressed | mds | pre | sparse_w | sparse_v]
    PoseidonLayout L;
    Fb io_tag;                              // SAFE IO-pattern tag in the capacity element
    int n_absorb;
    unsigned char kind[FOLD_RO_RATE];
    const Fb *step_consts;                  // FOLD_RO_RATE elements, Montgomery (CONST slots of this step)
    int challenge_bits;
    int mode;
    Fs *r_out;
    FoldRecord<Fb, Fs> *rec;
};

__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long *p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint4 ld_volatile_u4(const uint4 *p) {
    uint4 v;
    asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

template <class F>
__device__ __forceinline__ F shfl_fe_any(const F &x, int src_lane) {
    F r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = __shfl_sync(0xffffffffu, x.v[i], src_lane);
    return r;
}
template <class F>
__device__ __forceinline__ F shfl_down_fe_any(const F &x, int d) {
    F r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = __shfl_down_sync(0xffffffffu, x.v[i], d);
    return r;
}

// One width-25 Poseidon permutation by one warp (Neptune's optimised schedule, as poseidon_warp_kernel): lane i < 25 owns
// state element i.  Constants are read from global memory (L2 resident, read once per permutation).  Returns the lane's
// element of the permuted state.
template <class F>
__device__ F ro_permute_warp(const F *__restrict__ C, const PoseidonLayout &L, F s, int lane) {
    constexpr int T = FOLD_RO_RATE + 1;
    const int i = lane < T ? lane : T - 1;     // idle lanes mirror lane 24 (never read by the others)
    const int half = L.rf / 2;
    s = s + load_fe<F>(C + i);
    const F *key = C + T;
#pragma unroll 1
    for (int r = 0; r < L.rf; r++) {
        const bool last = r == L.rf - 1;
        {
            F x2 = s.sqr();
            F x4 = x2.sqr();
            s = x4 * s;
            if (!last) { s = s + load_fe<F>(key + i); key += T; }
        }
        {
            const F *M = C + (r == half - 1 ? L.off_pre : L.off_mds);
            F acc = F::zero();
            // 25 products: three lazy groups (9 + 8 + 8) so that one accumulator never exceeds its carry budget
#pragma unroll 1
            for (int m0 = 0; m0 < T; m0 += 9) {
                WideAcc<typename F::Params> w;
                w.clear();
                const int m1 = m0 + 9 < T ? m0 + 9 : T;
#pragma unroll 1
                for (int m = m0; m < m1; m++) w.mul_acc(shfl_fe_any(s, m), load_fe<F>(M + m * T + i));
                acc = acc + w.reduce();
            }
            s = acc;
        }
        if (r != half - 1) continue;
        const F *w = C + L.off_sw;
        const F *v = C + L.off_sv;
#pragma unroll 1
        for (int q = 0; q < L.rp; q++) {
            // product 1: lane 0 squares; the other lanes already form their term of <w, s'> (it does not depend on the S-box)
            const F wi = load_fe<F>(w + i);
            const F p1 = s * (i == 0 ? s : wi);
            F x4 = p1.sqr();                             // lane 0: x^4
            F x = x4 * s + load_fe<F>(key);              // lane 0: x^5 + key
            key++;
            x = shfl_fe_any(x, 0);
            // product 2: lane 0 forms its term with the S-box output; lane i > 0 its own update s_i + x v_(i-1)
            const F p2 = x * (i == 0 ? wi : load_fe<F>(v + (i > 0 ? i - 1 : 0)));
            F term = i == 0 ? p2 : p1;
            if (lane >= T) term = F::zero();
            const F upd = s + p2;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const F t2 = shfl_down_fe_any(term, d);
                if (lane + d < 32) term = term + t2;
            }
            s = i == 0 ? term : upd;
            w += T;
            v += T - 1;
        }
    }
    return s;
}

// One CTA, two warps.  Warp 0 / warp 1 handle comm_W / comm_T through exchange and summation; thread 0 normalises both with
// one inversion; warp 0 runs the sponge.
template <class C>
__global__ void __launch_bounds__(64) fold_challenge_kernel(ChallengeArgs<typename C::Base, typename C::Scalar> a) {
    using Fb = typename C::Base;
    using Fs = typename C::Scalar;
    using Pt = XYZZ<Fb>;
    __shared__ Pt sh_pt[2];
    __shared__ Fb sh_aff[4];
    __shared__ uint32_t sh_inf[2];
    __shared__ unsigned long long sh_seq;
    __shared__ uint32_t sh_status;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) { sh_seq = *a.seq + 1; *a.seq = sh_seq; sh_status = 0; }
    __syncthreads();
    const unsigned long long seq = sh_seq;

    // ---- this rank's partial (warp 0: W, warp 1: T)
    const Pt *mine = warp == 0 ? a.part_w : a.part_t;
    Pt pt = Pt::identity();
    if (a.world <= 1) {
        if (lane == 0 && mine) pt = load_xyzz(mine);
    } else {
        const int parity = (int)(seq & 1);
        // push my partial into slot[parity][rank] of every rank (own included); 8 x uint4 per point
        if (lane < 8) {
            uint4 word = make_uint4(0, 0, 0, 0);
            if (mine) word = reinterpret_cast<const uint4 *>(mine)[lane];
            for (int p = 0; p < a.world; p++) {
                XchgSlot<Fb> *dst = &a.peers[p]->slot[parity][a.rank];
                reinterpret_cast<uint4 *>(warp == 0 ? &dst->w : &dst->t)[lane] = word;
            }
        }
        __threadfence_system();
        __syncthreads();                     // both points of this rank are written and fenced
        if (warp == 0 && lane < a.world) st_release_sys(&a.peers[lane]->slot[parity][a.rank].flag, seq);
        // wait for every rank's flag in my own buffer (bounded: a peer that never arrives must not hang the GPU)
        if (lane < a.world) {
            const unsigned long long *flag = &a.peers[a.rank]->slot[parity][lane].flag;
            const unsigned long long t0 = globaltimer_ns();
            while (ld_acquire_sys(flag) < seq) {
                if (globaltimer_ns() - t0 > 4000000000ull) { sh_status = 1; break; }
                __nanosleep(200);
            }
        }
        __syncwarp();
        // lane p holds rank p's partial; butterfly sum (same association on every rank, the affine result is canonical anyway)
        if (lane < a.world) {
            const XchgSlot<Fb> *src = &a.peers[a.rank]->slot[parity][lane];
            const uint4 *q = reinterpret_cast<const uint4 *>(warp == 0 ? &src->w : &src->t);
            uint4 wd[8];
#pragma unroll
            for (int k = 0; k < 8; k++) wd[k] = ld_volatile_u4(q + k);
            const uint32_t *u = reinterpret_cast<const uint32_t *>(wd);
#pragma unroll
            for (int k = 0; k < 8; k++) { pt.x.v[k] = u[k]; pt.y.v[k] = u[8 + k]; pt.zz.v[k] = u[16 + k]; pt.zzz.v[k] = u[24 + k]; }
        }
        int span = 1;
        while (span < a.world) span <<= 1;
#pragma unroll 1
        for (int d = span >> 1; d > 0; d >>= 1) {
            const Pt p2 = shfl_xor_xyzz(pt, d);
            pt.add(p2);
        }
    }
    if (lane == 0) sh_pt[warp] = pt;
    __syncthreads();

    // ---- affine normalisation of both points with one inversion (thread 0)
    if (tid == 0) {
        const Pt pw = sh_pt[0], pc = sh_pt[1];
        const bool iw = pw.is_identity(), ic = pc.is_identity();
        const Fb zw = iw ? Fb::one() : pw.zzz, zc = ic ? Fb::one() : pc.zzz;
        const Fb inv = (zw * zc).inv_vartime();
        const Fb iwz = inv * zc, icz = inv * zw;          // 1 / ZZZ_w, 1 / ZZZ_t
        Fb x = Fb::zero(), y = Fb::zero();
        if (!iw) { const Fb zz_inv = (iwz * pw.zz).sqr(); x = pw.x * zz_inv; y = pw.y * iwz; }
        sh_aff[0] = x; sh_aff[1] = y;
        x = Fb::zero(); y = Fb::zero();
        if (!ic) { const Fb zz_inv = (icz * pc.zz).sqr(); x = pc.x * zz_inv; y = pc.y * icz; }
        sh_aff[2] = x; sh_aff[3] = y;
        sh_inf[0] = iw; sh_inf[1] = ic;
        a.rec->cw_x = sh_aff[0]; a.rec->cw_y = sh_aff[1]; a.rec->ct_x = sh_aff[2]; a.rec->ct_y = sh_aff[3];
        a.rec->cw_inf = iw; a.rec->ct_inf = ic;
        a.rec->status = sh_status;
        a.rec->seq = seq;
    }
    __syncthreads();
    if (a.mode != FOLD_MODE_FOLD || warp != 0) return;

    // ---- random oracle: SAFE sponge, capacity = IO tag, n_absorb rate elements, one permutation, squeeze element 1
    Fb s = Fb::zero();
    if (lane == 0) s = a.io_tag;
    else if (lane <= a.n_absorb) {
        switch (a.kind[lane - 1]) {
            case FOLD_RO_W_X: s = sh_aff[0]; break;
            case FOLD_RO_W_Y: s = sh_aff[1]; break;
            case FOLD_RO_W_INF: s = sh_inf[0] ? Fb::one() : Fb::zero(); break;
            case FOLD_RO_T_X: s = sh_aff[2]; break;
            case FOLD_RO_T_Y: s = sh_aff[3]; break;
            case FOLD_RO_T_INF: s = sh_inf[1] ? Fb::one() : Fb::zero(); break;
            default: s = load_fe<Fb>(a.step_consts + (lane - 1)); break;
        }
    }
    s = ro_permute_warp<Fb>(a.ro_consts, a.L, s, lane);
    if (lane == 1) {
        a.rec->hash = s;
        // the low `challenge_bits` bits of the canonical integer, re-read as an element of the witness field
        const Fb h = s.to_canonical();
        Fs raw = Fs::zero();
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int lo = 32 * k;
            uint32_t w = h.v[k];
            if (a.challenge_bits <= lo) w = 0;
            else if (a.challenge_bits < lo + 32) w &= (1u << (a.challenge_bits - lo)) - 1u;
            raw.v[k] = w;
        }
        if (!raw.is_reduced()) raw.final_sub();        // only possible when challenge_bits is close to the field size
        const Fs r = Fs::from_canonical(raw);
        a.rec->r = r;
        store_fe(a.r_out, r);
    }
}

// comm_W1 += r comm_W2, comm_E1 += r comm_T (thread 0 / thread 32), r = 128-bit (or wider) canonical scalar.
// Off the critical chain (side stream): plain double-and-add over the bits of r with an affine addend.
template <class C>
__global__ void __launch_bounds__(64) fold_commitments_kernel(XYZZ<typename C::Base> *run_w, XYZZ<typename C::Base> *run_e,
                                                              FoldRecord<typename C::Base, typename C::Scalar> *rec, int init) {
    using Fb = typename C::Base;
    using Fs = typename C::Scalar;
    using Pt = XYZZ<Fb>;
    const int which = threadIdx.x >> 5;
    if (threadIdx.x & 31) return;
    Affine<Fb> q;
    q.x = which == 0 ? rec->cw_x : rec->ct_x;
    q.y = which == 0 ? rec->cw_y : rec->ct_y;
    Pt *run = which == 0 ? run_w : run_e;
    Pt acc;
    if (init) {
        // RecursiveSNARK::new: the running instance is the first fresh instance (comm_E = identity)
        acc = which == 0 ? Pt::from_affine(q) : Pt::identity();
    } else {
        const Fs k = rec->r.to_canonical();
        acc = Pt::identity();
        int top = 255;
        while (top >= 0 && !((k.v[top >> 5] >> (top & 31)) & 1u)) top--;
#pragma unroll 1
        for (int b = top; b >= 0; b--) {
            acc = acc.dbl();
            if ((k.v[b >> 5] >> (b & 31)) & 1u) acc.add_affine(q);
        }
        Pt cur = *run;
        cur.add(acc);
        acc = cur;
    }
    *run = acc;
    Affine<Fb> af;
    af.x = Fb::zero();
    af.y = Fb::zero();
    if (!acc.is_identity()) {
        const Fb zi = acc.zzz.inv_vartime();
        const Fb zz_inv = (zi * acc.zz).sqr();
        af.x = acc.x * zz_inv;
        af.y = acc.y * zi;
    }
    if (which == 0) { rec->uw_x = af.x; rec->uw_y = af.y; rec->uw_inf = acc.is_identity(); }
    else { rec->ue_x = af.x; rec->ue_y = af.y; rec->ue_inf = acc.is_identity(); }
}

// ----------------------------------------------------------------------------- host side
struct FoldSpan { uint64_t first, row_elems, stride, rows; };

struct FoldSlotBatch {
    int arity = 0;                 // 0 = bit decomposition
    size_t count = 0;
    DevBuf d_offsets;              // u64 element offsets into W
    DevBuf d_pre[FOLD_MAX_DEPTH];  // preimages / values per fresh buffer
    void *h_pre[FOLD_MAX_DEPTH] = {nullptr, nullptr, nullptr, nullptr};   // pinned
    size_t bytes() const { return count * (size_t)(arity ? arity : 1) * 32; }
};

struct FoldConfigHost {
    int curve_id = 0, depth = 2, world = 1, rank = 0;
    uint64_t n_w = 0, n_x = 0, n_rows = 0;
    int latency_sms = 0;
};

struct FoldResultHost {
    uint8_t comm_w[96], comm_t[96], r[32], run_comm_w[96], run_comm_e[96], hash[32];
    int status;
    unsigned long long seq;
};

// curve-independent interface behind the C ABI
struct FoldCtxBase {
    virtual ~FoldCtxBase() {}
    virtual int init(const FoldConfigHost &cfg, const uint64_t *const row_ptr[3], const uint32_t *const col[3], const uint8_t *const val[3], int fmt,
                     lurk_msm_ctx *ck_w, lurk_msm_ctx *ck_t) = 0;
    virtual int add_slot_batch(int arity, size_t count, const uint64_t *offsets) = 0;
    virtual int set_spans(int n, const FoldSpan *spans) = 0;
    virtual int set_ro(int n_absorb, const int *kinds, int challenge_bits) = 0;
    virtual int host_buffer(int b, int which, void **ptr, size_t *bytes) = 0;
    virtual int device_buffer(int b, int which, void **ptr, size_t *bytes) = 0;
    virtual int exchange_handle(uint8_t out[64]) = 0;
    virtual int set_peers(const uint8_t *handles) = 0;
    virtual int set_running(const uint8_t *w, const uint8_t *e, const uint8_t *u, const uint8_t *x, const uint8_t *comm_w, const uint8_t *comm_e, int fmt) = 0;
    virtual int get_running(uint8_t *w, uint8_t *e, uint8_t *u, uint8_t *x, uint8_t *comm_w, uint8_t *comm_e, int fmt) = 0;
    virtual int stage_a(int b, int flags, int fmt) = 0;
    virtual int init_running(int b) = 0;
    virtual int stage_b_launch(int b) = 0;
    virtual int collect(int b, FoldResultHost *out, int fmt) = 0;
    virtual int check_running(unsigned long long *bad_rows, int *comm_w_ok, int *comm_e_ok) = 0;
    virtual int stats(unsigned *launches_a, unsigned *launches_b, float *acc_w_ms, float *acc_t_ms) = 0;
    virtual int sync() = 0;
};

enum { FOLD_BUF_GLUE = -1, FOLD_BUF_X2 = -2, FOLD_BUF_RO = -3, FOLD_BUF_W2 = -4, FOLD_BUF_T = -5, FOLD_BUF_Z1 = -6, FOLD_BUF_E1 = -7 };
enum { FOLD_INPUTS_RESIDENT = 1 };

template <class C> FoldCtxBase *make_fold_ctx();

#define LURK_FOLD_EXTERN(C) extern template FoldCtxBase *make_fold_ctx<C>();

}  // namespace lurk
