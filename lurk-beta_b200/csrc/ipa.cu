// N4 -- the folding rounds of the inner-product argument behind the C ABI (include/lurk_b200.h): Arecibo
// provider::ipa_pc::InnerProductArgument::prove as `compress` reaches it for the secondary circuit (EE2) and for the Pasta cycle
// (reference src/proof/nova.rs:57-71, 341-356).  Split from sumcheck.cu to keep the two translation units' nvcc time apart.
//   ipa_fold_scalars / _bases    a' = x a_lo + y a_hi;  G' = x G_lo + y G_hi (interleaved double-and-add, uniform branches).
//   ipa_weighted / weights_update the prover's own path: commitments of a round as Pippenger passes over the fixed key.
//   ipa_s_kernel                 the verifier's s = tensor of (1 / r_j, r_j) and <b, s> in one pass, for ck_hat = commit(ck, s).
#include "common.cuh"
#include "sumcheck.cuh"
#include "sc_scratch.cuh"
#include "pcs.cuh"
#include "tensor.cuh"

#include <algorithm>
#include <thread>
#include <vector>

namespace lurk {

// ------------------------------------------------------------------------------------------------ IPA folds
template <class F>
__global__ void __launch_bounds__(256) ipa_fold_scalars_kernel(F *a, size_t half, F x, F y) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x)
        store_fe(a + i, ipa_fold_scalar(load_fe<F>(a + i), load_fe<F>(a + i + half), x, y));
}
struct Scalar256 { uint32_t w[8]; };
template <class F>
__global__ void __launch_bounds__(128) ipa_fold_bases_kernel(Affine<F> *g, size_t half, const __grid_constant__ Scalar256 x, const __grid_constant__ Scalar256 y) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x) {
        Affine<F> p, q;
        p.x = load_fe<F>(&g[i].x); p.y = load_fe<F>(&g[i].y);
        q.x = load_fe<F>(&g[i + half].x); q.y = load_fe<F>(&g[i + half].y);
        const Affine<F> r = ipa_fold_point(p, q, x.w, y.w);
        store_fe(&g[i].x, r.x);
        store_fe(&g[i].y, r.y);
    }
}

// Fixed-base multiplication of ck_c on the host (the c_L ck_c / c_R ck_c terms, 2 per round): 4-bit windows, 64 mixed additions
// per product instead of a 254-step double-and-add.
template <class Fb>
struct HostFixedBase {
    std::vector<Affine<Fb>> table;     // table[w * 15 + d - 1] = d 16^w P
    explicit HostFixedBase(const Affine<Fb> &p) : table(64 * 15) {
        std::vector<XYZZ<Fb>> pts(64 * 15);
        Affine<Fb> base = p;
        for (int w = 0; w < 64; w++) {
            XYZZ<Fb> acc = XYZZ<Fb>::identity();
            for (int d = 1; d <= 15; d++) { acc.add_affine(base); pts[w * 15 + d - 1] = acc; }
            XYZZ<Fb> nb = acc;
            nb.add_affine(base);
            base = nb.to_affine();
        }
        std::vector<Fb> pref(pts.size());
        Fb run = Fb::one();
        for (size_t i = 0; i < pts.size(); i++) { pref[i] = run; if (!pts[i].is_identity()) run = run * pts[i].zzz; }
        Fb inv = run.inv();
        for (size_t i = pts.size(); i-- > 0;) {
            if (pts[i].is_identity()) { table[i].x = Fb::zero(); table[i].y = Fb::zero(); continue; }
            const Fb zi = inv * pref[i];
            inv = inv * pts[i].zzz;
            const Fb zz_inv = (zi * pts[i].zz).sqr();
            table[i].x = pts[i].x * zz_inv;
            table[i].y = pts[i].y * zi;
        }
    }
    XYZZ<Fb> mul(const uint32_t k[8]) const {       // k canonical
        XYZZ<Fb> acc = XYZZ<Fb>::identity();
        for (int w = 0; w < 64; w++) {
            const uint32_t d = (k[w >> 3] >> (4 * (w & 7))) & 15u;
            if (d) acc.add_affine(table[w * 15 + d - 1]);
        }
        return acc;
    }
};

// The prover never needs the folded key itself, only commitments under it: with W_j[idx] = prod_{k < j} (bit_k(idx) ? r_k : 1 / r_k)
// (bit_k = the k-th bit of idx from the top) the folded key of round j is G_j[i] = sum_{idx = i mod m} W_j[idx] G[idx], m = n / 2^j, so
//     L_j = <a_lo, G_j,hi> = sum_{idx : idx mod m >= m/2} W_j[idx] a_j[idx mod m - m/2] G[idx]      (R_j alike on the low halves)
// -- one Pippenger pass over the ORIGINAL key per commitment (the bucket sort drops the zero half) instead of m / 2 latency-bound
// 254-bit double-scalar multiplications per round; the key is not consumed and a fixed-base table of it can be reused.
template <class F>
__global__ void __launch_bounds__(256) ipa_weighted_kernel(const F *__restrict__ w, const F *__restrict__ a, size_t n, size_t m, F *__restrict__ sl, F *__restrict__ sr) {
    const size_t half = m / 2;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (size_t)gridDim.x * blockDim.x) {
        const size_t i = idx & (m - 1);
        const F wi = load_fe<F>(w + idx);
        if (i >= half) { store_fe(sl + idx, wi * load_fe<F>(a + (i - half))); store_fe(sr + idx, F::zero()); }
        else { store_fe(sr + idx, wi * load_fe<F>(a + (i + half))); store_fe(sl + idx, F::zero()); }
    }
}
// W_{j+1}[idx] = W_j[idx] * (idx mod m >= m/2 ? r : 1/r)
template <class F>
__global__ void __launch_bounds__(256) ipa_weights_update_kernel(F *w, size_t n, size_t m, F r, F r_inv) {
    const size_t half = m / 2;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (size_t)gridDim.x * blockDim.x)
        store_fe(w + idx, load_fe<F>(w + idx) * (((idx & (m - 1)) >= half) ? r : r_inv));
}
template <class F>
__global__ void __launch_bounds__(256) fill_one_kernel(F *w, size_t n) {
    const F one = F::one();
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (size_t)gridDim.x * blockDim.x) store_fe(w + idx, one);
}

// The key weights, the clone, the side stream and the event come from the arena A, grown where the one-shot entry point allocated them.
template <class C>
static int ipa_prove(lurk_msm_ctx *ck, PcsArena &A, const uint8_t *gc_bytes, void *d_a, void *d_b, int log_n, lurk_challenge_fn challenge, void *user,
                     uint8_t *L_out, uint8_t *R_out, uint8_t *a_final, uint8_t *b_final, int fmt, cudaStream_t s) {
    using Fb = typename C::Base;
    using Fs = typename C::Scalar;
    Affine<Fb> gc;
    if (!fe_in(gc_bytes, fmt, gc.x) || !fe_in(gc_bytes + 32, fmt, gc.y)) { set_error("ck_c is not reduced"); return LURK_ERR_RANGE; }
    const HostFixedBase<Fb> gc_mul(gc);
    ScScratch<Fs> sc;
    LURK_TRY(sc.init(s));
    Fs *a = static_cast<Fs *>(d_a), *b = static_cast<Fs *>(d_b);
    const size_t n = (size_t)1 << log_n;
    LURK_TRY(PcsArena::grow(A.weights, 3 * n * sizeof(Fs)));
    Fs *W = A.weights.as<Fs>(), *sl = W + n, *sr = W + 2 * n;
    fill_one_kernel<Fs><<<sc_grid(n, 256), 256, 0, s>>>(W, n);
    LURK_CUDA_TRY(cudaGetLastError());
    // L and R of a round are independent: the second one runs on a clone of the context (same resident key, own scratch) and a side stream
    LURK_TRY(A.clones(ck, 1));
    MsmCloneGuard &ck_r = A.clone[0];
    StreamGuard &s_r = A.side[0];
    LURK_TRY(A.event());
    EventGuard &weighted = A.ready;
    size_t m = n;
    for (int round = 0; round < log_n; round++) {
        const size_t half = m / 2;
        Fs cl, cr;
        LURK_TRY(dot_dev<Fs>(a, b + half, half, &cl, sc, s));
        LURK_TRY(dot_dev<Fs>(a + half, b, half, &cr, sc, s));
        ipa_weighted_kernel<Fs><<<sc_grid(n, 256), 256, 0, s>>>(W, a, n, m, sl, sr);
        LURK_CUDA_TRY(cudaGetLastError());
        LURK_CUDA_TRY(cudaEventRecord(weighted.e, s));
        LURK_CUDA_TRY(cudaStreamWaitEvent(s_r.s, weighted.e, 0));
        uint8_t parts[2][96];
        LURK_TRY(lurk_msm_ctx_launch_dev(ck, sl, n, LURK_FMT_MONTGOMERY, s));
        LURK_TRY(lurk_msm_ctx_launch_dev(ck_r.c, sr, n, LURK_FMT_MONTGOMERY, s_r.s));
        LURK_TRY(lurk_msm_ctx_finish(ck, parts[0]));
        LURK_TRY(lurk_msm_ctx_finish(ck_r.c, parts[1]));        // both passes are complete before anything below touches sl / sr / a
        uint8_t lr[192];
        for (int side = 0; side < 2; side++) {
            // L = <a_lo, G_hi> + c_L ck_c,  R = <a_hi, G_lo> + c_R ck_c  (G = the folded key of this round, never materialised)
            const uint8_t *part = parts[side];
            XYZZ<Fb> acc = XYZZ<Fb>::identity();
            Fb z;
            memcpy(z.v, part + 64, 32);
            if (!z.is_zero()) { Affine<Fb> p; memcpy(p.x.v, part, 32); memcpy(p.y.v, part + 32, 32); acc.add_affine(p); }
            const Fs c = (side == 0 ? cl : cr).to_canonical();
            acc.add(gc_mul.mul(c.v));
            point_to_bytes_fmt(acc, fmt, lr + 96 * side);
        }
        if (L_out) memcpy(L_out + 96 * (size_t)round, lr, 96);
        if (R_out) memcpy(R_out + 96 * (size_t)round, lr + 96, 96);
        uint8_t rbytes[32];
        int rc = challenge(user, round, lr, 192, rbytes);
        if (rc != 0) { set_error("challenge callback failed in round %d (%d)", round, rc); return LURK_ERR_ARG; }
        Fs r;
        if (!fe_in(rbytes, fmt, r) || r.is_zero()) { set_error("challenge of round %d is zero or not reduced", round); return LURK_ERR_RANGE; }
        const Fs r_inv = r.inv();
        // a' = a_lo r + a_hi r^-1;  b' = b_lo r^-1 + b_hi r;  key weights: low half r^-1, high half r
        ipa_fold_scalars_kernel<Fs><<<sc_grid(half, 256), 256, 0, s>>>(a, half, r, r_inv);
        ipa_fold_scalars_kernel<Fs><<<sc_grid(half, 256), 256, 0, s>>>(b, half, r_inv, r);
        ipa_weights_update_kernel<Fs><<<sc_grid(n, 256), 256, 0, s>>>(W, n, m, r, r_inv);
        LURK_CUDA_TRY(cudaGetLastError());
        m = half;
    }
    Fs fin[2];
    LURK_CUDA_TRY(cudaMemcpyAsync(&fin[0], a, sizeof(Fs), cudaMemcpyDeviceToHost, s));
    LURK_CUDA_TRY(cudaMemcpyAsync(&fin[1], b, sizeof(Fs), cudaMemcpyDeviceToHost, s));
    LURK_CUDA_TRY(cudaStreamSynchronize(s));
    if (a_final) fe_out(fin[0], fmt, a_final);
    if (b_final) fe_out(fin[1], fmt, b_final);
    return LURK_OK;
}

// ------------------------------------------------------------------------------------------------ the verifier
// s[i] = prod_j (bit_j(i) ? r_j : 1 / r_j) -- the prover's key weights after its last round -- from product-tensor tables in shared memory
// (tensor.cuh), written for the commitment ck_hat = commit(ck, s), and b_hat = <b, s> accumulated in the same pass.
template <class F>
struct IpaSArgs {
    TensorSpec<F> t;
    const F *b;
    F *s;
    size_t n;
    F *partial;
    unsigned *counter;
    F *result;
};

template <class F>
__global__ void __launch_bounds__(256) ipa_s_kernel(const __grid_constant__ IpaSArgs<F> a) {
    extern __shared__ uint4 ipa_tensor_smem[];
    F *tab = reinterpret_cast<F *>(ipa_tensor_smem);
    const int groups = tensor_groups(a.t.l);
    tensor_build(a.t, tab);
    __syncthreads();
    F acc[1] = {F::zero()};
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (size_t)gridDim.x * blockDim.x) {
        const F v = tensor_at(tab, groups, i);
        store_fe(a.s + i, v);
        acc[0] += load_fe<F>(a.b + i) * v;
    }
    grid_sum<F, 1>(acc, a.partial, a.counter, a.result);
}

// sum_{lo <= k < hi} scalars[k] P_k on the host: Straus, 4-bit windows, the 252 doublings shared by all terms of the range
template <class Fb, class Fs>
static XYZZ<Fb> host_straus(const std::vector<XYZZ<Fb>> &pts, const std::vector<Fs> &scalars, size_t lo, size_t hi) {
    const size_t n = hi - lo;
    std::vector<XYZZ<Fb>> tab(n * 16);
    std::vector<Fs> k(n);
    for (size_t i = 0; i < n; i++) {
        k[i] = scalars[lo + i].to_canonical();
        tab[16 * i] = XYZZ<Fb>::identity();
        for (int d = 1; d < 16; d++) { tab[16 * i + d] = tab[16 * i + d - 1]; tab[16 * i + d].add(pts[lo + i]); }
    }
    XYZZ<Fb> acc = XYZZ<Fb>::identity();
    for (int w = 63; w >= 0; w--) {
        for (int t = 0; t < 4; t++) acc = acc.dbl();
        for (size_t i = 0; i < n; i++) {
            const uint32_t d = (k[i].v[w >> 3] >> (4 * (w & 7))) & 15u;
            if (d) acc.add(tab[16 * i + d]);
        }
    }
    return acc;
}

// sum_k scalars[k] P_k: the terms split over host threads (the window additions dominate: 64 per term against 256 shared doublings)
template <class Fb, class Fs>
static XYZZ<Fb> host_msm(const std::vector<XYZZ<Fb>> &pts, const std::vector<Fs> &scalars) {
    const size_t n = pts.size();
    const size_t parts = std::max<size_t>(1, std::min<size_t>({(n + 3) / 4, 16, std::max(1u, std::thread::hardware_concurrency())}));
    std::vector<XYZZ<Fb>> partial(parts);
    std::vector<std::thread> pool;
    for (size_t t = 1; t < parts; t++)
        pool.emplace_back([&, t] { partial[t] = host_straus(pts, scalars, n * t / parts, n * (t + 1) / parts); });
    partial[0] = host_straus(pts, scalars, 0, n / parts);
    for (std::thread &th : pool) th.join();
    XYZZ<Fb> acc = partial[0];
    for (size_t t = 1; t < parts; t++) acc.add(partial[t]);
    return acc;
}

template <class Fb>
static bool same_point(const XYZZ<Fb> &p, const XYZZ<Fb> &q) {
    if (p.is_identity() || q.is_identity()) return p.is_identity() && q.is_identity();
    const Affine<Fb> a = p.to_affine(), b = q.to_affine();
    return a.x == b.x && a.y == b.y;
}

template <class C>
static int ipa_verify(lurk_msm_ctx *ck, const uint8_t *gc_bytes, const uint8_t *comm_bytes, const uint8_t *c_bytes, const void *d_b, int log_n,
                      const uint8_t *L, const uint8_t *R, const uint8_t *a_bytes, lurk_challenge_fn challenge, void *user, int *accepted,
                      uint8_t *ck_hat_out, uint8_t *b_hat_out, int fmt, cudaStream_t s) {
    using Fb = typename C::Base;
    using Fs = typename C::Scalar;
    *accepted = 0;
    const Affine<Fb> g = curve_generator<C>();
    const Fb b = g.y.sqr() - g.x.sqr() * g.x;
    uint8_t gc3[96] = {0};
    memcpy(gc3, gc_bytes, 64);
    bool gc_identity = true;
    for (int i = 0; i < 64; i++) gc_identity &= gc_bytes[i] == 0;
    if (!gc_identity) fe_out(Fb::one(), fmt, gc3 + 64);
    XYZZ<Fb> gc, comm;
    if (!point_in(gc3, fmt, b, gc)) { set_error("ck_c is not a reduced point on the curve"); return LURK_ERR_RANGE; }
    if (!point_in(comm_bytes, fmt, b, comm)) { set_error("comm is not a point of the header's form on the curve"); return LURK_ERR_RANGE; }
    Fs c, a_hat;
    if (!fe_in(c_bytes, fmt, c) || !fe_in(a_bytes, fmt, a_hat)) { set_error("c or a_final is not reduced"); return LURK_ERR_RANGE; }
    // every point is checked before the first transcript call: pts = comm, ck_c, L_0, R_0, L_1, R_1, ..
    std::vector<XYZZ<Fb>> pts{comm, gc};
    for (int j = 0; j < log_n; j++) {
        XYZZ<Fb> Lj, Rj;
        if (!point_in(L + 96 * (size_t)j, fmt, b, Lj) || !point_in(R + 96 * (size_t)j, fmt, b, Rj)) {
            set_error("L or R of round %d is not a point of the header's form on the curve", j);
            return LURK_ERR_RANGE;
        }
        pts.push_back(Lj);
        pts.push_back(Rj);
    }
    std::vector<Fs> sc(pts.size());
    sc[0] = Fs::one();
    TensorSpec<Fs> t;
    memset(&t, 0, sizeof t);
    t.l = log_n;
    for (int j = 0; j < log_n; j++) {
        uint8_t lr[192], rb[32];
        memcpy(lr, L + 96 * (size_t)j, 96);
        memcpy(lr + 96, R + 96 * (size_t)j, 96);
        const int rc = challenge(user, j, lr, 192, rb);
        if (rc != 0) { set_error("challenge callback failed in round %d (%d)", j, rc); return LURK_ERR_ARG; }
        Fs r;
        if (!fe_in(rb, fmt, r) || r.is_zero()) { set_error("challenge of round %d is zero or not reduced", j); return LURK_ERR_RANGE; }
        const Fs r_inv = r.inv();
        t.hi[j] = r;
        t.lo[j] = r_inv;
        sc[2 + 2 * j] = r * r;
        sc[3 + 2 * j] = r_inv * r_inv;
    }
    // s and b_hat, then ck_hat = commit(ck, s) on the key context.  b_hat is read as soon as the s pass ends, so that the other side of
    // the check, Q = comm + (c - a_hat b_hat) ck_c + sum_j (r_j^2 L_j + r_j^-2 R_j), is computed while the commitment runs -- by the
    // point-combination kernel on a stream of the greatest priority, whose one CTA takes the first SM the commitment's kernels free (or by
    // the host Straus, for a short Q); after it only a_hat ck_hat == Q is left.
    const size_t n = (size_t)1 << log_n;
    StreamBuf sbuf;
    LURK_TRY(sbuf.alloc(n * sizeof(Fs), s));
    ScScratch<Fs> scr;
    LURK_TRY(scr.init(s));
    IpaSArgs<Fs> a;
    a.t = t;
    a.b = static_cast<const Fs *>(d_b);
    a.s = static_cast<Fs *>(sbuf.p);
    a.n = n;
    a.partial = scr.partial;
    a.counter = scr.counter;
    a.result = scr.result;
    const size_t smem = (size_t)tensor_groups(log_n) * TENSOR_GROUP * sizeof(Fs);
    LURK_CUDA_TRY(cudaFuncSetAttribute(ipa_s_kernel<Fs>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ipa_s_kernel<Fs><<<sc_grid(n, 256), 256, smem, s>>>(a);
    LURK_CUDA_TRY(cudaGetLastError());
    EventGuard s_done;
    LURK_TRY(s_done.create());
    LURK_CUDA_TRY(cudaEventRecord(s_done.e, s));
    LURK_TRY(lurk_msm_ctx_launch_dev(ck, sbuf.p, n, LURK_FMT_MONTGOMERY, s));
    LURK_CUDA_TRY(cudaEventSynchronize(s_done.e));
    const Fs b_hat = *static_cast<const Fs *>(scr.pinned);
    sc[1] = c - a_hat * b_hat;
    std::vector<const uint8_t *> q_pts{comm_bytes, gc3};
    for (int j = 0; j < log_n; j++) {
        q_pts.push_back(L + 96 * (size_t)j);
        q_pts.push_back(R + 96 * (size_t)j);
    }
    std::vector<uint8_t> q_sc(32 * sc.size());
    for (size_t k = 0; k < sc.size(); k++) fe_out(sc[k], fmt, q_sc.data() + 32 * k);
    uint8_t q_bytes[96];
    const PointGroup q_group{q_pts.data(), q_sc.data(), (int)q_pts.size(), q_bytes};
    StreamGuard q_stream;
    int q_rc = q_stream.create_urgent();
    if (q_rc == LURK_OK) q_rc = point_combination_groups(C::ID, &q_group, 1, fmt, false, q_stream.s);
    uint8_t hat[96];
    LURK_TRY(lurk_msm_ctx_finish(ck, hat));            // the key context is left with nothing pending, whatever became of Q
    LURK_TRY(q_rc);
    XYZZ<Fb> q;
    point_in(q_bytes, fmt, b, q);
    XYZZ<Fb> ck_hat = XYZZ<Fb>::identity();
    Fb z;
    memcpy(z.v, hat + 64, 32);
    if (!z.is_zero()) { Affine<Fb> p; memcpy(p.x.v, hat, 32); memcpy(p.y.v, hat + 32, 32); ck_hat = XYZZ<Fb>::from_affine(p); }
    *accepted = same_point(host_msm(std::vector<XYZZ<Fb>>{ck_hat}, std::vector<Fs>{a_hat}), q) ? 1 : 0;
    if (ck_hat_out) point_to_bytes_fmt(ck_hat, fmt, ck_hat_out);
    if (b_hat_out) fe_out(b_hat, fmt, b_hat_out);
    return LURK_OK;
}

int ipa_prove_arena(int curve_id, lurk_msm_ctx *ck, PcsArena &a, const uint8_t *gc_bytes, void *d_a, void *d_b, int log_n, lurk_challenge_fn challenge,
                    void *user, uint8_t *L_out, uint8_t *R_out, uint8_t *a_final, uint8_t *b_final, int fmt, cudaStream_t s) {
    return dispatch_curve(curve_id, [&](auto c) {
        return ipa_prove<decltype(c)>(ck, a, gc_bytes, d_a, d_b, log_n, challenge, user, L_out, R_out, a_final, b_final, fmt, s);
    });
}

int ipa_verify_checked(int curve_id, lurk_msm_ctx *ck, const uint8_t *gc_bytes, const uint8_t *comm, const uint8_t *c, const void *d_b, int log_n,
                       const uint8_t *L, const uint8_t *R, const uint8_t *a_final, lurk_challenge_fn challenge, void *user, int *accepted, int fmt,
                       cudaStream_t s) {
    return dispatch_curve(curve_id, [&](auto cv) {
        return ipa_verify<decltype(cv)>(ck, gc_bytes, comm, c, d_b, log_n, L, R, a_final, challenge, user, accepted, nullptr, nullptr, fmt, s);
    });
}

bool points_valid(int curve_id, const uint8_t *const *points, int count, int fmt) {
    return dispatch_curve(curve_id, [&](auto c) {
        using C = decltype(c);
        const typename C::Base b = curve_b<C>();
        XYZZ<typename C::Base> p;
        for (int k = 0; k < count; k++)
            if (!points[k] || !point_in(points[k], fmt, b, p)) return 0;
        return 1;
    }) == 1;
}

// x | y -> x | y | z of the header's form
template <class Fb>
static void affine_to_96(const uint8_t *xy, int fmt, uint8_t out[96]) {
    memset(out, 0, 96);
    memcpy(out, xy, 64);
    bool identity = true;
    for (int i = 0; i < 64; i++) identity &= xy[i] == 0;
    if (!identity) fe_out(Fb::one(), fmt, out + 64);
}

bool affine_valid(int curve_id, const uint8_t *xy, int fmt) {
    return dispatch_curve(curve_id, [&](auto c) {
        using C = decltype(c);
        uint8_t p96[96];
        affine_to_96<typename C::Base>(xy, fmt, p96);
        XYZZ<typename C::Base> p;
        return point_in(p96, fmt, curve_b<C>(), p) ? 1 : 0;
    }) == 1;
}

int point_combination(int curve_id, const uint8_t *const *points, const uint8_t *scalars, int count, int fmt, uint8_t out[96]) {
    return dispatch_curve(curve_id, [&](auto c) {
        using C = decltype(c);
        using Fb = typename C::Base;
        using Fs = typename C::Scalar;
        const Fb b = curve_b<C>();
        std::vector<XYZZ<Fb>> pts(count);
        std::vector<Fs> sc(count);
        for (int k = 0; k < count; k++) {
            if (!point_in(points[k], fmt, b, pts[k])) { set_error("point %d is not a point of the header's form on the curve", k); return LURK_ERR_RANGE; }
            if (!fe_in(scalars + 32 * (size_t)k, fmt, sc[k])) { set_error("scalar %d is not reduced", k); return LURK_ERR_RANGE; }
        }
        point_to_bytes_fmt(host_msm(pts, sc), fmt, out);
        return LURK_OK;
    });
}

int scale_affine(int curve_id, const uint8_t *xy, const uint8_t *r, int fmt, uint8_t out[64]) {
    return dispatch_curve(curve_id, [&](auto c) {
        uint8_t p96[96], q96[96];
        affine_to_96<typename decltype(c)::Base>(xy, fmt, p96);
        const uint8_t *pts[1] = {p96};
        LURK_TRY(point_combination(curve_id, pts, r, 1, fmt, q96));
        memcpy(out, q96, 64);                   // the identity is (0, 0) in both forms
        return LURK_OK;
    });
}

}  // namespace lurk

using namespace lurk;

extern "C" {

int lurk_ipa_fold_scalars_dev(int field_id, void *d_a, size_t n, const uint8_t x[32], const uint8_t y[32], int fmt, void *stream) {
    if (!d_a || !x || !y || n < 2 || (n & (n - 1))) { set_error("bad argument (n must be a power of two >= 2)"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    return dispatch_field(field_id, [&](auto f) {
        using F = decltype(f);
        F fx, fy;
        if (!fe_in(x, fmt, fx) || !fe_in(y, fmt, fy)) { set_error("scalar is not reduced"); return LURK_ERR_RANGE; }
        ipa_fold_scalars_kernel<F><<<sc_grid(n / 2, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<F *>(d_a), n / 2, fx, fy);
        LURK_CUDA_TRY(cudaGetLastError());
        return LURK_OK;
    });
}

int lurk_ipa_fold_bases_dev(int curve_id, void *d_bases_mont, size_t n, const uint8_t x[32], const uint8_t y[32], int fmt, void *stream) {
    if (!d_bases_mont || !x || !y || n < 2 || (n & (n - 1))) { set_error("bad argument (n must be a power of two >= 2)"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    return dispatch_curve(curve_id, [&](auto c) {
        using C = decltype(c);
        using Fs = typename C::Scalar;
        using Fb = typename C::Base;
        Fs fx, fy;
        if (!fe_in(x, fmt, fx) || !fe_in(y, fmt, fy)) { set_error("scalar is not reduced"); return LURK_ERR_RANGE; }
        Scalar256 sx, sy;
        const Fs cx = fx.to_canonical(), cy = fy.to_canonical();
        for (int i = 0; i < 8; i++) { sx.w[i] = cx.v[i]; sy.w[i] = cy.v[i]; }
        ipa_fold_bases_kernel<Fb><<<sc_grid(n / 2, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<Affine<Fb> *>(d_bases_mont), n / 2, sx, sy);
        LURK_CUDA_TRY(cudaGetLastError());
        return LURK_OK;
    });
}

int lurk_ipa_prove_dev(int curve_id, lurk_msm_ctx *ck, const uint8_t ck_c[64], void *d_a, void *d_b, int log_n, lurk_challenge_fn challenge,
                       void *user, uint8_t *L_out, uint8_t *R_out, uint8_t a_final[32], uint8_t b_final[32], int fmt, void *stream) {
    if (!ck || !ck_c || !d_a || !d_b || !challenge) { set_error("null argument"); return LURK_ERR_ARG; }
    if (log_n < 0 || log_n > 30) { set_error("bad log_n %d", log_n); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    int ck_curve = -1;
    size_t ck_n = 0;
    LURK_TRY(lurk_msm_ctx_info(ck, &ck_curve, &ck_n));
    if (ck_curve != curve_id || ck_n < ((size_t)1 << log_n)) {
        set_error("commitment key: curve %d with %zu bases, need curve %d with >= 2^%d", ck_curve, ck_n, curve_id, log_n);
        return LURK_ERR_ARG;
    }
    PcsArena arena;           // per call: allocated and freed as the prover goes, as always
    return ipa_prove_arena(curve_id, ck, arena, ck_c, d_a, d_b, log_n, challenge, user, L_out, R_out, a_final, b_final, fmt,
                           static_cast<cudaStream_t>(stream));
}

int lurk_ipa_verify_dev(int curve_id, lurk_msm_ctx *ck, const uint8_t ck_c[64], const uint8_t comm[96], const uint8_t c[32], const void *d_b,
                        int log_n, const uint8_t *L, const uint8_t *R, const uint8_t a_final[32], lurk_challenge_fn challenge, void *user,
                        int *accepted, uint8_t ck_hat_out[96], uint8_t b_hat_out[32], int fmt, void *stream) {
    if (!ck || !ck_c || !comm || !c || !d_b || !a_final || !challenge || !accepted) { set_error("null argument"); return LURK_ERR_ARG; }
    if (log_n < 0 || log_n > 30) { set_error("bad log_n %d", log_n); return LURK_ERR_ARG; }
    if (log_n > 0 && (!L || !R)) { set_error("null L / R"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    int ck_curve = -1;
    size_t ck_n = 0;
    LURK_TRY(lurk_msm_ctx_info(ck, &ck_curve, &ck_n));
    if (ck_curve != curve_id || ck_n < ((size_t)1 << log_n)) {
        set_error("commitment key: curve %d with %zu bases, need curve %d with >= 2^%d", ck_curve, ck_n, curve_id, log_n);
        return LURK_ERR_ARG;
    }
    return dispatch_curve(curve_id, [&](auto cv) {
        return ipa_verify<decltype(cv)>(ck, ck_c, comm, c, d_b, log_n, L, R, a_final, challenge, user, accepted, ck_hat_out, b_hat_out, fmt,
                                        static_cast<cudaStream_t>(stream));
    });
}

}  // extern "C"
