// The KZG side of the BN256 path behind the C ABI (include/lurk_b200.h, N3 / N4):
//   lurk_ck_powers_dev        powers-of-tau commitment key  g, beta g, ..., beta^(n-1) g  (Arecibo hyperkzg CommitmentKey::setup ->
//                             UniversalKZGParam::gen_srs_for_testing; public_params of Bn256EngineKZG, reference src/proof/nova.rs:65-71,196-216)
//   lurk_hyperkzg_prove_dev   provider::hyperkzg::EvaluationEngine::prove -- the polynomial-commitment opening at the end of `compress`
//                             (src/proof/nova.rs:341-356) for the primary BN256 circuit: l - 1 folds of the polynomial + their commitments,
//                             3 l evaluations, the batched polynomial, three witness polynomials (linear recurrences) + their commitments.
// Every vector stays in HBM; per call the host sees 3 challenges' worth of messages ((l - 1) + 3 points, 3 l field elements).
// Kernels: thread-per-segment (32 elements) loops from kzg.cuh; the recurrences use the up-sweep / down-sweep of kzg.cuh; commitments
// go through the library's own Pippenger (lurk_msm_ctx_*) on device pointers.
#include "common.cuh"
#include "kzg.cuh"
#include "pcs.cuh"
#include "reduce.cuh"
#include "sc_scratch.cuh"

#include <algorithm>
#include <vector>

namespace lurk {

static inline int kzg_grid(size_t n, int block) {
    size_t want = (n + block - 1) / block;
    size_t cap = (size_t)sm_count() * 8;
    return (int)(want < cap ? (want ? want : 1) : cap);
}

// ------------------------------------------------------------------------------------------------ N3: powers of tau
template <class Fb, class Fs>
__global__ void __launch_bounds__(128) kzg_powers_kernel(const Affine<Fb> *__restrict__ table, Fs beta, size_t n, Affine<Fb> *__restrict__ out) {
    constexpr int PT = 4;      // points per thread: one inversion for four normalisations
    const size_t groups = (n + PT - 1) / PT;
    for (size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += (size_t)gridDim.x * blockDim.x) {
        const size_t i0 = g * PT;
        Fs s = kzg_pow_small(beta, i0);
        XYZZ<Fb> pts[PT];
        Fb pref[PT];
        Fb run = Fb::one();
#pragma unroll
        for (int k = 0; k < PT; k++) {
            const Fs c = s.to_canonical();
            pts[k] = kzg_fixed_base_mul(table, c.v);
            pref[k] = run;
            if (!pts[k].is_identity()) run = run * pts[k].zzz;
            s = s * beta;
        }
        Fb inv = run.inv();
#pragma unroll
        for (int k = PT - 1; k >= 0; k--) {
            Affine<Fb> a;
            if (pts[k].is_identity()) { a.x = Fb::zero(); a.y = Fb::zero(); }
            else {
                const Fb zi = inv * pref[k];          // 1 / ZZZ_k
                inv = inv * pts[k].zzz;
                const Fb zz_inv = (zi * pts[k].zz).sqr();
                a.x = pts[k].x * zz_inv;
                a.y = pts[k].y * zi;
            }
            if (i0 + k < n) { store_fe(&out[i0 + k].x, a.x); store_fe(&out[i0 + k].y, a.y); }
        }
    }
}

// table[w * 255 + d - 1] = d 2^(8w) g, affine Montgomery, built on the host (8160 points, one batched inversion)
template <class Fb>
static void kzg_build_table(const Affine<Fb> &g, std::vector<Affine<Fb>> &table) {
    const int N = KZG_WINDOWS * 255;
    std::vector<XYZZ<Fb>> pts(N);
    Affine<Fb> base = g;
    for (int w = 0; w < KZG_WINDOWS; w++) {
        XYZZ<Fb> acc = XYZZ<Fb>::identity();
        for (int d = 1; d <= 255; d++) { acc.add_affine(base); pts[w * 255 + d - 1] = acc; }
        XYZZ<Fb> nb = acc;
        nb.add_affine(base);                      // 256 base
        base = nb.to_affine();
    }
    table.resize(N);
    std::vector<Fb> pref(N);
    Fb run = Fb::one();
    for (int i = 0; i < N; i++) { pref[i] = run; if (!pts[i].is_identity()) run = run * pts[i].zzz; }
    Fb inv = run.inv();
    for (int i = N - 1; i >= 0; i--) {
        if (pts[i].is_identity()) { table[i].x = Fb::zero(); table[i].y = Fb::zero(); continue; }
        const Fb zi = inv * pref[i];
        inv = inv * pts[i].zzz;
        const Fb zz_inv = (zi * pts[i].zz).sqr();
        table[i].x = pts[i].x * zz_inv;
        table[i].y = pts[i].y * zi;
    }
}

template <class C>
static int ck_powers(const uint8_t *g_bytes, const uint8_t *beta_bytes, size_t n, void *d_out, int fmt, cudaStream_t s) {
    using Fb = typename C::Base;
    using Fs = typename C::Scalar;
    Affine<Fb> g;
    Fs beta;
    memcpy(g.x.v, g_bytes, 32); memcpy(g.y.v, g_bytes + 32, 32); memcpy(beta.v, beta_bytes, 32);
    if (!g.x.is_reduced() || !g.y.is_reduced() || !beta.is_reduced()) { set_error("generator or beta is not reduced"); return LURK_ERR_RANGE; }
    if (fmt == LURK_FMT_CANONICAL) { g.x = Fb::from_canonical(g.x); g.y = Fb::from_canonical(g.y); beta = Fs::from_canonical(beta); }
    if (!g.is_identity()) {
        const Fb b = C::ID == 0 ? Fb::from_u64(3) : C::ID == 1 ? Fb::from_u64(17).neg() : Fb::from_u64(5);
        if (g.y.sqr() != g.x.sqr() * g.x + b) { set_error("generator is not on the curve"); return LURK_ERR_RANGE; }
    }
    if (n == 0) return LURK_OK;
    std::vector<Affine<Fb>> table;
    kzg_build_table(g, table);
    DevBuf d_table;
    LURK_TRY(d_table.alloc(table.size() * sizeof(Affine<Fb>)));
    LURK_CUDA_TRY(cudaMemcpyAsync(d_table.p, table.data(), table.size() * sizeof(Affine<Fb>), cudaMemcpyHostToDevice, s));
    kzg_powers_kernel<Fb, Fs><<<kzg_grid((n + 3) / 4, 128), 128, 0, s>>>(d_table.as<Affine<Fb>>(), beta, n, static_cast<Affine<Fb> *>(d_out));
    LURK_CUDA_TRY(cudaGetLastError());
    LURK_CUDA_TRY(cudaStreamSynchronize(s));      // the table dies with this frame
    return LURK_OK;
}

// ------------------------------------------------------------------------------------------------ N4: HyperKZG prover kernels
template <class F>
__global__ void __launch_bounds__(256) kzg_fold_kernel(const F *__restrict__ in, F *__restrict__ out, size_t half, F x) {
    for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < half; j += (size_t)gridDim.x * blockDim.x)
        store_fe(out + j, kzg_fold_low(load_fe<F>(in + 2 * j), load_fe<F>(in + 2 * j + 1), x));
}

template <class F>
struct Tri { F v[3]; };

// up-sweep of one level: out[y][s] = sum_{k in segment s} in[y][k] v_y^(k - s L)
template <class F>
__global__ void __launch_bounds__(256) kzg_up_kernel(const F *__restrict__ in, size_t in_stride, size_t len, const __grid_constant__ Tri<F> v,
                                                     F *__restrict__ out, size_t out_stride) {
    const size_t nseg = (len + KZG_SEG - 1) / KZG_SEG;
    const int y = blockIdx.y;
    for (size_t s = (size_t)blockIdx.x * blockDim.x + threadIdx.x; s < nseg; s += (size_t)gridDim.x * blockDim.x) {
        const size_t lo = s * KZG_SEG, hi = lo + KZG_SEG < len ? lo + KZG_SEG : len;
        store_fe(out + y * out_stride + s, kzg_seg_horner(in + y * in_stride, lo, hi, v.v[y]));
    }
}
// down-sweep of one level: every segment re-runs the recurrence from H of the level above (upper[y][s + 1], 0 for the last segment)
template <class F>
__global__ void __launch_bounds__(256) kzg_down_kernel(const F *in, size_t in_stride, size_t len, const __grid_constant__ Tri<F> v, const F *__restrict__ upper,
                                                       size_t upper_stride, F *out, size_t out_stride, size_t shift) {
    const size_t nseg = (len + KZG_SEG - 1) / KZG_SEG;
    const int y = blockIdx.y;
    for (size_t s = (size_t)blockIdx.x * blockDim.x + threadIdx.x; s < nseg; s += (size_t)gridDim.x * blockDim.x) {
        const size_t lo = s * KZG_SEG, hi = lo + KZG_SEG < len ? lo + KZG_SEG : len;
        const F carry = (upper && s + 1 < nseg) ? load_fe<F>(upper + y * upper_stride + s + 1) : F::zero();
        kzg_seg_down(in + y * in_stride, lo, hi, v.v[y], carry, out + y * out_stride, shift);
    }
}

// B[k] = sum_{j : (n >> j) > k} qpow[j] P_j[k]
template <class F>
struct BatchArgs { F qpow[32]; int l; };
template <class F>
__global__ void __launch_bounds__(256) kzg_batch_kernel(const F *__restrict__ polys, size_t n, const __grid_constant__ BatchArgs<F> a, F *__restrict__ out) {
    for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (size_t)gridDim.x * blockDim.x) {
        F acc = load_fe<F>(polys + k);                 // q^0 = 1
        for (int j = 1; j < a.l && (n >> j) > k; j++) acc += a.qpow[j] * load_fe<F>(polys + kzg_poly_offset(n, j) + k);
        store_fe(out + k, acc);
    }
}

// evaluations P_j(u_y): one CTA per 8192-element chunk of a polynomial, threads own 32-element segments
constexpr int KZG_CHUNK = 256 * KZG_SEG;
struct EvalChunk { uint32_t poly, idx; };
template <class F>
struct EvalArgs { F u[3], u_seg[3], u_chunk[3]; };
template <class F>
__global__ void __launch_bounds__(256) kzg_eval_chunk_kernel(const F *__restrict__ polys, size_t n, const EvalChunk *__restrict__ chunks, size_t nchunks,
                                                             const __grid_constant__ EvalArgs<F> a, F *__restrict__ partial) {
    __shared__ F sh[8];
    const int y = blockIdx.y;
    const EvalChunk c = chunks[blockIdx.x];
    const size_t len = n >> c.poly;
    const F *base = polys + kzg_poly_offset(n, (int)c.poly);
    const size_t lo = (size_t)c.idx * KZG_CHUNK + (size_t)threadIdx.x * KZG_SEG;
    F val = F::zero();
    if (lo < len) {
        const size_t hi = lo + KZG_SEG < len ? lo + KZG_SEG : len;
        val = kzg_seg_horner(base, lo, hi, a.u[y]) * kzg_pow_small(a.u_seg[y], threadIdx.x);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) val = val + shfl_down_fe(val, off);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = val;
    __syncthreads();
    if (threadIdx.x == 0) {
        F s = sh[0];
        for (int w = 1; w < 8; w++) s = s + sh[w];
        store_fe(partial + (size_t)y * nchunks + blockIdx.x, s * kzg_pow_small(a.u_chunk[y], c.idx));
    }
}
// v[y][j] = sum of the partials of polynomial j
template <class F>
__global__ void kzg_eval_sum_kernel(const F *__restrict__ partial, size_t nchunks, const uint32_t *__restrict__ first, int l, F *__restrict__ v) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 3 * l) return;
    const int y = t / l, j = t % l;
    F s = F::zero();
    for (uint32_t c = first[j]; c < first[j + 1]; c++) s = s + load_fe<F>(partial + (size_t)y * nchunks + c);
    store_fe(v + t, s);
}

// lurk_msm_ctx_run_dev takes ONE format for the scalars and the result: the vectors here are Montgomery, the caller may want canonical
template <class Fb>
static void points_to_fmt(uint8_t *pts96, int count, int fmt) {
    if (fmt != LURK_FMT_CANONICAL) return;
    for (int j = 0; j < count; j++)
        for (int c = 0; c < 3; c++) { Fb t; memcpy(t.v, pts96 + 96 * j + 32 * c, 32); t = t.to_canonical(); memcpy(pts96 + 96 * j + 32 * c, t.v, 32); }
}

// H(i) = sum_{k >= i} B[k] u_y^(k - i) for the three points; h_y[i - 1] = H(i) (i >= 1), h_y[n - 1] = 0.  h: 3 arrays of n.
template <class F>
static int kzg_witness_polys(const F *d_B, size_t n, const F u[3], F *d_h, DevBuf &scratch, cudaStream_t s) {
    std::vector<size_t> lens{n};
    while (lens.back() > (size_t)KZG_SEG) lens.push_back((lens.back() + KZG_SEG - 1) / KZG_SEG);
    const int K = (int)lens.size() - 1;                    // levels above level 0
    size_t total = 0;
    std::vector<size_t> off(K + 1, 0);
    for (int k = 1; k <= K; k++) { off[k] = total; total += 3 * lens[k]; }
    LURK_TRY(PcsArena::grow(scratch, std::max<size_t>(total, 1) * sizeof(F)));
    F *Y = scratch.as<F>();
    std::vector<Tri<F>> mult(K + 1);
    for (int y = 0; y < 3; y++) mult[0].v[y] = u[y];
    for (int k = 1; k <= K; k++)
        for (int y = 0; y < 3; y++) mult[k].v[y] = kzg_pow_small(mult[k - 1].v[y], KZG_SEG);
    LURK_CUDA_TRY(cudaMemsetAsync(d_h, 0, 3 * n * sizeof(F), s));
    auto level_in = [&](int k) -> const F * { return k == 0 ? d_B : Y + off[k]; };
    auto stride = [&](int k) -> size_t { return k == 0 ? 0 : lens[k]; };
    for (int k = 0; k < K; k++) {
        dim3 grid(kzg_grid(lens[k + 1], 256), 3);
        kzg_up_kernel<F><<<grid, 256, 0, s>>>(level_in(k), stride(k), lens[k], mult[k], Y + off[k + 1], lens[k + 1]);
    }
    for (int k = K; k >= 0; k--) {
        dim3 grid(kzg_grid((lens[k] + KZG_SEG - 1) / KZG_SEG, 256), 3);
        const F *upper = k == K ? nullptr : Y + off[k + 1];
        F *out = k == 0 ? d_h : Y + off[k];
        kzg_down_kernel<F><<<grid, 256, 0, s>>>(level_in(k), stride(k), lens[k], mult[k], upper, k == K ? 0 : lens[k + 1], out, k == 0 ? n : lens[k],
                                                k == 0 ? 1 : 0);
    }
    LURK_CUDA_TRY(cudaGetLastError());
    return LURK_OK;
}

// Every buffer, clone, stream and event comes from the arena A, grown where the one-shot entry point allocated it.
template <class C>
static int hyperkzg_prove(lurk_msm_ctx *ck, PcsArena &A, const void *d_poly, const uint8_t *point, int l, lurk_challenge_fn challenge, void *user,
                          uint8_t *com_out, uint8_t *w_out, uint8_t *v_out, int fmt, cudaStream_t s) {
    using F = typename C::Scalar;
    const size_t n = (size_t)1 << l;
    std::vector<F> x(l);
    for (int i = 0; i < l; i++)
        if (!fe_in(point + 32 * i, fmt, x[i])) { set_error("point[%d] is not reduced", i); return LURK_ERR_RANGE; }
    // Phase 1: P_0 = the polynomial, P_{i+1}[j] = P_i[2j] + x[l-1-i] (P_i[2j+1] - P_i[2j]); commitments of P_1 .. P_{l-1}
    LURK_TRY(PcsArena::grow(A.polys, 2 * n * sizeof(F)));
    F *polys = A.polys.as<F>();
    if (d_poly != polys) LURK_CUDA_TRY(cudaMemcpyAsync(polys, d_poly, n * sizeof(F), cudaMemcpyDeviceToDevice, s));
    for (int i = 0; i + 1 < l; i++) {
        const size_t half = n >> (i + 1);
        kzg_fold_kernel<F><<<kzg_grid(half, 256), 256, 0, s>>>(polys + kzg_poly_offset(n, i), polys + kzg_poly_offset(n, i + 1), half, x[l - 1 - i]);
    }
    LURK_CUDA_TRY(cudaGetLastError());
    // the l - 1 commitments are independent and mostly short (latency-bound Pippenger chains): three of them in flight, on the context and
    // two clones of it (same resident key, own scratch), each on its own stream
    LURK_TRY(A.event());
    LURK_TRY(A.clones(ck, 2));
    EventGuard &ready = A.ready;
    lurk_msm_ctx *ctxs[3] = {ck, A.clone[0].c, A.clone[1].c};
    cudaStream_t streams[3] = {s, A.side[0].s, A.side[1].s};
    LURK_CUDA_TRY(cudaEventRecord(ready.e, s));
    for (int k = 1; k < 3; k++) LURK_CUDA_TRY(cudaStreamWaitEvent(streams[k], ready.e, 0));
    std::vector<uint8_t> com((size_t)std::max(l - 1, 1) * 96);
    {
        int pending[3] = {0, 0, 0};
        for (int j = 1; j < l; j++) {
            const int k = j % 3;
            if (pending[k]) LURK_TRY(lurk_msm_ctx_finish(ctxs[k], com.data() + 96 * (size_t)(pending[k] - 1)));
            LURK_TRY(lurk_msm_ctx_launch_dev(ctxs[k], polys + kzg_poly_offset(n, j), n >> j, LURK_FMT_MONTGOMERY, streams[k]));
            pending[k] = j;
        }
        for (int k = 0; k < 3; k++)
            if (pending[k]) LURK_TRY(lurk_msm_ctx_finish(ctxs[k], com.data() + 96 * (size_t)(pending[k] - 1)));
    }
    points_to_fmt<typename C::Base>(com.data(), l - 1, fmt);
    if (com_out && l > 1) memcpy(com_out, com.data(), (size_t)(l - 1) * 96);
    // Phase 2: r from the commitments; u = (r, -r, r^2)
    uint8_t rb[32];
    int rc = challenge(user, 0, com.data(), (size_t)(l - 1) * 96, rb);
    if (rc != 0) { set_error("challenge callback failed (commitments, %d)", rc); return LURK_ERR_ARG; }
    F u[3];
    if (!fe_in(rb, fmt, u[0])) { set_error("challenge r is not reduced"); return LURK_ERR_RANGE; }
    u[1] = u[0].neg();
    u[2] = u[0].sqr();
    // Phase 3a: v[y][j] = P_j(u_y)
    std::vector<EvalChunk> chunks;
    std::vector<uint32_t> first(l + 1, 0);
    for (int j = 0; j < l; j++) {
        first[j] = (uint32_t)chunks.size();
        const size_t len = n >> j, nc = (len + KZG_CHUNK - 1) / KZG_CHUNK;
        for (size_t c = 0; c < nc; c++) chunks.push_back({(uint32_t)j, (uint32_t)c});
    }
    first[l] = (uint32_t)chunks.size();
    const size_t nchunks = chunks.size();
    DevBuf &d_chunks = A.chunks, &d_first = A.first, &d_partial = A.partial, &d_v = A.v;
    LURK_TRY(PcsArena::grow(d_chunks, nchunks * sizeof(EvalChunk)));
    LURK_TRY(PcsArena::grow(d_first, (l + 1) * sizeof(uint32_t)));
    LURK_TRY(PcsArena::grow(d_partial, 3 * nchunks * sizeof(F)));
    LURK_TRY(PcsArena::grow(d_v, (size_t)3 * l * sizeof(F)));
    LURK_CUDA_TRY(cudaMemcpyAsync(d_chunks.p, chunks.data(), nchunks * sizeof(EvalChunk), cudaMemcpyHostToDevice, s));
    LURK_CUDA_TRY(cudaMemcpyAsync(d_first.p, first.data(), (l + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    EvalArgs<F> ea;
    for (int y = 0; y < 3; y++) { ea.u[y] = u[y]; ea.u_seg[y] = kzg_pow_small(u[y], KZG_SEG); ea.u_chunk[y] = kzg_pow_small(u[y], KZG_CHUNK); }
    kzg_eval_chunk_kernel<F><<<dim3((unsigned)nchunks, 3), 256, 0, s>>>(polys, n, d_chunks.as<EvalChunk>(), nchunks, ea, d_partial.as<F>());
    kzg_eval_sum_kernel<F><<<(3 * l + 63) / 64, 64, 0, s>>>(d_partial.as<F>(), nchunks, d_first.as<uint32_t>(), l, d_v.as<F>());
    LURK_CUDA_TRY(cudaGetLastError());
    std::vector<F> v((size_t)3 * l);
    LURK_CUDA_TRY(cudaMemcpyAsync(v.data(), d_v.p, v.size() * sizeof(F), cudaMemcpyDeviceToHost, s));
    LURK_CUDA_TRY(cudaStreamSynchronize(s));
    std::vector<uint8_t> vb(v.size() * 32);
    for (size_t i = 0; i < v.size(); i++) fe_out(v[i], fmt, vb.data() + 32 * i);
    if (v_out) memcpy(v_out, vb.data(), vb.size());
    uint8_t qb[32];
    rc = challenge(user, 1, vb.data(), vb.size(), qb);
    if (rc != 0) { set_error("challenge callback failed (evaluations, %d)", rc); return LURK_ERR_ARG; }
    F q;
    if (!fe_in(qb, fmt, q)) { set_error("challenge q is not reduced"); return LURK_ERR_RANGE; }
    // Phase 3b: B = sum_j q^j P_j; witness polynomials of B at u_0, u_1, u_2 and their commitments
    BatchArgs<F> ba;
    memset(&ba, 0, sizeof ba);
    ba.l = l;
    ba.qpow[0] = F::one();
    for (int j = 1; j < l; j++) ba.qpow[j] = ba.qpow[j - 1] * q;
    DevBuf &d_B = A.B, &d_h = A.h, &scan_scratch = A.scan;
    LURK_TRY(PcsArena::grow(d_B, n * sizeof(F)));
    LURK_TRY(PcsArena::grow(d_h, 3 * n * sizeof(F)));
    kzg_batch_kernel<F><<<kzg_grid(n, 256), 256, 0, s>>>(polys, n, ba, d_B.as<F>());
    LURK_CUDA_TRY(cudaGetLastError());
    LURK_TRY(kzg_witness_polys<F>(d_B.as<F>(), n, u, d_h.as<F>(), scan_scratch, s));
    uint8_t w[3 * 96];
    LURK_CUDA_TRY(cudaEventRecord(ready.e, s));
    for (int k = 1; k < 3; k++) LURK_CUDA_TRY(cudaStreamWaitEvent(streams[k], ready.e, 0));
    for (int y = 0; y < 3; y++) LURK_TRY(lurk_msm_ctx_launch_dev(ctxs[y], d_h.as<F>() + (size_t)y * n, n, LURK_FMT_MONTGOMERY, streams[y]));
    for (int y = 0; y < 3; y++) LURK_TRY(lurk_msm_ctx_finish(ctxs[y], w + 96 * y));
    points_to_fmt<typename C::Base>(w, 3, fmt);
    if (w_out) memcpy(w_out, w, sizeof w);
    uint8_t ignored[32];
    rc = challenge(user, 2, w, sizeof w, ignored);       // keeps the caller's transcript in the verifier's state
    if (rc != 0) { set_error("challenge callback failed (witness commitments, %d)", rc); return LURK_ERR_ARG; }
    return LURK_OK;
}

int hyperkzg_prove_arena(int curve_id, lurk_msm_ctx *ck, PcsArena &a, const void *d_poly, const uint8_t *point, int l, lurk_challenge_fn challenge,
                         void *user, uint8_t *com_out, uint8_t *w_out, uint8_t *v_out, int fmt, cudaStream_t s) {
    return dispatch_curve(curve_id, [&](auto c) {
        return hyperkzg_prove<decltype(c)>(ck, a, d_poly, point, l, challenge, user, com_out, w_out, v_out, fmt, s);
    });
}

}  // namespace lurk

using namespace lurk;

extern "C" {

int lurk_ck_powers_dev(int curve_id, const uint8_t g[64], const uint8_t beta[32], size_t n, void *d_bases_mont, int fmt, void *stream) {
    if (!g || !beta || (n && !d_bases_mont)) { set_error("null argument"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    return dispatch_curve(curve_id, [&](auto c) { return ck_powers<decltype(c)>(g, beta, n, d_bases_mont, fmt, static_cast<cudaStream_t>(stream)); });
}

int lurk_hyperkzg_prove_dev(int curve_id, lurk_msm_ctx *ck, const void *d_poly, const uint8_t *point, int num_vars, lurk_challenge_fn challenge,
                            void *user, uint8_t *com_out, uint8_t *w_out, uint8_t *v_out, int fmt, void *stream) {
    if (!ck || !d_poly || !point || !challenge) { set_error("null argument"); return LURK_ERR_ARG; }
    if (num_vars < 1 || num_vars > 30) { set_error("bad number of variables %d", num_vars); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    int ck_curve = -1;
    size_t ck_n = 0;
    LURK_TRY(lurk_msm_ctx_info(ck, &ck_curve, &ck_n));
    if (ck_curve != curve_id || ck_n < ((size_t)1 << num_vars)) {
        set_error("commitment key: curve %d with %zu bases, need curve %d with >= 2^%d", ck_curve, ck_n, curve_id, num_vars);
        return LURK_ERR_ARG;
    }
    PcsArena arena;           // per call: allocated and freed as the prover goes, as always
    return hyperkzg_prove_arena(curve_id, ck, arena, d_poly, point, num_vars, challenge, user, com_out, w_out, v_out, fmt, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
