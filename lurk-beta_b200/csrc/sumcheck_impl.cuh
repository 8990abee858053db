// The N4 templates behind the sum-check, eq-table, inner-product and batch_eval_reduce entry points: shared by sumcheck.cu (the
// primitives of the C ABI) and spartan.cu (the Spartan prover context, which calls them directly instead of going back through the
// argument checks of the extern "C" layer every round).
#pragma once
#include "common.cuh"
#include "sumcheck.cuh"
#include "reduce.cuh"
#include "sc_scratch.cuh"

#include <algorithm>
#include <cstring>
#include <vector>

namespace lurk {

// ------------------------------------------------------------------------------------------------ sum-check round
template <class F>
struct ScArgs {
    F *poly[4];
    size_t len;          // length of every polynomial on entry
    F r;                 // BIND: the previous round's challenge (Montgomery)
    F *partial;          // grid x EVALS
    unsigned *counter;
    F *result;           // EVALS
};

template <class F, int KIND, bool BIND>
__global__ void __launch_bounds__(256, 2) sc_round_kernel(const __grid_constant__ ScArgs<F> a) {
    constexpr int K = ScShape<KIND>::POLYS, E = ScShape<KIND>::EVALS;
    F acc[E];
#pragma unroll
    for (int e = 0; e < E; e++) acc[e] = F::zero();
    const size_t half = BIND ? a.len / 4 : a.len / 2;     // index pairs of THIS round
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x) {
        F lo[K], hi[K];
#pragma unroll
        for (int k = 0; k < K; k++) {
            if (BIND) {
                const F l0 = load_fe<F>(a.poly[k] + i), l1 = load_fe<F>(a.poly[k] + i + a.len / 2);
                const F h0 = load_fe<F>(a.poly[k] + i + a.len / 4), h1 = load_fe<F>(a.poly[k] + i + a.len / 4 + a.len / 2);
                lo[k] = sc_bind(l0, l1, a.r);
                hi[k] = sc_bind(h0, h1, a.r);
                store_fe(a.poly[k] + i, lo[k]);                 // only this thread ever touches these four slots
                store_fe(a.poly[k] + i + a.len / 4, hi[k]);
            } else {
                lo[k] = load_fe<F>(a.poly[k] + i);
                hi[k] = load_fe<F>(a.poly[k] + i + half);
            }
        }
        sc_accumulate<F, KIND>(lo, hi, acc);
    }
    grid_sum<F, E>(acc, a.partial, a.counter, a.result);
}

// the last bind (length 2 -> 1): the final evaluations of the K polynomials
template <class F>
__global__ void sc_final_bind_kernel(const __grid_constant__ ScArgs<F> a, int k_polys) {
    if (threadIdx.x < k_polys && blockIdx.x == 0) {
        F v = sc_bind(load_fe<F>(a.poly[threadIdx.x]), load_fe<F>(a.poly[threadIdx.x] + 1), a.r);
        store_fe(a.poly[threadIdx.x], v);
        store_fe(&a.result[threadIdx.x], v);
    }
}

// ------------------------------------------------------------------------------------------------ eq table
template <class F>
struct EqArgs { F tau[32], one_minus[32]; int l; };

template <class F, int LOW>
__global__ void __launch_bounds__(128) eq_kernel(const __grid_constant__ EqArgs<F> a, F *__restrict__ out, int to_canonical) {
    const int high = a.l - LOW;
    const size_t groups = (size_t)1 << high;
    for (size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += (size_t)gridDim.x * blockDim.x) {
        F vals[1 << LOW];
        F v = F::one();
        for (int j = 0; j < high; j++) v = v * (((g >> (high - 1 - j)) & 1) ? a.tau[j] : a.one_minus[j]);
        vals[0] = v;
#pragma unroll
        for (int j = 0; j < LOW; j++) {
#pragma unroll
            for (int t = (1 << j) - 1; t >= 0; t--) {
                const F hi = vals[t] * a.tau[high + j];
                vals[2 * t + 1] = hi;
                vals[2 * t] = vals[t] - hi;
            }
        }
#pragma unroll
        for (int t = 0; t < (1 << LOW); t++) store_fe(out + (g << LOW) + t, to_canonical ? vals[t].to_canonical() : vals[t]);
    }
}

// ------------------------------------------------------------------------------------------------ host-side helpers
// SumcheckProof::prove_quad_batch / prove_cubic_with_additive_term_batch (the BatchedRelaxedR1CSSNARK of SuperNova's `compress`,
// reference src/proof/supernova.rs:293-317) -- and, with one instance and coefficient 1, the plain prove_quad /
// prove_cubic_with_additive_term.  Instance i has its own polynomials of 2^nr[i] elements and joins in round max - nr[i]; until then
// its round polynomial is the constant 2^(remaining - nr[i] - 1) claim_i.  The round message is sum_i coeff_i s_i(X).
constexpr int SC_MAX_INSTANCES = 60;
template <class F, int KIND>
static int sumcheck_prove_batch(int n_inst, void *const *d_polys, const int *nr, const uint8_t *claims_in, const uint8_t *coeffs_in,
                                lurk_challenge_fn challenge, void *user, uint8_t *round_evals, uint8_t *challenges, uint8_t *final_evals, int fmt,
                                cudaStream_t s) {
    constexpr int K = ScShape<KIND>::POLYS, E = ScShape<KIND>::EVALS, DEG1 = E + 1;
    std::vector<F> claim(n_inst), coeff(n_inst);
    int max_rounds = 0;
    for (int i = 0; i < n_inst; i++) {
        if (!fe_in(claims_in + 32 * i, fmt, claim[i])) { set_error("claim %d is not reduced", i); return LURK_ERR_RANGE; }
        if (coeffs_in) { if (!fe_in(coeffs_in + 32 * i, fmt, coeff[i])) { set_error("coefficient %d is not reduced", i); return LURK_ERR_RANGE; } }
        else coeff[i] = F::one();
        max_rounds = std::max(max_rounds, nr[i]);
    }
    ScScratch<F> sc;
    LURK_TRY(sc.init(s));
    std::vector<ScArgs<F>> args(n_inst);
    std::vector<size_t> cur(n_inst);
    for (int i = 0; i < n_inst; i++) {
        memset(&args[i], 0, sizeof(ScArgs<F>));
        for (int k = 0; k < K; k++) args[i].poly[k] = static_cast<F *>(d_polys[i * K + k]);
        args[i].partial = sc.partial; args[i].counter = sc.counter; args[i].result = sc.result + 4 * i;
        args[i].r = F::zero();
        cur[i] = (size_t)1 << nr[i];
    }
    const F two = F::from_u64(2);
    auto pow2 = [&](int k) { F r = F::one(); for (int j = 0; j < k; j++) r = r * two; return r; };
    F e = F::zero();
    for (int i = 0; i < n_inst; i++) e += coeff[i] * claim[i] * pow2(max_rounds - nr[i]);
    F r_prev = F::zero();
    const ScLagrange<F> lagrange(DEG1);
    for (int round = 0; round < max_rounds; round++) {
        const int remaining = max_rounds - round;
        for (int i = 0; i < n_inst; i++) {
            if (remaining > nr[i]) continue;
            ScArgs<F> &a = args[i];
            const int grid = sc_grid(cur[i] / 2, 256);
            if (remaining == nr[i]) {                  // the instance's first round: evaluate only
                a.len = cur[i];
                sc_round_kernel<F, KIND, false><<<grid, 256, 0, s>>>(a);
            } else {                                   // bind the previous challenge, then evaluate
                a.len = cur[i] << 1;
                a.r = r_prev;
                sc_round_kernel<F, KIND, true><<<grid, 256, 0, s>>>(a);
            }
        }
        LURK_CUDA_TRY(cudaGetLastError());
        LURK_CUDA_TRY(cudaStreamSynchronize(s));       // the result slots are pinned host memory
        F comb[E];
        for (int t = 0; t < E; t++) comb[t] = F::zero();
        for (int i = 0; i < n_inst; i++) {
            if (remaining > nr[i]) {
                const F c = coeff[i] * claim[i] * pow2(remaining - nr[i] - 1);
                for (int t = 0; t < E; t++) comb[t] += c;
            } else {
                const F *res = static_cast<const F *>(sc.pinned) + 4 * i;
                for (int t = 0; t < E; t++) comb[t] += coeff[i] * res[t];
            }
        }
        // s(0), s(1) = claim - s(0), s(2)[, s(3)]
        F evals[DEG1];
        evals[0] = comb[0];
        evals[1] = e - comb[0];
        for (int t = 1; t < E; t++) evals[t + 1] = comb[t];
        uint8_t msg[DEG1 * 32], rbytes[32];
        for (int t = 0; t < DEG1; t++) fe_out(evals[t], fmt, msg + 32 * t);
        if (round_evals) memcpy(round_evals + (size_t)round * DEG1 * 32, msg, DEG1 * 32);
        int rc = challenge(user, round, msg, DEG1 * 32, rbytes);
        if (rc != 0) { set_error("challenge callback failed in round %d (%d)", round, rc); return LURK_ERR_ARG; }
        F r;
        if (!fe_in(rbytes, fmt, r)) { set_error("challenge of round %d is not reduced", round); return LURK_ERR_RANGE; }
        if (challenges) memcpy(challenges + (size_t)round * 32, rbytes, 32);
        e = lagrange.eval(evals, r);
        r_prev = r;
        for (int i = 0; i < n_inst; i++)
            if (remaining <= nr[i]) cur[i] >>= 1;
    }
    // final evaluations: the last bind of every instance that took part; instances without variables are their single element
    for (int i = 0; i < n_inst; i++) {
        if (nr[i] == 0) {
            for (int k = 0; k < K; k++) LURK_CUDA_TRY(cudaMemcpyAsync(sc.result + 4 * i + k, args[i].poly[k], sizeof(F), cudaMemcpyDeviceToHost, s));
        } else {
            args[i].len = 2;
            args[i].r = r_prev;
            sc_final_bind_kernel<F><<<1, 32, 0, s>>>(args[i], K);
        }
    }
    LURK_CUDA_TRY(cudaGetLastError());
    LURK_CUDA_TRY(cudaStreamSynchronize(s));
    if (final_evals)
        for (int i = 0; i < n_inst; i++)
            for (int k = 0; k < K; k++) fe_out(static_cast<const F *>(sc.pinned)[4 * i + k], fmt, final_evals + 32 * (i * K + k));
    return LURK_OK;
}

template <class F>
static int eq_launch(const EqArgs<F> &a, F *out, int to_canonical, cudaStream_t s) {
    const int l = a.l;
    switch (std::min(l, 4)) {
        case 0: eq_kernel<F, 0><<<1, 128, 0, s>>>(a, out, to_canonical); break;
        case 1: eq_kernel<F, 1><<<1, 128, 0, s>>>(a, out, to_canonical); break;
        case 2: eq_kernel<F, 2><<<1, 128, 0, s>>>(a, out, to_canonical); break;
        case 3: eq_kernel<F, 3><<<1, 128, 0, s>>>(a, out, to_canonical); break;
        default: eq_kernel<F, 4><<<sc_grid((size_t)1 << (l - 4), 128), 128, 0, s>>>(a, out, to_canonical); break;
    }
    LURK_CUDA_TRY(cudaGetLastError());
    return LURK_OK;
}

template <class F>
static int eq_evals(const uint8_t *tau, int l, void *d_out, int fmt, cudaStream_t s) {
    EqArgs<F> a;
    memset(&a, 0, sizeof a);
    a.l = l;
    for (int j = 0; j < l; j++) {
        if (!fe_in(tau + 32 * j, fmt, a.tau[j])) { set_error("tau[%d] is not reduced", j); return LURK_ERR_RANGE; }
        a.one_minus[j] = F::one() - a.tau[j];
    }
    return eq_launch<F>(a, static_cast<F *>(d_out), fmt == LURK_FMT_CANONICAL, s);
}

// ------------------------------------------------------------------------------------------------ batch_eval_reduce
// The joint polynomial of the reduction in one pass: out[k] = sum_{t : k < len_t} w_t P_t[k] for k < out_len.  The terms are sorted by
// length, longest first, so a thread stops at the first one that no longer reaches its index; every output is written once and every
// input element read once: 32 (sum_t len_t + out_len) bytes, one product per term -- HBM-bound.  The table rides in the kernel
// parameters (60 x 48 bytes), read as uniform constant-bank loads.
template <class F>
struct CombineArgs {
    struct Term { const F *poly; size_t len; F w; } term[SC_MAX_INSTANCES];
    int n;
    size_t out_len;
};

template <class F>
__global__ void __launch_bounds__(256) poly_combine_kernel(const __grid_constant__ CombineArgs<F> a, F *__restrict__ out) {
    for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < a.out_len; k += (size_t)gridDim.x * blockDim.x) {
        F acc = F::zero();
        for (int t = 0; t < a.n && k < a.term[t].len; t++) acc += a.term[t].w * load_fe<F>(a.term[t].poly + k);
        store_fe(out + k, acc);
    }
}

// the sum-check's rounds 0 .. m-1 are rounds 1 .. m of the reduction's transcript
struct ShiftedChallenge { lurk_challenge_fn fn; void *user; };
static int shifted_challenge(void *user, int round, const uint8_t *message, size_t message_len, uint8_t challenge_out[32]) {
    const ShiftedChallenge *c = static_cast<const ShiftedChallenge *>(user);
    return c->fn(c->user, round + 1, message, message_len, challenge_out);
}

// Arecibo's batch_eval_reduce (spartan/mod.rs in the public crate, not under the reference checkout; restated): claims P_i(x_i) = e_i
// -> rho; the batched quadratic sum-check of sum_i rho^i sum_y P_i(y) eq(x_i, y), instance i joining in round m - n_i, gives r and the
// L_i = P_i(r[m - n_i:]); -> gamma.  PolyEvalInstance / PolyEvalWitness::batch_diff_size then treat P_i as zero-padded at the top to
// 2^m elements, so the joint claim is sum_i gamma^i prod_{j < m - n_i} (1 - r_j) L_i about sum_i gamma^i P_i.
template <class F>
static int batch_eval_reduce(int n, const void *const *d_polys, const int *nv, const uint8_t *points, const uint8_t *evals_in,
                             lurk_challenge_fn challenge, void *user, uint8_t *round_evals, uint8_t *r_out, uint8_t *claims_left,
                             uint8_t *weights, uint8_t *joint_eval, void *d_joint, int fmt, cudaStream_t s) {
    int m = 0;
    size_t total = 0, at = 0;
    std::vector<EqArgs<F>> eq(n);
    for (int i = 0; i < n; i++) {
        F e;
        if (!fe_in(evals_in + 32 * i, fmt, e)) { set_error("evaluation %d is not reduced", i); return LURK_ERR_RANGE; }
        if (nv[i] > 32) { set_error("claim %d has %d variables; the eq table takes at most 32", i, nv[i]); return LURK_ERR_ARG; }
        memset(&eq[i], 0, sizeof(EqArgs<F>));
        eq[i].l = nv[i];
        for (int j = 0; j < nv[i]; j++, at++) {
            if (!fe_in(points + 32 * at, fmt, eq[i].tau[j])) { set_error("point %d, coordinate %d is not reduced", i, j); return LURK_ERR_RANGE; }
            eq[i].one_minus[j] = F::one() - eq[i].tau[j];
        }
        m = std::max(m, nv[i]);
        total += (size_t)1 << nv[i];
    }
    uint8_t cb[32];
    F rho, gamma;
    int rc = challenge(user, 0, evals_in, (size_t)n * 32, cb);
    if (rc != 0) { set_error("challenge callback failed in round 0 (%d)", rc); return LURK_ERR_ARG; }
    if (!fe_in(cb, fmt, rho)) { set_error("challenge of round 0 is not reduced"); return LURK_ERR_RANGE; }

    // working copies (the sum-check binds in place) and eq(x_i) beside them: [P_0 .. P_{n-1} | eq_0 .. eq_{n-1}]
    StreamBuf work;
    LURK_TRY(work.alloc(2 * total * sizeof(F), s));
    F *base = static_cast<F *>(work.p);
    std::vector<void *> polys(2 * n);
    std::vector<uint8_t> coeffs(32 * (size_t)n);
    F c = F::one();
    for (size_t i = 0, off = 0; i < (size_t)n; off += (size_t)1 << nv[i], i++) {
        const size_t len = (size_t)1 << nv[i];
        polys[2 * i] = base + off;
        polys[2 * i + 1] = base + total + off;
        LURK_CUDA_TRY(cudaMemcpyAsync(polys[2 * i], d_polys[i], len * sizeof(F), cudaMemcpyDeviceToDevice, s));
        LURK_TRY(eq_launch<F>(eq[i], static_cast<F *>(polys[2 * i + 1]), 0, s));
        fe_out(c, fmt, coeffs.data() + 32 * i);
        c = c * rho;
    }
    std::vector<uint8_t> r_bytes(32 * (size_t)std::max(m, 1)), fin(64 * (size_t)n);
    ShiftedChallenge shifted{challenge, user};
    LURK_TRY((sumcheck_prove_batch<F, SC_QUAD>(n, polys.data(), nv, evals_in, coeffs.data(), shifted_challenge, &shifted, round_evals,
                                               r_bytes.data(), fin.data(), fmt, s)));

    // round m + 1: the L_i -> gamma
    std::vector<uint8_t> left(32 * (size_t)n);
    for (int i = 0; i < n; i++) memcpy(left.data() + 32 * i, fin.data() + 64 * i, 32);
    rc = challenge(user, m + 1, left.data(), left.size(), cb);
    if (rc != 0) { set_error("challenge callback failed in round %d (%d)", m + 1, rc); return LURK_ERR_ARG; }
    if (!fe_in(cb, fmt, gamma)) { set_error("challenge of round %d is not reduced", m + 1); return LURK_ERR_RANGE; }

    std::vector<F> r(m);
    for (int j = 0; j < m; j++) fe_in(r_bytes.data() + 32 * j, fmt, r[j]);
    CombineArgs<F> args;
    memset(&args, 0, sizeof args);
    args.n = n;
    args.out_len = (size_t)1 << m;
    std::vector<int> order(n);
    for (int i = 0; i < n; i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return nv[a] > nv[b]; });
    std::vector<F> w(n);
    F joint = F::zero();
    w[0] = F::one();
    for (int i = 1; i < n; i++) w[i] = w[i - 1] * gamma;
    for (int i = 0; i < n; i++) {
        F L, scale = w[i];
        fe_in(left.data() + 32 * i, fmt, L);
        for (int j = 0; j < m - nv[i]; j++) scale = scale * (F::one() - r[j]);
        joint += scale * L;
    }
    for (int t = 0; t < n; t++) {
        const int i = order[t];
        args.term[t].poly = static_cast<const F *>(d_polys[i]);
        args.term[t].len = (size_t)1 << nv[i];
        args.term[t].w = w[i];
    }
    poly_combine_kernel<F><<<sc_grid(args.out_len, 256), 256, 0, s>>>(args, static_cast<F *>(d_joint));
    LURK_CUDA_TRY(cudaGetLastError());
    if (r_out) memcpy(r_out, r_bytes.data(), 32 * (size_t)m);
    if (claims_left) memcpy(claims_left, left.data(), left.size());
    if (weights)
        for (int i = 0; i < n; i++) fe_out(w[i], fmt, weights + 32 * i);
    if (joint_eval) fe_out(joint, fmt, joint_eval);
    return LURK_OK;
}

}  // namespace lurk
