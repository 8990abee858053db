// N4 -- the data-parallel half of `compress` behind the C ABI (include/lurk_b200.h, "N4"): sum-check prover rounds over
// device-resident multilinear polynomials and the folding rounds of the inner-product argument, i.e. the loops of Arecibo's
// SumcheckProof::prove_quad / prove_cubic_with_additive_term and InnerProductArgument::prove as RelaxedR1CSSNARK::prove runs
// them (reached from reference src/proof/nova.rs:341-356, supernova.rs:293-317).  The Fiat-Shamir transcript stays with the
// caller: every round hands its message to a callback and gets the challenge back (32 bytes in, <= 192 bytes out per round).
//
// Kernels (all grid-stride, 256-thread CTAs, grid <= 4 CTAs per SM, 128-bit loads / stores of 32-byte elements):
//   sc_round_kernel<KIND, BIND>  one pass per round: [bind the previous challenge into all K polynomials in place] + this round's
//                                s(0), s(2)[, s(3)] -- the bind of round j and the evaluation of round j + 1 read the same data,
//                                fusing them moves 3 n / 2 elements per polynomial and round instead of 2 n (and halves the launches).
//                                Bytes per index pair: K x (4 x 32 read + 2 x 32 written); products: K x 2 + 2 (quad: 4) / 6 (cubic).
//   eq_kernel                    EqPolynomial::evals: 16 outputs per thread (prefix product over the high bits, doubling over the low 4).
//   dot_kernel (sc_scratch.cuh)  inner product (MultilinearPolynomial::evaluate = <Z, eq(r)>, IPA's c_L / c_R).
//   poly_combine_kernel          batch_eval_reduce's joint polynomial sum_i gamma^i P_i in one pass (one read per input, one write per
//                                output) instead of n - 1 AXPY passes over the output.
// The inner-product argument lives in ipa.cu.
// Reductions: per-thread modular sums -> warp shuffles -> shared memory -> one partial per CTA -> the last CTA to finish adds the
// partials (single launch, no second kernel, no atomics on field elements).
#include "sumcheck_impl.cuh"

using namespace lurk;

extern "C" {

int lurk_sumcheck_prove_batch_dev(int field_id, int kind, int n_instances, void *const *d_polys, const int *num_rounds, const uint8_t *claims,
                                  const uint8_t *coeffs, lurk_challenge_fn challenge, void *user, uint8_t *round_evals, uint8_t *challenges,
                                  uint8_t *final_evals, int fmt, void *stream) {
    if (!d_polys || !claims || !challenge || !num_rounds) { set_error("null argument"); return LURK_ERR_ARG; }
    if (kind != LURK_SUMCHECK_QUAD && kind != LURK_SUMCHECK_CUBIC) { set_error("unknown sum-check kind %d", kind); return LURK_ERR_ARG; }
    if (n_instances < 1 || n_instances > SC_MAX_INSTANCES) { set_error("1..%d instances, got %d", SC_MAX_INSTANCES, n_instances); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    const int k = kind == LURK_SUMCHECK_QUAD ? 2 : 4;
    for (int i = 0; i < n_instances; i++) {
        if (num_rounds[i] < 0 || num_rounds[i] > 40) { set_error("bad number of rounds %d (instance %d)", num_rounds[i], i); return LURK_ERR_ARG; }
        for (int j = 0; j < k; j++)
            if (!d_polys[i * k + j]) { set_error("polynomial %d of instance %d is null", j, i); return LURK_ERR_ARG; }
    }
    LURK_TRY(require_gpu());
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    return dispatch_field(field_id, [&](auto f) {
        using F = decltype(f);
        return kind == LURK_SUMCHECK_QUAD
                   ? sumcheck_prove_batch<F, SC_QUAD>(n_instances, d_polys, num_rounds, claims, coeffs, challenge, user, round_evals, challenges, final_evals, fmt, s)
                   : sumcheck_prove_batch<F, SC_CUBIC>(n_instances, d_polys, num_rounds, claims, coeffs, challenge, user, round_evals, challenges, final_evals, fmt, s);
    });
}

int lurk_sumcheck_prove_dev(int field_id, int kind, void *const *d_polys, int num_rounds, const uint8_t claim[32], lurk_challenge_fn challenge,
                            void *user, uint8_t *round_evals, uint8_t *challenges, uint8_t *final_evals, int fmt, void *stream) {
    return lurk_sumcheck_prove_batch_dev(field_id, kind, 1, d_polys, &num_rounds, claim, nullptr, challenge, user, round_evals, challenges, final_evals,
                                         fmt, stream);
}

int lurk_batch_eval_reduce_dev(int field_id, int n_claims, const void *const *d_polys, const int *num_vars, const uint8_t *points,
                               const uint8_t *evals, lurk_challenge_fn challenge, void *user, uint8_t *round_evals, uint8_t *r_out,
                               uint8_t *claims_left, uint8_t *weights, uint8_t joint_eval[32], void *d_joint, int fmt, void *stream) {
    if (!d_polys || !num_vars || !evals || !challenge || !d_joint) { set_error("null argument"); return LURK_ERR_ARG; }
    if (n_claims < 1 || n_claims > SC_MAX_INSTANCES) { set_error("1..%d claims, got %d", SC_MAX_INSTANCES, n_claims); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    int m = 0;
    for (int i = 0; i < n_claims; i++) {
        if (num_vars[i] < 0 || num_vars[i] > 40) { set_error("bad number of variables %d (claim %d)", num_vars[i], i); return LURK_ERR_ARG; }
        if (!d_polys[i]) { set_error("polynomial %d is null", i); return LURK_ERR_ARG; }
        m = std::max(m, num_vars[i]);
    }
    if (m > 0 && !points) { set_error("null points"); return LURK_ERR_ARG; }
    // d_joint is written while the P_i are read: it must not overlap any of them
    const uintptr_t j0 = reinterpret_cast<uintptr_t>(d_joint), j1 = j0 + ((uintptr_t)32 << m);
    for (int i = 0; i < n_claims; i++) {
        const uintptr_t p0 = reinterpret_cast<uintptr_t>(d_polys[i]), p1 = p0 + ((uintptr_t)32 << num_vars[i]);
        if (p0 < j1 && j0 < p1) { set_error("d_joint overlaps polynomial %d", i); return LURK_ERR_ARG; }
    }
    LURK_TRY(require_gpu());
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    return dispatch_field(field_id, [&](auto f) {
        return batch_eval_reduce<decltype(f)>(n_claims, d_polys, num_vars, points, evals, challenge, user, round_evals, r_out, claims_left, weights,
                                              joint_eval, d_joint, fmt, s);
    });
}

int lurk_eq_evals_dev(int field_id, const uint8_t *tau, int num_vars, void *d_out, int fmt, void *stream) {
    if ((num_vars && !tau) || !d_out) { set_error("null argument"); return LURK_ERR_ARG; }
    if (num_vars < 0 || num_vars > 32) { set_error("bad number of variables %d", num_vars); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    return dispatch_field(field_id, [&](auto f) { return eq_evals<decltype(f)>(tau, num_vars, d_out, fmt, static_cast<cudaStream_t>(stream)); });
}

int lurk_inner_product_dev(int field_id, const void *d_a, const void *d_b, size_t n, uint8_t out[32], int fmt, void *stream) {
    if (!out || (n && (!d_a || !d_b))) { set_error("null argument"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    return dispatch_field(field_id, [&](auto f) {
        using F = decltype(f);
        ScScratch<F> sc;
        LURK_TRY(sc.init(s));
        F r = F::zero();
        if (n) LURK_TRY(dot_dev<F>(d_a, d_b, n, &r, sc, s));
        fe_out(r, fmt, out);
        return LURK_OK;
    });
}

}  // extern "C"
