// N4 -- the compressed verifier (include/lurk_b200.h, "Compressed verifier"): CompressedSNARK::verify (reference src/proof/nova.rs:358-373,
// supernova.rs:304-317) as one C-ABI call, for the proof lurk_compress_prove_dev writes.  Per circuit: the Spartan verifier of spartan.cu
// (its one device step is the matrix-evaluation pass), then the opening: the joint commitment sum_i weights_i C_i and the inner-product
// verifier of ipa.cu on eq(r) in stream-ordered scratch, or HyperKZG's verifier -- the fold consistency of the evaluations and the two G1
// points of the batched pairing check, the joint commitment folded into the first; the pairing itself is the caller's callback.  The point
// combinations go through point_combination_groups (pointcomb.cu): the device for the long ones, the host Straus for the short.  The secondary
// circuit runs on a pooled library thread and a stream forked from the caller's while the primary runs on the calling thread -- Arecibo's
// rayon::join of S1::verify and S2::verify.  No kernels of its own.
#include "msm_impl.cuh"
#include "pcs.cuh"
#include "sc_scratch.cuh"
#include "worker.cuh"

#include <mutex>
#include <string>
#include <vector>

namespace lurk {

int spartan_verify_precheck(int n, lurk_spartan_ctx *const *ctxs, const uint8_t *u, const uint8_t *const *X, const lurk_spartan_proof *proof,
                            int rounds_fmt, lurk_spartan_challenge_fn fn, const int *accepted, int fmt);                              // spartan.cu
int spartan_verify_checked(int n, lurk_spartan_ctx *const *ctxs, const uint8_t *u, const uint8_t *const *X, lurk_spartan_proof *proof, int rounds_fmt,
                           lurk_spartan_challenge_fn fn, void *user, int *accepted, int fmt, cudaStream_t s, bool batched);            // spartan.cu

namespace {

constexpr int CV_MAX_PRIMARY = 30;

// one circuit of a call, as the checks leave it
struct Side {
    const char *name;
    int idx, n = 0, field = 0, curve = 0, m = 0;
    bool batched = false;
    std::vector<lurk_spartan_ctx *> sp;
    const lurk_compress_vk_pcs *pcs = nullptr;
    const uint8_t *u = nullptr;
    std::vector<const uint8_t *> X, comms;       // comms = [comm_W_0 .., comm_E_0 ..]
    const lurk_compress_circuit_proof *proof = nullptr;
};

struct Transcript { lurk_compress_challenge_fn fn; void *user; int circuit, round_offset; };
int snark_challenge(void *user, int phase, int round, const uint8_t *msg, size_t len, uint8_t out[32]) {
    const Transcript *t = static_cast<const Transcript *>(user);
    return t->fn(t->user, t->circuit, phase, round, msg, len, out);
}
int pcs_challenge(void *user, int round, const uint8_t *msg, size_t len, uint8_t out[32]) {
    const Transcript *t = static_cast<const Transcript *>(user);
    return t->fn(t->user, t->circuit, LURK_SPARTAN_PCS, round + t->round_offset, msg, len, out);
}
template <class F>
int ask_pcs(const Transcript &t, int round, const uint8_t *msg, size_t len, int fmt, F &out) {
    uint8_t b[32];
    const int rc = t.fn(t.user, t.circuit, LURK_SPARTAN_PCS, round, msg, len, b);
    if (rc != 0) { set_error("challenge callback failed in phase %d, round %d (%d)", LURK_SPARTAN_PCS, round, rc); return LURK_ERR_ARG; }
    if (!fe_in(b, fmt, out)) { set_error("challenge of phase %d, round %d is not reduced", LURK_SPARTAN_PCS, round); return LURK_ERR_RANGE; }
    return LURK_OK;
}

bool all_reduced(int field, const uint8_t *p, size_t count, int fmt) {
    return dispatch_field(field, [&](auto f) {
        using F = decltype(f);
        F x;
        for (size_t k = 0; k < count; k++)
            if (!fe_in(p + 32 * k, fmt, x)) return 0;
        return 1;
    }) == 1;
}

bool points_at(int curve, const uint8_t *p, size_t count, int fmt) {
    for (size_t k = 0; k < count; k++) {
        const uint8_t *q = p + 96 * k;
        if (!points_valid(curve, &q, 1, fmt)) return false;
    }
    return true;
}

// the checks that read the contexts and keys (LURK_ERR_ARG), after the GPU check, before any range check
int check_side(Side &c, int fmt) {
    c.field = -1;
    for (int i = 0; i < c.n; i++) {
        int field = -1, lr = 0, lv = 0;
        LURK_TRY(lurk_spartan_ctx_info(c.sp[i], &field, &lr, &lv, nullptr));
        if (i && field != c.field) { set_error("%s context %d is over field %d, context 0 over field %d", c.name, i, field, c.field); return LURK_ERR_ARG; }
        c.field = field;
        c.m = std::max(c.m, std::max(lr, lv));
    }
    c.curve = c.field;                    // LURK_CURVE_* whose scalar field is LURK_FIELD_* of the same number
    const lurk_compress_circuit_proof &p = *c.proof;
    if (c.pcs->kind == LURK_PCS_IPA) {
        lurk_msm_ctx *ck = c.pcs->ck;
        int dev = -1;
        LURK_CUDA_TRY(cudaGetDevice(&dev));
        if (ck->curve_id != c.curve) { set_error("%s key is on curve %d, the circuit's field %d needs curve %d", c.name, ck->curve_id, c.field, c.curve); return LURK_ERR_ARG; }
        if (ck->n < ((size_t)1 << c.m)) { set_error("%s key has %zu bases, the joint polynomial needs 2^%d", c.name, ck->n, c.m); return LURK_ERR_ARG; }
        if (ck->device != dev) { set_error("%s key belongs to device %d, device %d is current", c.name, ck->device, dev); return LURK_ERR_ARG; }
        if (ck->pending) { set_error("%s key: a launch is pending on the key context", c.name); return LURK_ERR_ARG; }
        if (!p.L || !p.R || !p.a_final) { set_error("%s circuit: null L, R or a_final", c.name); return LURK_ERR_ARG; }
    } else if ((c.m > 1 && !p.com) || !p.v || !p.w) {
        set_error("%s circuit: null com, v or w", c.name);
        return LURK_ERR_ARG;
    }
    return LURK_OK;
}

// the range checks (LURK_ERR_RANGE) of one circuit: u, X, the Spartan proof, the commitments, the opening's fields, the key's points
int check_side_ranges(const Side &c, int rounds_fmt, int fmt) {
    const int dummy = 0;
    LURK_TRY(spartan_verify_precheck(c.n, c.sp.data(), c.u, c.X.data(), &c.proof->snark, rounds_fmt, snark_challenge, &dummy, fmt));
    if (!points_valid(c.curve, c.comms.data(), (int)c.comms.size(), fmt)) {
        set_error("%s circuit: a commitment is not a point of the header's form on curve %d", c.name, c.curve);
        return LURK_ERR_RANGE;
    }
    const lurk_compress_circuit_proof &p = *c.proof;
    const size_t m = (size_t)c.m;
    if (c.pcs->kind == LURK_PCS_IPA) {
        if (!points_at(c.curve, p.L, m, fmt) || !points_at(c.curve, p.R, m, fmt)) { set_error("%s circuit: an L or R is not a point of the header's form", c.name); return LURK_ERR_RANGE; }
        if (!all_reduced(c.field, p.a_final, 1, fmt)) { set_error("%s circuit: a_final is not reduced", c.name); return LURK_ERR_RANGE; }
        if (!affine_valid(c.curve, c.pcs->ck_c, fmt)) { set_error("%s ck_c is not a reduced point on the curve", c.name); return LURK_ERR_RANGE; }
    } else {
        if (!points_at(c.curve, p.com, m - 1, fmt)) { set_error("%s circuit: a com is not a point of the header's form", c.name); return LURK_ERR_RANGE; }
        if (!points_at(c.curve, p.w, 3, fmt)) { set_error("%s circuit: a w is not a point of the header's form", c.name); return LURK_ERR_RANGE; }
        if (!all_reduced(c.field, p.v, 3 * m, fmt)) { set_error("%s circuit: an element of v is not reduced", c.name); return LURK_ERR_RANGE; }
        if (!affine_valid(c.curve, c.pcs->g, fmt)) { set_error("%s g is not a reduced point on the curve", c.name); return LURK_ERR_RANGE; }
    }
    return LURK_OK;
}

// HyperKZG's verifier (provider::hyperkzg::EvaluationEngine::verify) on the host, the pairing left to the callback
// (the joint commitment comm = sum_i weights_i C_i never reaches HyperKZG's transcript: its term dsum comm of P is taken as the terms
// dsum weights_i C_i)
template <class F>
int hyperkzg_verify(const Side &c, const Transcript &t, const uint8_t *weights, const uint8_t *r_bytes, const uint8_t je_bytes[32],
                    lurk_pairing_check_fn pairing, int fmt, lurk_compress_verdict &v, cudaStream_t s) {
    const lurk_compress_circuit_proof &p = *c.proof;
    const int l = c.m;
    F r, q, d, je;
    LURK_TRY(ask_pcs<F>(t, 0, p.com, (size_t)(l - 1) * 96, fmt, r));
    std::vector<F> x(l), val(3 * (size_t)l);
    for (int i = 0; i < l; i++) fe_in(r_bytes + 32 * i, fmt, x[i]);
    for (size_t k = 0; k < val.size(); k++) fe_in(p.v + 32 * k, fmt, val[k]);
    fe_in(je_bytes, fmt, je);
    // 2 r Y[i+1] = r (1 - x) (v0[i] + v1[i]) + x (v0[i] - v1[i]), x = point[l - 1 - i], Y = v[2] | joint_eval
    const F *v0 = val.data(), *v1 = v0 + l, *v2 = v1 + l;
    const F two_r = r + r;
    v.eval_ok = 1;
    for (int i = 0; i < l && v.eval_ok; i++) {
        const F &xi = x[l - 1 - i];
        const F y = i + 1 < l ? v2[i + 1] : je;
        v.eval_ok = two_r * y == r * (F::one() - xi) * (v0[i] + v1[i]) + xi * (v0[i] - v1[i]);
    }
    if (!v.eval_ok) return LURK_OK;
    LURK_TRY(ask_pcs<F>(t, 1, p.v, 3 * (size_t)l * 32, fmt, q));
    LURK_TRY(ask_pcs<F>(t, 2, p.w, 3 * 96, fmt, d));
    // P = sum_t d^t (B - B(u_t) G + u_t w_t) over [com_0 = comm = sum_i weights_i C_i, com_1 .., G, w_0, w_1, w_2];  Q = sum_t d^t w_t
    const F u[3] = {r, r.neg(), r.sqr()}, dt[3] = {F::one(), d, d.sqr()};
    const F dsum = dt[0] + dt[1] + dt[2];
    std::vector<const uint8_t *> pts(c.comms);
    std::vector<F> sc;
    for (size_t i = 0; i < c.comms.size(); i++) {
        F wi;
        fe_in(weights + 32 * i, fmt, wi);
        sc.push_back(dsum * wi);
    }
    F qj = F::one(), bu = F::zero();
    for (int j = 0; j < l; j++, qj = qj * q) {
        if (j) {
            pts.push_back(p.com + 96 * (size_t)(j - 1));
            sc.push_back(dsum * qj);
        }
        for (int k = 0; k < 3; k++) bu += dt[k] * qj * val[(size_t)k * l + j];
    }
    uint8_t g96[96] = {0};
    memcpy(g96, c.pcs->g, 64);
    bool identity = true;
    for (int k = 0; k < 64; k++) identity &= c.pcs->g[k] == 0;
    if (!identity) LURK_TRY(dispatch_field(c.curve ^ 1, [&](auto f) { fe_out(decltype(f)::one(), fmt, g96 + 64); return LURK_OK; }));
    pts.push_back(g96);
    sc.push_back(bu.neg());
    for (int k = 0; k < 3; k++) {
        pts.push_back(p.w + 96 * k);
        sc.push_back(dt[k] * u[k]);
    }
    std::vector<uint8_t> sb(32 * sc.size());
    for (size_t k = 0; k < sc.size(); k++) fe_out(sc[k], fmt, sb.data() + 32 * k);
    uint8_t P[96], Q[96], db[96];
    for (int k = 0; k < 3; k++) fe_out(dt[k], fmt, db + 32 * k);
    const PointGroup pq[2] = {{pts.data(), sb.data(), (int)pts.size(), P}, {pts.data() + pts.size() - 3, db, 3, Q}};
    LURK_TRY(point_combination_groups(c.curve, pq, 2, fmt, false, s));
    int holds = 0;
    const int rc = pairing(t.user, c.idx, P, Q, &holds);
    if (rc != 0) { set_error("pairing callback failed (%d)", rc); return LURK_ERR_ARG; }
    v.opening_ok = holds != 0;
    return LURK_OK;
}

// steps 1 to 3 of one circuit on stream s; the verdict's fields stay -1 past the first failing check
int verify_side(const Side &c, lurk_compress_challenge_fn fn, lurk_pairing_check_fn pairing, void *user, int rounds_fmt, int fmt, cudaStream_t s,
                lurk_compress_verdict &v) {
    Transcript t{fn, user, c.idx, 0};
    std::vector<uint8_t> r(32 * (size_t)c.m), weights(64 * (size_t)c.n);
    uint8_t je[32];
    lurk_spartan_proof sp = c.proof->snark;       // read; the derived fields go to the call's own buffers, never the caller's
    sp.r_x = sp.r_y = nullptr;
    sp.r = r.data();
    sp.weights = weights.data();
    sp.joint_eval = je;
    int acc = 0;
    LURK_TRY(spartan_verify_checked(c.n, c.sp.data(), c.u, c.X.data(), &sp, rounds_fmt, snark_challenge, &t, &acc, fmt, s, c.batched));
    v.snark_ok = acc;
    if (!acc) return LURK_OK;
    if (c.pcs->kind == LURK_PCS_HYPERKZG)
        return dispatch_field(c.field, [&](auto f) { return hyperkzg_verify<decltype(f)>(c, t, weights.data(), r.data(), je, pairing, fmt, v, s); });
    // IPA: comm | joint_eval -> the scale of ck_c;  b = eq(r)
    uint8_t comm[96];
    const PointGroup joint{c.comms.data(), weights.data(), (int)c.comms.size(), comm};
    LURK_TRY(point_combination_groups(c.curve, &joint, 1, fmt, false, s));
    uint8_t msg[128], rb[32], gc[64];
    memcpy(msg, comm, 96);
    memcpy(msg + 96, je, 32);
    const int rc = fn(user, c.idx, LURK_SPARTAN_PCS, 0, msg, sizeof msg, rb);
    if (rc != 0) { set_error("challenge callback failed in phase %d, round 0 (%d)", LURK_SPARTAN_PCS, rc); return LURK_ERR_ARG; }
    LURK_TRY(scale_affine(c.curve, c.pcs->ck_c, rb, fmt, gc));
    StreamBuf b;
    LURK_TRY(b.alloc((size_t)32 << c.m, s));
    LURK_TRY(dispatch_field(c.field, [&](auto f) {
        using F = decltype(f);
        std::vector<uint8_t> rm(r.size());
        F x;
        for (int j = 0; j < c.m; j++) { fe_in(r.data() + 32 * j, fmt, x); fe_out(x, LURK_FMT_MONTGOMERY, rm.data() + 32 * j); }
        return lurk_eq_evals_dev(c.field, rm.data(), c.m, b.p, LURK_FMT_MONTGOMERY, s);
    }));
    v.eval_ok = 1;
    t.round_offset = 1;
    const lurk_compress_circuit_proof &p = *c.proof;
    LURK_TRY(ipa_verify_checked(c.curve, c.pcs->ck, gc, comm, je, b.p, c.m, p.L, p.R, p.a_final, pcs_challenge, &t, &acc, fmt, s));
    v.opening_ok = acc;
    return LURK_OK;
}

// idle secondary threads, kept for the life of the process so that each keeps its reduction scratch between calls
struct WorkerPool {
    std::mutex mu;
    std::vector<Worker *> idle;
    Worker *acquire() {
        std::lock_guard<std::mutex> g(mu);
        if (idle.empty()) return new Worker();
        Worker *w = idle.back();
        idle.pop_back();
        return w;
    }
    void release(Worker *w) {
        std::lock_guard<std::mutex> g(mu);
        idle.push_back(w);
    }
};
WorkerPool &worker_pool() {
    static WorkerPool *pool = new WorkerPool();     // never destroyed: its threads wait idle until the process ends
    return *pool;
}

int bad_pcs(const char *name, const lurk_compress_vk_pcs *pcs, lurk_pairing_check_fn pairing) {
    if (!pcs) { set_error("%s: null evaluation engine", name); return LURK_ERR_ARG; }
    if (pcs->kind == LURK_PCS_IPA) {
        if (!pcs->ck || !pcs->ck_c) { set_error("%s: IPA needs ck and ck_c", name); return LURK_ERR_ARG; }
    } else if (pcs->kind == LURK_PCS_HYPERKZG) {
        if (!pcs->g) { set_error("%s: HyperKZG needs g", name); return LURK_ERR_ARG; }
        if (!pairing) { set_error("%s: HyperKZG needs a pairing callback", name); return LURK_ERR_ARG; }
    } else {
        set_error("%s: unknown evaluation engine %d", name, pcs->kind);
        return LURK_ERR_ARG;
    }
    return LURK_OK;
}

}  // namespace
}  // namespace lurk

using namespace lurk;

extern "C" {

int lurk_compress_verify(int n_primary, lurk_spartan_ctx *const *primary, lurk_spartan_ctx *secondary, const lurk_compress_vk_pcs *pcs_primary,
                         const lurk_compress_vk_pcs *pcs_secondary, const uint8_t *u, const uint8_t *const *X, const uint8_t *const *comm_W,
                         const uint8_t *const *comm_E, const uint8_t u2[32], const uint8_t *X2, const uint8_t comm_W2[96], const uint8_t comm_E2[96],
                         const lurk_compress_proof *proof, int rounds_fmt, lurk_compress_challenge_fn challenge, lurk_pairing_check_fn pairing,
                         void *user, int flags, lurk_compress_verdict out[2], int *accepted, int fmt, void *stream) {
    // host-only checks that read no context
    if (!out || !accepted) { set_error("null verdict array or accepted"); return LURK_ERR_ARG; }
    *accepted = 0;
    for (int k = 0; k < 2; k++) out[k].snark_ok = out[k].eval_ok = out[k].opening_ok = -1;
    if (n_primary < 1 || n_primary > CV_MAX_PRIMARY) { set_error("1..%d primary contexts, got %d", CV_MAX_PRIMARY, n_primary); return LURK_ERR_ARG; }
    if (flags & ~(LURK_COMPRESS_SEQUENTIAL | LURK_COMPRESS_BATCHED)) { set_error("unknown flags 0x%x", flags); return LURK_ERR_ARG; }
    if (!(flags & LURK_COMPRESS_BATCHED) && n_primary != 1) { set_error("a plain (Nova) primary proof has one instance, got %d", n_primary); return LURK_ERR_ARG; }
    if (!primary || !secondary) { set_error("null Spartan context array or secondary context"); return LURK_ERR_ARG; }
    LURK_TRY(bad_pcs("primary", pcs_primary, pairing));
    LURK_TRY(bad_pcs("secondary", pcs_secondary, pairing));
    if (!challenge) { set_error("null challenge callback"); return LURK_ERR_ARG; }
    if (!proof) { set_error("null proof"); return LURK_ERR_ARG; }
    if (!u || !X || !comm_W || !comm_E) { set_error("null primary instance array"); return LURK_ERR_ARG; }
    for (int i = 0; i < n_primary; i++)
        if (!comm_W[i] || !comm_E[i]) { set_error("null comm_W / comm_E of primary instance %d", i); return LURK_ERR_ARG; }
    if (!u2 || !comm_W2 || !comm_E2) { set_error("null u2 / comm_W2 / comm_E2 of the secondary instance"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    if (rounds_fmt != LURK_SPARTAN_ROUNDS_EVALS && rounds_fmt != LURK_SPARTAN_ROUNDS_COMPRESSED) { set_error("unknown rounds_fmt %d", rounds_fmt); return LURK_ERR_ARG; }
    for (int i = 0; i < n_primary; i++) {
        if (!primary[i]) { set_error("null primary context %d", i); return LURK_ERR_ARG; }
        if (primary[i] == secondary) { set_error("primary context %d is also the secondary context", i); return LURK_ERR_ARG; }
        for (int k = 0; k < i; k++)
            if (primary[k] == primary[i]) { set_error("primary contexts %d and %d are the same context", k, i); return LURK_ERR_ARG; }
    }
    if (pcs_primary->kind == LURK_PCS_IPA && pcs_secondary->kind == LURK_PCS_IPA && pcs_primary->ck == pcs_secondary->ck) {
        set_error("the primary and the secondary key are the same context");
        return LURK_ERR_ARG;
    }
    LURK_TRY(require_gpu());
    Side c[2];
    c[0].name = "primary";
    c[0].idx = 0;
    c[0].n = n_primary;
    c[0].batched = (flags & LURK_COMPRESS_BATCHED) != 0;
    c[0].sp.assign(primary, primary + n_primary);
    c[0].pcs = pcs_primary;
    c[0].u = u;
    c[0].X.assign(X, X + n_primary);
    c[0].comms.assign(comm_W, comm_W + n_primary);
    c[0].comms.insert(c[0].comms.end(), comm_E, comm_E + n_primary);
    c[0].proof = &proof->primary;
    c[1].name = "secondary";
    c[1].idx = 1;
    c[1].n = 1;
    c[1].sp = {secondary};
    c[1].pcs = pcs_secondary;
    c[1].u = u2;
    c[1].X = {X2};
    c[1].comms = {comm_W2, comm_E2};
    c[1].proof = &proof->secondary;
    // the checks that read the contexts and keys, then every range check: all before the first callback and any device work
    for (Side &s : c) LURK_TRY(check_side(s, fmt));
    if (c[1].field != (c[0].field ^ 1)) {
        set_error("the secondary circuit is over field %d; the cycle partner of the primary's field %d is %d", c[1].field, c[0].field, c[0].field ^ 1);
        return LURK_ERR_ARG;
    }
    for (const Side &s : c) LURK_TRY(check_side_ranges(s, rounds_fmt, fmt));

    const bool sequential = (flags & LURK_COMPRESS_SEQUENTIAL) != 0;
    const cudaStream_t s0 = static_cast<cudaStream_t>(stream);
    int dev = 0;
    LURK_CUDA_TRY(cudaGetDevice(&dev));
    StreamGuard side;
    EventGuard fork, join;
    if (!sequential) {
        // the secondary's stream follows whatever the caller queued on `stream` before the call
        LURK_TRY(side.create());
        LURK_TRY(fork.create());
        LURK_TRY(join.create());
        LURK_CUDA_TRY(cudaEventRecord(fork.e, s0));
        LURK_CUDA_TRY(cudaStreamWaitEvent(side.s, fork.e, 0));
    }
    const cudaStream_t st[2] = {s0, sequential ? s0 : side.s};
    int rc[2] = {LURK_OK, LURK_OK};
    std::string msg[2];
    auto run = [&](int k) {
        cudaSetDevice(dev);
        rc[k] = verify_side(c[k], challenge, pairing, user, rounds_fmt, fmt, st[k], out[k]);
        if (rc[k] != LURK_OK) {
            msg[k] = lurk_last_error();
            cudaStreamSynchronize(st[k]);        // nothing of a failed circuit stays queued behind the call
            cudaGetLastError();
        }
    };
    if (sequential) {
        run(0);
        if (rc[0] == LURK_OK) run(1);
    } else {
        Worker *w = worker_pool().acquire();
        w->post([&] { run(1); });
        run(0);
        w->wait();
        worker_pool().release(w);
        // the secondary's stream joins the caller's, errors included
        cudaEventRecord(join.e, side.s);
        cudaStreamWaitEvent(s0, join.e, 0);
    }
    for (int k = 0; k < 2; k++)
        if (rc[k] != LURK_OK) {
            set_error("%s circuit: %s", c[k].name, msg[k].c_str());
            return rc[k];
        }
    int all = 1;
    for (int k = 0; k < 2; k++) all &= out[k].snark_ok == 1 && out[k].eval_ok == 1 && out[k].opening_ok == 1;
    *accepted = all;
    return LURK_OK;
}

int lurk_point_combination(int curve_id, const uint8_t *points_xyz, const uint8_t *scalars, size_t count, int fmt, uint8_t out_xyz[96]) {
    if (!out_xyz || (count && (!points_xyz || !scalars))) { set_error("null argument"); return LURK_ERR_ARG; }
    if (count > (1u << 24)) { set_error("at most 2^24 terms, got %zu", count); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    if (curve_id < LURK_CURVE_BN254_G1 || curve_id > LURK_CURVE_VESTA) { set_error("unknown curve id %d", curve_id); return LURK_ERR_ARG; }
    std::vector<const uint8_t *> pts(count);
    for (size_t k = 0; k < count; k++) pts[k] = points_xyz + 96 * k;
    return point_combination(curve_id, pts.data(), scalars, (int)count, fmt, out_xyz);
}

}  // extern "C"
