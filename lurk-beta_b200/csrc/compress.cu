// N4 -- the compress context (include/lurk_b200.h, "Compress context"): CompressedSNARK::prove (reference src/proof/nova.rs:341-356,
// supernova.rs:293-317) as one C-ABI call.  Per circuit: the Spartan prover of spartan.cu writes the joint polynomial of batch_eval_reduce
// straight into the opening's arena (P_0 of HyperKZG's fold chain, or a of the inner-product argument), the joint commitment
// sum_i weights_i C_i is formed (2n points, point_combination_groups of pointcomb.cu), and the opening runs on the arena (kzg.cu /
// ipa.cu).  The primary and the secondary circuit run at once on two library-owned host threads -- Arecibo's rayon::join(S1::prove,
// S2::prove) -- which keep their thread-local reduction scratch (sc_scratch.cuh) for the life of the context.  No kernels of its own:
// every device step is one of the existing provers'.
#include "common.cuh"
#include "pcs.cuh"
#include "sc_scratch.cuh"
#include "worker.cuh"

#include <algorithm>
#include <string>
#include <vector>

namespace lurk {

int spartan_prove_checked(int n, lurk_spartan_ctx *const *ctxs, const void *const *d_z, const void *const *d_E, lurk_spartan_challenge_fn fn, void *user,
                          lurk_spartan_proof *out, void *d_joint, int fmt, cudaStream_t s, bool batched);     // spartan.cu
int refuse_verifier_only(const lurk_spartan_ctx *ctx, const char *who);                                       // spartan.cu

constexpr int CP_MAX_PRIMARY = 30;

struct Circuit {
    std::vector<lurk_spartan_ctx *> sp;
    int field = 0, curve = 0, kind = 0, m = 0;     // m = log2 of the joint polynomial's length
    uint8_t ck_c[2][64] = {};                       // IPA: ck_c in LURK_FMT_CANONICAL | LURK_FMT_MONTGOMERY
    MsmCloneGuard ck;                               // the context's own clone of the key; before `arena`, whose clones it must outlive
    PcsArena arena;
};

struct CircuitChallenge { lurk_compress_challenge_fn fn; void *user; int circuit, round_offset; };
static int snark_challenge(void *user, int phase, int round, const uint8_t *msg, size_t len, uint8_t out[32]) {
    const CircuitChallenge *c = static_cast<const CircuitChallenge *>(user);
    return c->fn(c->user, c->circuit, phase, round, msg, len, out);
}
static int pcs_challenge(void *user, int round, const uint8_t *msg, size_t len, uint8_t out[32]) {
    const CircuitChallenge *c = static_cast<const CircuitChallenge *>(user);
    return c->fn(c->user, c->circuit, LURK_SPARTAN_PCS, round + c->round_offset, msg, len, out);
}

// the instances of one circuit in a call
struct CircuitInputs {
    int n;
    const void *const *d_z, *const *d_E;
    const uint8_t *const *comm_W, *const *comm_E;
    bool batched;
};

// RelaxedR1CSSNARK::prove (or the batched one) with the joint polynomial written into the arena, the joint commitment, the opening
static int prove_circuit(Circuit &c, int idx, const CircuitInputs &in, lurk_compress_challenge_fn fn, void *user, lurk_compress_circuit_proof *out,
                         int fmt, cudaStream_t s) {
    const size_t n = (size_t)1 << c.m;
    LURK_TRY(PcsArena::grow(c.arena.polys, 2 * n * 32));
    void *d_joint = c.arena.polys.p;
    // r, weights and joint_eval are needed here whether or not the caller wants them
    lurk_spartan_proof sp;
    if (out) sp = out->snark;
    else memset(&sp, 0, sizeof sp);
    std::vector<uint8_t> r(32 * (size_t)c.m), weights(64 * (size_t)in.n);
    uint8_t je[32];
    uint8_t *want_r = sp.r, *want_w = sp.weights, *want_je = sp.joint_eval;
    sp.r = r.data();
    sp.weights = weights.data();
    sp.joint_eval = je;
    CircuitChallenge cc{fn, user, idx, 0};
    LURK_TRY(spartan_prove_checked(in.n, c.sp.data(), in.d_z, in.d_E, snark_challenge, &cc, &sp, d_joint, fmt, s, in.batched));
    if (want_r) memcpy(want_r, r.data(), r.size());
    if (want_w) memcpy(want_w, weights.data(), weights.size());
    if (want_je) memcpy(want_je, je, 32);
    std::vector<const uint8_t *> pts(2 * (size_t)in.n);
    for (int i = 0; i < in.n; i++) { pts[i] = in.comm_W[i]; pts[in.n + i] = in.comm_E[i]; }
    uint8_t comm[96];
    const PointGroup joint{pts.data(), weights.data(), 2 * in.n, comm};
    LURK_TRY(point_combination_groups(c.curve, &joint, 1, fmt, false, s));
    if (out && out->comm) memcpy(out->comm, comm, 96);
    if (c.kind == LURK_PCS_HYPERKZG)
        return hyperkzg_prove_arena(c.curve, c.ck.c, c.arena, d_joint, r.data(), c.m, pcs_challenge, &cc, out ? out->com : nullptr, out ? out->w : nullptr,
                                    out ? out->v : nullptr, fmt, s);
    // IPA: comm | joint_eval -> the scale of ck_c;  a = the joint polynomial, b = eq(r)
    uint8_t msg[128], rb[32], gc[64];
    memcpy(msg, comm, 96);
    memcpy(msg + 96, je, 32);
    const int rc = fn(user, idx, LURK_SPARTAN_PCS, 0, msg, sizeof msg, rb);
    if (rc != 0) { set_error("challenge callback failed in phase %d, round 0 (%d)", LURK_SPARTAN_PCS, rc); return LURK_ERR_ARG; }
    LURK_TRY(scale_affine(c.curve, c.ck_c[fmt], rb, fmt, gc));
    void *d_b = static_cast<uint8_t *>(d_joint) + 32 * n;
    LURK_TRY(dispatch_field(c.field, [&](auto f) {
        using F = decltype(f);
        std::vector<uint8_t> rm(r.size());
        F x;
        for (int j = 0; j < c.m; j++) { fe_in(r.data() + 32 * j, fmt, x); fe_out(x, LURK_FMT_MONTGOMERY, rm.data() + 32 * j); }
        return lurk_eq_evals_dev(c.field, rm.data(), c.m, d_b, LURK_FMT_MONTGOMERY, s);
    }));
    cc.round_offset = 1;
    return ipa_prove_arena(c.curve, c.ck.c, c.arena, gc, d_joint, d_b, c.m, pcs_challenge, &cc, out ? out->L : nullptr, out ? out->R : nullptr,
                           out ? out->a_final : nullptr, out ? out->b_final : nullptr, fmt, s);
}

}  // namespace lurk

using namespace lurk;

struct lurk_compress_ctx {
    Circuit c[2];
    int device = 0;
    StreamGuard stream;          // the secondary proof's
    EventGuard inputs;
    Worker worker[2];            // last: joined before anything they use is released
};

static int bad_fmt(int fmt) {
    if (fmt == LURK_FMT_CANONICAL || fmt == LURK_FMT_MONTGOMERY) return LURK_OK;
    set_error("bad format %d", fmt);
    return LURK_ERR_ARG;
}

// host-only checks of one circuit's contexts and evaluation engine; fills what the context keeps of them
static int check_circuit(const char *name, int n, lurk_spartan_ctx *const *sp, const lurk_compress_pcs *pcs, int fmt, Circuit &c) {
    int m = 0;
    for (int i = 0; i < n; i++) {
        int field = -1, lr = 0, lv = 0;
        LURK_TRY(lurk_spartan_ctx_info(sp[i], &field, &lr, &lv, nullptr));
        if (i && field != c.field) { set_error("%s context %d is over field %d, context 0 over field %d", name, i, field, c.field); return LURK_ERR_ARG; }
        c.field = field;
        m = std::max(m, std::max(lr, lv));
        c.sp.push_back(sp[i]);
    }
    c.m = m;
    c.curve = c.field;                         // LURK_CURVE_* whose scalar field is LURK_FIELD_* of the same number
    c.kind = pcs->kind;
    int ck_curve = -1;
    size_t ck_n = 0;
    LURK_TRY(lurk_msm_ctx_info(pcs->ck, &ck_curve, &ck_n));
    if (ck_curve != c.curve) { set_error("%s key is on curve %d, the circuit's field %d needs curve %d", name, ck_curve, c.field, c.curve); return LURK_ERR_ARG; }
    if (ck_n < ((size_t)1 << m)) { set_error("%s key has %zu bases, the joint polynomial needs 2^%d", name, ck_n, m); return LURK_ERR_ARG; }
    if (c.kind == LURK_PCS_IPA) {
        if (!affine_valid(c.curve, pcs->ck_c, fmt)) { set_error("%s ck_c is not a reduced point on the curve", name); return LURK_ERR_RANGE; }
        // the base field of curve k is field k ^ 1
        LURK_TRY(dispatch_field(c.curve ^ 1, [&](auto f) {
            using F = decltype(f);
            F x;
            for (int k = 0; k < 2; k++) {
                fe_in(pcs->ck_c + 32 * k, fmt, x);
                fe_out(x, LURK_FMT_CANONICAL, c.ck_c[LURK_FMT_CANONICAL] + 32 * k);
                fe_out(x, LURK_FMT_MONTGOMERY, c.ck_c[LURK_FMT_MONTGOMERY] + 32 * k);
            }
            return LURK_OK;
        }));
    }
    return LURK_OK;
}

extern "C" {

int lurk_compress_ctx_create(int n_primary, lurk_spartan_ctx *const *primary, lurk_spartan_ctx *secondary, const lurk_compress_pcs *pcs_primary,
                             const lurk_compress_pcs *pcs_secondary, int fmt, lurk_compress_ctx **out) {
    if (!out) { set_error("null out"); return LURK_ERR_ARG; }
    *out = nullptr;
    if (n_primary < 1 || n_primary > CP_MAX_PRIMARY) { set_error("1..%d primary contexts, got %d", CP_MAX_PRIMARY, n_primary); return LURK_ERR_ARG; }
    if (!primary || !secondary) { set_error("null Spartan context array or secondary context"); return LURK_ERR_ARG; }
    if (!pcs_primary || !pcs_secondary) { set_error("null evaluation engine"); return LURK_ERR_ARG; }
    LURK_TRY(bad_fmt(fmt));
    const lurk_compress_pcs *pcs[2] = {pcs_primary, pcs_secondary};
    for (int k = 0; k < 2; k++) {
        const char *name = k ? "secondary" : "primary";
        if (pcs[k]->kind != LURK_PCS_HYPERKZG && pcs[k]->kind != LURK_PCS_IPA) { set_error("%s: unknown evaluation engine %d", name, pcs[k]->kind); return LURK_ERR_ARG; }
        if (!pcs[k]->ck) { set_error("%s: null key context", name); return LURK_ERR_ARG; }
        if (pcs[k]->kind == LURK_PCS_IPA && !pcs[k]->ck_c) { set_error("%s: IPA needs ck_c", name); return LURK_ERR_ARG; }
    }
    for (int i = 0; i < n_primary; i++) {
        if (!primary[i]) { set_error("null primary context %d", i); return LURK_ERR_ARG; }
        if (primary[i] == secondary) { set_error("primary context %d is also the secondary context", i); return LURK_ERR_ARG; }
        for (int k = 0; k < i; k++)
            if (primary[k] == primary[i]) { set_error("primary contexts %d and %d are the same context", k, i); return LURK_ERR_ARG; }
    }
    if (pcs_primary->ck == pcs_secondary->ck) { set_error("the primary and the secondary key are the same context"); return LURK_ERR_ARG; }
    for (int i = 0; i < n_primary; i++) LURK_TRY(refuse_verifier_only(primary[i], "lurk_compress_ctx_create (primary)"));
    LURK_TRY(refuse_verifier_only(secondary, "lurk_compress_ctx_create (secondary)"));
    LURK_TRY(require_gpu());
    lurk_compress_ctx *ctx = new lurk_compress_ctx();
    int rc = check_circuit("primary", n_primary, primary, pcs_primary, fmt, ctx->c[0]);
    if (rc == LURK_OK) rc = check_circuit("secondary", 1, &secondary, pcs_secondary, fmt, ctx->c[1]);
    if (rc == LURK_OK && ctx->c[1].field != (ctx->c[0].field ^ 1)) {
        set_error("the secondary circuit is over field %d; the cycle partner of the primary's field %d is %d", ctx->c[1].field, ctx->c[0].field,
                  ctx->c[0].field ^ 1);
        rc = LURK_ERR_ARG;
    }
    // the first device work: the clones of the keys, the worker stream
    if (rc == LURK_OK) rc = lurk_msm_ctx_clone(pcs_primary->ck, &ctx->c[0].ck.c);
    if (rc == LURK_OK) rc = lurk_msm_ctx_clone(pcs_secondary->ck, &ctx->c[1].ck.c);
    if (rc == LURK_OK && cudaGetDevice(&ctx->device) != cudaSuccess) { set_error("cudaGetDevice failed"); rc = LURK_ERR_CUDA; }
    if (rc == LURK_OK) rc = ctx->stream.create();
    if (rc == LURK_OK) rc = ctx->inputs.create();
    if (rc != LURK_OK) { delete ctx; return rc; }
    *out = ctx;
    return LURK_OK;
}

void lurk_compress_ctx_destroy(lurk_compress_ctx *ctx) { delete ctx; }

int lurk_compress_ctx_info(lurk_compress_ctx *ctx, size_t *device_bytes, size_t *joint_len_primary, size_t *joint_len_secondary) {
    if (!ctx) { set_error("null context"); return LURK_ERR_ARG; }
    if (device_bytes) *device_bytes = ctx->c[0].arena.device_bytes() + ctx->c[1].arena.device_bytes();
    if (joint_len_primary) *joint_len_primary = (size_t)1 << ctx->c[0].m;
    if (joint_len_secondary) *joint_len_secondary = (size_t)1 << ctx->c[1].m;
    return LURK_OK;
}

int lurk_compress_prove_dev(lurk_compress_ctx *ctx, int n_primary, const void *const *d_z, const void *const *d_E, const uint8_t *const *comm_W,
                            const uint8_t *const *comm_E, const void *d_z2, const void *d_E2, const uint8_t comm_W2[96], const uint8_t comm_E2[96],
                            lurk_compress_challenge_fn challenge, void *user, int flags, lurk_compress_proof *out, int fmt, void *stream) {
    if (!ctx) { set_error("null context"); return LURK_ERR_ARG; }
    if (!challenge) { set_error("null challenge callback"); return LURK_ERR_ARG; }
    LURK_TRY(bad_fmt(fmt));
    if (flags & ~(LURK_COMPRESS_SEQUENTIAL | LURK_COMPRESS_BATCHED)) { set_error("unknown flags 0x%x", flags); return LURK_ERR_ARG; }
    if (n_primary < 1 || n_primary > CP_MAX_PRIMARY) { set_error("1..%d primary instances, got %d", CP_MAX_PRIMARY, n_primary); return LURK_ERR_ARG; }
    if (!(flags & LURK_COMPRESS_BATCHED) && n_primary != 1) { set_error("a plain (Nova) primary proof has one instance, got %d", n_primary); return LURK_ERR_ARG; }
    if (!d_z || !d_E || !comm_W || !comm_E) { set_error("null primary instance array"); return LURK_ERR_ARG; }
    for (int i = 0; i < n_primary; i++)
        if (!d_z[i] || !d_E[i] || !comm_W[i] || !comm_E[i]) { set_error("null d_z / d_E / comm_W / comm_E of primary instance %d", i); return LURK_ERR_ARG; }
    if (!d_z2 || !d_E2 || !comm_W2 || !comm_E2) { set_error("null d_z2 / d_E2 / comm_W2 / comm_E2 of the secondary instance"); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    if (n_primary != (int)ctx->c[0].sp.size()) { set_error("%d primary instances for %zu primary contexts", n_primary, ctx->c[0].sp.size()); return LURK_ERR_ARG; }
    int dev = -1;
    LURK_CUDA_TRY(cudaGetDevice(&dev));
    if (dev != ctx->device) { set_error("the context belongs to device %d, device %d is current", ctx->device, dev); return LURK_ERR_ARG; }
    const uint8_t *const cw2[1] = {comm_W2}, *const ce2[1] = {comm_E2};
    if (!points_valid(ctx->c[0].curve, comm_W, n_primary, fmt) || !points_valid(ctx->c[0].curve, comm_E, n_primary, fmt)) {
        set_error("primary circuit: a commitment is not a point of the header's form on curve %d", ctx->c[0].curve);
        return LURK_ERR_RANGE;
    }
    if (!points_valid(ctx->c[1].curve, cw2, 1, fmt) || !points_valid(ctx->c[1].curve, ce2, 1, fmt)) {
        set_error("secondary circuit: a commitment is not a point of the header's form on curve %d", ctx->c[1].curve);
        return LURK_ERR_RANGE;
    }
    const cudaStream_t s[2] = {static_cast<cudaStream_t>(stream), ctx->stream.s};
    // the secondary's stream follows whatever the caller queued on `stream` before the call
    LURK_CUDA_TRY(cudaEventRecord(ctx->inputs.e, s[0]));
    LURK_CUDA_TRY(cudaStreamWaitEvent(s[1], ctx->inputs.e, 0));
    const void *const z2[1] = {d_z2}, *const e2[1] = {d_E2};
    const CircuitInputs in[2] = {{n_primary, d_z, d_E, comm_W, comm_E, (flags & LURK_COMPRESS_BATCHED) != 0}, {1, z2, e2, cw2, ce2, false}};
    int rc[2] = {LURK_OK, LURK_OK};
    std::string msg[2];
    auto run = [&](int k) {
        cudaSetDevice(ctx->device);
        rc[k] = prove_circuit(ctx->c[k], k, in[k], challenge, user, out ? (k ? &out->secondary : &out->primary) : nullptr, fmt, s[k]);
        if (rc[k] != LURK_OK) {
            msg[k] = lurk_last_error();
            cudaStreamSynchronize(s[k]);        // nothing of a failed proof stays queued behind the call
            cudaGetLastError();
        }
    };
    if (flags & LURK_COMPRESS_SEQUENTIAL) {
        ctx->worker[0].post([&] { run(0); if (rc[0] == LURK_OK) run(1); });
        ctx->worker[0].wait();
    } else {
        ctx->worker[0].post([&] { run(0); });
        ctx->worker[1].post([&] { run(1); });
        ctx->worker[0].wait();
        ctx->worker[1].wait();
    }
    for (int k = 0; k < 2; k++)
        if (rc[k] != LURK_OK) {
            set_error("%s circuit: %s", k ? "secondary" : "primary", msg[k].c_str());
            return rc[k];
        }
    return LURK_OK;
}

}  // extern "C"
