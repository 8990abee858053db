// C-ABI front end of the fold context (S5/S6 in include/lurk_b200.h); the per-curve implementation is in foldctx_inst.cu.
#include "foldctx_impl.cuh"

namespace lurk {
LURK_FOLD_EXTERN(CurveBn254G1)
LURK_FOLD_EXTERN(CurveGrumpkin)
LURK_FOLD_EXTERN(CurvePallas)
LURK_FOLD_EXTERN(CurveVesta)
}  // namespace lurk

using namespace lurk;

struct lurk_fold_ctx {
    FoldCtxBase *impl = nullptr;
    int world = 1;
};

#define FOLD_CHECK(ctx)                                                  \
    do {                                                                 \
        if (!(ctx) || !(ctx)->impl) { set_error("null fold context"); return LURK_ERR_ARG; } \
    } while (0)

extern "C" {

int lurk_fold_ctx_create(const lurk_fold_config *cfg, lurk_msm_ctx *ck_w, lurk_msm_ctx *ck_t, lurk_fold_ctx **out) {
    if (!out) { set_error("null out"); return LURK_ERR_ARG; }
    *out = nullptr;
    if (!cfg || !ck_w || !ck_t) { set_error("null argument"); return LURK_ERR_ARG; }
    if (cfg->depth < 1 || cfg->depth > FOLD_MAX_DEPTH) { set_error("depth %d not in 1..%d", cfg->depth, FOLD_MAX_DEPTH); return LURK_ERR_ARG; }
    if (cfg->world < 1 || cfg->world > FOLD_MAX_WORLD || cfg->rank < 0 || cfg->rank >= cfg->world) { set_error("bad world / rank"); return LURK_ERR_ARG; }
    if (cfg->fmt != LURK_FMT_CANONICAL && cfg->fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", cfg->fmt); return LURK_ERR_ARG; }
    if (cfg->n_w + 1 + cfg->n_x >= (1ull << 32) || cfg->n_rows >= (1ull << 32)) { set_error("instance too large"); return LURK_ERR_ARG; }
    if (cfg->latency_sms < 0 || cfg->latency_sms % 8) { set_error("latency_sms must be a multiple of 8"); return LURK_ERR_ARG; }
    for (int m = 0; m < 3; m++)
        if (!cfg->row_ptr[m] || (cfg->n_rows && cfg->row_ptr[m][cfg->n_rows] && (!cfg->col[m] || !cfg->val[m]))) { set_error("null matrix %d", m); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    FoldCtxBase *impl = nullptr;
    int rc = dispatch_curve(cfg->curve_id, [&](auto c) { impl = make_fold_ctx<decltype(c)>(); return LURK_OK; });
    if (rc != LURK_OK) return rc;
    FoldConfigHost h;
    h.curve_id = cfg->curve_id; h.depth = cfg->depth; h.world = cfg->world; h.rank = cfg->rank;
    h.n_w = cfg->n_w; h.n_x = cfg->n_x; h.n_rows = cfg->n_rows; h.latency_sms = cfg->latency_sms;
    rc = impl->init(h, cfg->row_ptr, cfg->col, cfg->val, cfg->fmt, ck_w, ck_t);
    if (rc != LURK_OK) { delete impl; return rc; }
    lurk_fold_ctx *ctx = new lurk_fold_ctx();
    ctx->impl = impl;
    ctx->world = cfg->world;
    *out = ctx;
    return LURK_OK;
}

void lurk_fold_ctx_destroy(lurk_fold_ctx *ctx) {
    if (!ctx) return;
    delete ctx->impl;
    delete ctx;
}

int lurk_fold_ctx_add_slot_batch(lurk_fold_ctx *ctx, int arity, size_t count, const uint64_t *offsets) {
    FOLD_CHECK(ctx);
    if (count && !offsets) { set_error("null offsets"); return LURK_ERR_ARG; }
    return ctx->impl->add_slot_batch(arity, count, offsets);
}
int lurk_fold_ctx_add_sha256_batch(lurk_fold_ctx *ctx, int n, size_t count, const uint64_t *offsets) {
    FOLD_CHECK(ctx);
    if (count && !offsets) { set_error("null offsets"); return LURK_ERR_ARG; }
    return ctx->impl->add_sha256_batch(n, count, offsets);
}
int lurk_fold_ctx_add_trie_batch(lurk_fold_ctx *ctx, int op, int height, size_t count, const uint64_t *offsets) {
    FOLD_CHECK(ctx);
    if (count && !offsets) { set_error("null offsets"); return LURK_ERR_ARG; }
    return ctx->impl->add_trie_batch(op, height, count, offsets);
}
int lurk_fold_ctx_set_spans(lurk_fold_ctx *ctx, int n_spans, const lurk_fold_span *spans) {
    FOLD_CHECK(ctx);
    if (n_spans && !spans) { set_error("null spans"); return LURK_ERR_ARG; }
    static_assert(sizeof(lurk_fold_span) == sizeof(FoldSpan), "span layout");
    return ctx->impl->set_spans(n_spans, reinterpret_cast<const FoldSpan *>(spans));
}
int lurk_fold_ctx_set_ro(lurk_fold_ctx *ctx, int n_absorb, const int *kinds, int challenge_bits) {
    FOLD_CHECK(ctx);
    if (!kinds) { set_error("null kinds"); return LURK_ERR_ARG; }
    return ctx->impl->set_ro(n_absorb, kinds, challenge_bits);
}
int lurk_fold_ctx_host_buffer(lurk_fold_ctx *ctx, int b, int which, void **ptr, size_t *bytes) {
    FOLD_CHECK(ctx);
    return ctx->impl->host_buffer(b, which, ptr, bytes);
}
int lurk_fold_ctx_device_buffer(lurk_fold_ctx *ctx, int b, int which, void **d_ptr, size_t *bytes) {
    FOLD_CHECK(ctx);
    return ctx->impl->device_buffer(b, which, d_ptr, bytes);
}
int lurk_fold_ctx_exchange_handle(lurk_fold_ctx *ctx, uint8_t handle[64]) {
    FOLD_CHECK(ctx);
    if (!handle) { set_error("null handle"); return LURK_ERR_ARG; }
    return ctx->impl->exchange_handle(handle);
}
int lurk_fold_ctx_set_peers(lurk_fold_ctx *ctx, const uint8_t *handles) {
    FOLD_CHECK(ctx);
    if (!handles && ctx->world > 1) { set_error("null handles"); return LURK_ERR_ARG; }
    return ctx->impl->set_peers(handles);
}
int lurk_fold_ctx_set_running(lurk_fold_ctx *ctx, const uint8_t *W, const uint8_t *E, const uint8_t u[32], const uint8_t *X,
                              const uint8_t comm_W[96], const uint8_t comm_E[96], int fmt) {
    FOLD_CHECK(ctx);
    if (!u || !comm_W || !comm_E) { set_error("null argument"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    return ctx->impl->set_running(W, E, u, X, comm_W, comm_E, fmt);
}
int lurk_fold_ctx_get_running(lurk_fold_ctx *ctx, uint8_t *W, uint8_t *E, uint8_t u[32], uint8_t *X, uint8_t comm_W[96], uint8_t comm_E[96],
                              int fmt) {
    FOLD_CHECK(ctx);
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    return ctx->impl->get_running(W, E, u, X, comm_W, comm_E, fmt);
}
int lurk_fold_ctx_stage_a(lurk_fold_ctx *ctx, int b, int flags, int fmt) {
    FOLD_CHECK(ctx);
    return ctx->impl->stage_a(b, flags, fmt);
}
int lurk_fold_ctx_init_running(lurk_fold_ctx *ctx, int b) {
    FOLD_CHECK(ctx);
    return ctx->impl->init_running(b);
}
int lurk_fold_ctx_stage_b_launch(lurk_fold_ctx *ctx, int b) {
    FOLD_CHECK(ctx);
    return ctx->impl->stage_b_launch(b);
}
int lurk_fold_ctx_collect(lurk_fold_ctx *ctx, int b, lurk_fold_result *out, int fmt) {
    FOLD_CHECK(ctx);
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    FoldResultHost h;
    int rc = ctx->impl->collect(b, out ? &h : nullptr, fmt);
    if (out && (rc == LURK_OK || rc == LURK_ERR_CUDA)) {
        memcpy(out->comm_W, h.comm_w, 96); memcpy(out->comm_T, h.comm_t, 96); memcpy(out->r, h.r, 32);
        memcpy(out->running_comm_W, h.run_comm_w, 96); memcpy(out->running_comm_E, h.run_comm_e, 96); memcpy(out->ro_hash, h.hash, 32);
        out->status = h.status;
        out->seq = h.seq;
    }
    return rc;
}
int lurk_fold_ctx_check_running(lurk_fold_ctx *ctx, uint64_t *bad_rows, int *comm_W_ok, int *comm_E_ok) {
    FOLD_CHECK(ctx);
    unsigned long long bad = 0;
    int rc = ctx->impl->check_running(&bad, comm_W_ok, comm_E_ok);
    if (bad_rows) *bad_rows = bad;
    return rc;
}
int lurk_fold_ctx_stats(lurk_fold_ctx *ctx, unsigned *launches_a, unsigned *launches_b, float *accumulate_w_ms, float *accumulate_t_ms) {
    FOLD_CHECK(ctx);
    return ctx->impl->stats(launches_a, launches_b, accumulate_w_ms, accumulate_t_ms);
}
int lurk_fold_ctx_sync(lurk_fold_ctx *ctx) {
    FOLD_CHECK(ctx);
    return ctx->impl->sync();
}

}  // extern "C"
