// C-ABI front end of the Pedersen commitment (S4 in include/lurk_b200.h); the kernels and the per-curve pipeline are in
// msm_impl.cuh and are compiled once per curve in msm_inst.cu.
#include "msm_impl.cuh"

namespace lurk {
LURK_MSM_EXTERN(CurveBn254G1)
LURK_MSM_EXTERN(CurveGrumpkin)
LURK_MSM_EXTERN(CurvePallas)
LURK_MSM_EXTERN(CurveVesta)
}  // namespace lurk

using namespace lurk;

extern "C" {

int lurk_msm_ctx_create_dev(int curve_id, const void *d_bases_mont, size_t n, lurk_msm_ctx **out) {
    if (!out) { set_error("null out"); return LURK_ERR_ARG; }
    *out = nullptr;
    if (curve_id < 0 || curve_id > 3) { set_error("unknown curve id %d", curve_id); return LURK_ERR_ARG; }
    if (n >= ((size_t)1 << 31)) { set_error("commitment key too large"); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    lurk_msm_ctx *ctx = new lurk_msm_ctx();
    ctx->curve_id = curve_id;
    ctx->n = n;
    ctx->d_bases = const_cast<void *>(d_bases_mont);
    cudaGetDevice(&ctx->device);
    *out = ctx;
    return LURK_OK;
}

int lurk_msm_ctx_create(int curve_id, const uint8_t *bases_affine, size_t n, int fmt, lurk_msm_ctx **out) {
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    if (n && !bases_affine) { set_error("null bases"); return LURK_ERR_ARG; }
    LURK_TRY(lurk_msm_ctx_create_dev(curve_id, nullptr, n, out));
    if (n == 0) return LURK_OK;
    int rc = dispatch_curve(curve_id, [&](auto c) { return ctx_upload<decltype(c)>(*out, bases_affine, n, fmt); });
    if (rc != LURK_OK) { lurk_msm_ctx_destroy(*out); *out = nullptr; }
    return rc;
}

int lurk_msm_ctx_set_profiling(lurk_msm_ctx *ctx, int enable) {
    if (!ctx) { set_error("null context"); return LURK_ERR_ARG; }
    std::lock_guard<std::mutex> g(ctx->mu);
    if (enable && !ctx->ev0) {
        LURK_CUDA_TRY(cudaEventCreate(&ctx->ev0));
        LURK_CUDA_TRY(cudaEventCreate(&ctx->ev1));
        LURK_CUDA_TRY(cudaEventCreate(&ctx->ev_sort));
    }
    ctx->profile = enable != 0;
    return LURK_OK;
}
int lurk_msm_ctx_last_profile(lurk_msm_ctx *ctx, float *accumulate_ms, unsigned *kernel_launches) {
    if (!ctx) { set_error("null context"); return LURK_ERR_ARG; }
    if (accumulate_ms) *accumulate_ms = ctx->last_accumulate_ms;
    if (kernel_launches) *kernel_launches = ctx->last_launches;
    return LURK_OK;
}

int lurk_msm_ctx_last_sort_ms(lurk_msm_ctx *ctx, float *sort_ms) {
    if (!ctx || !sort_ms) { set_error("null argument"); return LURK_ERR_ARG; }
    std::lock_guard<std::mutex> g(ctx->mu);
    *sort_ms = 0.f;
    if (ctx->pending) { set_error("a launch is pending on this context"); return LURK_ERR_ARG; }
    if (ctx->ev_sort) LURK_CUDA_TRY(cudaEventElapsedTime(sort_ms, ctx->ev_sort, ctx->ev0));
    return LURK_OK;
}

int lurk_msm_ctx_info(lurk_msm_ctx *ctx, int *curve_id, size_t *n) {
    if (!ctx) { set_error("null context"); return LURK_ERR_ARG; }
    if (curve_id) *curve_id = ctx->curve_id;
    if (n) *n = ctx->n;
    return LURK_OK;
}

void lurk_msm_ctx_destroy(lurk_msm_ctx *ctx) {
    if (!ctx) return;
    if (ctx->ev0) { cudaEventDestroy(ctx->ev0); cudaEventDestroy(ctx->ev1); }
    if (ctx->ev_sort) cudaEventDestroy(ctx->ev_sort);
    if (ctx->done) cudaEventDestroy(ctx->done);
    if (ctx->ev_fork) { cudaEventDestroy(ctx->ev_fork); cudaEventDestroy(ctx->ev_join); }
    if (ctx->owns_bases && ctx->d_bases) cudaFree(ctx->d_bases);
    if (ctx->owns_table && ctx->d_table) cudaFree(ctx->d_table);
    delete ctx;
}

int lurk_msm_ctx_run_dev(lurk_msm_ctx *ctx, const void *d_scalars, size_t n, int fmt, uint8_t out_xyz[96], void *stream) {
    if (!ctx || !out_xyz) { set_error("null argument"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    if (n > ctx->n) { set_error("%zu scalars for a commitment key of %zu bases", n, ctx->n); return LURK_ERR_ARG; }
    std::lock_guard<std::mutex> g(ctx->mu);
    return dispatch_curve(ctx->curve_id, [&](auto c) { return msm_run<decltype(c)>(ctx, d_scalars, n, fmt, out_xyz, (cudaStream_t)stream); });
}

int lurk_msm_ctx_launch_dev(lurk_msm_ctx *ctx, const void *d_scalars, size_t n, int fmt, void *stream) {
    if (!ctx) { set_error("null argument"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    if (n > ctx->n) { set_error("%zu scalars for a commitment key of %zu bases", n, ctx->n); return LURK_ERR_ARG; }
    std::lock_guard<std::mutex> g(ctx->mu);
    return dispatch_curve(ctx->curve_id, [&](auto c) { return msm_launch<decltype(c)>(ctx, d_scalars, n, fmt, (cudaStream_t)stream, true); });
}
int lurk_msm_ctx_finish(lurk_msm_ctx *ctx, uint8_t out_xyz[96]) {
    if (!ctx || !out_xyz) { set_error("null argument"); return LURK_ERR_ARG; }
    std::lock_guard<std::mutex> g(ctx->mu);
    return dispatch_curve(ctx->curve_id, [&](auto c) { return msm_finish<decltype(c)>(ctx, out_xyz); });
}
int lurk_msm_ctx_precompute(lurk_msm_ctx *ctx) {
    if (!ctx) { set_error("null context"); return LURK_ERR_ARG; }
    std::lock_guard<std::mutex> g(ctx->mu);
    if (ctx->d_table || ctx->n == 0) return LURK_OK;
    if (ctx->pending) { set_error("a launch is pending on this context"); return LURK_ERR_ARG; }
    return dispatch_curve(ctx->curve_id, [&](auto cv) { return msm_precompute<decltype(cv)>(ctx, 0); });
}

int lurk_msm_ctx_precompute_window(lurk_msm_ctx *ctx, int c) {
    if (!ctx) { set_error("null context"); return LURK_ERR_ARG; }
    std::lock_guard<std::mutex> g(ctx->mu);
    if (ctx->d_table) { set_error("the context already has a fixed-base table"); return LURK_ERR_ARG; }
    if (ctx->n == 0) return LURK_OK;
    if (ctx->pending) { set_error("a launch is pending on this context"); return LURK_ERR_ARG; }
    if (c <= 0) { set_error("window width %d out of range", c); return LURK_ERR_ARG; }
    return dispatch_curve(ctx->curve_id, [&](auto cv) { return msm_precompute<decltype(cv)>(ctx, c); });
}

int lurk_msm_ctx_clone(lurk_msm_ctx *ctx, lurk_msm_ctx **out) {
    if (!ctx || !out) { set_error("null argument"); return LURK_ERR_ARG; }
    std::lock_guard<std::mutex> g(ctx->mu);        // a concurrent lurk_msm_ctx_precompute publishes d_table under it
    lurk_msm_ctx *c = new lurk_msm_ctx();
    c->curve_id = ctx->curve_id;
    c->device = ctx->device;
    c->n = ctx->n;
    c->d_bases = ctx->d_bases;     // shared, not owned: the parent must outlive its clones
    c->owns_bases = false;
    c->d_table = ctx->d_table;
    c->owns_table = false;
    c->fixed_c = ctx->fixed_c;
    *out = c;
    return LURK_OK;
}

int lurk_msm_ctx_run(lurk_msm_ctx *ctx, const uint8_t *scalars, size_t n, int fmt, uint8_t out_xyz[96]) {
    if (!ctx || !out_xyz || (n && !scalars)) { set_error("null argument"); return LURK_ERR_ARG; }
    if (n > ctx->n) { set_error("%zu scalars for a commitment key of %zu bases", n, ctx->n); return LURK_ERR_ARG; }
    if (n == 0) { memset(out_xyz, 0, 96); return LURK_OK; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    std::lock_guard<std::mutex> g(ctx->mu);
    if (ctx->pending) { set_error("a launch is already pending on this context (call lurk_msm_ctx_finish)"); return LURK_ERR_ARG; }
    LURK_TRY(ctx_check_device(ctx));
    if (ctx->scratch.scalars.bytes < n * 32) LURK_TRY(ctx->scratch.scalars.alloc(n * 32));
    // upload through two pinned staging buffers: the memcpy out of the caller's pageable memory overlaps the DMA
    MsmScratch &S = ctx->scratch;
    const size_t STAGE = (size_t)8 << 20;
    if (!S.stage_stream) LURK_CUDA_TRY(cudaStreamCreateWithFlags(&S.stage_stream, cudaStreamNonBlocking));
    cudaStream_t hs = S.stage_stream;      // not the legacy default stream: that one serialises against every other stream
    if (!S.h_stage[0]) {
        for (int k = 0; k < 2; k++) {
            LURK_CUDA_TRY(cudaMallocHost(&S.h_stage[k], STAGE));
            LURK_CUDA_TRY(cudaEventCreateWithFlags(&S.stage_done[k], cudaEventDisableTiming));
        }
    }
    const size_t total = n * 32;
    int k = 0;
    for (size_t off = 0; off < total; off += STAGE, k ^= 1) {
        const size_t len = std::min(STAGE, total - off);
        LURK_CUDA_TRY(cudaEventSynchronize(S.stage_done[k]));      // the previous DMA out of this buffer is complete
        memcpy(S.h_stage[k], scalars + off, len);
        LURK_CUDA_TRY(cudaMemcpyAsync((uint8_t *)S.scalars.p + off, S.h_stage[k], len, cudaMemcpyHostToDevice, hs));
        LURK_CUDA_TRY(cudaEventRecord(S.stage_done[k], hs));
    }
    int bad = 0;
    LURK_TRY(dispatch_curve(ctx->curve_id, [&](auto c) {
        using Fs = typename decltype(c)::Scalar;
        return check_reduced_dev<Fs>(ctx->scratch.scalars.p, n, hs, &bad);
    }));
    if (bad) { set_error("%d scalar(s) are not reduced below the group order", bad); return LURK_ERR_RANGE; }
    return dispatch_curve(ctx->curve_id, [&](auto c) { return msm_run<decltype(c)>(ctx, ctx->scratch.scalars.p, n, fmt, out_xyz, hs); });
}

int lurk_msm(int curve_id, const uint8_t *bases_affine, const uint8_t *scalars, size_t n, int fmt, uint8_t out_xyz[96]) {
    lurk_msm_ctx *ctx = nullptr;
    LURK_TRY(lurk_msm_ctx_create(curve_id, bases_affine, n, fmt, &ctx));
    int rc = lurk_msm_ctx_run(ctx, scalars, n, fmt, out_xyz);
    lurk_msm_ctx_destroy(ctx);
    return rc;
}

int lurk_synthetic_bases(int curve_id, uint64_t start, size_t n, int fmt, uint8_t *bases_out) {
    if (!bases_out && n) { set_error("null output"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    return dispatch_curve(curve_id, [&](auto c) {
        using Cv = decltype(c);
        using Fb = typename Cv::Base;
        const Affine<Fb> g = curve_generator<Cv>();
        const size_t BATCH = 1 << 12;
        unsigned nthreads = std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
        const size_t nbatches = (n + BATCH - 1) / BATCH;
        std::atomic<size_t> next{0};
        auto worker = [&]() {
            std::vector<XYZZ<Fb>> pts(BATCH);
            std::vector<Fb> pref(BATCH);
            for (;;) {
                size_t b = next.fetch_add(1);
                if (b >= nbatches) break;
                size_t lo = b * BATCH, m = std::min(BATCH, n - lo);
                // [start + lo + 1] G by double-and-add, then a running sum
                uint64_t k = start + lo + 1;
                XYZZ<Fb> acc = XYZZ<Fb>::identity();
                for (int bit = 63; bit >= 0; bit--) { acc = acc.dbl(); if ((k >> bit) & 1) acc.add_affine(g); }
                for (size_t i = 0; i < m; i++) { pts[i] = acc; acc.add_affine(g); }
                // one inversion per batch (Montgomery's trick on the ZZZ coordinates)
                Fb run = Fb::one();
                for (size_t i = 0; i < m; i++) { pref[i] = run; run = run * pts[i].zzz; }
                Fb inv = run.inv();
                for (size_t i = m; i-- > 0;) {
                    Fb zi = inv * pref[i];            // 1 / ZZZ_i
                    inv = inv * pts[i].zzz;
                    Fb zz_inv = (zi * pts[i].zz).sqr();
                    Fb x = pts[i].x * zz_inv, y = pts[i].y * zi;
                    if (fmt == LURK_FMT_CANONICAL) { x = x.to_canonical(); y = y.to_canonical(); }
                    memcpy(bases_out + 64 * (lo + i), x.v, 32);
                    memcpy(bases_out + 64 * (lo + i) + 32, y.v, 32);
                }
            }
        };
        std::vector<std::thread> pool;
        for (unsigned t = 1; t < nthreads; t++) pool.emplace_back(worker);
        worker();
        for (auto &t : pool) t.join();
        return LURK_OK;
    });
}

int lurk_point_sum(int curve_id, const uint8_t *points_xyz, size_t count, int fmt, uint8_t out_xyz[96]) {
    if (!out_xyz || (count && !points_xyz)) { set_error("null argument"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    return dispatch_curve(curve_id, [&](auto c) {
        using Fb = typename decltype(c)::Base;
        XYZZ<Fb> acc = XYZZ<Fb>::identity();
        for (size_t i = 0; i < count; i++) {
            const uint8_t *p = points_xyz + 96 * i;
            Fb x, y, z;
            memcpy(x.v, p, 32); memcpy(y.v, p + 32, 32); memcpy(z.v, p + 64, 32);
            if (!x.is_reduced() || !y.is_reduced()) { set_error("point %zu is not reduced", i); return LURK_ERR_RANGE; }
            if (z.is_zero()) continue;
            Affine<Fb> a;
            a.x = fmt == LURK_FMT_CANONICAL ? Fb::from_canonical(x) : x;
            a.y = fmt == LURK_FMT_CANONICAL ? Fb::from_canonical(y) : y;
            acc.add_affine(a);
        }
        point_to_bytes(acc, fmt, out_xyz);
        return LURK_OK;
    });
}

}  // extern "C"
