// N3 -- commitment-key generation behind the C ABI (include/lurk_b200.h, "N3"): the GPU half of Arecibo
// `CommitmentKey::setup(label, n)` -> `DlogGroup::from_label` as `public_params` reaches it (reference src/proof/nova.rs:196-216,
// supernova.rs:117-137; cached by src/public_parameters/mod.rs:20-71 because it takes minutes on the CPU).
//
// Data flow of lurk_ck_generate_dev: the SHAKE256 stream is inherently sequential, so a host thread squeezes it in chunks of
// 2^16 x 32 bytes into two pinned buffers while the GPU maps the previous chunk: H2D copy and kernel of chunk k run under the
// squeeze of chunk k + 1.  The key is written where the commitment contexts read it (n x 64 bytes, Montgomery, device memory:
// lurk_msm_ctx_create_dev) and never crosses PCIe.  One thread per point, persistent grid of 4 CTAs of 128 threads per SM.
#include "common.cuh"
#include "h2c_params.h"

#include <algorithm>

namespace lurk {

template <class F>
__global__ void __launch_bounds__(128) h2c_kernel(const __grid_constant__ H2cParams<F> P, const uint8_t *__restrict__ msgs, uint32_t msg_len,
                                                  size_t n, Affine<F> *__restrict__ out, int to_canonical) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        alignas(16) uint8_t m[H2C_MAX_MSG];      // the 16-byte copies below need it
        const uint8_t *src = msgs + i * msg_len;
        if ((msg_len & 15u) == 0 && (reinterpret_cast<uintptr_t>(msgs) & 15u) == 0) {
            for (uint32_t k = 0; k < msg_len; k += 16) *reinterpret_cast<uint4 *>(m + k) = *reinterpret_cast<const uint4 *>(src + k);
        } else {
            for (uint32_t k = 0; k < msg_len; k++) m[k] = src[k];
        }
        Affine<F> pt = hash_to_curve_point(P, m, msg_len);
        if (to_canonical) { pt.x = pt.x.to_canonical(); pt.y = pt.y.to_canonical(); }
        store_fe(&out[i].x, pt.x);
        store_fe(&out[i].y, pt.y);
    }
}

template <class C>
static int h2c_launch(const H2cParams<typename C::Base> &P, const uint8_t *d_msgs, uint32_t msg_len, size_t n, void *d_out, int to_canonical,
                      cudaStream_t s) {
    using F = typename C::Base;
    if (n == 0) return LURK_OK;
    const size_t want = (n + 127) / 128;
    const int grid = (int)std::min<size_t>(want, (size_t)sm_count() * 4);
    h2c_kernel<F><<<grid, 128, 0, s>>>(P, d_msgs, msg_len, n, reinterpret_cast<Affine<F> *>(d_out), to_canonical);
    LURK_CUDA_TRY(cudaGetLastError());
    return LURK_OK;
}

struct PinnedBuf {
    void *p = nullptr;
    ~PinnedBuf() { if (p) cudaFreeHost(p); }
    int alloc(size_t n) { LURK_CUDA_TRY(cudaHostAlloc(&p, n, cudaHostAllocDefault)); return LURK_OK; }
};
struct EventPair {
    cudaEvent_t e[2] = {nullptr, nullptr};
    ~EventPair() { for (auto x : e) if (x) cudaEventDestroy(x); }
};

template <class C>
static int ck_generate_dev(const uint8_t *label, size_t label_len, size_t first, size_t n, void *d_bases, int to_canonical, cudaStream_t s) {
    H2cParams<typename C::Base> P;
    if (!h2c_make_params<C>("from_uniform_bytes", 32, P)) { set_error("hash-to-curve parameters"); return LURK_ERR_ARG; }
    const size_t CHUNK = (size_t)1 << 16;
    PinnedBuf pin[2];
    DevBuf stage[2];
    EventPair copied;
    const int nbuf = n > CHUNK ? 2 : 1;
    for (int k = 0; k < nbuf; k++) {
        LURK_TRY(pin[k].alloc(32 * std::min(n, CHUNK)));
        LURK_TRY(stage[k].alloc(32 * std::min(n, CHUNK)));
        LURK_CUDA_TRY(cudaEventCreateWithFlags(&copied.e[k], cudaEventDisableTiming));
    }
    Shake256 xof;
    xof.absorb(label, label_len);
    for (size_t skip = first; skip;) {                   // a rank's slice of a sharded key starts in the middle of the stream
        uint8_t drop[4096];
        size_t k = std::min<size_t>(skip, sizeof drop / 32);
        xof.squeeze(drop, 32 * k);
        skip -= k;
    }
    size_t chunk_no = 0;
    for (size_t lo = 0; lo < n; lo += CHUNK, chunk_no++) {
        const size_t m = std::min(CHUNK, n - lo);
        const int k = (int)(chunk_no & 1);
        if (chunk_no >= 2) LURK_CUDA_TRY(cudaEventSynchronize(copied.e[k]));   // the pinned buffer is free again
        xof.squeeze(static_cast<uint8_t *>(pin[k].p), 32 * m);
        // the kernel that read stage[k] two chunks ago precedes this copy in stream order
        LURK_CUDA_TRY(cudaMemcpyAsync(stage[k].p, pin[k].p, 32 * m, cudaMemcpyHostToDevice, s));
        LURK_CUDA_TRY(cudaEventRecord(copied.e[k], s));
        LURK_TRY(h2c_launch<C>(P, stage[k].as<uint8_t>(), 32, m, static_cast<uint8_t *>(d_bases) + 64 * lo, to_canonical, s));
    }
    LURK_CUDA_TRY(cudaStreamSynchronize(s));   // the staging buffers die with this frame
    return LURK_OK;
}

}  // namespace lurk

using namespace lurk;

extern "C" {

size_t lurk_ck_size(size_t num_cons, size_t num_vars, size_t ck_floor) {
    size_t m = std::max(std::max(num_cons, num_vars), std::max(ck_floor, (size_t)1));
    size_t p = 1;
    while (p < m) p <<= 1;
    return p;
}

int lurk_shake256(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_len) {
    if ((in_len && !in) || (out_len && !out)) { set_error("null argument"); return LURK_ERR_ARG; }
    Shake256 x;
    x.absorb(in, in_len);
    x.squeeze(out, out_len);
    return LURK_OK;
}

int lurk_hash_to_curve_batch_dev(int curve_id, const char *domain_prefix, const void *d_messages, size_t msg_len, size_t n, void *d_points,
                                 int fmt, void *stream) {
    if (!domain_prefix || (n && (!d_messages || !d_points))) { set_error("null argument"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    return dispatch_curve(curve_id, [&](auto c) {
        using C = decltype(c);
        H2cParams<typename C::Base> P;
        if (!h2c_make_params<C>(domain_prefix, msg_len, P)) {
            set_error("domain prefix / message length do not fit one BLAKE2b block (msg_len %zu)", msg_len);
            return LURK_ERR_ARG;
        }
        return h2c_launch<C>(P, static_cast<const uint8_t *>(d_messages), (uint32_t)msg_len, n, d_points, fmt == LURK_FMT_CANONICAL,
                             static_cast<cudaStream_t>(stream));
    });
}

int lurk_hash_to_curve_batch(int curve_id, const char *domain_prefix, const uint8_t *messages, size_t msg_len, size_t n, int fmt,
                             uint8_t *points_out) {
    if (!domain_prefix || (n && (!messages || !points_out))) { set_error("null argument"); return LURK_ERR_ARG; }
    if (curve_id < 0 || curve_id > 3) { set_error("unknown curve id %d", curve_id); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    if (n == 0) return LURK_OK;
    DevBuf d_in, d_out;
    LURK_TRY(d_in.alloc(std::max<size_t>(n * msg_len, 16)));
    LURK_TRY(d_out.alloc(n * 64));
    cudaStream_t s;
    LURK_CUDA_TRY(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    int rc = LURK_OK;
    auto run = [&]() -> int {
        if (msg_len) LURK_CUDA_TRY(cudaMemcpyAsync(d_in.p, messages, n * msg_len, cudaMemcpyHostToDevice, s));
        LURK_TRY(lurk_hash_to_curve_batch_dev(curve_id, domain_prefix, d_in.p, msg_len, n, d_out.p, fmt, s));
        LURK_CUDA_TRY(cudaMemcpyAsync(points_out, d_out.p, n * 64, cudaMemcpyDeviceToHost, s));
        LURK_CUDA_TRY(cudaStreamSynchronize(s));
        return LURK_OK;
    };
    rc = run();
    cudaStreamDestroy(s);
    return rc;
}

int lurk_ck_generate_range_dev(int curve_id, const uint8_t *label, size_t label_len, size_t first, size_t n, void *d_bases_mont,
                               void *stream) {
    if ((label_len && !label) || (n && !d_bases_mont)) { set_error("null argument"); return LURK_ERR_ARG; }
    if (curve_id < 0 || curve_id > 3) { set_error("unknown curve id %d", curve_id); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    return dispatch_curve(curve_id, [&](auto c) {
        return ck_generate_dev<decltype(c)>(label, label_len, first, n, d_bases_mont, 0, static_cast<cudaStream_t>(stream));
    });
}
int lurk_ck_generate_dev(int curve_id, const uint8_t *label, size_t label_len, size_t n, void *d_bases_mont, void *stream) {
    return lurk_ck_generate_range_dev(curve_id, label, label_len, 0, n, d_bases_mont, stream);
}

int lurk_ck_generate(int curve_id, const uint8_t *label, size_t label_len, size_t n, int fmt, uint8_t *bases_out) {
    if ((label_len && !label) || (n && !bases_out)) { set_error("null argument"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    if (curve_id < 0 || curve_id > 3) { set_error("unknown curve id %d", curve_id); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    if (n == 0) return LURK_OK;
    DevBuf d_out;
    LURK_TRY(d_out.alloc(n * 64));
    cudaStream_t s;
    LURK_CUDA_TRY(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    int rc = dispatch_curve(curve_id, [&](auto c) {
        return ck_generate_dev<decltype(c)>(label, label_len, 0, n, d_out.p, fmt == LURK_FMT_CANONICAL, s);
    });
    if (rc == LURK_OK) {
        cudaError_t e = cudaMemcpyAsync(bases_out, d_out.p, n * 64, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) { set_error("copy of the key failed: %s", cudaGetErrorString(e)); rc = LURK_ERR_CUDA; }
    }
    cudaStreamDestroy(s);
    return rc;
}

}  // extern "C"
