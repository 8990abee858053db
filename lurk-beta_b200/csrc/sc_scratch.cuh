// Shared by sumcheck.cu and ipa.cu: grid sizing, the per-thread reduction scratch, byte <-> field helpers and the inner-product kernel.
#pragma once
#include "common.cuh"
#include "reduce.cuh"

namespace lurk {

// RAII for the side streams / cloned commitment contexts that let independent Pippenger passes of one prover call overlap
struct StreamGuard {
    cudaStream_t s = nullptr;
    ~StreamGuard() { if (s) cudaStreamDestroy(s); }
    int create() { LURK_CUDA_TRY(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking)); return LURK_OK; }
    // the device's greatest priority: its CTAs are placed before those of default-priority streams as SMs free up
    int create_urgent() {
        int least = 0, greatest = 0;
        LURK_CUDA_TRY(cudaDeviceGetStreamPriorityRange(&least, &greatest));
        LURK_CUDA_TRY(cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, greatest));
        return LURK_OK;
    }
};
struct EventGuard { cudaEvent_t e = nullptr; ~EventGuard() { if (e) cudaEventDestroy(e); } int create() { LURK_CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); return LURK_OK; } };
struct MsmCloneGuard { lurk_msm_ctx *c = nullptr; ~MsmCloneGuard() { if (c) lurk_msm_ctx_destroy(c); } };
// stream-ordered scratch, freed (in stream order) when the call returns
struct StreamBuf {
    void *p = nullptr;
    cudaStream_t s = nullptr;
    ~StreamBuf() { if (p) cudaFreeAsync(p, s); }
    int alloc(size_t bytes, cudaStream_t st) { s = st; LURK_CUDA_TRY(cudaMallocAsync(&p, bytes ? bytes : 16, st)); return LURK_OK; }
};

static inline int sc_grid(size_t n, int block) {
    size_t want = (n + block - 1) / block;
    size_t cap = (size_t)sm_count() * 4;
    return (int)(want < cap ? (want ? want : 1) : cap);
}

// Scratch of the reductions: per-CTA partials, the ticket counter, the result slots and their pinned mirror.  One per host thread
// and device, kept for the life of the thread: allocating (and above all freeing) device / pinned memory inside every call would
// synchronise the whole device each time.  Every field element is 32 bytes, so the pool is type-agnostic.
struct ScPool {
    void *dev = nullptr, *pinned = nullptr;
    int device = -1;
    ~ScPool() { if (dev) cudaFree(dev); if (pinned) cudaFreeHost(pinned); }
};
static ScPool &sc_pool() {
    static thread_local ScPool pool;
    return pool;
}
template <class F>
struct ScScratch {
    F *partial = nullptr, *result = nullptr;
    unsigned *counter = nullptr;
    void *pinned = nullptr;
    int init(cudaStream_t s) {
        ScPool &pool = sc_pool();
        const size_t cap = (size_t)sm_count() * 4;
        int dev = -1;
        LURK_CUDA_TRY(cudaGetDevice(&dev));
        if (pool.device != dev) {
            if (pool.dev) { cudaFree(pool.dev); pool.dev = nullptr; }
            if (pool.pinned) { cudaFreeHost(pool.pinned); pool.pinned = nullptr; }
            LURK_CUDA_TRY(cudaMalloc(&pool.dev, 32 * (cap * 3 + 8) + 64));
            LURK_CUDA_TRY(cudaHostAlloc(&pool.pinned, 32 * 256, cudaHostAllocDefault));
            pool.device = dev;
        }
        partial = static_cast<F *>(pool.dev);
        counter = reinterpret_cast<unsigned *>(partial + cap * 3 + 8);
        pinned = pool.pinned;
        // the result slots ARE the pinned host buffer (unified addressing: the last CTA stores <= 128 bytes across PCIe), so a round
        // costs one launch + one stream synchronisation and no copy
        result = static_cast<F *>(pool.pinned);
        LURK_CUDA_TRY(cudaMemsetAsync(counter, 0, 64, s));     // a kernel that died mid-way must not poison the next call
        return LURK_OK;
    }
    // waits for the kernel that wrote result[0..k)
    int fetch(int k, F *out, cudaStream_t s) {
        LURK_CUDA_TRY(cudaStreamSynchronize(s));
        memcpy(out, pinned, sizeof(F) * k);
        return LURK_OK;
    }
};

template <class F>
static inline void fe_out(const F &x_mont, int fmt, uint8_t *out) {
    F v = fmt == LURK_FMT_CANONICAL ? x_mont.to_canonical() : x_mont;
    memcpy(out, v.v, 32);
}
template <class F>
static inline bool fe_in(const uint8_t *in, int fmt, F &x_mont) {
    F v;
    memcpy(v.v, in, 32);
    if (!v.is_reduced()) return false;
    x_mont = fmt == LURK_FMT_CANONICAL ? F::from_canonical(v) : v;
    return true;
}

template <class F>
__global__ void __launch_bounds__(256) dot_kernel(const F *__restrict__ x, const F *__restrict__ y, size_t n, F *partial, unsigned *counter, F *result) {
    F acc[1] = {F::zero()};
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        acc[0] += load_fe<F>(x + i) * load_fe<F>(y + i);
    grid_sum<F, 1>(acc, partial, counter, result);
}

template <class F>
static int dot_dev(const void *d_x, const void *d_y, size_t n, F *out, ScScratch<F> &sc, cudaStream_t s) {
    dot_kernel<F><<<sc_grid(n, 256), 256, 0, s>>>(static_cast<const F *>(d_x), static_cast<const F *>(d_y), n, sc.partial, sc.counter, sc.result);
    LURK_CUDA_TRY(cudaGetLastError());
    return sc.fetch(1, out, s);
}

}  // namespace lurk
