// Shared plumbing of liblurk_b200: error reporting, CUDA call checking, field/curve dispatch.
#pragma once
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <vector>

#include "../../include/lurk_b200.h"
#include "curve.cuh"

namespace lurk {

void set_error(const char *fmt, ...);
int require_gpu();   // LURK_OK or LURK_ERR_NOGPU (message set)

#define LURK_CUDA_TRY(expr)                                                                          \
    do {                                                                                             \
        cudaError_t e__ = (expr);                                                                    \
        if (e__ != cudaSuccess) {                                                                    \
            ::lurk::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
            return e__ == cudaErrorMemoryAllocation ? LURK_ERR_OOM : LURK_ERR_CUDA;                  \
        }                                                                                            \
    } while (0)

#define LURK_TRY(expr)              \
    do {                            \
        int rc__ = (expr);          \
        if (rc__ != LURK_OK) return rc__; \
    } while (0)

// RAII device / pinned buffers for the host-buffer entry points
struct DevBuf {
    void *p = nullptr;
    size_t bytes = 0;
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf() { if (p) cudaFree(p); }
    int alloc(size_t n) {
        if (p) { cudaFree(p); p = nullptr; }
        bytes = 0;                       // stays 0 when cudaMalloc fails: `bytes >= want` must never hide a null buffer
        if (n == 0) return LURK_OK;
        LURK_CUDA_TRY(cudaMalloc(&p, n));
        bytes = n;
        return LURK_OK;
    }
    template <class T> T *as() const { return reinterpret_cast<T *>(p); }
};

template <class Fn>
int dispatch_field(int field_id, Fn &&fn) {
    switch (field_id) {
        case LURK_FIELD_BN254_FR: return fn(Fe<Bn254Fr>());
        case LURK_FIELD_BN254_FQ: return fn(Fe<Bn254Fq>());
        case LURK_FIELD_PALLAS_FQ: return fn(Fe<PallasFq>());
        case LURK_FIELD_PALLAS_FP: return fn(Fe<PallasFp>());
    }
    set_error("unknown field id %d", field_id);
    return LURK_ERR_ARG;
}
template <class Fn>
int dispatch_curve(int curve_id, Fn &&fn) {
    switch (curve_id) {
        case LURK_CURVE_BN254_G1: return fn(CurveBn254G1());
        case LURK_CURVE_GRUMPKIN: return fn(CurveGrumpkin());
        case LURK_CURVE_PALLAS: return fn(CurvePallas());
        case LURK_CURVE_VESTA: return fn(CurveVesta());
    }
    set_error("unknown curve id %d", curve_id);
    return LURK_ERR_ARG;
}

inline int sm_count() {
    static int n = 0;
    if (!n) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
    }
    return n;
}

// element-wise helpers implemented in fold.cu
template <class F> int convert_dev(const void *d_in, size_t n, int to_fmt, void *d_out, cudaStream_t s);
// returns number of elements >= p in a raw host/device buffer check (device side), used by host entry points
template <class F> int check_reduced_dev(const void *d_in, size_t n, cudaStream_t s, int *bad_host);
template <class F> int check_reduced_accumulate_dev(const void *d_in, size_t n, cudaStream_t s, int *d_bad);

}  // namespace lurk
