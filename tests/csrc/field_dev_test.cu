// Operation-level harness of lurk-beta_b200/csrc/field.cuh: every field operation, the lazy dot product WideAcc and its two users
// mul_sub_mul (curve.cuh) and ipa_fold_scalar (sumcheck.cuh), run element by element over arrays of raw 256-bit operands.
//
// nvcc builds it for sm_90a with the library's flags (libfield_dev_test.so, not linked into liblurk_b200.so): the device code is what
// ptxas made of the carry chains, condition code and all.  g++ builds the same file with -x c++ -DLURK_HOST_EMULATE_CC (the carry flag
// emulated) or without it (the host's 64-bit product), so the CPU suite runs the identical cases through both host paths.
// Test-only, not part of the product.
//
// fdt_run(field, op, k, n, in, out): case i reads width(op, k) elements of 32 bytes from in + 32 * width * i and writes one element.
// Operands are raw words (Montgomery form where the operation expects it); nothing is converted on the way in or out.
#include "field.cuh"
#include "curve.cuh"
#include "sumcheck.cuh"
#include <cstddef>
#include <cstring>
#if defined(__CUDACC__)
#include <cuda_runtime.h>
#include <vector>
#include "spmv3.cuh"
#endif

using namespace lurk;

enum {
    OP_MUL, OP_SQR, OP_ADD, OP_SUB, OP_NEG, OP_DBL, OP_POW5, OP_INV, OP_INV_VARTIME, OP_FROM_CANONICAL, OP_TO_CANONICAL,
    OP_FINAL_SUB, OP_IS_REDUCED, OP_MUL_SUB_MUL, OP_IPA_FOLD, OP_DOT, OP_DOT4, OP_CSR_ROW, OP_COUNT
};

extern "C" int fdt_width(int op, int k) {
    switch (op) {
        case OP_MUL: case OP_ADD: case OP_SUB: return 2;
        case OP_MUL_SUB_MUL: case OP_IPA_FOLD: return 4;
        case OP_DOT: case OP_DOT4: return k >= 1 && k <= 15 ? 2 * k : -1;
        case OP_CSR_ROW: return k >= 1 && k <= 64 ? 2 * k : -1;
    }
    return op >= 0 && op < OP_COUNT ? 1 : -1;
}

template <class F>
LURK_HD F ld(const uint32_t *p) { F x; for (int i = 0; i < 8; i++) x.v[i] = p[i]; return x; }

// k <= 15 pairs a[0..k), b[0..k) through one WideAcc: reduce() with its default ROUNDS (what the kernels call), or reduce<4>
template <class F, bool FOUR>
LURK_HD F dot(const uint32_t *in, int k) {
    WideAcc<typename F::Params> acc;
    acc.clear();
    for (int j = 0; j < k; j++) acc.mul_acc(ld<F>(in + 8 * j), ld<F>(in + 8 * (k + j)));
    return FOUR ? acc.template reduce<4>() : acc.reduce();
}

template <class F>
LURK_HD F eval(int op, int k, const uint32_t *in) {
    const F a = ld<F>(in);
    switch (op) {
        case OP_MUL: return a * ld<F>(in + 8);
        case OP_SQR: return a.sqr();
        case OP_ADD: return a + ld<F>(in + 8);
        case OP_SUB: return a - ld<F>(in + 8);
        case OP_NEG: return a.neg();
        case OP_DBL: return a.dbl();
        case OP_POW5: return a.pow5();
        case OP_INV: return a.inv();
        case OP_INV_VARTIME: return a.inv_vartime();
        case OP_FROM_CANONICAL: return F::from_canonical(a);
        case OP_TO_CANONICAL: return a.to_canonical();
        case OP_FINAL_SUB: { F r = a; r.final_sub(); return r; }
        case OP_IS_REDUCED: { F r = F::zero(); r.v[0] = a.is_reduced() ? 1u : 0u; return r; }
        case OP_MUL_SUB_MUL: return mul_sub_mul(a, ld<F>(in + 8), ld<F>(in + 16), ld<F>(in + 24));
        case OP_IPA_FOLD: return ipa_fold_scalar(a, ld<F>(in + 8), ld<F>(in + 16), ld<F>(in + 24));
        case OP_DOT: return dot<F, false>(in, k);
        default: return dot<F, true>(in, k);
    }
}

#if defined(__CUDACC__)
template <class F>
__global__ void __launch_bounds__(256) fdt_kernel(int op, int k, int width, size_t n, const uint32_t *__restrict__ in, uint32_t *__restrict__ out) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const F r = eval<F>(op, k, in + 8 * width * i);
        for (int w = 0; w < 8; w++) out[8 * i + w] = r.v[w];
    }
}
// csr_row_dot (spmv3.cuh) on row i = (val[i k .. i k + k), z[i k .. i k + k)): the single-product shortcut, groups of 8
template <class F>
__global__ void __launch_bounds__(256) fdt_csr_kernel(CsrDev M, size_t n, const F *__restrict__ z, F *__restrict__ out) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) store_fe(out + i, csr_row_dot(M, i, z));
}

template <class F>
static int run(int op, int k, size_t n, const uint8_t *in, uint8_t *out) {
    const int width = fdt_width(op, k);
    uint32_t *d_in = nullptr, *d_out = nullptr;
    std::vector<uint8_t> val, z;
    std::vector<uint64_t> rp;
    std::vector<uint32_t> col;
    void *d_rp = nullptr, *d_col = nullptr;
    cudaError_t e = cudaMalloc(&d_in, 32 * width * n + 32);
    if (e == cudaSuccess) e = cudaMalloc(&d_out, 32 * n + 32);
    if (e == cudaSuccess && op == OP_CSR_ROW) {
        // the row's values and z entries, each contiguous; z is indexed through col
        val.resize(32 * k * n); z.resize(32 * k * n); rp.resize(n + 1); col.resize(k * n);
        for (size_t i = 0; i < n; i++) {
            memcpy(&val[32 * k * i], in + 32 * width * i, 32 * k);
            memcpy(&z[32 * k * i], in + 32 * width * i + 32 * k, 32 * k);
            rp[i] = (uint64_t)k * i;
            for (int j = 0; j < k; j++) col[k * i + j] = (uint32_t)(k * i + j);
        }
        rp[n] = (uint64_t)k * n;
        e = cudaMemcpy(d_in, val.data(), val.size(), cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemcpy((uint8_t *)d_in + val.size(), z.data(), z.size(), cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMalloc(&d_rp, 8 * (n + 1));
        if (e == cudaSuccess) e = cudaMalloc(&d_col, 4 * k * n);
        if (e == cudaSuccess) e = cudaMemcpy(d_rp, rp.data(), 8 * (n + 1), cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemcpy(d_col, col.data(), 4 * k * n, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) {
            CsrDev M{(const uint64_t *)d_rp, (const uint32_t *)d_col, d_in};
            fdt_csr_kernel<F><<<(unsigned)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096), 256>>>(M, n, (const F *)((uint8_t *)d_in + val.size()), (F *)d_out);
            e = cudaGetLastError();
        }
    } else if (e == cudaSuccess) {
        e = cudaMemcpy(d_in, in, 32 * width * n, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) {
            fdt_kernel<F><<<(unsigned)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096), 256>>>(op, k, width, n, d_in, d_out);
            e = cudaGetLastError();
        }
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(out, d_out, 32 * n, cudaMemcpyDeviceToHost);
    cudaFree(d_in); cudaFree(d_out); cudaFree(d_rp); cudaFree(d_col);
    return e == cudaSuccess ? 0 : -100 - (int)e;
}
#else
template <class F>
static int run(int op, int k, size_t n, const uint8_t *in, uint8_t *out) {
    if (op == OP_CSR_ROW) return -2;        // csr_row_dot is device code only
    const int width = fdt_width(op, k);
    for (size_t i = 0; i < n; i++) {
        uint32_t w[8 * 30];
        memcpy(w, in + 32 * width * i, 32 * width);
        const F r = eval<F>(op, k, w);
        memcpy(out + 32 * i, r.v, 32);
    }
    return 0;
}
#endif

// 0 on success, -1 bad op / k, -2 op not available in this build, -3 bad field, <= -100 a CUDA error
extern "C" int fdt_run(int field, int op, int k, size_t n, const uint8_t *in, uint8_t *out) {
    if (fdt_width(op, k) < 0) return -1;
    if (n == 0) return 0;
    switch (field) {
        case 0: return run<Fe<Bn254Fr>>(op, k, n, in, out);
        case 1: return run<Fe<Bn254Fq>>(op, k, n, in, out);
        case 2: return run<Fe<PallasFq>>(op, k, n, in, out);
        case 3: return run<Fe<PallasFp>>(op, k, n, in, out);
    }
    return -3;
}
