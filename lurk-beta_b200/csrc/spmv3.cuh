// The three R1CS products A z, B z, C z in one launch: shared by the fold context (foldctx_impl.cuh) and the Spartan prover context
// (spartan.cu), which both keep the matrices as CSR over the columns of z = (W, u, X).  r1cs_sat_kernel is the same pass with the
// relaxed R1CS check in place of the stores: the fold context's check_running and the recursive verifier (recursive.cu).
#pragma once
#include "common.cuh"

namespace lurk {

struct CsrDev {
    const uint64_t *row_ptr;
    const uint32_t *col;
    const void *val;
};

// row i of M times z: lazy accumulation, one Montgomery reduction per group of <= 8 products
template <class F>
__device__ __forceinline__ F csr_row_dot(const CsrDev &M, size_t i, const F *__restrict__ z) {
    const F *val = (const F *)M.val;
    const uint64_t k0 = M.row_ptr[i], k1 = M.row_ptr[i + 1];
    F acc = F::zero();
    if (k1 - k0 == 1) {
        acc = load_fe<F>(val + k0) * load_fe<F>(z + M.col[k0]);
    } else if (k1 > k0) {
        for (uint64_t k = k0; k < k1;) {
            WideAcc<typename F::Params> w;
            w.clear();
            const uint64_t ke = k1 - k > 8 ? k + 8 : k1;
            for (; k < ke; k++) w.mul_acc(load_fe<F>(val + k), load_fe<F>(z + M.col[k]));
            acc = acc + w.reduce();
        }
    }
    return acc;
}

// y_m = M_m z for the three R1CS matrices in one launch (blockIdx.y = matrix), one row per thread
template <class F>
__global__ void __launch_bounds__(256) spmv3_kernel(CsrDev A, CsrDev B, CsrDev C, size_t rows, const F *__restrict__ z, F *__restrict__ ya,
                                                    F *__restrict__ yb, F *__restrict__ yc) {
    const CsrDev M = blockIdx.y == 0 ? A : (blockIdx.y == 1 ? B : C);
    F *y = blockIdx.y == 0 ? ya : (blockIdx.y == 1 ? yb : yc);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += (size_t)gridDim.x * blockDim.x)
        store_fe(y + i, csr_row_dot(M, i, z));
}

// The failing rows of one instance: count[0] = how many, count[1] = the first (UINT64_MAX when every row holds).
struct SatCount {
    unsigned long long bad, first;
};

// (A z)∘(B z) = u (C z) + E row by row, with the three products formed in registers and never stored: no O(rows) scratch.  u is z[n_w];
// E == nullptr is a strict instance (E = 0).  With `kept_a` the vectors the folds keep current (kept_a, kept_b, kept_c) must also equal
// the fresh products.  One row per thread; each warp adds its count and offers its first failing row once, after the loop.
template <class F>
__global__ void __launch_bounds__(256) r1cs_sat_kernel(CsrDev A, CsrDev B, CsrDev C, size_t rows, const F *__restrict__ z, uint64_t n_w,
                                                       const F *__restrict__ e, const F *__restrict__ kept_a, const F *__restrict__ kept_b,
                                                       const F *__restrict__ kept_c, SatCount *out) {
    const F u = load_fe<F>(z + n_w);
    unsigned bad = 0;
    unsigned long long first = ~0ull;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += (size_t)gridDim.x * blockDim.x) {
        const F a = csr_row_dot(A, i, z), b = csr_row_dot(B, i, z), c = csr_row_dot(C, i, z);
        F rhs = u * c;
        if (e) rhs = rhs + load_fe<F>(e + i);
        bool ok = a * b == rhs;
        if (kept_a) ok = ok && a == load_fe<F>(kept_a + i) && b == load_fe<F>(kept_b + i) && c == load_fe<F>(kept_c + i);
        if (!ok) {
            bad++;
            if (first == ~0ull) first = i;      // grid-stride rows only grow
        }
    }
    bad = __reduce_add_sync(0xffffffffu, bad);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const unsigned long long o = __shfl_xor_sync(0xffffffffu, first, off);
        first = o < first ? o : first;
    }
    if ((threadIdx.x & 31) == 0 && bad) {
        atomicAdd(&out->bad, (unsigned long long)bad);
        atomicMin(&out->first, first);
    }
}

// Resets *d_out and enqueues r1cs_sat_kernel on s; the grid is the fold's (8 CTAs of 256 per SM at most).
template <class F>
int r1cs_sat_launch(const CsrDev M[3], size_t rows, const F *z, uint64_t n_w, const F *e, const F *const kept[3], SatCount *d_out, cudaStream_t s) {
    LURK_CUDA_TRY(cudaMemsetAsync(&d_out->bad, 0, sizeof d_out->bad, s));
    LURK_CUDA_TRY(cudaMemsetAsync(&d_out->first, 0xff, sizeof d_out->first, s));
    if (!rows) return LURK_OK;
    const size_t want = (rows + 255) / 256, cap = (size_t)sm_count() * 8;
    r1cs_sat_kernel<F><<<(unsigned)(want < cap ? want : cap), 256, 0, s>>>(M[0], M[1], M[2], rows, z, n_w, e, kept ? kept[0] : nullptr,
                                                                           kept ? kept[1] : nullptr, kept ? kept[2] : nullptr, d_out);
    LURK_CUDA_TRY(cudaGetLastError());
    return LURK_OK;
}

}  // namespace lurk
