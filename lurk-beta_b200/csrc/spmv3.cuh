// The three R1CS products A z, B z, C z in one launch: shared by the fold context (foldctx_impl.cuh) and the Spartan prover context
// (spartan.cu), which both keep the matrices as CSR over the columns of z = (W, u, X).
#pragma once
#include "common.cuh"

namespace lurk {

struct CsrDev {
    const uint64_t *row_ptr;
    const uint32_t *col;
    const void *val;
};

// y_m = M_m z for the three R1CS matrices in one launch (blockIdx.y = matrix), one row per thread
template <class F>
__global__ void __launch_bounds__(256) spmv3_kernel(CsrDev A, CsrDev B, CsrDev C, size_t rows, const F *__restrict__ z, F *__restrict__ ya,
                                                    F *__restrict__ yb, F *__restrict__ yc) {
    const CsrDev M = blockIdx.y == 0 ? A : (blockIdx.y == 1 ? B : C);
    F *y = blockIdx.y == 0 ? ya : (blockIdx.y == 1 ? yb : yc);
    const F *val = (const F *)M.val;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += (size_t)gridDim.x * blockDim.x) {
        const uint64_t k0 = M.row_ptr[i], k1 = M.row_ptr[i + 1];
        F acc = F::zero();
        if (k1 - k0 == 1) {
            acc = load_fe<F>(val + k0) * load_fe<F>(z + M.col[k0]);
        } else if (k1 > k0) {
            // lazy accumulation: one Montgomery reduction per group of <= 8 products
            for (uint64_t k = k0; k < k1;) {
                WideAcc<typename F::Params> w;
                w.clear();
                const uint64_t ke = k1 - k > 8 ? k + 8 : k1;
                for (; k < ke; k++) w.mul_acc(load_fe<F>(val + k), load_fe<F>(z + M.col[k]));
                acc = acc + w.reduce();
            }
        }
        store_fe(y + i, acc);
    }
}

}  // namespace lurk
