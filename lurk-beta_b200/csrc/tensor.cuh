// Product-tensor lookup of the verifier kernels: T(idx) = prod_j (bit_j(idx) ? hi_j : lo_j) over an l-bit index, bit 0 = the TOP
// bit (Arecibo's variable order).  eq(r, idx) is the case lo_j = 1 - r_j, hi_j = r_j; the IPA verifier's s the case lo_j = 1 / r_j,
// hi_j = r_j.  The product factors over groups of 8 index bits: group g covers index bits 8g .. 8g + 7 (counted from the least
// significant) and its table holds the 256 partial products of those bits, so T(idx) = prod_g table_g[(idx >> 8g) & 255] -- at most four
// tables of 8 KB in shared memory instead of a 2^l-entry table in HBM, and ceil(l / 8) - 1 products per lookup.
#pragma once
#include "field.cuh"

namespace lurk {

constexpr int TENSOR_MAX_VARS = 32;
constexpr int TENSOR_GROUP_BITS = 8;
constexpr int TENSOR_GROUP = 1 << TENSOR_GROUP_BITS;

template <class F>
struct TensorSpec {
    F lo[TENSOR_MAX_VARS], hi[TENSOR_MAX_VARS];
    int l;
};

// l = 0 keeps one table of ones: T() = 1
LURK_HD int tensor_groups(int l) { return l ? (l + TENSOR_GROUP_BITS - 1) / TENSOR_GROUP_BITS : 1; }

// every thread of the CTA takes part; the caller synchronises before the first lookup
template <class F>
__device__ void tensor_build(const TensorSpec<F> &t, F *tab) {
    const int groups = tensor_groups(t.l);
    for (int k = threadIdx.x; k < groups * TENSOR_GROUP; k += blockDim.x) {
        const int g = k / TENSOR_GROUP, e = k % TENSOR_GROUP;
        const int w = min(TENSOR_GROUP_BITS, t.l - TENSOR_GROUP_BITS * g);
        F v = F::one();
        for (int b = 0; b < w; b++) {
            const int j = t.l - 1 - (TENSOR_GROUP_BITS * g + b);      // index bit 8g + b <-> variable l - 1 - (8g + b)
            v = v * (((e >> b) & 1) ? t.hi[j] : t.lo[j]);
        }
        tab[k] = v;
    }
}

template <class F>
__device__ __forceinline__ F tensor_at(const F *tab, int groups, uint64_t idx) {
    F v = tab[idx & (TENSOR_GROUP - 1)];
    for (int g = 1; g < groups; g++) v = v * tab[g * TENSOR_GROUP + ((idx >> (TENSOR_GROUP_BITS * g)) & (TENSOR_GROUP - 1))];
    return v;
}

}  // namespace lurk
