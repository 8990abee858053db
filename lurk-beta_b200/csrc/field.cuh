// 256-bit prime-field arithmetic in Montgomery form, 8 x 32-bit limbs, written for sm_90a.
//
// The same templates compile for the host (carry flag emulated) so that the exact algorithm that runs on
// the GPU is unit-tested on CPU and is reused by the host-side code of the library (Poseidon constant
// generation, final MSM window combine, affine normalisation).
//
// Multiplication keeps two interleaved accumulators ("even" / "odd" columns) so that every 32x32->64 product
// is a mad.lo.cc/madc.hi.cc pair on adjacent words, which ptxas fuses into one IMAD.WIDE.U32 with carry-in
// and carry-out: ~128 IMAD.WIDE + 8 IMAD per 256-bit Montgomery product.  Word-serial (CIOS-style)
// reduction is interleaved with the row products; the accumulators swap roles at every row instead of
// shifting registers.
//
// Element layout in memory: 32 bytes, little-endian limbs.  "canonical" = plain integer < p (what
// ff::PrimeField::to_repr gives, reference src/field.rs:72-81); "Montgomery" = x*2^256 mod p (what
// pasta_curves / halo2curves keep in memory as [u64; 4]).
#pragma once
#include <cstdint>
#include <cstring>

#if defined(__CUDACC__)
#define LURK_HD __host__ __device__ __forceinline__
#define LURK_D __device__ __forceinline__
#else
#define LURK_HD inline
#define LURK_D inline
#endif

#include "field_consts.cuh"

namespace lurk {

// ----------------------------------------------------------------------------- carry-chain primitives
namespace cc {
#if defined(__CUDA_ARCH__)
LURK_D uint32_t add_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
LURK_D uint32_t addc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
LURK_D uint32_t addc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
LURK_D uint32_t sub_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
LURK_D uint32_t subc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
LURK_D uint32_t subc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
LURK_D uint32_t mul_lo(uint32_t a, uint32_t b) { uint32_t r; asm volatile("mul.lo.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
LURK_D uint32_t mul_hi(uint32_t a, uint32_t b) { uint32_t r; asm volatile("mul.hi.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
LURK_D uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("mad.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
LURK_D uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
LURK_D uint32_t mad_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("mad.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
LURK_D uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
LURK_D uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.hi.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
#else
// host emulation of the PTX condition-code register
inline uint32_t &cf() { static thread_local uint32_t f = 0; return f; }
inline uint32_t add_cc(uint32_t a, uint32_t b) { uint64_t s = (uint64_t)a + b; cf() = (uint32_t)(s >> 32); return (uint32_t)s; }
inline uint32_t addc_cc(uint32_t a, uint32_t b) { uint64_t s = (uint64_t)a + b + cf(); cf() = (uint32_t)(s >> 32); return (uint32_t)s; }
inline uint32_t addc(uint32_t a, uint32_t b) { return a + b + cf(); }
inline uint32_t sub_cc(uint32_t a, uint32_t b) { uint64_t d = (uint64_t)a - b; cf() = (uint32_t)(d >> 63); return (uint32_t)d; }
inline uint32_t subc_cc(uint32_t a, uint32_t b) { uint64_t d = (uint64_t)a - b - cf(); cf() = (uint32_t)(d >> 63); return (uint32_t)d; }
inline uint32_t subc(uint32_t a, uint32_t b) { return a - b - cf(); }
inline uint32_t mul_lo(uint32_t a, uint32_t b) { return a * b; }
inline uint32_t mul_hi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
inline uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint64_t s = (uint64_t)(a * b) + c; cf() = (uint32_t)(s >> 32); return (uint32_t)s; }
inline uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint64_t s = (uint64_t)(a * b) + c + cf(); cf() = (uint32_t)(s >> 32); return (uint32_t)s; }
inline uint32_t mad_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint64_t s = (((uint64_t)a * b) >> 32) + c; cf() = (uint32_t)(s >> 32); return (uint32_t)s; }
inline uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint64_t s = (((uint64_t)a * b) >> 32) + c + cf(); cf() = (uint32_t)(s >> 32); return (uint32_t)s; }
inline uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { return (uint32_t)(((uint64_t)a * b) >> 32) + c + cf(); }
#endif
}  // namespace cc

// ----------------------------------------------------------------------------- field element
template <class P>
struct alignas(16) Fe {
    uint32_t v[8];
    using Params = P;

    LURK_HD static Fe zero() { Fe r; for (int i = 0; i < 8; i++) r.v[i] = 0; return r; }
    LURK_HD static Fe one() { Fe r; for (int i = 0; i < 8; i++) r.v[i] = P::ONE(i); return r; }
    LURK_HD static Fe rr() { Fe r; for (int i = 0; i < 8; i++) r.v[i] = P::RR(i); return r; }
    LURK_HD static Fe modulus_raw() { Fe r; for (int i = 0; i < 8; i++) r.v[i] = P::MOD(i); return r; }

    LURK_HD bool is_zero() const { uint32_t o = 0; for (int i = 0; i < 8; i++) o |= v[i]; return o == 0; }
    LURK_HD bool operator==(const Fe &b) const { uint32_t o = 0; for (int i = 0; i < 8; i++) o |= v[i] ^ b.v[i]; return o == 0; }
    LURK_HD bool operator!=(const Fe &b) const { return !(*this == b); }

    // r = (r >= p) ? r - p : r
    LURK_HD void final_sub() {
        uint32_t t[8];
        t[0] = cc::sub_cc(v[0], P::MOD(0));
#pragma unroll
        for (int i = 1; i < 8; i++) t[i] = cc::subc_cc(v[i], P::MOD(i));
        uint32_t borrow = cc::subc(0, 0);   // 0xffffffff when v < p
#pragma unroll
        for (int i = 0; i < 8; i++) v[i] = borrow ? v[i] : t[i];
    }
    // raw (possibly unreduced 256-bit) comparison against p: true when value < p
    LURK_HD bool is_reduced() const {
        uint32_t t = cc::sub_cc(v[0], P::MOD(0));
#pragma unroll
        for (int i = 1; i < 8; i++) t = cc::subc_cc(v[i], P::MOD(i));
        (void)t;
        return cc::subc(0, 0) != 0;
    }

    LURK_HD friend Fe operator+(const Fe &a, const Fe &b) {
        Fe r;
        r.v[0] = cc::add_cc(a.v[0], b.v[0]);
#pragma unroll
        for (int i = 1; i < 7; i++) r.v[i] = cc::addc_cc(a.v[i], b.v[i]);
        r.v[7] = cc::addc(a.v[7], b.v[7]);   // p < 2^255: no carry out
        r.final_sub();
        return r;
    }
    LURK_HD friend Fe operator-(const Fe &a, const Fe &b) {
        Fe r;
        r.v[0] = cc::sub_cc(a.v[0], b.v[0]);
#pragma unroll
        for (int i = 1; i < 8; i++) r.v[i] = cc::subc_cc(a.v[i], b.v[i]);
        uint32_t borrow = cc::subc(0, 0);
        r.v[0] = cc::add_cc(r.v[0], P::MOD(0) & borrow);
#pragma unroll
        for (int i = 1; i < 7; i++) r.v[i] = cc::addc_cc(r.v[i], P::MOD(i) & borrow);
        r.v[7] = cc::addc(r.v[7], P::MOD(7) & borrow);
        return r;
    }
    LURK_HD Fe neg() const { return zero() - *this; }
    LURK_HD Fe dbl() const { return *this + *this; }

    // ---- Montgomery product -------------------------------------------------------------------------
    // acc[0..7] = (a[0], a[2], a[4], a[6]) * bi as four (lo, hi) pairs
    LURK_HD static void mul_n(uint32_t *acc, const uint32_t *a, uint32_t bi) {
#pragma unroll
        for (int j = 0; j < 8; j += 2) { acc[j] = cc::mul_lo(a[j], bi); acc[j + 1] = cc::mul_hi(a[j], bi); }
    }
    // acc[0..7] += (a[0], a[2], a[4], a[6]) * bi, one carry chain; carry-out stays in the flag
    LURK_HD static void cmad_n(uint32_t *acc, const uint32_t *a, uint32_t bi) {
        acc[0] = cc::mad_lo_cc(a[0], bi, acc[0]);
        acc[1] = cc::madc_hi_cc(a[0], bi, acc[1]);
#pragma unroll
        for (int j = 2; j < 8; j += 2) { acc[j] = cc::madc_lo_cc(a[j], bi, acc[j]); acc[j + 1] = cc::madc_hi_cc(a[j], bi, acc[j + 1]); }
    }
    // same with the modulus as the multiplicand (compile-time words become immediates)
    template <int OFF>
    LURK_HD static void cmad_mod(uint32_t *acc, uint32_t mi) {
        acc[0] = cc::mad_lo_cc(P::MOD(OFF), mi, acc[0]);
        acc[1] = cc::madc_hi_cc(P::MOD(OFF), mi, acc[1]);
#pragma unroll
        for (int j = 2; j < 8; j += 2) { acc[j] = cc::madc_lo_cc(P::MOD(OFF + j), mi, acc[j]); acc[j + 1] = cc::madc_hi_cc(P::MOD(OFF + j), mi, acc[j + 1]); }
    }
    // odd <- (odd >> 64) + (a[0], a[2], a[4], a[6]) * bi, consuming the incoming carry flag
    LURK_HD static void madc_n_rshift(uint32_t *odd, const uint32_t *a, uint32_t bi) {
#pragma unroll
        for (int j = 0; j < 6; j += 2) { odd[j] = cc::madc_lo_cc(a[j], bi, odd[j + 2]); odd[j + 1] = cc::madc_hi_cc(a[j], bi, odd[j + 3]); }
        odd[6] = cc::madc_lo_cc(a[6], bi, 0);
        odd[7] = cc::madc_hi(a[6], bi, 0);
    }
    // one row: acc += a*bi; acc += m*p with m chosen so the low word vanishes.  `even` holds columns 0..7,
    // `odd` columns 1..8 of the running sum; the caller swaps them row by row (that is the 32-bit shift).
    template <bool FIRST>
    LURK_HD static void mad_row_redc(uint32_t *even, uint32_t *odd, const uint32_t *a, uint32_t bi) {
        if (FIRST) {
            mul_n(odd, a + 1, bi);
            mul_n(even, a, bi);
        } else {
            even[0] = cc::add_cc(even[0], odd[1]);
            madc_n_rshift(odd, a + 1, bi);
            cmad_n(even, a, bi);
            odd[7] = cc::addc(odd[7], 0);
        }
        uint32_t mi = even[0] * P::M0;
        cmad_mod<1>(odd, mi);
        cmad_mod<0>(even, mi);
        odd[7] = cc::addc(odd[7], 0);
    }

    LURK_HD friend Fe operator*(const Fe &a, const Fe &b) {
#if !defined(__CUDA_ARCH__) && !defined(LURK_HOST_EMULATE_CC)
        return host_mul(a, b);   // host code takes the native 64-bit path (see below)
#else
        uint32_t even[8], odd[8];
        mad_row_redc<true>(even, odd, a.v, b.v[0]);
        mad_row_redc<false>(odd, even, a.v, b.v[1]);
#pragma unroll
        for (int i = 2; i < 8; i += 2) {
            mad_row_redc<false>(even, odd, a.v, b.v[i]);
            mad_row_redc<false>(odd, even, a.v, b.v[i + 1]);
        }
        Fe r;
        r.v[0] = cc::add_cc(even[0], odd[1]);
#pragma unroll
        for (int i = 1; i < 7; i++) r.v[i] = cc::addc_cc(even[i], odd[i + 1]);
        r.v[7] = cc::addc(even[7], 0);
        r.final_sub();
        return r;
#endif
    }
#if !defined(__CUDA_ARCH__)
    // Host-only 4x64-bit CIOS product.  The library's host code (constant generation, final MSM window combine,
    // affine normalisation) uses this; tests define LURK_HOST_EMULATE_CC to run the GPU limb algorithm instead.
    static Fe host_mul(const Fe &a, const Fe &b) {
        typedef unsigned __int128 u128;
        uint64_t A[4], B[4], M[4], t[6] = {0, 0, 0, 0, 0, 0};
        for (int i = 0; i < 4; i++) {
            A[i] = (uint64_t)a.v[2 * i] | ((uint64_t)a.v[2 * i + 1] << 32);
            B[i] = (uint64_t)b.v[2 * i] | ((uint64_t)b.v[2 * i + 1] << 32);
            M[i] = (uint64_t)P::MOD(2 * i) | ((uint64_t)P::MOD(2 * i + 1) << 32);
        }
        uint64_t inv = 1;
        for (int i = 0; i < 6; i++) inv *= 2 - M[0] * inv;
        inv = 0 - inv;
        for (int i = 0; i < 4; i++) {
            uint64_t c = 0;
            for (int j = 0; j < 4; j++) { u128 s = (u128)A[j] * B[i] + t[j] + c; t[j] = (uint64_t)s; c = (uint64_t)(s >> 64); }
            u128 s = (u128)t[4] + c; t[4] = (uint64_t)s; t[5] = (uint64_t)(s >> 64);
            uint64_t m = t[0] * inv;
            s = (u128)m * M[0] + t[0]; c = (uint64_t)(s >> 64);
            for (int j = 1; j < 4; j++) { s = (u128)m * M[j] + t[j] + c; t[j - 1] = (uint64_t)s; c = (uint64_t)(s >> 64); }
            s = (u128)t[4] + c; t[3] = (uint64_t)s; t[4] = t[5] + (uint64_t)(s >> 64);
        }
        bool ge = t[4] != 0;
        if (!ge) {
            ge = true;
            for (int i = 3; i >= 0; i--) { if (t[i] > M[i]) break; if (t[i] < M[i]) { ge = false; break; } }
        }
        if (ge) { uint64_t br = 0; for (int i = 0; i < 4; i++) { u128 d = (u128)t[i] - M[i] - br; t[i] = (uint64_t)d; br = (uint64_t)(d >> 64) & 1; } }
        Fe r;
        for (int i = 0; i < 4; i++) { r.v[2 * i] = (uint32_t)t[i]; r.v[2 * i + 1] = (uint32_t)(t[i] >> 32); }
        return r;
    }
#endif
    // No dedicated squaring (36 word products + doubling instead of 64): the extra carry/shift work lands on the ALU
    // pipe and as IMAD.MOV on the FMA pipe, which ate the saving in an earlier measurement.
    LURK_HD Fe sqr() const { return *this * *this; }
    LURK_HD Fe pow5() const { Fe x2 = sqr(); Fe x4 = x2.sqr(); return x4 * *this; }

    LURK_HD Fe &operator+=(const Fe &b) { *this = *this + b; return *this; }
    LURK_HD Fe &operator-=(const Fe &b) { *this = *this - b; return *this; }
    LURK_HD Fe &operator*=(const Fe &b) { *this = *this * b; return *this; }

    // ---- representation changes ---------------------------------------------------------------------
    // canonical integer (must be < p) -> Montgomery
    LURK_HD static Fe from_canonical(const Fe &raw) { return raw * rr(); }
    // Montgomery -> canonical integer
    LURK_HD Fe to_canonical() const {
        Fe o = zero();
        o.v[0] = 1;
        return *this * o;
    }
    LURK_HD static Fe from_u64(uint64_t x) {
        Fe r = zero();
        r.v[0] = (uint32_t)x;
        r.v[1] = (uint32_t)(x >> 32);
        return from_canonical(r);
    }

    // exponentiation by a raw 256-bit exponent (host-side use: inversion, roots of unity)
    LURK_HD Fe pow_raw(const uint32_t e[8]) const {
        Fe acc = one(), base = *this;
        for (int i = 0; i < 256; i++) {
            if ((e[i >> 5] >> (i & 31)) & 1) acc = acc * base;
            base = base.sqr();
        }
        return acc;
    }
    // Variable-time inversion by the binary extended Euclidean algorithm (shifts, adds and compares only: ~6x fewer
    // dependent multiplier instructions than Fermat for a single thread, which is what the one-thread affine
    // normalisation on the fold's critical chain needs).  Montgomery form in and out; 0 -> 0.
    // Invariants: x1 * a == u, x2 * a == v (mod p) with a the raw input; gcd(a, p) = 1 so the loop ends with u or v = 1.
    LURK_HD Fe inv_vartime() const {
        if (is_zero()) return zero();
        uint32_t u[8], w[8];
        Fe x1 = zero(), x2 = zero();
        x1.v[0] = 1;
#pragma unroll
        for (int i = 0; i < 8; i++) { u[i] = v[i]; w[i] = P::MOD(i); }
        auto is_one = [](const uint32_t *a) { uint32_t o = a[0] ^ 1u; for (int i = 1; i < 8; i++) o |= a[i]; return o == 0; };
        auto shr1 = [](uint32_t *a) { for (int i = 0; i < 7; i++) a[i] = (a[i] >> 1) | (a[i + 1] << 31); a[7] >>= 1; };
        auto halve = [&](Fe &x) {                 // x / 2 mod p on a raw value < p (p < 2^255: x + p cannot overflow)
            if (x.v[0] & 1u) {
                x.v[0] = cc::add_cc(x.v[0], P::MOD(0));
                for (int i = 1; i < 7; i++) x.v[i] = cc::addc_cc(x.v[i], P::MOD(i));
                x.v[7] = cc::addc(x.v[7], P::MOD(7));
            }
            shr1(x.v);
        };
        auto sub_raw = [](uint32_t *a, const uint32_t *b) {   // a -= b, returns the borrow mask
            a[0] = cc::sub_cc(a[0], b[0]);
            for (int i = 1; i < 8; i++) a[i] = cc::subc_cc(a[i], b[i]);
            return cc::subc(0, 0);
        };
        auto geq = [](const uint32_t *a, const uint32_t *b) {
            for (int i = 7; i >= 0; i--) { if (a[i] > b[i]) return true; if (a[i] < b[i]) return false; }
            return true;
        };
        while (!is_one(u) && !is_one(w)) {
            while (!(u[0] & 1u)) { shr1(u); halve(x1); }
            while (!(w[0] & 1u)) { shr1(w); halve(x2); }
            if (geq(u, w)) { sub_raw(u, w); x1 = x1 - x2; }
            else { sub_raw(w, u); x2 = x2 - x1; }
        }
        // raw inverse X = (aR)^-1; the Montgomery form of the inverse is a^-1 R = X R^2 = mont(X, R^3)
        const Fe r3 = rr() * rr();
        return (is_one(u) ? x1 : x2) * r3;
    }
    // Fermat inversion; 0 -> 0
    LURK_HD Fe inv() const {
        uint32_t e[8];
        e[0] = cc::sub_cc(P::MOD(0), 2);
#pragma unroll
        for (int i = 1; i < 8; i++) e[i] = cc::subc_cc(P::MOD(i), 0);
        return pow_raw(e);
    }
};

// ----------------------------------------------------------------------------- wide reduction
// Word-serial Montgomery reduction of a 17-word value t (t[16] small): returns t / 2^256 mod p, fully reduced.
// Row carries that leave an 8-word window go to r[] (columns 8..16): they never feed a reduction multiplier.
// The value before the conditional subtractions must be < (ROUNDS + 1) p.
template <class P, int ROUNDS>
LURK_HD Fe<P> redc17(uint32_t *t) {
    uint32_t r[9];
#pragma unroll
    for (int k = 0; k < 9; k++) r[k] = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        uint32_t mi = t[i] * P::M0;
        Fe<P>::template cmad_mod<0>(t + i, mi);
        r[i] = cc::addc(r[i], 0);
        Fe<P>::template cmad_mod<1>(t + i + 1, mi);
        r[i + 1] = cc::addc(r[i + 1], 0);
    }
    t[8] = cc::add_cc(t[8], r[0]);
#pragma unroll
    for (int k = 1; k < 8; k++) t[8 + k] = cc::addc_cc(t[8 + k], r[k]);
    t[16] = cc::addc(t[16], r[8]);
#pragma unroll
    for (int round = 0; round < ROUNDS; round++) {
        uint32_t d[9];
        d[0] = cc::sub_cc(t[8], P::MOD(0));
#pragma unroll
        for (int k = 1; k < 8; k++) d[k] = cc::subc_cc(t[8 + k], P::MOD(k));
        d[8] = cc::subc_cc(t[16], 0);
        uint32_t borrow = cc::subc(0, 0);
#pragma unroll
        for (int k = 0; k < 9; k++) t[8 + k] = borrow ? t[8 + k] : d[k];
    }
    Fe<P> out;
#pragma unroll
    for (int k = 0; k < 8; k++) out.v[k] = t[8 + k];
    return out;
}

// ----------------------------------------------------------------------------- lazy dot products
// Accumulates up to 9 full 256x256-bit products and performs ONE Montgomery reduction at the end:
//     reduce() = (sum_k a_k * b_k) / 2^256  mod p        (fully reduced)
// which is the Montgomery-form dot product when the inputs are in Montgomery form.  A Poseidon MDS row costs
// t*64 + 72 IMAD.WIDE this way instead of t*137.  Products are accumulated in the same even/odd column split as
// the Montgomery product; carries that leave an 8-word row go to small per-column counters instead of rippling
// (they only ever land on columns >= 8, which no reduction multiplier depends on).
template <class P>
struct WideAcc {
    uint32_t e[17];   // columns 0..16
    uint32_t o[16];   // columns 1..16
    uint32_t ce[5];   // pending carries into e[8], e[10], e[12], e[14], e[16]
    uint32_t co[4];   // pending carries into o[8], o[10], o[12], o[14]

    LURK_HD void clear() {
#pragma unroll
        for (int i = 0; i < 17; i++) e[i] = 0;
#pragma unroll
        for (int i = 0; i < 16; i++) o[i] = 0;
#pragma unroll
        for (int i = 0; i < 5; i++) ce[i] = 0;
#pragma unroll
        for (int i = 0; i < 4; i++) co[i] = 0;
    }

    template <int I>
    LURK_HD void row(const uint32_t *a, uint32_t bi) {
        if (I % 2 == 0) {
            Fe<P>::cmad_n(e + I, a, bi);
            ce[I / 2] = cc::addc(ce[I / 2], 0);
            Fe<P>::cmad_n(o + I, a + 1, bi);
            co[I / 2] = cc::addc(co[I / 2], 0);
        } else {
            Fe<P>::cmad_n(e + I + 1, a + 1, bi);
            ce[(I + 1) / 2] = cc::addc(ce[(I + 1) / 2], 0);
            Fe<P>::cmad_n(o + I - 1, a, bi);
            co[(I - 1) / 2] = cc::addc(co[(I - 1) / 2], 0);
        }
    }
    // += a * b (plain 256-bit integers, each < 2^256)
    LURK_HD void mul_acc(const Fe<P> &a, const Fe<P> &b) {
        row<0>(a.v, b.v[0]); row<1>(a.v, b.v[1]); row<2>(a.v, b.v[2]); row<3>(a.v, b.v[3]);
        row<4>(a.v, b.v[4]); row<5>(a.v, b.v[5]); row<6>(a.v, b.v[6]); row<7>(a.v, b.v[7]);
    }

    // k accumulated products give a value < (k p / 2^256 + 1) p before the final conditional subtractions:
    // ROUNDS = 3 is enough for k <= 11 (Pasta, p/2^256 = 0.25) or k <= 15 (BN254, 0.19); use ROUNDS = 4 up to k = 15.
    template <int ROUNDS = 3>
    LURK_HD Fe<P> reduce() {
        // fold the pending carries
        e[8] = cc::add_cc(e[8], ce[0]);   e[9] = cc::addc_cc(e[9], 0);
        e[10] = cc::addc_cc(e[10], ce[1]); e[11] = cc::addc_cc(e[11], 0);
        e[12] = cc::addc_cc(e[12], ce[2]); e[13] = cc::addc_cc(e[13], 0);
        e[14] = cc::addc_cc(e[14], ce[3]); e[15] = cc::addc_cc(e[15], 0);
        e[16] = cc::addc(e[16], ce[4]);
        o[8] = cc::add_cc(o[8], co[0]);   o[9] = cc::addc_cc(o[9], 0);
        o[10] = cc::addc_cc(o[10], co[1]); o[11] = cc::addc_cc(o[11], 0);
        o[12] = cc::addc_cc(o[12], co[2]); o[13] = cc::addc_cc(o[13], 0);
        o[14] = cc::addc_cc(o[14], co[3]); o[15] = cc::addc(o[15], 0);
        // merge the column split: t = e + (o << 32)
        uint32_t t[17];
        t[0] = e[0];
        t[1] = cc::add_cc(e[1], o[0]);
#pragma unroll
        for (int k = 2; k < 16; k++) t[k] = cc::addc_cc(e[k], o[k - 1]);
        t[16] = cc::addc(e[16], o[15]);
        return redc17<P, ROUNDS>(t);
    }
};

// 128-bit vectorised global access of one 32-byte element
template <class F>
LURK_D F load_fe(const void *p) {
#if defined(__CUDA_ARCH__)
    const uint4 *q = reinterpret_cast<const uint4 *>(p);
    uint4 lo = q[0], hi = q[1];
    F r;
    r.v[0] = lo.x; r.v[1] = lo.y; r.v[2] = lo.z; r.v[3] = lo.w;
    r.v[4] = hi.x; r.v[5] = hi.y; r.v[6] = hi.z; r.v[7] = hi.w;
    return r;
#else
    F r; memcpy(r.v, p, 32); return r;
#endif
}
template <class F>
LURK_D void store_fe(void *p, const F &x) {
#if defined(__CUDA_ARCH__)
    uint4 *q = reinterpret_cast<uint4 *>(p);
    q[0] = make_uint4(x.v[0], x.v[1], x.v[2], x.v[3]);
    q[1] = make_uint4(x.v[4], x.v[5], x.v[6], x.v[7]);
#else
    memcpy(p, x.v, 32);
#endif
}

}  // namespace lurk
