// The opening provers' scratch (HyperKZG: kzg.cu, the inner-product argument: ipa.cu) as an object the caller can keep, and the host
// point arithmetic the compress context (compress.cu) needs around them.  lurk_hyperkzg_prove_dev / lurk_ipa_prove_dev build a fresh
// arena per call, so they allocate what they always did, where they always did; lurk_compress_ctx keeps one per circuit, grown by its
// first proof and reused by every later one (no cudaMalloc / cudaFree, no stream or clone creation on the proving path).
#pragma once
#include "common.cuh"
#include "sc_scratch.cuh"

namespace lurk {

struct PcsArena {
    // declared in the order the one-shot HyperKZG prover created them, so that they are released in the order it released them
    DevBuf polys;                 // HyperKZG: the fold chain P_0 | P_1 | .. (2n);  compress's IPA: a (n) | b (n)
    MsmCloneGuard clone[2];       // clones of the key context (own scratch, same resident key): HyperKZG 2, IPA 1
    StreamGuard side[2];
    EventGuard ready;
    DevBuf chunks, first, partial, v;     // HyperKZG: the evaluation chunks and their partial sums
    DevBuf B, h, scan;            // HyperKZG: the batched polynomial (n), the witness polynomials (3n), the up-sweep levels
    DevBuf weights;               // IPA: the key weights W | sl | sr (3n)
    // the buffer holds at least `bytes`; a fresh DevBuf gets exactly `bytes` (what the one-shot entry points allocated)
    static int grow(DevBuf &b, size_t bytes) { return b.bytes >= bytes ? LURK_OK : b.alloc(bytes); }
    int clones(lurk_msm_ctx *ck, int k) {
        for (int i = 0; i < k; i++) {
            if (!clone[i].c) LURK_TRY(lurk_msm_ctx_clone(ck, &clone[i].c));
            if (!side[i].s) LURK_TRY(side[i].create());
        }
        return LURK_OK;
    }
    int event() { return ready.e ? LURK_OK : ready.create(); }
    size_t device_bytes() const {
        return polys.bytes + B.bytes + h.bytes + scan.bytes + chunks.bytes + first.bytes + partial.bytes + v.bytes + weights.bytes;
    }
};

// provider::hyperkzg::EvaluationEngine::prove on the arena; d_poly may be the arena's P_0 (the joint polynomial written in place), then
// the copy into P_0 is skipped.  `ck` has been checked by the caller (curve, >= 2^l bases).
int hyperkzg_prove_arena(int curve_id, lurk_msm_ctx *ck, PcsArena &a, const void *d_poly, const uint8_t *point, int l, lurk_challenge_fn challenge,
                         void *user, uint8_t *com_out, uint8_t *w_out, uint8_t *v_out, int fmt, cudaStream_t s);
// InnerProductArgument::prove's rounds on the arena; d_a / d_b consumed as by lurk_ipa_prove_dev
int ipa_prove_arena(int curve_id, lurk_msm_ctx *ck, PcsArena &a, const uint8_t *gc_bytes, void *d_a, void *d_b, int log_n, lurk_challenge_fn challenge,
                    void *user, uint8_t *L_out, uint8_t *R_out, uint8_t *a_final, uint8_t *b_final, int fmt, cudaStream_t s);
// InnerProductArgument::verify as lurk_ipa_verify_dev runs it, for a caller that has checked the key (curve, >= 2^log_n bases) and the pointers
int ipa_verify_checked(int curve_id, lurk_msm_ctx *ck, const uint8_t *gc_bytes, const uint8_t *comm, const uint8_t *c, const void *d_b, int log_n,
                       const uint8_t *L, const uint8_t *R, const uint8_t *a_final, lurk_challenge_fn challenge, void *user, int *accepted, int fmt,
                       cudaStream_t s);
// b of y^2 = x^3 + b
template <class C>
static typename C::Base curve_b() {
    const Affine<typename C::Base> g = curve_generator<C>();
    return g.y.sqr() - g.x.sqr() * g.x;
}
// a 96-byte point x | y | z of the header's convention (z = 1, or x = y = z = 0 for the identity), on the curve y^2 = x^3 + b
template <class Fb>
static bool point_in(const uint8_t *in, int fmt, const Fb &b, XYZZ<Fb> &out) {
    Affine<Fb> p;
    Fb z;
    if (!fe_in(in, fmt, p.x) || !fe_in(in + 32, fmt, p.y) || !fe_in(in + 64, fmt, z)) return false;
    if (z.is_zero()) { out = XYZZ<Fb>::identity(); return p.x.is_zero() && p.y.is_zero(); }
    if (z != Fb::one() || p.y.sqr() != p.x.sqr() * p.x + b) return false;
    out = XYZZ<Fb>::from_affine(p);
    return true;
}
// the point in that form: x | y | 1, or 0 | 0 | 0
template <class Fb>
static void point_to_bytes_fmt(const XYZZ<Fb> &p, int fmt, uint8_t out[96]) {
    memset(out, 0, 96);
    if (p.is_identity()) return;
    Affine<Fb> a = p.to_affine();
    Fb one = Fb::one();
    if (fmt == LURK_FMT_CANONICAL) { a.x = a.x.to_canonical(); a.y = a.y.to_canonical(); one = one.to_canonical(); }
    memcpy(out, a.x.v, 32); memcpy(out + 32, a.y.v, 32); memcpy(out + 64, one.v, 32);
}

// every 96-byte point x | y | z of the header's form (z = 1 on the curve, or the identity 0 | 0 | 0), in `fmt`; host only
bool points_valid(int curve_id, const uint8_t *const *points, int count, int fmt);
// an affine point x | y (identity = (0, 0)) of the curve, in `fmt`; host only
bool affine_valid(int curve_id, const uint8_t *xy, int fmt);
// out = sum_k scalars[k] points[k] (points as points_valid takes them, scalars 32 bytes each), a 96-byte point in `fmt`; host only
int point_combination(int curve_id, const uint8_t *const *points, const uint8_t *scalars, int count, int fmt, uint8_t out[96]);
// r ck_c for the affine ck_c (x | y, `fmt`) and the scalar r (`fmt`) as an affine x | y in `fmt`; host only
int scale_affine(int curve_id, const uint8_t *xy, const uint8_t *r, int fmt, uint8_t out[64]);

// Batched point combination (pointcomb.cu).  One group: out = sum_k scalars[k] points[k], as point_combination takes and writes them.
struct PointGroup {
    const uint8_t *const *points;
    const uint8_t *scalars;
    int count;
    uint8_t *out;
};
constexpr int PC_MAX_TERMS = LURK_POINT_COMBINATION_MAX_TERMS;     // per group on the device
// Every group checked first (the messages of point_combination, with the group's index), then: the groups of at least
// PC_DEVICE_MIN_TERMS terms (every group with `all_device`) combined by one kernel on `s` while the host combines the others.
// Returns when all are written; the bytes are point_combination's.
int point_combination_groups(int curve_id, const PointGroup *groups, int n_groups, int fmt, bool all_device, cudaStream_t s);

}  // namespace lurk
