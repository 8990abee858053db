// The satisfiability half of RecursiveSNARK::verify (Proof::verify on a Recursive proof, reference src/proof/nova.rs:358-373,
// supernova.rs:304-317) as one C-ABI call: R1CSShape::is_sat_relaxed on every running instance and is_sat on the secondary's last
// fresh instance, i.e. per instance one r1cs_sat_kernel pass over the shape (spmv3.cuh) and the recomputed commit(W) / commit(E) on the
// borrowed key.  Every distinct key gets a stream forked from the caller's and a host thread that runs its instances one after the
// other (a key context holds one pending launch), so the primary and the secondary curve run at once -- Arecibo's rayon::join of the
// is_sat calls.  The RO hashes of RecursiveSNARK::verify stay with the caller.
#include "msm_impl.cuh"
#include "pcs.cuh"
#include "sc_scratch.cuh"
#include "spmv3.cuh"

#include <algorithm>
#include <array>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

namespace lurk {

void spartan_ctx_shape(const lurk_spartan_ctx *ctx, int *field_id, uint64_t *n_w, uint64_t *n_x, uint64_t *rows, CsrDev csr[3]);   // spartan.cu

constexpr int RV_MAX_INSTANCES = 32;       // 30 SuperNova primaries (the batched Spartan prover's limit) + the secondary's two

struct RvInst {
    int field = 0;
    uint64_t n_w = 0, n_x = 0, rows = 0;
    CsrDev csr[3];
    lurk_msm_ctx *ck = nullptr;
    const void *z = nullptr, *E = nullptr;   // device, Montgomery
    const uint8_t *comm_W = nullptr, *comm_E = nullptr;
    int key = 0;                             // index of its key's stream
    size_t z_len() const { return n_w + 1 + n_x; }
};

// host-only checks that read no context
static int check_pointers(int n, const lurk_recursive_instance *inst, const lurk_recursive_verdict *out, const int *accepted, int fmt) {
    if (n < 1 || n > RV_MAX_INSTANCES) { set_error("1..%d instances, got %d", RV_MAX_INSTANCES, n); return LURK_ERR_ARG; }
    if (!inst) { set_error("null instance array"); return LURK_ERR_ARG; }
    if (!out) { set_error("null verdict array"); return LURK_ERR_ARG; }
    if (!accepted) { set_error("null accepted"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    for (int i = 0; i < n; i++) {
        const lurk_recursive_instance &x = inst[i];
        if (!x.shape) { set_error("instance %d: null shape", i); return LURK_ERR_ARG; }
        if (!x.ck) { set_error("instance %d: null key context", i); return LURK_ERR_ARG; }
        if (!x.z) { set_error("instance %d: null z", i); return LURK_ERR_ARG; }
        if (!x.comm_W) { set_error("instance %d: null comm_W", i); return LURK_ERR_ARG; }
        if (!x.E != !x.comm_E) { set_error("instance %d: E and comm_E go together (both for a relaxed instance, neither for a strict one)", i); return LURK_ERR_ARG; }
    }
    return LURK_OK;
}

// the checks that read the shapes and keys: after the GPU check, before any device work
static int check_contexts(int n, const lurk_recursive_instance *inst, int fmt, std::vector<RvInst> &I, std::vector<lurk_msm_ctx *> &keys) {
    int dev = -1;
    LURK_CUDA_TRY(cudaGetDevice(&dev));
    I.resize(n);
    for (int i = 0; i < n; i++) {
        const lurk_recursive_instance &x = inst[i];
        RvInst &v = I[i];
        spartan_ctx_shape(x.shape, &v.field, &v.n_w, &v.n_x, &v.rows, v.csr);
        v.ck = x.ck;
        v.z = x.z;
        v.E = x.E;
        v.comm_W = x.comm_W;
        v.comm_E = x.comm_E;
        // LURK_CURVE_k's scalar field is LURK_FIELD_k
        if (x.ck->curve_id != v.field) {
            set_error("instance %d: the key is on curve %d, the shape's field %d needs curve %d", i, x.ck->curve_id, v.field, v.field);
            return LURK_ERR_ARG;
        }
        const uint64_t need = std::max(v.n_w, v.rows);
        if (x.ck->n < need) { set_error("instance %d: the key has %zu bases, the shape needs %llu", i, x.ck->n, (unsigned long long)need); return LURK_ERR_ARG; }
        if (x.ck->device != dev) { set_error("instance %d: the key belongs to device %d, device %d is current", i, x.ck->device, dev); return LURK_ERR_ARG; }
        if (x.ck->pending) { set_error("instance %d: a launch is pending on the key context", i); return LURK_ERR_ARG; }
        const uint8_t *pts[2] = {x.comm_W, x.comm_E};
        if (!points_valid(v.field, pts, x.comm_E ? 2 : 1, fmt)) {
            set_error("instance %d: a commitment is not a point of the header's form on curve %d", i, v.field);
            return LURK_ERR_RANGE;
        }
        v.key = (int)(std::find(keys.begin(), keys.end(), x.ck) - keys.begin());
        if (v.key == (int)keys.size()) keys.push_back(x.ck);
    }
    return LURK_OK;
}

// every element of z and E below p; u of every instance (Montgomery) into u_mont
static int check_ranges(const std::vector<RvInst> &I, std::array<uint8_t, 32> *u_mont, cudaStream_t s) {
    for (size_t i = 0; i < I.size(); i++) {
        const RvInst &v = I[i];
        int bad_z = 0, bad_e = 0;
        LURK_TRY(dispatch_field(v.field, [&](auto f) {
            using F = decltype(f);
            LURK_TRY(check_reduced_dev<F>(v.z, v.z_len(), s, &bad_z));
            if (v.E) LURK_TRY(check_reduced_dev<F>(v.E, v.rows, s, &bad_e));
            return LURK_OK;
        }));
        if (bad_z) { set_error("instance %zu: %d element(s) of z not reduced below the field modulus", i, bad_z); return LURK_ERR_RANGE; }
        if (bad_e) { set_error("instance %zu: %d element(s) of E not reduced below the field modulus", i, bad_e); return LURK_ERR_RANGE; }
        LURK_CUDA_TRY(cudaMemcpyAsync(u_mont[i].data(), static_cast<const uint8_t *>(v.z) + 32 * v.n_w, 32, cudaMemcpyDeviceToHost, s));
    }
    LURK_CUDA_TRY(cudaStreamSynchronize(s));
    return LURK_OK;
}

// a point as points_valid admits it (x | y | 1, or 0 | 0 | 0), in `fmt`, to the same form in Montgomery: the form a finished commitment
// over Montgomery scalars has, so the two compare as bytes
static void point_to_mont(int curve_id, const uint8_t in[96], int fmt, uint8_t out[96]) {
    dispatch_field(curve_id ^ 1, [&](auto f) {     // the base field of curve k is field k ^ 1
        using F = decltype(f);
        F x;
        for (int k = 0; k < 3; k++) {
            fe_in(in + 32 * k, fmt, x);
            fe_out(x, LURK_FMT_MONTGOMERY, out + 32 * k);
        }
        return LURK_OK;
    });
}

// commit(v) on the key against the expected point (Montgomery bytes)
static int commitment_holds(lurk_msm_ctx *ck, const void *v, size_t n, const uint8_t want[96], cudaStream_t s, int *ok) {
    uint8_t have[96];
    LURK_TRY(lurk_msm_ctx_launch_dev(ck, v, n, LURK_FMT_MONTGOMERY, s));
    LURK_TRY(lurk_msm_ctx_finish(ck, have));
    *ok = memcmp(have, want, 96) == 0;
    return LURK_OK;
}

// one key's instances, in order, on its stream: r1cs_sat_kernel, commit(W), commit(E)
static int run_key(const std::vector<RvInst> &I, int key, SatCount *d_count, lurk_recursive_verdict *out, int fmt, cudaStream_t s) {
    for (size_t i = 0; i < I.size(); i++) {
        const RvInst &v = I[i];
        if (v.key != key) continue;
        LURK_TRY(dispatch_field(v.field, [&](auto f) {
            using F = decltype(f);
            return r1cs_sat_launch<F>(v.csr, v.rows, static_cast<const F *>(v.z), v.n_w, static_cast<const F *>(v.E), nullptr, d_count + i, s);
        }));
        uint8_t want[96];
        point_to_mont(v.field, v.comm_W, fmt, want);
        LURK_TRY(commitment_holds(v.ck, v.z, v.n_w, want, s, &out[i].comm_W_ok));
        out[i].comm_E_ok = 1;
        if (v.E) {
            point_to_mont(v.field, v.comm_E, fmt, want);
            LURK_TRY(commitment_holds(v.ck, v.E, v.rows, want, s, &out[i].comm_E_ok));
        }
    }
    return LURK_OK;
}

// the device instances checked and in place: fork one stream per key, run, join, collect the verdicts
static int verify_dev(std::vector<RvInst> &I, const std::vector<lurk_msm_ctx *> &keys, const std::array<uint8_t, 32> *u_mont, lurk_recursive_verdict *out,
                      int *accepted, int fmt, cudaStream_t s) {
    const int n = (int)I.size(), nk = (int)keys.size();
    for (int i = 0; i < n; i++) {
        memset(&out[i], 0, sizeof out[i]);
        // a strict instance is (W, 1, X): its u slot must hold one
        out[i].u_ok = 1;
        if (!I[i].E)
            dispatch_field(I[i].field, [&](auto f) {
                using F = decltype(f);
                const F one = F::one();
                out[i].u_ok = memcmp(u_mont[i].data(), one.v, 32) == 0;
                return LURK_OK;
            });
    }
    StreamBuf counts;
    LURK_TRY(counts.alloc(sizeof(SatCount) * n, s));
    EventGuard fork;
    LURK_TRY(fork.create());
    LURK_CUDA_TRY(cudaEventRecord(fork.e, s));
    std::vector<StreamGuard> ks(nk);
    std::vector<EventGuard> join(nk);
    for (int k = 0; k < nk; k++) {
        LURK_TRY(ks[k].create());
        LURK_TRY(join[k].create());
        LURK_CUDA_TRY(cudaStreamWaitEvent(ks[k].s, fork.e, 0));
    }
    std::vector<int> rc(nk, LURK_OK);
    std::vector<std::string> msg(nk);
    int dev = 0;
    LURK_CUDA_TRY(cudaGetDevice(&dev));
    auto run = [&](int k) {
        cudaSetDevice(dev);
        rc[k] = run_key(I, k, static_cast<SatCount *>(counts.p), out, fmt, ks[k].s);
        if (rc[k] != LURK_OK) msg[k] = lurk_last_error();
    };
    std::vector<std::thread> th;
    for (int k = 1; k < nk; k++) th.emplace_back(run, k);
    run(0);
    for (std::thread &t : th) t.join();
    // join every key stream into the caller's, errors included: the scratch is freed in the caller's stream order
    for (int k = 0; k < nk; k++) {
        cudaEventRecord(join[k].e, ks[k].s);
        cudaStreamWaitEvent(s, join[k].e, 0);
    }
    std::vector<SatCount> cnt(n);
    const cudaError_t e = cudaMemcpyAsync(cnt.data(), counts.p, sizeof(SatCount) * n, cudaMemcpyDeviceToHost, s);
    const cudaError_t e2 = cudaStreamSynchronize(s);
    for (int k = 0; k < nk; k++)
        if (rc[k] != LURK_OK) {
            set_error("%s", msg[k].c_str());
            return rc[k];
        }
    LURK_CUDA_TRY(e);
    LURK_CUDA_TRY(e2);
    int all = 1;
    for (int i = 0; i < n; i++) {
        out[i].bad_rows = cnt[i].bad;
        out[i].first_bad_row = cnt[i].first;
        all &= out[i].bad_rows == 0 && out[i].u_ok && out[i].comm_W_ok && out[i].comm_E_ok;
    }
    *accepted = all;
    return LURK_OK;
}

}  // namespace lurk

using namespace lurk;

extern "C" {

int lurk_recursive_verify_dev(int n, const lurk_recursive_instance *inst, lurk_recursive_verdict *out, int *accepted, int fmt, void *stream) {
    LURK_TRY(check_pointers(n, inst, out, accepted, fmt));
    LURK_TRY(require_gpu());
    std::vector<RvInst> I;
    std::vector<lurk_msm_ctx *> keys;
    LURK_TRY(check_contexts(n, inst, fmt, I, keys));
    *accepted = 0;
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    std::vector<std::array<uint8_t, 32>> u(n);
    LURK_TRY(check_ranges(I, u.data(), s));
    return verify_dev(I, keys, u.data(), out, accepted, fmt, s);
}

int lurk_recursive_verify(int n, const lurk_recursive_instance *inst, lurk_recursive_verdict *out, int *accepted, int fmt, void *stream) {
    LURK_TRY(check_pointers(n, inst, out, accepted, fmt));
    LURK_TRY(require_gpu());
    std::vector<RvInst> I;
    std::vector<lurk_msm_ctx *> keys;
    LURK_TRY(check_contexts(n, inst, fmt, I, keys));
    *accepted = 0;
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    // each instance's z and E into stream-ordered scratch, range-checked as they are, then converted in place
    std::vector<StreamBuf> bufs(2 * (size_t)n);
    for (int i = 0; i < n; i++) {
        RvInst &v = I[i];
        const void *src[2] = {v.z, v.E};
        const size_t len[2] = {v.z_len(), v.E ? v.rows : 0};
        const void **dst[2] = {&v.z, &v.E};
        for (int k = 0; k < 2; k++) {
            if (!src[k]) continue;
            StreamBuf &b = bufs[2 * i + k];
            LURK_TRY(b.alloc(32 * len[k], s));
            if (len[k]) LURK_CUDA_TRY(cudaMemcpyAsync(b.p, src[k], 32 * len[k], cudaMemcpyHostToDevice, s));
            *dst[k] = b.p;
        }
    }
    std::vector<std::array<uint8_t, 32>> u(n);
    LURK_TRY(check_ranges(I, u.data(), s));
    if (fmt == LURK_FMT_CANONICAL)
        for (int i = 0; i < n; i++) {
            RvInst &v = I[i];
            LURK_TRY(dispatch_field(v.field, [&](auto f) {
                using F = decltype(f);
                LURK_TRY(convert_dev<F>(v.z, v.z_len(), LURK_FMT_MONTGOMERY, const_cast<void *>(v.z), s));
                if (v.E) LURK_TRY(convert_dev<F>(v.E, v.rows, LURK_FMT_MONTGOMERY, const_cast<void *>(v.E), s));
                // u as the device now holds it
                F x;
                fe_in(u[i].data(), LURK_FMT_CANONICAL, x);
                fe_out(x, LURK_FMT_MONTGOMERY, u[i].data());
                return LURK_OK;
            }));
        }
    return verify_dev(I, keys, u.data(), out, accepted, fmt, s);
}

}  // extern "C"
