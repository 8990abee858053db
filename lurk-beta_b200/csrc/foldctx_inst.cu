// Host side of the fold context for one curve (compiled once per curve: -DLURK_C=<curve>); see foldctx_impl.cuh.
#include "foldctx_impl.cuh"
#include "sha256.cuh"

#include <cuda.h>      // types of the green-context driver API only; entry points are resolved at run time
#include <cstring>

namespace lurk {
LURK_MSM_EXTERN(LURK_C)
#define LURK_FOLD_POSEIDON_EXTERN(F)                                                                          \
    extern template int launch_poseidon<F, true>(int, const void *, size_t, void *, int, int, cudaStream_t, const uint64_t *, const PoseidonGather *); \
    extern template int poseidon_instance_info<F>(int, const PoseidonParams<F> **, PoseidonLayout *);        \
    extern template int launch_bitdecomp<F>(const void *, size_t, void *, int, int, cudaStream_t, const uint64_t *); \
    extern template size_t sha256_block_len<F>(int);                                                          \
    extern template int launch_sha256_witness<F>(const void *, size_t, int, void *, const uint64_t *, int, int, cudaStream_t); \
    extern template size_t trie_block_len<F>(int, int);                                                       \
    extern template int launch_trie_witness<F>(int, int, const void *, size_t, void *, const uint64_t *, int, int, cudaStream_t);
LURK_FOLD_POSEIDON_EXTERN(Fe<Bn254Fr>)
LURK_FOLD_POSEIDON_EXTERN(Fe<Bn254Fq>)
LURK_FOLD_POSEIDON_EXTERN(Fe<PallasFq>)
LURK_FOLD_POSEIDON_EXTERN(Fe<PallasFp>)

static inline int fold_grid(size_t n, int block, int per_sm) {
    size_t want = (n + block - 1) / block;
    size_t cap = (size_t)sm_count() * per_sm;
    return (int)(want < cap ? (want ? want : 1) : cap);
}

// SAFE sponge IO-pattern tag of [Absorb(n), Squeeze(1)] with no domain separator (neptune sponge::api::IOPattern::value):
// x = 2^128 - 159; every op value v (Absorb(n) = n + 2^31, Squeeze(n) = n) and finally the domain separator (0) update
// x_i *= x; state += x_i * v in wrapping 128-bit arithmetic.
static inline unsigned __int128 safe_io_tag(uint32_t n_absorb, uint32_t n_squeeze) {
    typedef unsigned __int128 u128;
    const u128 x = (u128)0 - 159;
    u128 xi = 1, state = 0;
    auto update = [&](u128 a) { xi *= x; state += xi * a; };
    update((u128)n_absorb + ((u128)1 << 31));
    update((u128)n_squeeze);
    update(0);
    return state;
}

template <class C>
struct FoldCtx final : FoldCtxBase {
    using Fb = typename C::Base;
    using Fs = typename C::Scalar;
    using Pt = XYZZ<Fb>;
    using Rec = FoldRecord<Fb, Fs>;

    FoldConfigHost cfg;
    int field_id = 0;                       // witness field (LURK_FIELD_*), for the slot kernels' dispatch-free calls
    size_t nz = 0;                          // |z| = n_w + 1 + n_x
    int D = 2;
    lurk_msm_ctx *ckW[FOLD_MAX_DEPTH] = {nullptr, nullptr, nullptr, nullptr};
    lurk_msm_ctx *ckT = nullptr, *ckChk = nullptr, *ckChkW = nullptr, *ckWbase = nullptr;
    DevBuf z1, e1, T, mv1[3], z2[FOLD_MAX_DEPTH], mv2[FOLD_MAX_DEPTH][3];
    DevBuf csr_rp[3], csr_col[3], csr_val[3];
    CsrDev csr[3];
    DevBuf ro_img, step_consts[FOLD_MAX_DEPTH], r_dev, seq_dev, rec_dev[FOLD_MAX_DEPTH + 1], run_pts, xchg, bad_dev, dummy_w, dummy_p;
    bool dummy_ready = false;
    Rec *h_rec[FOLD_MAX_DEPTH + 1] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    void *h_glue[FOLD_MAX_DEPTH] = {nullptr, nullptr, nullptr, nullptr};
    void *h_x2[FOLD_MAX_DEPTH] = {nullptr, nullptr, nullptr, nullptr};
    void *h_ro[FOLD_MAX_DEPTH] = {nullptr, nullptr, nullptr, nullptr};
    size_t glue_elems = 0;
    std::vector<std::unique_ptr<FoldSlotBatch>> batches;
    std::vector<FoldSpan> spans;
    // RO
    PoseidonLayout roL{};
    Fb io_tag;
    int n_absorb = 0, challenge_bits = 128;
    unsigned char kinds[FOLD_RO_RATE];
    // exchange
    XchgBuf<Fb> *peers[FOLD_MAX_WORLD];
    bool peers_open[FOLD_MAX_WORLD];
    bool peers_set = false;
    // streams / events
    cudaStream_t sH = nullptr, sK[3] = {nullptr, nullptr, nullptr}, sA = nullptr, sB = nullptr, sC = nullptr, sT = nullptr;
    bool partitioned = false;
    cudaEvent_t ev_h2d[FOLD_MAX_DEPTH], ev_slot[FOLD_MAX_DEPTH][3], ev_cw[FOLD_MAX_DEPTH], ev_A[FOLD_MAX_DEPTH], ev_fold[FOLD_MAX_DEPTH],
        ev_chal[FOLD_MAX_DEPTH + 1], ev_done[FOLD_MAX_DEPTH + 1];
    bool fold_recorded[FOLD_MAX_DEPTH] = {false, false, false, false};
    bool a_recorded[FOLD_MAX_DEPTH] = {false, false, false, false};
    bool b_pending[FOLD_MAX_DEPTH + 1] = {false, false, false, false, false};
    bool running_set = false;
    bool mv1_valid = false;           // mv1 = (A z1, B z1, C z1) is kept current by the fold itself
    unsigned launches_a = 0, launches_b = 0;
    int device = 0;
    // green contexts (optional SM partition)
    void *green[2] = {nullptr, nullptr};
    int partition_sms[2] = {0, 0};

    FoldCtx() {
        for (int p = 0; p < FOLD_MAX_WORLD; p++) { peers[p] = nullptr; peers_open[p] = false; }
        for (int b = 0; b < FOLD_MAX_DEPTH; b++) {
            ev_h2d[b] = ev_cw[b] = ev_A[b] = ev_fold[b] = nullptr;
            for (int k = 0; k < 3; k++) ev_slot[b][k] = nullptr;
        }
        for (int b = 0; b <= FOLD_MAX_DEPTH; b++) ev_chal[b] = ev_done[b] = nullptr;
        memset(kinds, 0, sizeof kinds);
    }

    ~FoldCtx() override {
        cudaDeviceSynchronize();
        for (int p = 0; p < FOLD_MAX_WORLD; p++)
            if (peers_open[p]) cudaIpcCloseMemHandle(peers[p]);
        for (int b = 0; b < FOLD_MAX_DEPTH; b++) {
            if (ckW[b]) lurk_msm_ctx_destroy(ckW[b]);
            if (h_glue[b]) cudaFreeHost(h_glue[b]);
            if (h_x2[b]) cudaFreeHost(h_x2[b]);
            if (h_ro[b]) cudaFreeHost(h_ro[b]);
            for (cudaEvent_t e : {ev_h2d[b], ev_cw[b], ev_A[b], ev_fold[b], ev_slot[b][0], ev_slot[b][1], ev_slot[b][2]})
                if (e) cudaEventDestroy(e);
        }
        for (int b = 0; b <= FOLD_MAX_DEPTH; b++) {
            if (h_rec[b]) cudaFreeHost(h_rec[b]);
            if (ev_chal[b]) cudaEventDestroy(ev_chal[b]);
            if (ev_done[b]) cudaEventDestroy(ev_done[b]);
        }
        if (ckT) lurk_msm_ctx_destroy(ckT);
        if (ckChk) lurk_msm_ctx_destroy(ckChk);
        if (ckChkW) lurk_msm_ctx_destroy(ckChkW);
        if (ckWbase) lurk_msm_ctx_destroy(ckWbase);
        for (auto &sb : batches)
            for (int b = 0; b < FOLD_MAX_DEPTH; b++)
                if (sb->h_pre[b]) cudaFreeHost(sb->h_pre[b]);
        for (cudaStream_t s : {sH, sK[0], sK[1], sK[2], sA, sB, sC, partitioned ? sT : (cudaStream_t) nullptr})
            if (s) cudaStreamDestroy(s);
        green_destroy();
    }

    // ------------------------------------------------------------------------------------------ SM partition
    // Green contexts (CUDA driver API, resolved at run time so that the library still loads without libcuda): `latency_sms`
    // SMs for the latency-shaped kernels of the chain, the rest for the bucket-accumulation kernels and stage A.
    template <class Fn>
    static bool drv(const char *name, Fn *out) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) {
            cudaGetLastError();
            return false;
        }
        *out = reinterpret_cast<Fn>(p);
        return true;
    }
    void green_destroy() {
        typedef CUresult (*destroy_t)(CUgreenCtx);
        destroy_t fn = nullptr;
        if ((green[0] || green[1]) && drv("cuGreenCtxDestroy", &fn))
            for (void *g : green)
                if (g) fn((CUgreenCtx)g);
        green[0] = green[1] = nullptr;
    }
    // Splits the device into a tiny partition (`tiny_sms` SMs: the single-CTA kernels of the chain) and the rest (everything
    // else) and creates the streams of both.
    int green_streams(int tiny_sms, cudaStream_t *tiny, int n_tiny, cudaStream_t *big_hi, cudaStream_t *big_lo, int n_lo) {
        typedef CUresult (*get_res_t)(CUdevice, CUdevResource *, CUdevResourceType);
        typedef CUresult (*split_t)(CUdevResource *, unsigned *, const CUdevResource *, CUdevResource *, unsigned, unsigned);
        typedef CUresult (*gen_desc_t)(CUdevResourceDesc *, CUdevResource *, unsigned);
        typedef CUresult (*green_create_t)(CUgreenCtx *, CUdevResourceDesc, CUdevice, unsigned);
        typedef CUresult (*green_stream_t)(CUstream *, CUgreenCtx, unsigned, int);
        get_res_t get_res; split_t split; gen_desc_t gen_desc; green_create_t green_create; green_stream_t green_stream;
        if (!drv("cuDeviceGetDevResource", &get_res) || !drv("cuDevSmResourceSplitByCount", &split) ||
            !drv("cuDevResourceGenerateDesc", &gen_desc) || !drv("cuGreenCtxCreate", &green_create) ||
            !drv("cuGreenCtxStreamCreate", &green_stream))
            return LURK_ERR_CUDA;
        CUdevResource all, part, rest;
        if (get_res((CUdevice)device, &all, CU_DEV_RESOURCE_TYPE_SM)) return LURK_ERR_CUDA;
        unsigned groups = 1;
        if (split(&part, &groups, &all, &rest, 0, (unsigned)tiny_sms) || groups != 1) return LURK_ERR_CUDA;
        CUdevResourceDesc desc[2] = {nullptr, nullptr};
        if (gen_desc(&desc[0], &part, 1) || gen_desc(&desc[1], &rest, 1)) return LURK_ERR_CUDA;
        if (green_create((CUgreenCtx *)&green[0], desc[0], (CUdevice)device, CU_GREEN_CTX_DEFAULT_STREAM) ||
            green_create((CUgreenCtx *)&green[1], desc[1], (CUdevice)device, CU_GREEN_CTX_DEFAULT_STREAM)) { green_destroy(); return LURK_ERR_CUDA; }
        partition_sms[0] = (int)part.sm.smCount;
        partition_sms[1] = (int)rest.sm.smCount;
        int rc = 0;
        for (int k = 0; k < n_tiny; k++) rc |= green_stream((CUstream *)(tiny + k), (CUgreenCtx)green[0], CU_STREAM_NON_BLOCKING, -1);
        rc |= green_stream((CUstream *)big_hi, (CUgreenCtx)green[1], CU_STREAM_NON_BLOCKING, -1);
        for (int k = 0; k < n_lo; k++) rc |= green_stream((CUstream *)(big_lo + k), (CUgreenCtx)green[1], CU_STREAM_NON_BLOCKING, 0);
        if (rc) { green_destroy(); return LURK_ERR_CUDA; }
        return LURK_OK;
    }

    // ------------------------------------------------------------------------------------------ creation
    int init(const FoldConfigHost &c, const uint64_t *const row_ptr[3], const uint32_t *const col[3], const uint8_t *const val[3], int fmt,
             lurk_msm_ctx *ck_w, lurk_msm_ctx *ck_t) override {
        cfg = c;
        D = c.depth;
        nz = (size_t)c.n_w + 1 + (size_t)c.n_x;
        field_id = C::ID == 0 ? LURK_FIELD_BN254_FR : C::ID == 1 ? LURK_FIELD_BN254_FQ : C::ID == 2 ? LURK_FIELD_PALLAS_FQ : LURK_FIELD_PALLAS_FP;
        LURK_CUDA_TRY(cudaGetDevice(&device));
        if (ck_w->curve_id != C::ID || ck_t->curve_id != C::ID) { set_error("commitment key belongs to another curve"); return LURK_ERR_ARG; }
        if (ck_w->n < c.n_w || ck_t->n < c.n_rows) { set_error("commitment key shorter than the witness / the constraint count"); return LURK_ERR_ARG; }
        if (ck_w->device != device || ck_t->device != device) { set_error("commitment key lives on another device"); return LURK_ERR_ARG; }
        // fixed-base tables: the device-side finish of a commitment needs one bucket set (msm_horner_kernel)
        LURK_TRY(lurk_msm_ctx_precompute(ck_w));
        if (ck_t != ck_w) LURK_TRY(lurk_msm_ctx_precompute(ck_t));
        {
            // commit(W2 - D): after the dummy-witness offset only ~a third of the scalars are non-zero, so the 2^(c-1)-bucket
            // reduction weighs more against the per-window additions than for a dense vector: own narrower table when it pays
            const int want = std::min(ck_w->fixed_c, FOLD_W_WINDOW);
            LURK_TRY(lurk_msm_ctx_clone(ck_w, &ckWbase));
            if (want != ck_w->fixed_c && c.n_w) {
                ckWbase->n = c.n_w;
                ckWbase->d_table = nullptr;
                ckWbase->owns_table = false;
                ckWbase->fixed_c = 0;
                LURK_TRY(msm_precompute<C>(ckWbase, want));
            }
            for (int b = 0; b < D; b++) LURK_TRY(lurk_msm_ctx_clone(ckWbase, &ckW[b]));
        }
        LURK_TRY(lurk_msm_ctx_clone(ck_t, &ckT));
        {
            // commit(T) sits on the sequential chain: a narrower window than the throughput optimum shortens the bucket
            // reduction (2^(c-1) buckets on the critical path) at the price of a few more additions per scalar; the context
            // gets its own table over exactly n_rows bases
            const int want = std::min(ck_t->fixed_c, FOLD_T_WINDOW);   // never wider than the key's own choice
            if (want != ck_t->fixed_c && c.n_rows) {
                ckT->n = c.n_rows;
                ckT->d_table = nullptr;
                ckT->owns_table = false;
                ckT->fixed_c = 0;
                LURK_TRY(msm_precompute<C>(ckT, want));
            }
        }
        LURK_TRY(lurk_msm_ctx_clone(ck_t, &ckChk));
        LURK_TRY(lurk_msm_ctx_clone(ck_w, &ckChkW));     // check_running must not touch a prefetched commit(W2)
        for (int b = 0; b < D; b++) lurk_msm_ctx_set_profiling(ckW[b], 1);
        lurk_msm_ctx_set_profiling(ckT, 1);

        // streams: the chain gets the high priority; optional SM partition
        int lo = 0, hi = 0;
        LURK_CUDA_TRY(cudaDeviceGetStreamPriorityRange(&lo, &hi));
        if (c.latency_sms > 0) {
            cudaStream_t tiny[2] = {nullptr, nullptr}, big_lo[4] = {nullptr, nullptr, nullptr, nullptr};
            if (green_streams(c.latency_sms, tiny, 2, &sB, big_lo, 4) != LURK_OK) {
                set_error("SM partitioning (green contexts) is not available on this driver");
                return LURK_ERR_CUDA;
            }
            sT = tiny[0]; sC = tiny[1];
            sK[0] = big_lo[0]; sK[1] = big_lo[1]; sK[2] = big_lo[2]; sA = big_lo[3];
            partitioned = true;
        } else {
            LURK_CUDA_TRY(cudaStreamCreateWithPriority(&sB, cudaStreamNonBlocking, hi));
            for (int k = 0; k < 3; k++) LURK_CUDA_TRY(cudaStreamCreateWithPriority(&sK[k], cudaStreamNonBlocking, lo));
            LURK_CUDA_TRY(cudaStreamCreateWithPriority(&sA, cudaStreamNonBlocking, lo));
            LURK_CUDA_TRY(cudaStreamCreateWithPriority(&sC, cudaStreamNonBlocking, lo));
            sT = sB;                       // no partition: the single-CTA kernels stay on the chain's stream
        }
        LURK_CUDA_TRY(cudaStreamCreateWithPriority(&sH, cudaStreamNonBlocking, lo));
        if (partitioned) {
            for (lurk_msm_ctx *m : {ckW[0], ckW[1], ckW[2], ckW[3], ckT, ckChk, ckChkW}) {
                if (!m) continue;
                m->tiny_stream = sT;
                LURK_CUDA_TRY(cudaEventCreateWithFlags(&m->ev_fork, cudaEventDisableTiming));
                LURK_CUDA_TRY(cudaEventCreateWithFlags(&m->ev_join, cudaEventDisableTiming));
            }
        }
        auto mkev = [](cudaEvent_t *e) { return cudaEventCreateWithFlags(e, cudaEventDisableTiming); };
        for (int b = 0; b < D; b++) {
            LURK_CUDA_TRY(mkev(&ev_h2d[b])); LURK_CUDA_TRY(mkev(&ev_cw[b])); LURK_CUDA_TRY(mkev(&ev_A[b])); LURK_CUDA_TRY(mkev(&ev_fold[b]));
            for (int k = 0; k < 3; k++) LURK_CUDA_TRY(mkev(&ev_slot[b][k]));
        }
        for (int b = 0; b <= D; b++) { LURK_CUDA_TRY(mkev(&ev_chal[b])); LURK_CUDA_TRY(mkev(&ev_done[b])); }

        // vectors
        LURK_TRY(z1.alloc(nz * sizeof(Fs)));
        LURK_TRY(e1.alloc((size_t)c.n_rows * sizeof(Fs)));
        LURK_TRY(T.alloc((size_t)c.n_rows * sizeof(Fs)));
        for (int m = 0; m < 3; m++) LURK_TRY(mv1[m].alloc((size_t)c.n_rows * sizeof(Fs)));
        const Fs one = Fs::one();
        for (int b = 0; b < D; b++) {
            LURK_TRY(z2[b].alloc(nz * sizeof(Fs)));
            LURK_CUDA_TRY(cudaMemset(z2[b].p, 0, nz * sizeof(Fs)));
            LURK_CUDA_TRY(cudaMemcpy(z2[b].as<Fs>() + c.n_w, &one, sizeof(Fs), cudaMemcpyHostToDevice));   // u2 = 1
            for (int m = 0; m < 3; m++) LURK_TRY(mv2[b][m].alloc((size_t)c.n_rows * sizeof(Fs)));
            LURK_TRY(step_consts[b].alloc(FOLD_RO_RATE * sizeof(Fb)));
            LURK_CUDA_TRY(cudaMemset(step_consts[b].p, 0, FOLD_RO_RATE * sizeof(Fb)));
            LURK_CUDA_TRY(cudaMallocHost(&h_ro[b], FOLD_RO_RATE * 32));
            memset(h_ro[b], 0, FOLD_RO_RATE * 32);
            if (c.n_x) { LURK_CUDA_TRY(cudaMallocHost(&h_x2[b], (size_t)c.n_x * 32)); memset(h_x2[b], 0, (size_t)c.n_x * 32); }
        }
        LURK_CUDA_TRY(cudaMemset(z1.p, 0, nz * sizeof(Fs)));
        LURK_CUDA_TRY(cudaMemset(e1.p, 0, (size_t)c.n_rows * sizeof(Fs)));
        for (int b = 0; b <= D; b++) {
            LURK_TRY(rec_dev[b].alloc(sizeof(Rec)));
            LURK_CUDA_TRY(cudaMemset(rec_dev[b].p, 0, sizeof(Rec)));
            LURK_CUDA_TRY(cudaMallocHost((void **)&h_rec[b], sizeof(Rec)));
            memset(h_rec[b], 0, sizeof(Rec));
        }
        LURK_TRY(r_dev.alloc(sizeof(Fs)));
        LURK_TRY(seq_dev.alloc(sizeof(unsigned long long)));
        LURK_CUDA_TRY(cudaMemset(seq_dev.p, 0, sizeof(unsigned long long)));
        LURK_TRY(run_pts.alloc(2 * sizeof(Pt)));
        LURK_CUDA_TRY(cudaMemset(run_pts.p, 0, 2 * sizeof(Pt)));
        LURK_TRY(bad_dev.alloc(sizeof(SatCount)));
        LURK_TRY(xchg.alloc(sizeof(XchgBuf<Fb>)));
        LURK_CUDA_TRY(cudaMemset(xchg.p, 0, sizeof(XchgBuf<Fb>)));
        peers[c.rank] = xchg.as<XchgBuf<Fb>>();

        // R1CS matrices
        for (int m = 0; m < 3; m++) {
            const size_t nnz = c.n_rows ? (size_t)row_ptr[m][c.n_rows] : 0;
            for (size_t k = 0; k < nnz; k++)
                if (col[m][k] >= nz) { set_error("matrix %d: column %u out of range", m, col[m][k]); return LURK_ERR_ARG; }
            LURK_TRY(csr_rp[m].alloc(((size_t)c.n_rows + 1) * sizeof(uint64_t)));
            LURK_TRY(csr_col[m].alloc(std::max<size_t>(1, nnz) * sizeof(uint32_t)));
            LURK_TRY(csr_val[m].alloc(std::max<size_t>(1, nnz) * sizeof(Fs)));
            LURK_CUDA_TRY(cudaMemcpy(csr_rp[m].p, row_ptr[m], ((size_t)c.n_rows + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice));
            if (nnz) {
                LURK_CUDA_TRY(cudaMemcpy(csr_col[m].p, col[m], nnz * sizeof(uint32_t), cudaMemcpyHostToDevice));
                LURK_CUDA_TRY(cudaMemcpy(csr_val[m].p, val[m], nnz * sizeof(Fs), cudaMemcpyHostToDevice));
                int bad = 0;
                LURK_TRY(check_reduced_dev<Fs>(csr_val[m].p, nnz, sB, &bad));
                if (bad) { set_error("matrix %d: %d coefficient(s) not reduced", m, bad); return LURK_ERR_RANGE; }
                if (fmt == LURK_FMT_CANONICAL) LURK_TRY(convert_dev<Fs>(csr_val[m].p, nnz, LURK_FMT_MONTGOMERY, csr_val[m].p, sB));
            }
            csr[m].row_ptr = csr_rp[m].as<uint64_t>();
            csr[m].col = csr_col[m].as<uint32_t>();
            csr[m].val = csr_val[m].p;
        }
        LURK_CUDA_TRY(cudaStreamSynchronize(sB));

        // random oracle constants: width 25 (arity 24), Neptune Strength::Standard; the capacity element carries the IO tag
        const PoseidonParams<Fb> *pp = nullptr;
        LURK_TRY(poseidon_instance_info<Fb>(FOLD_RO_RATE, &pp, &roL));
        std::vector<Fb> flat = pp->flat();
        LURK_TRY(ro_img.alloc(flat.size() * sizeof(Fb)));
        LURK_CUDA_TRY(cudaMemcpy(ro_img.p, flat.data(), flat.size() * sizeof(Fb), cudaMemcpyHostToDevice));
        // default pattern = Arecibo NIFS::prove: pp_digest, U2 = (comm_W, X[0], X[1]), comm_T
        const int def[9] = {FOLD_RO_CONST, FOLD_RO_W_X, FOLD_RO_W_Y, FOLD_RO_W_INF, FOLD_RO_CONST, FOLD_RO_CONST, FOLD_RO_T_X, FOLD_RO_T_Y, FOLD_RO_T_INF};
        return set_ro(9, def, 128);
    }

    int set_ro(int n, const int *k, int bits) override {
        if (n < 1 || n > FOLD_RO_RATE || bits < 1 || bits > 250) { set_error("RO pattern: 1..24 absorbed elements, 1..250 challenge bits"); return LURK_ERR_ARG; }
        for (int i = 0; i < n; i++)
            if (k[i] < FOLD_RO_CONST || k[i] > FOLD_RO_T_INF) { set_error("RO pattern: unknown slot kind %d", k[i]); return LURK_ERR_ARG; }
        n_absorb = n;
        challenge_bits = bits;
        memset(kinds, 0, sizeof kinds);
        for (int i = 0; i < n; i++) kinds[i] = (unsigned char)k[i];
        const unsigned __int128 tag = safe_io_tag((uint32_t)n, 1);
        Fb raw = Fb::zero();
        for (int i = 0; i < 4; i++) raw.v[i] = (uint32_t)(tag >> (32 * i));
        io_tag = Fb::from_canonical(raw);
        return LURK_OK;
    }

    int add_slot_batch(int arity, size_t count, const uint64_t *offsets) override {
        if (arity != 0 && arity != 3 && arity != 4 && arity != 6 && arity != 8) { set_error("slot arity %d", arity); return LURK_ERR_ARG; }
        size_t blk = 0;
        if (arity) {
            PoseidonLayout L;
            LURK_TRY(poseidon_instance_info<Fs>(arity, nullptr, &L));
            blk = (size_t)L.block_elems;
        } else {
            uint32_t mod[8];
            for (int i = 0; i < 8; i++) mod[i] = Fs::Params::MOD(i);
            blk = (size_t)bitdecomp_block_host(mod);
        }
        for (size_t k = 0; k < count; k++)
            if (offsets[k] + blk > cfg.n_w) { set_error("slot block %zu does not fit into W", k); return LURK_ERR_ARG; }
        auto sb = std::make_unique<FoldSlotBatch>();
        sb->arity = arity;
        return add_batch(std::move(sb), count, offsets);
    }
    int add_sha256_batch(int n, size_t count, const uint64_t *offsets) override {
        const size_t blk = sha256_block_len<Fs>(n);
        if (!blk) { set_error("SHA-256 coprocessor arity %d: 1..%d", n, LURK_SHA256_MAX_N); return LURK_ERR_ARG; }
        for (size_t k = 0; k < count; k++)
            if (offsets[k] + blk > cfg.n_w) { set_error("SHA-256 block %zu does not fit into W", k); return LURK_ERR_ARG; }
        auto sb = std::make_unique<FoldSlotBatch>();
        sb->sha_n = n;
        return add_batch(std::move(sb), count, offsets);
    }
    int add_trie_batch(int op, int height, size_t count, const uint64_t *offsets) override {
        const size_t blk = trie_block_len<Fs>(op, height);
        if (!blk) { set_error("trie op %d / height %d: op 0 (lookup) or 1 (insert), height 1..%d", op, height, LURK_TRIE_MAX_HEIGHT); return LURK_ERR_ARG; }
        for (size_t k = 0; k < count; k++)
            if (offsets[k] + blk > cfg.n_w) { set_error("trie block %zu does not fit into W", k); return LURK_ERR_ARG; }
        auto sb = std::make_unique<FoldSlotBatch>();
        sb->trie_op = op;
        sb->trie_h = height;
        return add_batch(std::move(sb), count, offsets);
    }
    int add_batch(std::unique_ptr<FoldSlotBatch> sb, size_t count, const uint64_t *offsets) {
        sb->count = count;
        LURK_TRY(sb->d_offsets.alloc(std::max<size_t>(1, count) * sizeof(uint64_t)));
        if (count) LURK_CUDA_TRY(cudaMemcpy(sb->d_offsets.p, offsets, count * sizeof(uint64_t), cudaMemcpyHostToDevice));
        for (int b = 0; b < D; b++) {
            LURK_TRY(sb->d_pre[b].alloc(std::max<size_t>(32, sb->bytes())));
            LURK_CUDA_TRY(cudaMemset(sb->d_pre[b].p, 0, std::max<size_t>(32, sb->bytes())));
            LURK_CUDA_TRY(cudaMallocHost(&sb->h_pre[b], std::max<size_t>(32, sb->bytes())));
            memset(sb->h_pre[b], 0, std::max<size_t>(32, sb->bytes()));
        }
        batches.push_back(std::move(sb));
        return (int)batches.size() - 1;
    }

    int set_spans(int n, const FoldSpan *sp) override {
        if (n < 0 || n > FOLD_MAX_SPANS) { set_error("at most %d spans", FOLD_MAX_SPANS); return LURK_ERR_ARG; }
        size_t total = 0;
        for (int i = 0; i < n; i++) {
            const FoldSpan &s = sp[i];
            if (s.rows == 0 || s.row_elems == 0) { set_error("empty span"); return LURK_ERR_ARG; }
            if (s.rows > 1 && s.stride < s.row_elems) { set_error("span rows overlap"); return LURK_ERR_ARG; }
            if (s.first + (s.rows - 1) * s.stride + s.row_elems > cfg.n_w) { set_error("span %d leaves W", i); return LURK_ERR_ARG; }
            total += (size_t)s.rows * s.row_elems;
        }
        spans.assign(sp, sp + n);
        for (int b = 0; b < D; b++) {
            if (h_glue[b]) { cudaFreeHost(h_glue[b]); h_glue[b] = nullptr; }
            if (total) { LURK_CUDA_TRY(cudaMallocHost(&h_glue[b], total * 32)); memset(h_glue[b], 0, total * 32); }
        }
        glue_elems = total;
        return LURK_OK;
    }

    int chk_b(int b) const {
        if (b < 0 || b >= D) { set_error("fresh-instance buffer %d out of range (depth %d)", b, D); return LURK_ERR_ARG; }
        return LURK_OK;
    }

    int host_buffer(int b, int which, void **ptr, size_t *bytes) override {
        LURK_TRY(chk_b(b));
        void *p = nullptr;
        size_t n = 0;
        if (which >= 0) {
            if (which >= (int)batches.size()) { set_error("no slot batch %d", which); return LURK_ERR_ARG; }
            p = batches[which]->h_pre[b]; n = batches[which]->bytes();
        } else if (which == FOLD_BUF_GLUE) { p = h_glue[b]; n = glue_elems * 32; }
        else if (which == FOLD_BUF_X2) { p = h_x2[b]; n = (size_t)cfg.n_x * 32; }
        else if (which == FOLD_BUF_RO) { p = h_ro[b]; n = FOLD_RO_RATE * 32; }
        else { set_error("no host buffer %d", which); return LURK_ERR_ARG; }
        if (ptr) *ptr = p;
        if (bytes) *bytes = n;
        return LURK_OK;
    }
    int device_buffer(int b, int which, void **ptr, size_t *bytes) override {
        void *p = nullptr;
        size_t n = 0;
        if (which >= 0) {
            LURK_TRY(chk_b(b));
            if (which >= (int)batches.size()) { set_error("no slot batch %d", which); return LURK_ERR_ARG; }
            p = batches[which]->d_pre[b].p; n = batches[which]->bytes();
        } else if (which == FOLD_BUF_W2) { LURK_TRY(chk_b(b)); p = z2[b].p; n = nz * 32; }
        else if (which == FOLD_BUF_RO) { LURK_TRY(chk_b(b)); p = step_consts[b].p; n = FOLD_RO_RATE * 32; }
        else if (which == FOLD_BUF_T) { p = T.p; n = (size_t)cfg.n_rows * 32; }
        else if (which == FOLD_BUF_Z1) { p = z1.p; n = nz * 32; }
        else if (which == FOLD_BUF_E1) { p = e1.p; n = (size_t)cfg.n_rows * 32; }
        else { set_error("no device buffer %d", which); return LURK_ERR_ARG; }
        if (ptr) *ptr = p;
        if (bytes) *bytes = n;
        return LURK_OK;
    }

    // ------------------------------------------------------------------------------------------ exchange
    int exchange_handle(uint8_t out[64]) override {
        static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
        cudaIpcMemHandle_t h;
        LURK_CUDA_TRY(cudaIpcGetMemHandle(&h, xchg.p));
        memcpy(out, &h, 64);
        return LURK_OK;
    }
    int set_peers(const uint8_t *handles) override {
        if (cfg.world <= 1) return LURK_OK;
        for (int p = 0; p < cfg.world; p++) {
            if (p == cfg.rank) continue;
            cudaIpcMemHandle_t h;
            memcpy(&h, handles + 64 * p, 64);
            void *ptr = nullptr;
            LURK_CUDA_TRY(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
            peers[p] = (XchgBuf<Fb> *)ptr;
            peers_open[p] = true;
        }
        peers_set = true;
        return LURK_OK;
    }

    // ------------------------------------------------------------------------------------------ running instance
    static void point_bytes(const Fb &x, const Fb &y, uint32_t inf, int fmt, uint8_t out[96]) {
        memset(out, 0, 96);
        if (inf) return;
        Fb a = x, b = y, one = Fb::one();
        if (fmt == LURK_FMT_CANONICAL) { a = a.to_canonical(); b = b.to_canonical(); one = one.to_canonical(); }
        memcpy(out, a.v, 32); memcpy(out + 32, b.v, 32); memcpy(out + 64, one.v, 32);
    }
    static int point_from_bytes(const uint8_t in[96], int fmt, Pt *out) {
        Fb x, y, z;
        memcpy(x.v, in, 32); memcpy(y.v, in + 32, 32); memcpy(z.v, in + 64, 32);
        if (!x.is_reduced() || !y.is_reduced()) { set_error("point coordinate not reduced"); return LURK_ERR_RANGE; }
        if (z.is_zero()) { *out = Pt::identity(); return LURK_OK; }
        Affine<Fb> a;
        a.x = fmt == LURK_FMT_CANONICAL ? Fb::from_canonical(x) : x;
        a.y = fmt == LURK_FMT_CANONICAL ? Fb::from_canonical(y) : y;
        *out = Pt::from_affine(a);
        return LURK_OK;
    }

    int upload_vec(void *dst, const uint8_t *src, size_t n, int fmt) {
        if (!n) return LURK_OK;
        LURK_CUDA_TRY(cudaMemcpyAsync(dst, src, n * 32, cudaMemcpyHostToDevice, sB));
        int bad = 0;
        LURK_TRY(check_reduced_dev<Fs>(dst, n, sB, &bad));
        if (bad) { set_error("%d element(s) not reduced below the field modulus", bad); return LURK_ERR_RANGE; }
        if (fmt == LURK_FMT_CANONICAL) LURK_TRY(convert_dev<Fs>(dst, n, LURK_FMT_MONTGOMERY, dst, sB));
        return LURK_OK;
    }
    int set_running(const uint8_t *w, const uint8_t *e, const uint8_t *u, const uint8_t *x, const uint8_t *comm_w, const uint8_t *comm_e,
                    int fmt) override {
        LURK_TRY(sync());
        LURK_TRY(upload_vec(z1.p, w, cfg.n_w, fmt));
        LURK_TRY(upload_vec(z1.as<Fs>() + cfg.n_w, u, 1, fmt));
        LURK_TRY(upload_vec(z1.as<Fs>() + cfg.n_w + 1, x, cfg.n_x, fmt));
        LURK_TRY(upload_vec(e1.p, e, cfg.n_rows, fmt));
        Pt pts[2];
        LURK_TRY(point_from_bytes(comm_w, fmt, &pts[0]));
        LURK_TRY(point_from_bytes(comm_e, fmt, &pts[1]));
        LURK_CUDA_TRY(cudaMemcpyAsync(run_pts.p, pts, sizeof pts, cudaMemcpyHostToDevice, sB));
        LURK_CUDA_TRY(cudaStreamSynchronize(sB));
        running_set = true;
        mv1_valid = false;
        return LURK_OK;
    }
    int download_vec(uint8_t *dst, const void *src, size_t n, int fmt) {
        if (!n || !dst) return LURK_OK;
        if (fmt == LURK_FMT_MONTGOMERY) {
            LURK_CUDA_TRY(cudaMemcpyAsync(dst, src, n * 32, cudaMemcpyDeviceToHost, sB));
        } else {
            void *tmp = nullptr;
            LURK_CUDA_TRY(cudaMallocAsync(&tmp, n * 32, sB));
            int rc = convert_dev<Fs>(src, n, LURK_FMT_CANONICAL, tmp, sB);
            cudaError_t e = cudaMemcpyAsync(dst, tmp, n * 32, cudaMemcpyDeviceToHost, sB);
            cudaFreeAsync(tmp, sB);
            LURK_TRY(rc);
            LURK_CUDA_TRY(e);
        }
        return LURK_OK;
    }
    // checkpoint / resume (SURVEY.md section 5): the running instance is materialised on the host on demand
    int get_running(uint8_t *w, uint8_t *e, uint8_t *u, uint8_t *x, uint8_t *comm_w, uint8_t *comm_e, int fmt) override {
        LURK_TRY(sync());
        LURK_TRY(download_vec(w, z1.p, cfg.n_w, fmt));
        LURK_TRY(download_vec(u, z1.as<Fs>() + cfg.n_w, 1, fmt));
        LURK_TRY(download_vec(x, z1.as<Fs>() + cfg.n_w + 1, cfg.n_x, fmt));
        LURK_TRY(download_vec(e, e1.p, cfg.n_rows, fmt));
        Pt pts[2];
        LURK_CUDA_TRY(cudaMemcpyAsync(pts, run_pts.p, sizeof pts, cudaMemcpyDeviceToHost, sB));
        LURK_CUDA_TRY(cudaStreamSynchronize(sB));
        if (comm_w) point_to_bytes(pts[0], fmt, comm_w);
        if (comm_e) point_to_bytes(pts[1], fmt, comm_e);
        return LURK_OK;
    }

    // The constant part of every fresh witness: D = the slot blocks of a step whose slots are all dummies (all-zero preimages),
    // zero elsewhere.  Unused slots of a frame share one cached witness per slot type in the reference
    // (src/lem/multiframe.rs:553-577), so W2 - D vanishes on every dummy slot: commit(W2) = commit(W2 - D) + commit(D) with
    // commit(D) computed once here.  Built at the first stage A, when the slot batches are known.
    int prepare_dummy() {
        if (dummy_ready) return LURK_OK;
        dummy_ready = true;
        size_t nslots = 0;
        for (auto &sb : batches) nslots += sb->coprocessor() ? 0 : sb->count;   // coprocessor blocks are not part of D
        if (!nslots || !cfg.n_w) return LURK_OK;
        LURK_TRY(dummy_w.alloc((size_t)cfg.n_w * sizeof(Fs)));
        LURK_CUDA_TRY(cudaMemsetAsync(dummy_w.p, 0, (size_t)cfg.n_w * sizeof(Fs), sB));
        for (auto &sb : batches) {
            if (!sb->count || sb->coprocessor()) continue;
            void *zeros = nullptr;
            LURK_CUDA_TRY(cudaMallocAsync(&zeros, sb->bytes(), sB));
            LURK_CUDA_TRY(cudaMemsetAsync(zeros, 0, sb->bytes(), sB));
            int rc;
            if (sb->arity) {
                rc = launch_poseidon<Fs, true>(sb->arity, zeros, sb->count, dummy_w.p, LURK_FMT_MONTGOMERY, LURK_FMT_MONTGOMERY, sB, sb->d_offsets.as<uint64_t>());
            } else {
                uint32_t mod[8];
                for (int i = 0; i < 8; i++) mod[i] = Fs::Params::MOD(i);
                rc = launch_bitdecomp<Fs>(zeros, sb->count, dummy_w.p, bitdecomp_block_host(mod), LURK_FMT_MONTGOMERY, sB, sb->d_offsets.as<uint64_t>());
            }
            cudaFreeAsync(zeros, sB);
            LURK_TRY(rc);
        }
        uint8_t pt[96];
        LURK_TRY(msm_launch<C>(ckChkW, dummy_w.p, cfg.n_w, LURK_FMT_MONTGOMERY, sB, true));
        LURK_TRY(msm_finish<C>(ckChkW, pt));
        Fb z;
        memcpy(z.v, pt + 64, 32);
        if (z.is_zero()) return LURK_OK;               // commit(D) is the identity: nothing to gain
        LURK_TRY(dummy_p.alloc(64));
        LURK_CUDA_TRY(cudaMemcpy(dummy_p.p, pt, 64, cudaMemcpyHostToDevice));
        for (int k = 0; k < D; k++) { ckW[k]->d_sub = dummy_w.p; ckW[k]->d_offset = dummy_p.p; }
        return LURK_OK;
    }

    // ------------------------------------------------------------------------------------------ stage A
    int stage_a(int b, int flags, int fmt) override {
        LURK_TRY(chk_b(b));
        LURK_TRY(prepare_dummy());
        if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
        if (b_pending[b]) { set_error("buffer %d: the previous step's result has not been collected", b); return LURK_ERR_ARG; }
        const bool staged = !(flags & FOLD_INPUTS_RESIDENT);
        if (!staged && fmt != LURK_FMT_MONTGOMERY) { set_error("device-resident inputs are Montgomery form"); return LURK_ERR_ARG; }
        Fs *W2 = z2[b].as<Fs>();
        unsigned k = 0;
        if (fold_recorded[b]) LURK_CUDA_TRY(cudaStreamWaitEvent(sH, ev_fold[b], 0));   // W2[b] / mv2[b] may still be read by a fold
        if (staged) {
            for (auto &sb : batches)
                if (sb->count) LURK_CUDA_TRY(cudaMemcpyAsync(sb->d_pre[b].p, sb->h_pre[b], sb->bytes(), cudaMemcpyHostToDevice, sH));
            size_t off = 0;
            for (const FoldSpan &s : spans) {
                LURK_CUDA_TRY(cudaMemcpy2DAsync(W2 + s.first, s.stride * 32, (const uint8_t *)h_glue[b] + off * 32, s.row_elems * 32, s.row_elems * 32,
                                                s.rows, cudaMemcpyHostToDevice, sH));
                if (fmt == LURK_FMT_CANONICAL) {
                    span_to_mont_kernel<Fs><<<fold_grid(s.rows * s.row_elems, 256, 4), 256, 0, sH>>>(W2, s.first, s.row_elems, s.stride, s.rows);
                    k++;
                }
                off += s.rows * s.row_elems;
            }
            if (cfg.n_x) {
                LURK_CUDA_TRY(cudaMemcpyAsync(W2 + cfg.n_w + 1, h_x2[b], (size_t)cfg.n_x * 32, cudaMemcpyHostToDevice, sH));
                if (fmt == LURK_FMT_CANONICAL) { LURK_TRY(convert_dev<Fs>(W2 + cfg.n_w + 1, cfg.n_x, LURK_FMT_MONTGOMERY, W2 + cfg.n_w + 1, sH)); k++; }
            }
            LURK_CUDA_TRY(cudaMemcpyAsync(step_consts[b].p, h_ro[b], FOLD_RO_RATE * 32, cudaMemcpyHostToDevice, sH));
            if (fmt == LURK_FMT_CANONICAL) { LURK_TRY(convert_dev<Fb>(step_consts[b].p, FOLD_RO_RATE, LURK_FMT_MONTGOMERY, step_consts[b].p, sH)); k++; }
        }
        LURK_CUDA_TRY(cudaEventRecord(ev_h2d[b], sH));
        for (int s = 0; s < 3; s++) LURK_CUDA_TRY(cudaStreamWaitEvent(sK[s], ev_h2d[b], 0));
        LURK_CUDA_TRY(cudaStreamWaitEvent(sA, ev_h2d[b], 0));
        // slot witnesses, written in place into W2 (src/lem/multiframe.rs:520-592; one stream per slot type, round robin)
        int idx = 0;
        for (auto &sb : batches) {
            cudaStream_t st = sK[idx % 3];
            idx++;
            if (!sb->count) continue;
            if (sb->sha_n) {
                LURK_TRY(launch_sha256_witness<Fs>(sb->d_pre[b].p, sb->count, sb->sha_n, W2, sb->d_offsets.as<uint64_t>(), fmt, LURK_FMT_MONTGOMERY, st));
            } else if (sb->trie_h) {
                LURK_TRY(launch_trie_witness<Fs>(sb->trie_op, sb->trie_h, sb->d_pre[b].p, sb->count, W2, sb->d_offsets.as<uint64_t>(), fmt,
                                                 LURK_FMT_MONTGOMERY, st));
                k++;   // two launches: the Poseidon levels, then root, bits and picks
            } else if (sb->arity) {
                LURK_TRY((launch_poseidon<Fs, true>(sb->arity, sb->d_pre[b].p, sb->count, W2, fmt, LURK_FMT_MONTGOMERY, st, sb->d_offsets.as<uint64_t>())));
            } else {
                uint32_t mod[8];
                for (int i = 0; i < 8; i++) mod[i] = Fs::Params::MOD(i);
                LURK_TRY(bitdecomp_fold(sb->d_pre[b].p, sb->count, W2, bitdecomp_block_host(mod), fmt, st, sb->d_offsets.as<uint64_t>()));
            }
            k++;
        }
        for (int s = 0; s < 3; s++) LURK_CUDA_TRY(cudaEventRecord(ev_slot[b][s], sK[s]));
        for (int s = 1; s < 3; s++) LURK_CUDA_TRY(cudaStreamWaitEvent(sK[0], ev_slot[b][s], 0));
        // comm_W2 (this rank's share): result stays on the device for the challenge kernel
        LURK_TRY(msm_launch<C>(ckW[b], W2, cfg.n_w, LURK_FMT_MONTGOMERY, sK[0], false));
        k += ckW[b]->last_launches;
        LURK_CUDA_TRY(cudaEventRecord(ev_cw[b], partitioned ? sT : sK[0]));   // where msm_horner_kernel ran
        // A z2, B z2, C z2
        for (int s = 0; s < 3; s++) LURK_CUDA_TRY(cudaStreamWaitEvent(sA, ev_slot[b][s], 0));
        if (cfg.n_rows) {
            spmv3_kernel<Fs><<<dim3(fold_grid(cfg.n_rows, 256, 8), 3), 256, 0, sA>>>(csr[0], csr[1], csr[2], cfg.n_rows, z2[b].as<Fs>(), mv2[b][0].as<Fs>(),
                                                                                    mv2[b][1].as<Fs>(), mv2[b][2].as<Fs>());
            k++;
        }
        LURK_CUDA_TRY(cudaGetLastError());
        LURK_CUDA_TRY(cudaEventRecord(ev_A[b], sA));
        a_recorded[b] = true;
        launches_a = k;
        return LURK_OK;
    }

    // bit-decomposition slots: input format differs from the (always Montgomery) output only for canonical hosts
    int bitdecomp_fold(const void *d_vals, size_t n, void *d_base, int blk, int fmt, cudaStream_t st, const uint64_t *d_offs) {
        if (fmt == LURK_FMT_MONTGOMERY) return launch_bitdecomp<Fs>(d_vals, n, d_base, blk, LURK_FMT_MONTGOMERY, st, d_offs);
        // canonical values: convert in place first (the kernel takes one format for input and output)
        LURK_TRY(convert_dev<Fs>(d_vals, n, LURK_FMT_MONTGOMERY, const_cast<void *>(d_vals), st));
        return launch_bitdecomp<Fs>(d_vals, n, d_base, blk, LURK_FMT_MONTGOMERY, st, d_offs);
    }

    ChallengeArgs<Fb, Fs> challenge_args(const Pt *pw, const Pt *pt, int b, int rec_index, int mode) {
        ChallengeArgs<Fb, Fs> a;
        a.part_w = pw; a.part_t = pt;
        a.world = cfg.world; a.rank = cfg.rank;
        a.seq = seq_dev.as<unsigned long long>();
        for (int p = 0; p < FOLD_MAX_WORLD; p++) a.peers[p] = peers[p];
        a.ro_consts = ro_img.as<Fb>();
        a.L = roL;
        a.io_tag = io_tag;
        a.n_absorb = n_absorb;
        memcpy(a.kind, kinds, sizeof kinds);
        a.step_consts = step_consts[b].as<Fb>();
        a.challenge_bits = challenge_bits;
        a.mode = mode;
        a.r_out = r_dev.as<Fs>();
        a.rec = rec_dev[rec_index].as<Rec>();
        return a;
    }
    int need_peers() const {
        if (cfg.world > 1 && !peers_set) { set_error("sharded key: call lurk_fold_ctx_set_peers before the first step"); return LURK_ERR_ARG; }
        return LURK_OK;
    }

    // RecursiveSNARK::new (src/proof/nova.rs:286-288): the running instance becomes the first fresh instance (u = 1, E = 0)
    int init_running(int b) override {
        LURK_TRY(chk_b(b));
        LURK_TRY(need_peers());
        if (!a_recorded[b]) { set_error("buffer %d: stage A has not been enqueued", b); return LURK_ERR_ARG; }
        if (b_pending[b]) { set_error("buffer %d: result not collected", b); return LURK_ERR_ARG; }
        LURK_CUDA_TRY(cudaStreamWaitEvent(sB, ev_A[b], 0));
        LURK_CUDA_TRY(cudaMemcpyAsync(z1.p, z2[b].p, nz * sizeof(Fs), cudaMemcpyDeviceToDevice, sB));
        LURK_CUDA_TRY(cudaMemsetAsync(e1.p, 0, (size_t)cfg.n_rows * sizeof(Fs), sB));
        for (int m = 0; m < 3 && cfg.n_rows; m++)
            LURK_CUDA_TRY(cudaMemcpyAsync(mv1[m].p, mv2[b][m].p, (size_t)cfg.n_rows * sizeof(Fs), cudaMemcpyDeviceToDevice, sB));
        mv1_valid = true;
        LURK_CUDA_TRY(cudaStreamWaitEvent(sT, ev_cw[b], 0));
        fold_challenge_kernel<C><<<1, 64, 0, sT>>>(challenge_args(ckW[b]->scratch.result.template as<Pt>(), nullptr, b, b, FOLD_MODE_COMMIT_ONLY));
        LURK_CUDA_TRY(cudaGetLastError());
        LURK_CUDA_TRY(cudaEventRecord(ev_chal[b], sT));
        if (sT != sB) LURK_CUDA_TRY(cudaStreamWaitEvent(sB, ev_chal[b], 0));
        LURK_CUDA_TRY(cudaEventRecord(ev_fold[b], sB));     // after the last reader of W2[b] and of commit(W2[b])'s result
        fold_recorded[b] = true;
        LURK_CUDA_TRY(cudaStreamWaitEvent(sC, ev_chal[b], 0));
        fold_commitments_kernel<C><<<1, 64, 0, sC>>>(run_pts.as<Pt>(), run_pts.as<Pt>() + 1, rec_dev[b].as<Rec>(), 1);
        LURK_CUDA_TRY(cudaGetLastError());
        LURK_CUDA_TRY(cudaMemcpyAsync(h_rec[b], rec_dev[b].p, sizeof(Rec), cudaMemcpyDeviceToHost, sC));
        LURK_CUDA_TRY(cudaEventRecord(ev_done[b], sC));
        b_pending[b] = true;
        running_set = true;
        launches_b = 2;
        return LURK_OK;
    }

    // ------------------------------------------------------------------------------------------ stage B
    int stage_b_launch(int b) override {
        LURK_TRY(chk_b(b));
        LURK_TRY(need_peers());
        if (!running_set) { set_error("no running instance (lurk_fold_ctx_init_running or _set_running first)"); return LURK_ERR_ARG; }
        if (!a_recorded[b]) { set_error("buffer %d: stage A has not been enqueued", b); return LURK_ERR_ARG; }
        if (b_pending[b]) { set_error("buffer %d: the previous step's result has not been collected", b); return LURK_ERR_ARG; }
        unsigned k = 0;
        const size_t rows = cfg.n_rows;
        if (rows && !mv1_valid) {     // only after set_running: the fold keeps A z1, B z1, C z1 current by linearity
            spmv3_kernel<Fs><<<dim3(fold_grid(rows, 256, 8), 3), 256, 0, sB>>>(csr[0], csr[1], csr[2], rows, z1.as<Fs>(), mv1[0].as<Fs>(), mv1[1].as<Fs>(),
                                                                             mv1[2].as<Fs>());
            k++;
        }
        mv1_valid = true;
        LURK_CUDA_TRY(cudaStreamWaitEvent(sB, ev_A[b], 0));
        if (rows) {
            cross_term_dev_kernel<Fs><<<fold_grid(rows, 256, 8), 256, 0, sB>>>(mv1[0].as<Fs>(), mv1[1].as<Fs>(), mv1[2].as<Fs>(), mv2[b][0].as<Fs>(),
                                                                              mv2[b][1].as<Fs>(), mv2[b][2].as<Fs>(), z1.as<Fs>() + cfg.n_w,
                                                                              z2[b].as<Fs>() + cfg.n_w, rows, T.as<Fs>());
            k++;
        }
        LURK_TRY(msm_launch<C>(ckT, T.p, rows, LURK_FMT_MONTGOMERY, sB, false));
        k += rows ? ckT->last_launches : 0;
        // the finished partial commitments are on sT (the tiny partition's stream, or sB itself without a partition)
        if (sT != sB && !rows) {           // an empty T is produced by a memset on sB
            LURK_CUDA_TRY(cudaEventRecord(ev_chal[b], sB));
            LURK_CUDA_TRY(cudaStreamWaitEvent(sT, ev_chal[b], 0));
        }
        LURK_CUDA_TRY(cudaStreamWaitEvent(sT, ev_cw[b], 0));
        fold_challenge_kernel<C><<<1, 64, 0, sT>>>(challenge_args(ckW[b]->scratch.result.template as<Pt>(), ckT->scratch.result.template as<Pt>(), b, b,
                                                                  FOLD_MODE_FOLD));
        k++;
        LURK_CUDA_TRY(cudaEventRecord(ev_chal[b], sT));
        if (sT != sB) LURK_CUDA_TRY(cudaStreamWaitEvent(sB, ev_chal[b], 0));
        {
            FoldAxpyArgs<Fs> ax;
            ax.dst[0] = z1.as<Fs>(); ax.src[0] = z2[b].as<Fs>(); ax.end[0] = nz;
            ax.dst[1] = e1.as<Fs>(); ax.src[1] = T.as<Fs>(); ax.end[1] = nz + rows;
            for (int m = 0; m < 3; m++) { ax.dst[2 + m] = mv1[m].as<Fs>(); ax.src[2 + m] = mv2[b][m].as<Fs>(); ax.end[2 + m] = nz + (size_t)(2 + m) * rows; }
            fold_axpy_kernel<Fs><<<fold_grid(ax.end[4], 256, 8), 256, 0, sB>>>(ax, r_dev.as<Fs>());
            k++;
        }
        LURK_CUDA_TRY(cudaGetLastError());
        LURK_CUDA_TRY(cudaEventRecord(ev_fold[b], sB));
        fold_recorded[b] = true;
        // side stream: running commitments and the result record
        LURK_CUDA_TRY(cudaStreamWaitEvent(sC, ev_chal[b], 0));
        fold_commitments_kernel<C><<<1, 64, 0, sC>>>(run_pts.as<Pt>(), run_pts.as<Pt>() + 1, rec_dev[b].as<Rec>(), 0);
        k++;
        LURK_CUDA_TRY(cudaGetLastError());
        LURK_CUDA_TRY(cudaMemcpyAsync(h_rec[b], rec_dev[b].p, sizeof(Rec), cudaMemcpyDeviceToHost, sC));
        LURK_CUDA_TRY(cudaEventRecord(ev_done[b], sC));
        b_pending[b] = true;
        launches_b = k;
        return LURK_OK;
    }

    int collect(int b, FoldResultHost *out, int fmt) override {
        LURK_TRY(chk_b(b));
        if (!b_pending[b]) { set_error("buffer %d: nothing to collect", b); return LURK_ERR_ARG; }
        LURK_CUDA_TRY(cudaEventSynchronize(ev_done[b]));
        // the record is ready once the challenge is; the running instance only once the fold on sB has written z1, E1 and A z1 .. C z1.
        // Callers read Z1 / E1 right after collect (lurk_spartan_prove_dev, lurk_compress_prove_dev, lurk_recursive_verify_dev), on
        // streams the context does not know.
        LURK_CUDA_TRY(cudaEventSynchronize(ev_fold[b]));
        b_pending[b] = false;
        const Rec &r = *h_rec[b];
        if (out) {
            point_bytes(r.cw_x, r.cw_y, r.cw_inf, fmt, out->comm_w);
            point_bytes(r.ct_x, r.ct_y, r.ct_inf, fmt, out->comm_t);
            point_bytes(r.uw_x, r.uw_y, r.uw_inf, fmt, out->run_comm_w);
            point_bytes(r.ue_x, r.ue_y, r.ue_inf, fmt, out->run_comm_e);
            Fs rr = fmt == LURK_FMT_CANONICAL ? r.r.to_canonical() : r.r;
            memcpy(out->r, rr.v, 32);
            Fb hh = fmt == LURK_FMT_CANONICAL ? r.hash.to_canonical() : r.hash;
            memcpy(out->hash, hh.v, 32);
            out->status = (int)r.status;
            out->seq = r.seq;
        }
        if (r.status) { set_error("partial-commitment exchange timed out (a peer rank did not reach step %llu)", r.seq); return LURK_ERR_CUDA; }
        return LURK_OK;
    }

    // relaxed R1CS check of the running instance, on the device: residual rows and recomputed commitments
    int check_running(unsigned long long *bad_rows, int *comm_w_ok, int *comm_e_ok) override {
        LURK_TRY(need_peers());
        LURK_TRY(sync());
        const size_t rows = cfg.n_rows;
        // one pass with the products in registers; the vectors kept current by the folds (mv1) must equal the fresh products
        const Fs *kept[3] = {mv1[0].as<Fs>(), mv1[1].as<Fs>(), mv1[2].as<Fs>()};
        SatCount cnt{0, 0};
        LURK_TRY(r1cs_sat_launch<Fs>(csr, rows, z1.as<Fs>(), cfg.n_w, e1.as<Fs>(), mv1_valid ? kept : nullptr, bad_dev.as<SatCount>(), sB));
        LURK_CUDA_TRY(cudaMemcpyAsync(&cnt, bad_dev.p, sizeof cnt, cudaMemcpyDeviceToHost, sB));     // read after the synchronisation of sB below
        // commit(W1) with the W key, commit(E1) with the T key, exchanged and normalised like a step's commitments
        LURK_TRY(msm_launch<C>(ckChkW, z1.p, cfg.n_w, LURK_FMT_MONTGOMERY, sB, false));
        LURK_TRY(msm_launch<C>(ckChk, e1.p, rows, LURK_FMT_MONTGOMERY, sB, false));
        if (sT != sB) {                    // covers the empty-vector memsets, which stay on sB
            LURK_CUDA_TRY(cudaEventRecord(ev_chal[D], sB));
            LURK_CUDA_TRY(cudaStreamWaitEvent(sT, ev_chal[D], 0));
        }
        fold_challenge_kernel<C><<<1, 64, 0, sT>>>(challenge_args(ckChkW->scratch.result.template as<Pt>(), ckChk->scratch.result.template as<Pt>(), 0, D,
                                                                  FOLD_MODE_COMMIT_ONLY));
        LURK_CUDA_TRY(cudaGetLastError());
        LURK_CUDA_TRY(cudaMemcpyAsync(h_rec[D], rec_dev[D].p, sizeof(Rec), cudaMemcpyDeviceToHost, sT));
        Pt pts[2];
        LURK_CUDA_TRY(cudaMemcpyAsync(pts, run_pts.p, sizeof pts, cudaMemcpyDeviceToHost, sT));
        LURK_CUDA_TRY(cudaStreamSynchronize(sT));
        LURK_CUDA_TRY(cudaStreamSynchronize(sB));
        const Rec &r = *h_rec[D];
        if (r.status) { set_error("partial-commitment exchange timed out"); return LURK_ERR_CUDA; }
        uint8_t have[96], want[96];
        point_bytes(r.cw_x, r.cw_y, r.cw_inf, LURK_FMT_MONTGOMERY, have);
        point_to_bytes(pts[0], LURK_FMT_MONTGOMERY, want);
        if (comm_w_ok) *comm_w_ok = memcmp(have, want, 96) == 0;
        point_bytes(r.ct_x, r.ct_y, r.ct_inf, LURK_FMT_MONTGOMERY, have);
        point_to_bytes(pts[1], LURK_FMT_MONTGOMERY, want);
        if (comm_e_ok) *comm_e_ok = memcmp(have, want, 96) == 0;
        if (bad_rows) *bad_rows = cnt.bad;
        return LURK_OK;
    }

    int stats(unsigned *la, unsigned *lb, float *acc_w_ms, float *acc_t_ms) override {
        LURK_TRY(sync());
        if (la) *la = launches_a;
        if (lb) *lb = launches_b;
        float ms = 0.f;
        if (acc_w_ms) { *acc_w_ms = 0.f; if (ckW[0]->ev0 && cudaEventElapsedTime(&ms, ckW[0]->ev0, ckW[0]->ev1) == cudaSuccess) *acc_w_ms = ms; }
        if (acc_t_ms) { *acc_t_ms = 0.f; if (ckT->ev0 && cudaEventElapsedTime(&ms, ckT->ev0, ckT->ev1) == cudaSuccess) *acc_t_ms = ms; }
        cudaGetLastError();
        return LURK_OK;
    }

    int sync() override {
        for (cudaStream_t s : {sH, sK[0], sK[1], sK[2], sA, sB, sC, sT})
            if (s) LURK_CUDA_TRY(cudaStreamSynchronize(s));
        return LURK_OK;
    }
};

template <class C>
FoldCtxBase *make_fold_ctx() { return new FoldCtx<C>(); }
template FoldCtxBase *make_fold_ctx<LURK_C>();

}  // namespace lurk
