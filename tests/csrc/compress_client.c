/* A plain C99 client of the compress context (lurk_compress_ctx_*, lurk_compress_prove_dev; include/lurk_b200.h): what the Rust side of
 * CompressedSNARK::prove (src/proof/nova.rs:341-356) would do through bindgen.  It folds a small step circuit (satisfiable by
 * construction) on BN254 (primary, HyperKZG) and on Grumpkin (secondary, IPA) through two fold contexts -- the secondary's last fold is one
 * more stage_a + stage_b_launch + collect, as Arecibo folds l_u_secondary into r_U_secondary before S2::prove -- and proves both circuits
 * in one call from the LURK_FOLD_BUF_Z1 / LURK_FOLD_BUF_E1 buffers and the records' running commitments.  It checks what it can check by
 * itself: the shape of both transcripts, identical bytes from the concurrent and the sequential call, a failing secondary callback that
 * names the secondary circuit and leaves the context usable, and a key shorter than the joint polynomial refused at creation.
 * Without a GPU the refusals still hold and every entry point fails loudly with LURK_ERR_NOGPU. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "lurk_b200.h"

#define M 48      /* free ("slot") columns */
#define K 20      /* defined columns g_j = s_a(j) * s_b(j) */
#define NW (M + K)
#define ROWS (3 * K)
#define NX 2
#define LOGN 7    /* joint_len = 2^7: 2^6 rows, num_vars = 2^7 */

static int fail(int code, const char *what) {
    fprintf(stderr, "compress_client: %s (last error: %s)\n", what, lurk_last_error());
    return code;
}
static void put_u64(uint8_t *dst, uint64_t v) { int i; memset(dst, 0, 32); for (i = 0; i < 8; i++) dst[i] = (uint8_t)(v >> (8 * i)); }
static uint32_t rng_state = 4242;
static uint32_t rnd(void) { rng_state = rng_state * 1664525u + 1013904223u; return rng_state >> 8; }

/* a stand-in transcript per circuit: the challenge is a 62-bit mix of the phase, the round and the message (canonical, far below p) */
typedef struct { int calls[2][7]; int fail_circuit; } transcript;
static int challenge(void *user, int circuit, int phase, int round, const uint8_t *msg, size_t len, uint8_t out[32]) {
    transcript *t = (transcript *)user;
    uint64_t h = 1469598103934665603ull ^ (uint64_t)(circuit * 7919 + phase * 131 + round);
    size_t i;
    if (circuit < 0 || circuit > 1 || phase < 0 || phase > 6) return 1;
    t->calls[circuit][phase]++;
    if (circuit == t->fail_circuit && phase == LURK_SPARTAN_PCS) return 9;
    for (i = 0; i < len; i++) h = (h ^ msg[i]) * 1099511628211ull;
    put_u64(out, (h >> 2) | 1);
    return 0;
}

typedef struct {
    lurk_msm_ctx *ck;
    lurk_fold_ctx *fc;
    lurk_fold_result res;
} circuit;

/* a running instance of the step circuit after `steps` folds on `curve`; the key has 256 bases */
static int fold(circuit *c, int curve, int steps, const uint64_t *const rp[3], const uint32_t *const col[3], const uint8_t *const val[3],
                const int *a_of, const int *b_of) {
    uint8_t *bases = malloc(64 * 256);
    lurk_fold_config cfg;
    int m, step, i, j;
    if (!bases || lurk_synthetic_bases(curve, 0, 256, LURK_FMT_CANONICAL, bases) != LURK_OK) return 1;
    if (lurk_msm_ctx_create(curve, bases, 256, LURK_FMT_CANONICAL, &c->ck) != LURK_OK) return 1;
    free(bases);
    memset(&cfg, 0, sizeof cfg);
    cfg.curve_id = curve; cfg.depth = 1; cfg.n_w = NW; cfg.n_x = NX; cfg.n_rows = ROWS;
    for (m = 0; m < 3; m++) { cfg.row_ptr[m] = rp[m]; cfg.col[m] = col[m]; cfg.val[m] = val[m]; }
    cfg.fmt = LURK_FMT_CANONICAL; cfg.world = 1; cfg.rank = 0;
    if (lurk_fold_ctx_create(&cfg, c->ck, c->ck, &c->fc) != LURK_OK) return 1;
    lurk_fold_span span = {0, NW, NW, 1};
    if (lurk_fold_ctx_set_spans(c->fc, 1, &span) != LURK_OK) return 1;
    for (step = 0; step < steps; step++) {
        void *w, *x, *ro;
        size_t bytes;
        uint64_t s[M];
        if (lurk_fold_ctx_host_buffer(c->fc, 0, LURK_FOLD_BUF_GLUE, &w, &bytes) != LURK_OK || lurk_fold_ctx_host_buffer(c->fc, 0, LURK_FOLD_BUF_X2, &x, &bytes) != LURK_OK ||
            lurk_fold_ctx_host_buffer(c->fc, 0, LURK_FOLD_BUF_RO, &ro, &bytes) != LURK_OK)
            return 1;
        for (i = 0; i < M; i++) { s[i] = rnd() & 0xffff; put_u64((uint8_t *)w + 32 * i, s[i]); }
        for (j = 0; j < K; j++) put_u64((uint8_t *)w + 32 * (M + j), s[a_of[j]] * s[b_of[j]]);
        memset(ro, 0, 24 * 32);
        put_u64((uint8_t *)ro, 0xabcdef);
        for (i = 0; i < NX; i++) { uint64_t v = rnd(); put_u64((uint8_t *)x + 32 * i, v); put_u64((uint8_t *)ro + 32 * (4 + i), v); }
        if (lurk_fold_ctx_stage_a(c->fc, 0, 0, LURK_FMT_CANONICAL) != LURK_OK) return 1;
        if ((step == 0 ? lurk_fold_ctx_init_running(c->fc, 0) : lurk_fold_ctx_stage_b_launch(c->fc, 0)) != LURK_OK) return 1;
        if (lurk_fold_ctx_collect(c->fc, 0, &c->res, LURK_FMT_CANONICAL) != LURK_OK || c->res.status != 0) return 1;
    }
    return 0;
}

int main(void) {
    static uint64_t rp[3][ROWS + 1];
    static uint32_t col[3][2 * ROWS];
    static uint8_t val[3][2 * ROWS * 32];
    const uint64_t *rps[3];
    const uint32_t *cols[3];
    const uint8_t *vals[3];
    int a_of[K], b_of[K], m, j, r;
    size_t nnz[3] = {0, 0, 0};
    for (j = 0; j < K; j++) { a_of[j] = (int)(rnd() % M); b_of[j] = (int)(rnd() % M); }
    for (r = 0; r < ROWS; r++) {
        int kind = r / K;                  /* 0: definition, 1: the same with other coefficients, 2: linear row */
        j = r % K;
        for (m = 0; m < 3; m++) rp[m][r] = nnz[m];
        if (kind < 2) {
            uint64_t l = kind ? 2 : 1, mu = kind ? 3 : 1;
            col[0][nnz[0]] = (uint32_t)a_of[j]; put_u64(val[0] + 32 * nnz[0]++, l);
            col[1][nnz[1]] = (uint32_t)b_of[j]; put_u64(val[1] + 32 * nnz[1]++, mu);
            col[2][nnz[2]] = (uint32_t)(M + j); put_u64(val[2] + 32 * nnz[2]++, l * mu);
        } else {                           /* (s_a + x_0) * u = (s_a + x_0) */
            col[0][nnz[0]] = (uint32_t)a_of[j]; put_u64(val[0] + 32 * nnz[0]++, 1);
            col[0][nnz[0]] = NW + 1; put_u64(val[0] + 32 * nnz[0]++, 1);
            col[1][nnz[1]] = NW; put_u64(val[1] + 32 * nnz[1]++, 1);
            col[2][nnz[2]] = (uint32_t)a_of[j]; put_u64(val[2] + 32 * nnz[2]++, 1);
            col[2][nnz[2]] = NW + 1; put_u64(val[2] + 32 * nnz[2]++, 1);
        }
    }
    for (m = 0; m < 3; m++) { rp[m][ROWS] = nnz[m]; rps[m] = rp[m]; cols[m] = col[m]; vals[m] = val[m]; }

    /* refusals come before any device work, with or without a GPU */
    lurk_compress_ctx *cc = NULL;
    lurk_compress_pcs none = {LURK_PCS_HYPERKZG, NULL, NULL};
    lurk_compress_proof proof;
    transcript t;
    memset(&proof, 0, sizeof proof);
    memset(&t, 0, sizeof t);
    t.fail_circuit = -1;
    if (lurk_compress_ctx_create(0, NULL, NULL, &none, &none, LURK_FMT_CANONICAL, &cc) != LURK_ERR_ARG || cc) return fail(1, "no primary accepted");
    if (lurk_compress_prove_dev(NULL, 1, NULL, NULL, NULL, NULL, NULL, NULL, NULL, NULL, challenge, &t, 0, &proof, LURK_FMT_CANONICAL, NULL) != LURK_ERR_ARG)
        return fail(1, "null context accepted");
    if (lurk_compress_ctx_info(NULL, NULL, NULL, NULL) != LURK_ERR_ARG) return fail(1, "info without a context");

    lurk_spartan_ctx *sp1 = NULL, *sp2 = NULL;
    int rc = lurk_spartan_ctx_create(LURK_FIELD_BN254_FR, NW, NX, ROWS, rps, cols, vals, LURK_FMT_CANONICAL, &sp1);
    if (lurk_device_count() <= 0) {
        if (rc != LURK_ERR_NOGPU || sp1 != NULL) return fail(2, "context creation without a GPU must fail loudly");
        puts("compress_client ok (no GPU: compute entry points fail loudly)");
        return 0;
    }
    if (rc != LURK_OK || lurk_spartan_ctx_create(LURK_FIELD_BN254_FQ, NW, NX, ROWS, rps, cols, vals, LURK_FMT_CANONICAL, &sp2) != LURK_OK)
        return fail(3, "spartan ctx");

    /* the primary folds three steps; the secondary three, then its last fresh instance (l_u_secondary) is folded in: a fourth fold */
    circuit c1, c2;
    memset(&c1, 0, sizeof c1);
    memset(&c2, 0, sizeof c2);
    if (fold(&c1, LURK_CURVE_BN254_G1, 3, rps, cols, vals, a_of, b_of)) return fail(4, "primary folds");
    if (fold(&c2, LURK_CURVE_GRUMPKIN, 4, rps, cols, vals, a_of, b_of)) return fail(4, "secondary folds");

    uint8_t ck_c[64];
    if (lurk_synthetic_bases(LURK_CURVE_GRUMPKIN, 1000, 1, LURK_FMT_CANONICAL, ck_c) != LURK_OK) return fail(5, "ck_c");
    lurk_compress_pcs p1 = {LURK_PCS_HYPERKZG, c1.ck, NULL}, p2 = {LURK_PCS_IPA, c2.ck, ck_c};
    /* a key shorter than the joint polynomial is refused at creation */
    {
        uint8_t small[64 * 64];
        lurk_msm_ctx *short_ck = NULL;
        lurk_compress_pcs ps = {LURK_PCS_HYPERKZG, NULL, NULL};
        if (lurk_synthetic_bases(LURK_CURVE_BN254_G1, 0, 64, LURK_FMT_CANONICAL, small) != LURK_OK ||
            lurk_msm_ctx_create(LURK_CURVE_BN254_G1, small, 64, LURK_FMT_CANONICAL, &short_ck) != LURK_OK)
            return fail(6, "short key");
        ps.ck = short_ck;
        if (lurk_compress_ctx_create(1, &sp1, sp2, &ps, &p2, LURK_FMT_CANONICAL, &cc) != LURK_ERR_ARG || cc) return fail(6, "short key accepted");
        lurk_msm_ctx_destroy(short_ck);
    }
    if (lurk_compress_ctx_create(1, &sp1, sp2, &p1, &p2, LURK_FMT_CANONICAL, &cc) != LURK_OK) return fail(7, "compress ctx");
    size_t held = 1, jl1 = 0, jl2 = 0;
    if (lurk_compress_ctx_info(cc, &held, &jl1, &jl2) != LURK_OK || held != 0 || jl1 != ((size_t)1 << LOGN) || jl2 != ((size_t)1 << LOGN))
        return fail(7, "info before the first proof");

    void *z1, *e1, *z2, *e2;
    size_t b;
    if (lurk_fold_ctx_device_buffer(c1.fc, 0, LURK_FOLD_BUF_Z1, &z1, &b) != LURK_OK || lurk_fold_ctx_device_buffer(c1.fc, 0, LURK_FOLD_BUF_E1, &e1, &b) != LURK_OK ||
        lurk_fold_ctx_device_buffer(c2.fc, 0, LURK_FOLD_BUF_Z1, &z2, &b) != LURK_OK || lurk_fold_ctx_device_buffer(c2.fc, 0, LURK_FOLD_BUF_E1, &e2, &b) != LURK_OK)
        return fail(8, "device buffers");
    const void *zs[1] = {z1}, *es[1] = {e1};
    const uint8_t *cw[1] = {c1.res.running_comm_W}, *ce[1] = {c1.res.running_comm_E};
    static uint8_t comm[2][2][96], w[2][3 * 96], v[2][3 * LOGN * 32], L[2][LOGN * 96], R[2][LOGN * 96], af[2][32], je[2][2][32];
    int run;
    for (run = 0; run < 2; run++) {       /* concurrent, then sequential: the same bytes */
        memset(&proof, 0, sizeof proof);
        proof.primary.comm = comm[run][0]; proof.primary.w = w[run]; proof.primary.v = v[run]; proof.primary.snark.joint_eval = je[run][0];
        proof.secondary.comm = comm[run][1]; proof.secondary.L = L[run]; proof.secondary.R = R[run]; proof.secondary.a_final = af[run];
        proof.secondary.snark.joint_eval = je[run][1];
        memset(&t, 0, sizeof t);
        t.fail_circuit = -1;
        if (lurk_compress_prove_dev(cc, 1, zs, es, cw, ce, z2, e2, c2.res.running_comm_W, c2.res.running_comm_E, challenge, &t, run ? LURK_COMPRESS_SEQUENTIAL : 0,
                                    &proof, LURK_FMT_CANONICAL, NULL) != LURK_OK)
            return fail(9, "prove");
        for (j = 0; j < 2; j++)
            if (t.calls[j][LURK_SPARTAN_TAU] != 6 || t.calls[j][LURK_SPARTAN_OUTER] != 6 || t.calls[j][LURK_SPARTAN_CLAIMS] != 1 ||
                t.calls[j][LURK_SPARTAN_INNER] != 8 || t.calls[j][LURK_SPARTAN_BATCH_EVAL] != LOGN + 2)
                return fail(10, "Spartan transcript shape");
        if (t.calls[0][LURK_SPARTAN_PCS] != 3 || t.calls[1][LURK_SPARTAN_PCS] != 1 + LOGN) return fail(10, "opening transcript shape");
    }
    if (memcmp(comm[0], comm[1], sizeof comm[0]) || memcmp(w[0], w[1], sizeof w[0]) || memcmp(v[0], v[1], sizeof v[0]) || memcmp(L[0], L[1], sizeof L[0]) ||
        memcmp(R[0], R[1], sizeof R[0]) || memcmp(af[0], af[1], 32) || memcmp(je[0], je[1], sizeof je[0]))
        return fail(11, "concurrent and sequential proofs differ");
    if (lurk_compress_ctx_info(cc, &held, NULL, NULL) != LURK_OK || held == 0) return fail(12, "no arena after the first proof");
    /* a failing secondary callback: an error naming the secondary circuit; the context proves again afterwards */
    t.fail_circuit = 1;
    if (lurk_compress_prove_dev(cc, 1, zs, es, cw, ce, z2, e2, c2.res.running_comm_W, c2.res.running_comm_E, challenge, &t, 0, &proof, LURK_FMT_CANONICAL,
                                NULL) != LURK_ERR_ARG || !strstr(lurk_last_error(), "secondary"))
        return fail(13, "failing secondary callback");
    t.fail_circuit = -1;
    proof.primary.comm = comm[1][0];
    if (lurk_compress_prove_dev(cc, 1, zs, es, cw, ce, z2, e2, c2.res.running_comm_W, c2.res.running_comm_E, challenge, &t, 0, &proof, LURK_FMT_CANONICAL,
                                NULL) != LURK_OK || memcmp(comm[0][0], comm[1][0], 96))
        return fail(14, "the context after an error");
    lurk_compress_ctx_destroy(cc);
    lurk_fold_ctx_destroy(c1.fc);
    lurk_fold_ctx_destroy(c2.fc);
    lurk_msm_ctx_destroy(c1.ck);
    lurk_msm_ctx_destroy(c2.ck);
    lurk_spartan_ctx_destroy(sp1);
    lurk_spartan_ctx_destroy(sp2);
    puts("compress_client ok");
    return 0;
}
