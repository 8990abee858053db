/* A plain C99 client of the Spartan prover context (lurk_spartan_ctx_*, include/lurk_b200.h): what the Rust side of `compress`
 * (src/proof/nova.rs:341-356) would do through bindgen.  It folds a small step circuit (satisfiable by construction) through the fold
 * context and proves RelaxedR1CSSNARK straight from the running instance's device buffers LURK_FOLD_BUF_Z1 / LURK_FOLD_BUF_E1, with no
 * host copy of W or E, and checks what it can check by itself:
 *   - the transcript has the shape of the protocol: log_rows tau challenges and outer rounds, one claims message of 4 elements,
 *     log_vars + 1 inner rounds, m + 2 rounds of the evaluation-claim reduction;
 *   - the same call again gives the same bytes; a callback that fails aborts the proof with an error code.
 * Without a GPU the refusals still hold and creating a context fails loudly with LURK_ERR_NOGPU. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "lurk_b200.h"

#define M 48      /* free ("slot") columns */
#define K 20      /* defined columns g_j = s_a(j) * s_b(j) */
#define NW (M + K)
#define ROWS (3 * K)
#define NX 2

static int fail(int code, const char *what) {
    fprintf(stderr, "spartan_client: %s (last error: %s)\n", what, lurk_last_error());
    return code;
}
static void put_u64(uint8_t *dst, uint64_t v) { int i; memset(dst, 0, 32); for (i = 0; i < 8; i++) dst[i] = (uint8_t)(v >> (8 * i)); }
static uint32_t rng_state = 4242;
static uint32_t rnd(void) { rng_state = rng_state * 1664525u + 1013904223u; return rng_state >> 8; }

/* a stand-in transcript: the challenge is a 62-bit mix of the phase, the round and the message (canonical, far below p) */
typedef struct { int calls[6]; int fail_at_phase; } transcript;
static int challenge(void *user, int phase, int round, const uint8_t *msg, size_t len, uint8_t out[32]) {
    transcript *t = (transcript *)user;
    uint64_t h = 1469598103934665603ull ^ (uint64_t)(phase * 131 + round);
    size_t i;
    if (phase < 0 || phase > 5) return 1;
    t->calls[phase]++;
    if (phase == t->fail_at_phase) return 7;
    for (i = 0; i < len; i++) h = (h ^ msg[i]) * 1099511628211ull;
    put_u64(out, (h >> 2) | 1);
    return 0;
}

int main(void) {
    static uint64_t rp[3][ROWS + 1];
    static uint32_t col[3][2 * ROWS];
    static uint8_t val[3][2 * ROWS * 32];
    const uint64_t *rps[3];
    const uint32_t *cols[3];
    const uint8_t *vals[3];
    int a_of[K], b_of[K], m, j, r, step;
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
    lurk_spartan_ctx *sp = NULL;
    lurk_spartan_proof proof;
    memset(&proof, 0, sizeof proof);
    if (lurk_spartan_ctx_create(LURK_FIELD_BN254_FR, NW, NX, ROWS, rps, cols, vals, 5, &sp) != LURK_ERR_ARG || sp) return fail(1, "bad format accepted");
    if (lurk_spartan_ctx_create(LURK_FIELD_BN254_FR, NW, NX, 0, rps, cols, vals, LURK_FMT_CANONICAL, &sp) != LURK_ERR_ARG) return fail(1, "no rows accepted");
    if (lurk_spartan_prove_dev(NULL, NULL, NULL, challenge, NULL, &proof, NULL, LURK_FMT_CANONICAL, NULL) != LURK_ERR_ARG) return fail(1, "null context accepted");
    if (lurk_spartan_prove_batch_dev(31, NULL, NULL, NULL, challenge, NULL, &proof, NULL, LURK_FMT_CANONICAL, NULL) != LURK_ERR_ARG) return fail(1, "31 instances accepted");

    int rc = lurk_spartan_ctx_create(LURK_FIELD_BN254_FR, NW, NX, ROWS, rps, cols, vals, LURK_FMT_CANONICAL, &sp);
    if (lurk_device_count() <= 0) {
        if (rc != LURK_ERR_NOGPU || sp != NULL) return fail(2, "context creation without a GPU must fail loudly");
        puts("spartan_client ok (no GPU: compute entry points fail loudly)");
        return 0;
    }
    if (rc != LURK_OK) return fail(3, "spartan ctx");
    int log_rows = 0, log_vars = 0, field = -1;
    size_t joint_len = 0;
    if (lurk_spartan_ctx_info(sp, &field, &log_rows, &log_vars, &joint_len) != LURK_OK || field != LURK_FIELD_BN254_FR) return fail(4, "info");
    /* ROWS = 60 -> 2^6 rows; z = 68 + 1 + 2 -> num_vars = 2^7 */
    if (log_rows != 6 || log_vars != 7 || joint_len != 128) return fail(4, "shape");

    /* the running instance: three folds through the fold context */
    uint8_t *bases = malloc(64 * 256);
    lurk_msm_ctx *ck = NULL;
    if (lurk_synthetic_bases(LURK_CURVE_BN254_G1, 0, 256, LURK_FMT_CANONICAL, bases) != LURK_OK) return fail(5, "synthetic bases");
    if (lurk_msm_ctx_create(LURK_CURVE_BN254_G1, bases, 256, LURK_FMT_CANONICAL, &ck) != LURK_OK) return fail(5, "msm ctx");
    lurk_fold_config cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.curve_id = LURK_CURVE_BN254_G1; cfg.depth = 1; cfg.n_w = NW; cfg.n_x = NX; cfg.n_rows = ROWS;
    for (m = 0; m < 3; m++) { cfg.row_ptr[m] = rp[m]; cfg.col[m] = col[m]; cfg.val[m] = val[m]; }
    cfg.fmt = LURK_FMT_CANONICAL; cfg.world = 1; cfg.rank = 0;
    lurk_fold_ctx *fc = NULL;
    if (lurk_fold_ctx_create(&cfg, ck, ck, &fc) != LURK_OK) return fail(6, "fold ctx");
    lurk_fold_span span = {0, NW, NW, 1};
    if (lurk_fold_ctx_set_spans(fc, 1, &span) != LURK_OK) return fail(6, "spans");
    lurk_fold_result res;
    for (step = 0; step < 3; step++) {
        void *w, *x, *ro;
        size_t bytes;
        uint64_t s[M];
        int i;
        if (lurk_fold_ctx_host_buffer(fc, 0, LURK_FOLD_BUF_GLUE, &w, &bytes) != LURK_OK || lurk_fold_ctx_host_buffer(fc, 0, LURK_FOLD_BUF_X2, &x, &bytes) != LURK_OK ||
            lurk_fold_ctx_host_buffer(fc, 0, LURK_FOLD_BUF_RO, &ro, &bytes) != LURK_OK)
            return fail(7, "host buffers");
        for (i = 0; i < M; i++) { s[i] = rnd() & 0xffff; put_u64((uint8_t *)w + 32 * i, s[i]); }
        for (j = 0; j < K; j++) put_u64((uint8_t *)w + 32 * (M + j), s[a_of[j]] * s[b_of[j]]);
        memset(ro, 0, 24 * 32);
        put_u64((uint8_t *)ro, 0xabcdef);
        for (i = 0; i < NX; i++) { uint64_t v = rnd(); put_u64((uint8_t *)x + 32 * i, v); put_u64((uint8_t *)ro + 32 * (4 + i), v); }
        if (lurk_fold_ctx_stage_a(fc, 0, 0, LURK_FMT_CANONICAL) != LURK_OK) return fail(8, "stage A");
        if ((step == 0 ? lurk_fold_ctx_init_running(fc, 0) : lurk_fold_ctx_stage_b_launch(fc, 0)) != LURK_OK) return fail(8, "stage B");
        if (lurk_fold_ctx_collect(fc, 0, &res, LURK_FMT_CANONICAL) != LURK_OK || res.status != 0) return fail(8, "collect");
    }
    void *d_z = NULL, *d_E = NULL, *d_joint = NULL;
    size_t zb = 0, eb = 0, jb = 0;
    if (lurk_fold_ctx_device_buffer(fc, 0, LURK_FOLD_BUF_Z1, &d_z, &zb) != LURK_OK || lurk_fold_ctx_device_buffer(fc, 0, LURK_FOLD_BUF_E1, &d_E, &eb) != LURK_OK)
        return fail(9, "device buffers");
    /* device memory for the joint polynomial (2^7 elements): the running E of a second fold context with 200 empty rows */
    lurk_fold_config big = cfg;
    lurk_fold_ctx *holder = NULL;
    big.n_w = 200;
    big.n_rows = 200;
    {
        static uint64_t zrp[201];
        const uint64_t *zr[3];
        memset(zrp, 0, sizeof zrp);
        for (m = 0; m < 3; m++) { zr[m] = zrp; big.row_ptr[m] = zr[m]; big.col[m] = NULL; big.val[m] = NULL; }
        if (lurk_fold_ctx_create(&big, ck, ck, &holder) != LURK_OK) return fail(10, "holder ctx");
    }
    if (lurk_fold_ctx_device_buffer(holder, 0, LURK_FOLD_BUF_E1, &d_joint, &jb) != LURK_OK || jb < 32 * joint_len) return fail(10, "joint buffer");

    static uint8_t outer[6 * 4 * 32], inner[8 * 3 * 32], claims[4 * 32], red[7 * 3 * 32], rr[7 * 32], je[32], je2[32], left[2 * 32], w[2 * 32];
    transcript t;
    memset(&t, 0, sizeof t);
    t.fail_at_phase = -1;
    proof.outer_rounds = outer; proof.inner_rounds = inner; proof.claims = claims; proof.reduce_rounds = red; proof.r = rr;
    proof.joint_eval = je; proof.claims_left = left; proof.weights = w;
    if (lurk_spartan_prove_dev(sp, d_z, d_E, challenge, &t, &proof, d_joint, LURK_FMT_CANONICAL, NULL) != LURK_OK) return fail(11, "prove");
    if (t.calls[LURK_SPARTAN_TAU] != log_rows || t.calls[LURK_SPARTAN_OUTER_R] != 0 || t.calls[LURK_SPARTAN_OUTER] != log_rows ||
        t.calls[LURK_SPARTAN_CLAIMS] != 1 || t.calls[LURK_SPARTAN_INNER] != log_vars + 1 || t.calls[LURK_SPARTAN_BATCH_EVAL] != 7 + 2)
        return fail(12, "transcript shape");
    proof.joint_eval = je2;
    if (lurk_spartan_prove_dev(sp, d_z, d_E, challenge, &t, &proof, d_joint, LURK_FMT_CANONICAL, NULL) != LURK_OK || memcmp(je, je2, 32))
        return fail(13, "the same proof twice differs");
    t.fail_at_phase = LURK_SPARTAN_INNER;
    if (lurk_spartan_prove_dev(sp, d_z, d_E, challenge, &t, &proof, d_joint, LURK_FMT_CANONICAL, NULL) != LURK_ERR_ARG) return fail(14, "failing callback");
    /* d_joint over the running E is refused */
    if (lurk_spartan_prove_dev(sp, d_z, d_E, challenge, &t, &proof, d_E, LURK_FMT_CANONICAL, NULL) != LURK_ERR_ARG) return fail(15, "overlap accepted");
    lurk_fold_ctx_destroy(holder);
    lurk_fold_ctx_destroy(fc);
    lurk_msm_ctx_destroy(ck);
    lurk_spartan_ctx_destroy(sp);
    free(bases);
    puts("spartan_client ok");
    return 0;
}
