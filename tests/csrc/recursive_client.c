/* A plain C99 client of the recursive verifier (lurk_recursive_verify_dev / lurk_recursive_verify; include/lurk_b200.h): what the Rust
 * side of Proof::verify on a Recursive proof (src/proof/nova.rs:358-373) would do through bindgen.  It folds a small step circuit
 * (satisfiable by construction) on BN254 (primary) and on Grumpkin (secondary) through two fold contexts, stages the secondary's next
 * fresh instance without folding it (l_u_secondary), and verifies [r_U_primary, r_U_secondary, l_u_secondary] in one call straight from
 * LURK_FOLD_BUF_Z1 / _E1 / _W2, the secondary's shape a verifier-only context.  It checks that the call accepts and agrees with
 * lurk_fold_ctx_check_running, that swapped commitments are rejected with the right verdict, and that the host form agrees.
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
    fprintf(stderr, "recursive_client: %s (last error: %s)\n", what, lurk_last_error());
    return code;
}
static void put_u64(uint8_t *dst, uint64_t v) { int i; memset(dst, 0, 32); for (i = 0; i < 8; i++) dst[i] = (uint8_t)(v >> (8 * i)); }
static uint32_t rng_state = 4242;
static uint32_t rnd(void) { rng_state = rng_state * 1664525u + 1013904223u; return rng_state >> 8; }

typedef struct {
    lurk_msm_ctx *ck;
    lurk_fold_ctx *fc;
    lurk_fold_result res;
} circuit;

/* a running instance of the step circuit after `steps` folds on `curve` (with stage_only, the last step is staged in buffer 0 and not
 * folded); records in Montgomery form; the key has 256 bases */
static int fold(circuit *c, int curve, int steps, int stage_only, const uint64_t *const rp[3], const uint32_t *const col[3], const uint8_t *const val[3],
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
        if (step == steps - 1 && stage_only) return lurk_fold_ctx_sync(c->fc) != LURK_OK;     /* staged, not folded */
        if ((step == 0 ? lurk_fold_ctx_init_running(c->fc, 0) : lurk_fold_ctx_stage_b_launch(c->fc, 0)) != LURK_OK) return 1;
        if (lurk_fold_ctx_collect(c->fc, 0, &c->res, LURK_FMT_MONTGOMERY) != LURK_OK || c->res.status != 0) return 1;
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
    lurk_recursive_instance inst[3];
    lurk_recursive_verdict verdict[3];
    int accepted = 7;
    memset(inst, 0, sizeof inst);
    if (lurk_recursive_verify_dev(0, inst, verdict, &accepted, LURK_FMT_MONTGOMERY, NULL) != LURK_ERR_ARG) return fail(1, "no instance accepted");
    if (lurk_recursive_verify_dev(1, inst, verdict, &accepted, LURK_FMT_MONTGOMERY, NULL) != LURK_ERR_ARG || !strstr(lurk_last_error(), "shape"))
        return fail(1, "null shape accepted");

    lurk_spartan_ctx *sp1 = NULL, *sp2 = NULL;
    int rc = lurk_spartan_ctx_create(LURK_FIELD_BN254_FR, NW, NX, ROWS, rps, cols, vals, LURK_FMT_CANONICAL, &sp1);
    if (lurk_device_count() <= 0) {
        if (rc != LURK_ERR_NOGPU || sp1 != NULL) return fail(2, "context creation without a GPU must fail loudly");
        if (lurk_spartan_ctx_create_verifier(LURK_FIELD_BN254_FQ, NW, NX, ROWS, rps, cols, vals, LURK_FMT_CANONICAL, &sp2) != LURK_ERR_NOGPU || sp2)
            return fail(2, "verifier-only context creation without a GPU must fail loudly");
        puts("recursive_client ok (no GPU: compute entry points fail loudly)");
        return 0;
    }
    if (rc != LURK_OK || lurk_spartan_ctx_create_verifier(LURK_FIELD_BN254_FQ, NW, NX, ROWS, rps, cols, vals, LURK_FMT_CANONICAL, &sp2) != LURK_OK)
        return fail(3, "spartan ctx");

    /* three folds each; the secondary's fourth instance is staged and left unfolded: l_u_secondary */
    circuit c1, c2;
    memset(&c1, 0, sizeof c1);
    memset(&c2, 0, sizeof c2);
    if (fold(&c1, LURK_CURVE_BN254_G1, 3, 0, rps, cols, vals, a_of, b_of)) return fail(4, "primary folds");
    if (fold(&c2, LURK_CURVE_GRUMPKIN, 4, 1, rps, cols, vals, a_of, b_of)) return fail(4, "secondary folds");
    void *z1, *e1, *z2, *e2, *w2;
    size_t b;
    if (lurk_fold_ctx_device_buffer(c1.fc, 0, LURK_FOLD_BUF_Z1, &z1, &b) != LURK_OK || lurk_fold_ctx_device_buffer(c1.fc, 0, LURK_FOLD_BUF_E1, &e1, &b) != LURK_OK ||
        lurk_fold_ctx_device_buffer(c2.fc, 0, LURK_FOLD_BUF_Z1, &z2, &b) != LURK_OK || lurk_fold_ctx_device_buffer(c2.fc, 0, LURK_FOLD_BUF_E1, &e2, &b) != LURK_OK ||
        lurk_fold_ctx_device_buffer(c2.fc, 0, LURK_FOLD_BUF_W2, &w2, &b) != LURK_OK)
        return fail(5, "device buffers");
    /* comm_W of the fresh instance: the step's commitment, recomputed on the key (Montgomery, as the records) */
    uint8_t comm_w2[96];
    if (lurk_msm_ctx_run_dev(c2.ck, w2, NW, LURK_FMT_MONTGOMERY, comm_w2, NULL) != LURK_OK) return fail(5, "commit(W2)");
    lurk_recursive_instance good[3] = {{sp1, c1.ck, z1, e1, c1.res.running_comm_W, c1.res.running_comm_E},
                                       {sp2, c2.ck, z2, e2, c2.res.running_comm_W, c2.res.running_comm_E},
                                       {sp2, c2.ck, w2, NULL, comm_w2, NULL}};
    if (lurk_recursive_verify_dev(3, good, verdict, &accepted, LURK_FMT_MONTGOMERY, NULL) != LURK_OK) return fail(6, "verify");
    for (j = 0; j < 3; j++)
        if (verdict[j].bad_rows || verdict[j].first_bad_row != UINT64_MAX || !verdict[j].u_ok || !verdict[j].comm_W_ok || !verdict[j].comm_E_ok)
            return fail(6, "a verdict of a good proof fails");
    if (accepted != 1) return fail(6, "a good proof rejected");
    uint64_t bad_rows = 1;
    int okw = 0, oke = 0;
    if (lurk_fold_ctx_check_running(c1.fc, &bad_rows, &okw, &oke) != LURK_OK || bad_rows || !okw || !oke) return fail(7, "check_running disagrees");
    /* the primary's comm_W and comm_E swapped: rejected, both commitments named, the rows hold */
    memcpy(inst, good, sizeof inst);
    inst[0].comm_W = c1.res.running_comm_E;
    inst[0].comm_E = c1.res.running_comm_W;
    if (lurk_recursive_verify_dev(3, inst, verdict, &accepted, LURK_FMT_MONTGOMERY, NULL) != LURK_OK || accepted != 0) return fail(8, "swapped commitments accepted");
    if (verdict[0].bad_rows || verdict[0].comm_W_ok || verdict[0].comm_E_ok || !verdict[1].comm_W_ok || !verdict[2].u_ok) return fail(8, "verdicts of the swap");
    /* the host form, from the running instance the fold context hands out (canonical) */
    {
        static uint8_t W[NW * 32], E[ROWS * 32], z[(NW + 1 + NX) * 32], cw[96], ce[96];
        if (lurk_fold_ctx_get_running(c1.fc, W, E, z + NW * 32, z + (NW + 1) * 32, cw, ce, LURK_FMT_CANONICAL) != LURK_OK) return fail(9, "get_running");
        memcpy(z, W, sizeof W);
        lurk_recursive_instance h = {sp1, c1.ck, z, E, cw, ce};
        if (lurk_recursive_verify(1, &h, verdict, &accepted, LURK_FMT_CANONICAL, NULL) != LURK_OK || accepted != 1) return fail(9, "host form");
        E[32 * 3] ^= 1;
        if (lurk_recursive_verify(1, &h, verdict, &accepted, LURK_FMT_CANONICAL, NULL) != LURK_OK || accepted != 0 || verdict[0].bad_rows != 1 ||
            verdict[0].first_bad_row != 3 || verdict[0].comm_E_ok)
            return fail(9, "host form, one E row changed");
    }
    lurk_fold_ctx_destroy(c1.fc);
    lurk_fold_ctx_destroy(c2.fc);
    lurk_msm_ctx_destroy(c1.ck);
    lurk_msm_ctx_destroy(c2.ck);
    lurk_spartan_ctx_destroy(sp1);
    lurk_spartan_ctx_destroy(sp2);
    puts("recursive_client ok");
    return 0;
}
