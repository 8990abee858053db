/* A plain C99 client of the compressed verifier (lurk_compress_verify; include/lurk_b200.h): what the Rust side of
 * CompressedSNARK::verify (src/proof/nova.rs:358-373) would do through bindgen.  It folds a small step circuit (satisfiable by construction)
 * on BN254 (primary, HyperKZG, under a powers-of-tau key of known beta) and on Grumpkin (secondary, IPA), proves both circuits with the
 * compress context, and verifies the proof with the same native transcript.  The pairing callback checks P == beta Q in G1 with
 * lurk_point_combination, which is what e(P, H) == e(Q, beta H) means under a key of known beta.  It checks: the good proof is accepted by
 * the concurrent and the sequential call with the prover's transcript shape, a tampered a_final is rejected by the secondary's closing check
 * alone, a pairing callback that fails is an error naming the primary circuit, and the refusals come before any callback.
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
    fprintf(stderr, "compress_verify_client: %s (last error: %s)\n", what, lurk_last_error());
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

#define BETA 0x1234567fedcbull

/* beta P (96 bytes) with lurk_point_combination */
static int times_beta(const uint8_t P[96], uint8_t out[96]) {
    uint8_t b[32];
    put_u64(b, BETA);
    return lurk_point_combination(LURK_CURVE_BN254_G1, P, b, 1, LURK_FMT_CANONICAL, out);
}

/* the KZG key g, beta g, .., beta^255 g with g = (1, 2), BN254's generator */
static int kzg_bases(uint8_t *bases) {
    uint8_t p[96];
    int i;
    memset(p, 0, 96);
    p[0] = 1; p[32] = 2; p[64] = 1;
    for (i = 0; i < 256; i++) {
        memcpy(bases + 64 * i, p, 64);
        if (times_beta(p, p) != LURK_OK) return 1;
    }
    return 0;
}

/* the pairing check under the key of known beta: P == beta Q */
typedef struct { int calls, fail; } pairing_state;
typedef struct { transcript t; pairing_state *ps; } verifier_user;      /* the one user pointer of both callbacks */
static int pairing(void *user, int circuit, const uint8_t P[96], const uint8_t Q[96], int *holds) {
    pairing_state *s = ((verifier_user *)user)->ps;
    uint8_t bq[96];
    s->calls++;
    if (circuit != 0 || s->fail) return 7;
    if (times_beta(Q, bq) != LURK_OK) return 8;
    *holds = memcmp(P, bq, 96) == 0;
    return 0;
}

/* a running instance of the step circuit after `steps` folds on `curve`; the key has 256 bases (KZG powers on BN254) */
static int fold(circuit *c, int curve, int steps, const uint64_t *const rp[3], const uint32_t *const col[3], const uint8_t *const val[3],
                const int *a_of, const int *b_of) {
    uint8_t *bases = malloc(64 * 256);
    lurk_fold_config cfg;
    int m, step, i, j;
    if (!bases || (curve == LURK_CURVE_BN254_G1 ? kzg_bases(bases) : lurk_synthetic_bases(curve, 0, 256, LURK_FMT_CANONICAL, bases)) != LURK_OK) return 1;
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

    /* refusals come before any callback or device work, with or without a GPU */
    lurk_compress_vk_pcs none = {LURK_PCS_HYPERKZG, NULL, NULL, NULL};
    lurk_compress_proof proof;
    lurk_compress_verdict out[2];
    pairing_state ps = {0, 0};
    verifier_user vu;
    int accepted = -1;
    memset(&proof, 0, sizeof proof);
    memset(&vu, 0, sizeof vu);
    vu.t.fail_circuit = -1;
    vu.ps = &ps;
    if (lurk_compress_verify(0, NULL, NULL, &none, &none, NULL, NULL, NULL, NULL, NULL, NULL, NULL, NULL, &proof, 0, challenge, pairing, &vu, 0, out,
                             &accepted, LURK_FMT_CANONICAL, NULL) != LURK_ERR_ARG || accepted != 0 || out[0].snark_ok != -1)
        return fail(1, "no primary accepted");
    if (vu.t.calls[0][0] || ps.calls) return fail(1, "a callback before the refusal");

    lurk_spartan_ctx *sp1 = NULL, *sp2 = NULL;
    int rc = lurk_spartan_ctx_create(LURK_FIELD_BN254_FR, NW, NX, ROWS, rps, cols, vals, LURK_FMT_CANONICAL, &sp1);
    if (lurk_device_count() <= 0) {
        if (rc != LURK_ERR_NOGPU || sp1 != NULL) return fail(2, "context creation without a GPU must fail loudly");
        puts("compress_verify_client ok (no GPU: compute entry points fail loudly)");
        return 0;
    }
    if (rc != LURK_OK || lurk_spartan_ctx_create(LURK_FIELD_BN254_FQ, NW, NX, ROWS, rps, cols, vals, LURK_FMT_CANONICAL, &sp2) != LURK_OK)
        return fail(3, "spartan ctx");
    circuit c1, c2;
    memset(&c1, 0, sizeof c1);
    memset(&c2, 0, sizeof c2);
    if (fold(&c1, LURK_CURVE_BN254_G1, 3, rps, cols, vals, a_of, b_of)) return fail(4, "primary folds");
    if (fold(&c2, LURK_CURVE_GRUMPKIN, 4, rps, cols, vals, a_of, b_of)) return fail(4, "secondary folds");
    uint8_t ck_c[64];
    if (lurk_synthetic_bases(LURK_CURVE_GRUMPKIN, 1000, 1, LURK_FMT_CANONICAL, ck_c) != LURK_OK) return fail(5, "ck_c");
    lurk_compress_pcs p1 = {LURK_PCS_HYPERKZG, c1.ck, NULL}, p2 = {LURK_PCS_IPA, c2.ck, ck_c};
    lurk_compress_ctx *cc = NULL;
    if (lurk_compress_ctx_create(1, &sp1, sp2, &p1, &p2, LURK_FMT_CANONICAL, &cc) != LURK_OK) return fail(6, "compress ctx");
    void *z1, *e1, *z2, *e2;
    size_t b;
    if (lurk_fold_ctx_device_buffer(c1.fc, 0, LURK_FOLD_BUF_Z1, &z1, &b) != LURK_OK || lurk_fold_ctx_device_buffer(c1.fc, 0, LURK_FOLD_BUF_E1, &e1, &b) != LURK_OK ||
        lurk_fold_ctx_device_buffer(c2.fc, 0, LURK_FOLD_BUF_Z1, &z2, &b) != LURK_OK || lurk_fold_ctx_device_buffer(c2.fc, 0, LURK_FOLD_BUF_E1, &e2, &b) != LURK_OK)
        return fail(7, "device buffers");
    const void *zs[1] = {z1}, *es[1] = {e1};
    const uint8_t *cw[1] = {c1.res.running_comm_W}, *ce[1] = {c1.res.running_comm_E};
    /* the proof, every field the verifier reads */
    static uint8_t outer[2][LOGN * 4 * 32], claims[2][4 * 32], inner[2][(LOGN + 1) * 3 * 32], ew[2][32], red[2][LOGN * 3 * 32], left[2][2 * 32];
    static uint8_t com[(LOGN - 1) * 96], w[3 * 96], v[3 * LOGN * 32], L[LOGN * 96], R[LOGN * 96], af[32];
    lurk_compress_circuit_proof *cp[2] = {&proof.primary, &proof.secondary};
    for (j = 0; j < 2; j++) {
        cp[j]->snark.outer_rounds = outer[j]; cp[j]->snark.claims = claims[j]; cp[j]->snark.inner_rounds = inner[j]; cp[j]->snark.eval_W = ew[j];
        cp[j]->snark.reduce_rounds = red[j]; cp[j]->snark.claims_left = left[j];
    }
    proof.primary.com = com; proof.primary.w = w; proof.primary.v = v;
    proof.secondary.L = L; proof.secondary.R = R; proof.secondary.a_final = af;
    if (lurk_compress_prove_dev(cc, 1, zs, es, cw, ce, z2, e2, c2.res.running_comm_W, c2.res.running_comm_E, challenge, &vu.t, 0, &proof,
                                LURK_FMT_CANONICAL, NULL) != LURK_OK)
        return fail(8, "prove");
    transcript prover = vu.t;
    /* the instances: u and X of each running instance */
    uint8_t u1[32], x1[NX * 32], u2[32], x2[NX * 32];
    if (lurk_fold_ctx_get_running(c1.fc, NULL, NULL, u1, x1, NULL, NULL, LURK_FMT_CANONICAL) != LURK_OK ||
        lurk_fold_ctx_get_running(c2.fc, NULL, NULL, u2, x2, NULL, NULL, LURK_FMT_CANONICAL) != LURK_OK)
        return fail(9, "running instances");
    const uint8_t *xs[1] = {x1};
    lurk_compress_vk_pcs v1 = {LURK_PCS_HYPERKZG, NULL, NULL, NULL}, v2 = {LURK_PCS_IPA, c2.ck, ck_c, NULL};
    uint8_t g[64];
    memset(g, 0, 64);
    g[0] = 1; g[32] = 2;
    v1.g = g;
    int run;
    for (run = 0; run < 2; run++) {       /* concurrent, then sequential */
        memset(&vu.t, 0, sizeof vu.t);
        vu.t.fail_circuit = -1;
        ps.calls = 0;
        accepted = -1;
        if (lurk_compress_verify(1, &sp1, sp2, &v1, &v2, u1, xs, cw, ce, u2, x2, c2.res.running_comm_W, c2.res.running_comm_E, &proof,
                                 LURK_SPARTAN_ROUNDS_EVALS, challenge, pairing, &vu, run ? LURK_COMPRESS_SEQUENTIAL : 0, out, &accepted, LURK_FMT_CANONICAL, NULL) != LURK_OK)
            return fail(10, "verify");
        if (accepted != 1 || ps.calls != 1) return fail(11, "the good proof is not accepted");
        for (j = 0; j < 2; j++)
            if (out[j].snark_ok != 1 || out[j].eval_ok != 1 || out[j].opening_ok != 1) return fail(11, "a verdict of the good proof");
        if (memcmp(prover.calls, vu.t.calls, sizeof prover.calls)) return fail(12, "the verifier's transcript shape differs from the prover's");
    }
    /* a tampered a_final: the secondary's closing check alone fails */
    af[0] ^= 1;
    memset(&vu.t, 0, sizeof vu.t);
    vu.t.fail_circuit = -1;
    if (lurk_compress_verify(1, &sp1, sp2, &v1, &v2, u1, xs, cw, ce, u2, x2, c2.res.running_comm_W, c2.res.running_comm_E, &proof,
                             LURK_SPARTAN_ROUNDS_EVALS, challenge, pairing, &vu, 0, out, &accepted, LURK_FMT_CANONICAL, NULL) != LURK_OK || accepted != 0 ||
        out[0].opening_ok != 1 || out[1].snark_ok != 1 || out[1].eval_ok != 1 || out[1].opening_ok != 0)
        return fail(13, "tampered a_final");
    af[0] ^= 1;
    /* a pairing callback that fails: an error naming the primary circuit */
    ps.fail = 1;
    if (lurk_compress_verify(1, &sp1, sp2, &v1, &v2, u1, xs, cw, ce, u2, x2, c2.res.running_comm_W, c2.res.running_comm_E, &proof,
                             LURK_SPARTAN_ROUNDS_EVALS, challenge, pairing, &vu, 0, out, &accepted, LURK_FMT_CANONICAL, NULL) != LURK_ERR_ARG ||
        !strstr(lurk_last_error(), "primary"))
        return fail(14, "failing pairing callback");
    ps.fail = 0;
    /* HyperKZG without a pairing callback is refused before any callback */
    memset(&vu.t, 0, sizeof vu.t);
    vu.t.fail_circuit = -1;
    if (lurk_compress_verify(1, &sp1, sp2, &v1, &v2, u1, xs, cw, ce, u2, x2, c2.res.running_comm_W, c2.res.running_comm_E, &proof,
                             LURK_SPARTAN_ROUNDS_EVALS, challenge, NULL, &vu, 0, out, &accepted, LURK_FMT_CANONICAL, NULL) != LURK_ERR_ARG ||
        vu.t.calls[0][LURK_SPARTAN_TAU] != 0)
        return fail(15, "HyperKZG without a pairing callback");
    lurk_compress_ctx_destroy(cc);
    lurk_fold_ctx_destroy(c1.fc);
    lurk_fold_ctx_destroy(c2.fc);
    lurk_msm_ctx_destroy(c1.ck);
    lurk_msm_ctx_destroy(c2.ck);
    lurk_spartan_ctx_destroy(sp1);
    lurk_spartan_ctx_destroy(sp2);
    puts("compress_verify_client ok");
    return 0;
}
