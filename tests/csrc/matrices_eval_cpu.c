/*
 * Test infrastructure, NOT product code: an OpenMP port of oracle/spartan.py: matrices_eval -- the multilinear extensions of the R1CS
 * matrices A, B, C at (r_x, r_y) that Spartan's RelaxedR1CSSNARK::verify evaluates itself:
 *     M(r_x, r_y) = sum_{row, col} eq(r_x, row) M[row][col] eq(r_y, col'),   col' = col < n_w ? col : num_vars + (col - n_w)
 * (the column in the padded z = (W | 0.. | u | X | 0..)), r[0] <-> the top index bit.  Full eq tables, then the rows split over the threads,
 * each with its own three sums.  It is the full-size checker of the GPU kernel (the Python loop is too slow at 5 M non-zeros) and the CPU
 * baseline timed beside it.  Self-contained: the modulus comes from the caller; 4 x 64-bit Montgomery arithmetic with unsigned __int128.
 * Built by tests/matrices_eval_cpu.py into a temporary directory.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef unsigned __int128 u128;
typedef struct { uint64_t l[4]; } fe;
typedef struct { uint64_t p[4], inv; fe one, r2; } field;

static int ge(const uint64_t *a, const uint64_t *b) {
    for (int i = 3; i >= 0; i--)
        if (a[i] != b[i]) return a[i] > b[i];
    return 1;
}
static uint64_t sub_n(uint64_t *r, const uint64_t *a, const uint64_t *b) {
    uint64_t borrow = 0;
    for (int i = 0; i < 4; i++) { u128 d = (u128)a[i] - b[i] - borrow; r[i] = (uint64_t)d; borrow = (uint64_t)(d >> 64) & 1; }
    return borrow;
}
static uint64_t add_n(uint64_t *r, const uint64_t *a, const uint64_t *b) {
    uint64_t c = 0;
    for (int i = 0; i < 4; i++) { u128 s = (u128)a[i] + b[i] + c; r[i] = (uint64_t)s; c = (uint64_t)(s >> 64); }
    return c;
}
static void f_add(const field *f, fe *r, const fe *a, const fe *b) {
    uint64_t c = add_n(r->l, a->l, b->l);
    if (c || ge(r->l, f->p)) sub_n(r->l, r->l, f->p);
}
static void f_sub(const field *f, fe *r, const fe *a, const fe *b) {
    if (sub_n(r->l, a->l, b->l)) add_n(r->l, r->l, f->p);
}
static void f_mul(const field *f, fe *r, const fe *a, const fe *b) {
    uint64_t t[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 4; i++) {
        uint64_t c = 0;
        for (int j = 0; j < 4; j++) { u128 s = (u128)a->l[j] * b->l[i] + t[j] + c; t[j] = (uint64_t)s; c = (uint64_t)(s >> 64); }
        u128 s = (u128)t[4] + c; t[4] = (uint64_t)s; t[5] = (uint64_t)(s >> 64);
        const uint64_t m = t[0] * f->inv;
        s = (u128)m * f->p[0] + t[0]; c = (uint64_t)(s >> 64);
        for (int j = 1; j < 4; j++) { s = (u128)m * f->p[j] + t[j] + c; t[j - 1] = (uint64_t)s; c = (uint64_t)(s >> 64); }
        s = (u128)t[4] + c; t[3] = (uint64_t)s; t[4] = t[5] + (uint64_t)(s >> 64);
    }
    if (t[4] || ge(t, f->p)) sub_n(r->l, t, f->p); else memcpy(r->l, t, 32);
}
static void field_init(field *f, const uint8_t p_le[32]) {
    memcpy(f->p, p_le, 32);
    uint64_t inv = 1;
    for (int i = 0; i < 6; i++) inv *= 2 - f->p[0] * inv;     /* Newton: p^-1 mod 2^64 */
    f->inv = 0 - inv;
    uint64_t x[4] = {1, 0, 0, 0};                              /* R = 2^256 and R^2 mod p by doublings of 1 */
    for (int i = 0; i < 512; i++) {
        const uint64_t c = add_n(x, x, x);
        if (c || ge(x, f->p)) sub_n(x, x, f->p);
        if (i == 255) memcpy(f->one.l, x, 32);
    }
    memcpy(f->r2.l, x, 32);
}
static int load(const field *f, fe *r, const uint8_t *in) {     /* canonical bytes -> Montgomery; 0 when not reduced */
    fe t;
    memcpy(t.l, in, 32);
    if (ge(t.l, f->p)) return 0;
    f_mul(f, r, &t, &f->r2);
    return 1;
}

/* EqPolynomial::evals: 2^l entries, r[0] <-> the top bit, level by level between two buffers */
static fe *eq_table(const field *f, const fe *r, int l) {
    fe *t = (fe *)malloc(sizeof(fe) << l), *u = (fe *)malloc(sizeof(fe) << l);
    if (!t || !u) { free(t); free(u); return NULL; }
    t[0] = f->one;
    for (int j = 0; j < l; j++) {
        const long half = 1L << j;
#pragma omp parallel for schedule(static)
        for (long i = 0; i < half; i++) {
            fe hi, lo;
            f_mul(f, &hi, &t[i], &r[j]);
            f_sub(f, &lo, &t[i], &hi);
            u[2 * i] = lo;
            u[2 * i + 1] = hi;
        }
        fe *s = t; t = u; u = s;
    }
    free(u);
    return t;
}

/* out = A | B | C canonical (3 x 32 bytes).  Returns 0, -1 for a value >= p, -2 when out of memory. */
int matrices_eval_cpu(const uint8_t p_le[32], uint64_t rows, uint64_t n_w, uint64_t num_vars, const uint64_t *const rp[3],
                      const uint32_t *const col[3], const uint8_t *const val[3], const uint8_t *rx, int log_rows, const uint8_t *ry, int log_y,
                      uint8_t out[96], int nthreads) {
    field f;
    field_init(&f, p_le);
#ifdef _OPENMP
    if (nthreads > 0) omp_set_num_threads(nthreads);
#else
    (void)nthreads;
#endif
    fe x[64], y[64];
    for (int j = 0; j < log_rows; j++) if (!load(&f, &x[j], rx + 32 * j)) return -1;
    for (int j = 0; j < log_y; j++) if (!load(&f, &y[j], ry + 32 * j)) return -1;
    fe *ex = eq_table(&f, x, log_rows), *ey = eq_table(&f, y, log_y);
    if (!ex || !ey) { free(ex); free(ey); return -2; }
    int bad = 0;
    for (int m = 0; m < 3; m++) {
        fe total = {{0, 0, 0, 0}};
#pragma omp parallel
        {
            fe acc = {{0, 0, 0, 0}};
#pragma omp for schedule(dynamic, 4096)
            for (long i = 0; i < (long)rows; i++) {
                fe row = {{0, 0, 0, 0}};
                for (uint64_t k = rp[m][i]; k < rp[m][i + 1]; k++) {
                    fe v, t;
                    if (!load(&f, &v, val[m] + 32 * k)) { bad = 1; continue; }
                    const uint64_t c = col[m][k];
                    f_mul(&f, &t, &v, &ey[c < n_w ? c : num_vars + (c - n_w)]);
                    f_add(&f, &row, &row, &t);
                }
                fe t;
                f_mul(&f, &t, &row, &ex[i]);
                f_add(&f, &acc, &acc, &t);
            }
#pragma omp critical
            f_add(&f, &total, &total, &acc);
        }
        const fe one_raw = {{1, 0, 0, 0}};
        fe canon;
        f_mul(&f, &canon, &total, &one_raw);
        memcpy(out + 32 * m, canon.l, 32);
    }
    free(ex);
    free(ey);
    return bad ? -1 : 0;
}

int matrices_eval_cpu_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
