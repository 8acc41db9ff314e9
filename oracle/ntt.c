/*
 * ORACLE (test infrastructure, not product code): radix-2 NTT and coset low-degree extension.
 * Restates the published two-adic coset LDE used by Plonky3's TwoAdicFriPcs::commit
 * (coset_lde_batch then bit_reverse_rows; SURVEY.md App. C.1).  The reference tree has no source for
 * this stage (SURVEY.md §8 a6) => parity unpinned; self-checked against the O(n^2) DFT below.
 */
#include "oracle.h"
#include "bb31.h"
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

int orc_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

void orc_dft_naive(const uint32_t* in, uint32_t* out, unsigned log_n, uint32_t shift) {
    size_t n = (size_t)1 << log_n;
    uint32_t w = bb_root_of_unity(log_n);
    for (size_t k = 0; k < n; k++) {
        uint32_t x = bb_mul(shift, bb_pow(w, k)), acc = 0, xp = 1;
        for (size_t i = 0; i < n; i++) { acc = bb_add(acc, bb_mul(in[i], xp)); xp = bb_mul(xp, x); }
        out[k] = acc;
    }
}

static void bit_reverse_inplace(uint32_t* a, unsigned log_n) {
    size_t n = (size_t)1 << log_n;
    for (size_t i = 0; i < n; i++) { size_t j = bitrev32((uint32_t)i, log_n); if (i < j) { uint32_t t = a[i]; a[i] = a[j]; a[j] = t; } }
}

/* textbook iterative Cooley-Tukey: bit-reverse, then spans 1,2,4,... with twiddle w_{2s}^j */
static void ntt_core(uint32_t* a, unsigned log_n, uint32_t root) {
    size_t n = (size_t)1 << log_n;
    bit_reverse_inplace(a, log_n);
    for (unsigned s = 0; s < log_n; s++) {
        size_t half = (size_t)1 << s;
        uint32_t wm = bb_pow(root, n >> (s + 1));
        for (size_t blk = 0; blk < n; blk += 2 * half) {
            uint32_t w = 1;
            for (size_t j = 0; j < half; j++) {
                uint32_t u = a[blk + j], v = bb_mul(a[blk + j + half], w);
                a[blk + j] = bb_add(u, v);
                a[blk + j + half] = bb_sub(u, v);
                w = bb_mul(w, wm);
            }
        }
    }
}

void orc_ntt(uint32_t* a, unsigned log_n) { ntt_core(a, log_n, bb_root_of_unity(log_n)); }

void orc_intt(uint32_t* a, unsigned log_n) {
    size_t n = (size_t)1 << log_n;
    ntt_core(a, log_n, bb_inv(bb_root_of_unity(log_n)));
    uint32_t ninv = bb_inv((uint32_t)(n % BB_P));
    for (size_t i = 0; i < n; i++) a[i] = bb_mul(a[i], ninv);
}

void orc_lde_batch(const uint32_t* trace, unsigned log_n, size_t width, unsigned log_blowup, uint32_t shift, uint32_t* lde) {
    size_t n = (size_t)1 << log_n, m = n << log_blowup;
    unsigned log_m = log_n + log_blowup;
#pragma omp parallel
    {
        uint32_t* buf = (uint32_t*)malloc(m * sizeof(uint32_t));
#pragma omp for schedule(dynamic, 1)
        for (long c = 0; c < (long)width; c++) {
            memcpy(buf, trace + (size_t)c * n, n * sizeof(uint32_t));
            orc_intt(buf, log_n);                        /* coefficients */
            uint32_t sp = 1;
            for (size_t i = 0; i < n; i++) { buf[i] = bb_mul(buf[i], sp); sp = bb_mul(sp, shift); }   /* f(shift*x) */
            memset(buf + n, 0, (m - n) * sizeof(uint32_t));
            orc_ntt(buf, log_m);                          /* natural-order evals on shift*H' */
            uint32_t* out = lde + (size_t)c * m;
            for (size_t i = 0; i < m; i++) out[bitrev32((uint32_t)i, log_m)] = buf[i];   /* bit_reverse_rows */
        }
        free(buf);
    }
}

/* out[j] = (lo+hi)/2 + beta*(lo-hi)/(2 x_j), x_j = shift * w_len^{bitrev(j)}  (SURVEY.md App. C.5) */
void orc_fri_fold(const uint32_t* in, unsigned log_len, uint32_t shift, const uint32_t beta[4], uint32_t* out) {
    size_t half = (size_t)1 << (log_len - 1);
    uint32_t w = bb_root_of_unity(log_len);
    uint32_t two_inv = bb_inv(2);
    bb4_t b = {{beta[0], beta[1], beta[2], beta[3]}};
#pragma omp parallel for schedule(static) if (half >= 4096)
    for (long j = 0; j < (long)half; j++) {
        bb4_t lo, hi;
        memcpy(lo.c, in + 8 * (size_t)j, 16);
        memcpy(hi.c, in + 8 * (size_t)j + 4, 16);
        uint32_t x = bb_mul(shift, bb_pow(w, bitrev32((uint32_t)j, log_len - 1)));
        uint32_t hx = bb_mul(two_inv, bb_inv(x));
        bb4_t s = bb4_scale(bb4_add(lo, hi), two_inv);
        bb4_t d = bb4_scale(bb4_sub(lo, hi), hx);
        bb4_t r = bb4_add(s, bb4_mul(b, d));
        memcpy(out + 4 * (size_t)j, r.c, 16);
    }
}

/* ---- openings (SURVEY.md §8f-4, widened in round 1): f(zeta) for columns given as evaluations over shift*H (natural order).
   Restated independently of the GPU's barycentric formula: interpolate (iNTT of g(y) = f(shift*y)), then Horner at zeta/shift
   in the extension field.  out: [width][4]. */
void orc_eval_at_point(const uint32_t* mat, unsigned log_n, size_t width, uint32_t shift, const uint32_t zeta[4], uint32_t* out) {
    size_t n = (size_t)1 << log_n;
    bb4_t z = {{zeta[0], zeta[1], zeta[2], zeta[3]}};
    bb4_t zs = bb4_scale(z, bb_inv(shift));
#pragma omp parallel
    {
        uint32_t* buf = (uint32_t*)malloc(n * sizeof(uint32_t));
#pragma omp for schedule(dynamic, 1)
        for (long c = 0; c < (long)width; c++) {
            memcpy(buf, mat + (size_t)c * n, n * sizeof(uint32_t));
            orc_intt(buf, log_n);
            bb4_t acc = bb4_from_base(0);
            for (size_t i = n; i-- > 0;) {
                acc = bb4_mul(acc, zs);
                acc.c[0] = bb_add(acc.c[0], buf[i]);
            }
            memcpy(out + 4 * (size_t)c, acc.c, 16);
        }
        free(buf);
    }
}

/* reduced opening at one point over the LDE domain shift*H' (bit-reversed rows):
   ro[r] = ( sum_j gamma^j * (f_j[r] - y_j) ) / (x_r - zeta),   x_r = shift * w_m^{bitrev(r)},  j runs over all columns of all
   matrices in order.  mats: column-major, height m = 2^log_m.  ys: [total_width][4].  out: [m][4].
   Returns -1, and writes nothing, when zeta lies on shift*H' (x_r - zeta has no inverse at one row). */
int orc_deep_quotient(const uint32_t* const* mats, const size_t* widths, size_t n_mats, unsigned log_m, uint32_t shift,
                      const uint32_t zeta[4], const uint32_t gamma[4], const uint32_t* ys, uint32_t* out) {
    if (bb4_in_coset(zeta, shift, log_m)) return -1;
    size_t m = (size_t)1 << log_m, total = 0;
    for (size_t i = 0; i < n_mats; i++) total += widths[i];
    bb4_t g = {{gamma[0], gamma[1], gamma[2], gamma[3]}}, z = {{zeta[0], zeta[1], zeta[2], zeta[3]}};
    bb4_t* gp = (bb4_t*)malloc(total * sizeof(bb4_t));
    bb4_t cur = bb4_from_base(1), ysum = bb4_from_base(0);
    for (size_t j = 0; j < total; j++) {
        gp[j] = cur;
        bb4_t y;
        memcpy(y.c, ys + 4 * j, 16);
        ysum = bb4_add(ysum, bb4_mul(cur, y));
        cur = bb4_mul(cur, g);
    }
    uint32_t w = bb_root_of_unity(log_m);
#pragma omp parallel for schedule(static)
    for (long r = 0; r < (long)m; r++) {
        bb4_t acc = bb4_from_base(0);
        size_t j = 0;
        for (size_t i = 0; i < n_mats; i++)
            for (size_t c = 0; c < widths[i]; c++, j++) acc = bb4_add(acc, bb4_scale(gp[j], mats[i][c * m + (size_t)r]));
        acc = bb4_sub(acc, ysum);
        uint32_t x = bb_mul(shift, bb_pow(w, bitrev32((uint32_t)r, log_m)));
        bb4_t d = bb4_from_base(x);
        d = bb4_sub(d, z);
        bb4_t v = bb4_mul(acc, bb4_inv(d));
        memcpy(out + 4 * (size_t)r, v.c, 16);
    }
    free(gp);
    return 0;
}

/* reduced opening over several (column group, point) pairs:
   ro[r] = sum_g ( sum_{j in g} gamma_j * (f_j[r] - y_j) ) / (x_r - z_g),  gamma_j = the column's power of the batching challenge.
   cols[j]: one column of height 2^log_m (bit-reversed rows over shift*H'); gamma_pows, ys: [n_cols][4]; zs: [n_groups][4]; out [m][4]. */
void orc_deep_quotient_groups(const uint32_t* const* cols, const uint32_t* group_of_col, size_t n_cols, const uint32_t* zs, size_t n_groups,
                              unsigned log_m, uint32_t shift, const uint32_t* gamma_pows, const uint32_t* ys, uint32_t* out) {
    const size_t m = (size_t)1 << log_m;
    bb4_t* gp = (bb4_t*)malloc((n_cols ? n_cols : 1) * sizeof(bb4_t));
    bb4_t* ysum = (bb4_t*)calloc(n_groups, sizeof(bb4_t));
    for (size_t j = 0; j < n_cols; j++) {
        bb4_t y;
        memcpy(gp[j].c, gamma_pows + 4 * j, 16);
        memcpy(y.c, ys + 4 * j, 16);
        ysum[group_of_col[j]] = bb4_add(ysum[group_of_col[j]], bb4_mul(gp[j], y));
    }
    const uint32_t w = bb_root_of_unity(log_m);
#pragma omp parallel for schedule(static)
    for (long r = 0; r < (long)m; r++) {
        const uint32_t x = bb_mul(shift, bb_pow(w, bitrev32((uint32_t)r, log_m)));
        bb4_t total = bb4_from_base(0);
        for (size_t q = 0; q < n_groups; q++) {
            bb4_t acc = bb4_from_base(0);
            for (size_t j = 0; j < n_cols; j++)
                if (group_of_col[j] == q) acc = bb4_add(acc, bb4_scale(gp[j], cols[j][(size_t)r]));
            acc = bb4_sub(acc, ysum[q]);
            bb4_t d = bb4_from_base(x), z;
            memcpy(z.c, zs + 4 * q, 16);
            d = bb4_sub(d, z);
            total = bb4_add(total, bb4_mul(acc, bb4_inv(d)));
        }
        memcpy(out + 4 * (size_t)r, total.c, 16);
    }
    free(gp); free(ysum);
}
