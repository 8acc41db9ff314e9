/*
 * ORACLE (test infrastructure, not product code).  CPU restatement of BabyBear field
 * arithmetic in CANONICAL form (values in [0,p)), deliberately implemented with plain
 * 64-bit `%` so it shares no reduction trick with the CUDA path (which is Montgomery).
 *
 * Pins from the reference tree:
 *   p = 2013265921: /root/reference/number/src/baby_bear.rs:46-55  ((p-1)/2 = 0x3c000000)
 *   canonical-u32 serialisation: /root/reference/number/src/plonky3_macros.rs:38-59
 *   from(i64 < 0) = p + n:      /root/reference/number/src/plonky3_macros.rs:156-170
 * Extension field F_p[x]/(x^4 - 11) is the Plonky3 BabyBear binomial extension
 * (SURVEY.md App. B/C; not present in the reference tree => parity unpinned for Ext4).
 */
#ifndef PB_ORACLE_BB31_H
#define PB_ORACLE_BB31_H
#include <stdint.h>
#include <stddef.h>

#define BB_P 2013265921u
#define BB_GENERATOR 31u          /* multiplicative generator of F_p^* */
#define BB_TWO_ADICITY 27
#define BB_EXT_W 11u              /* x^4 = 11 */

static inline uint32_t bb_add(uint32_t a, uint32_t b) { uint32_t s = a + b; return s >= BB_P ? s - BB_P : s; }
static inline uint32_t bb_sub(uint32_t a, uint32_t b) { return a >= b ? a - b : a + BB_P - b; }
static inline uint32_t bb_neg(uint32_t a) { return a ? BB_P - a : 0; }
static inline uint32_t bb_mul(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) % BB_P); }
static inline uint32_t bb_pow(uint32_t a, uint64_t e) {
    uint32_t r = 1;
    while (e) { if (e & 1) r = bb_mul(r, a); a = bb_mul(a, a); e >>= 1; }
    return r;
}
static inline uint32_t bb_inv(uint32_t a) { return bb_pow(a, BB_P - 2); }   /* inv(0) = 0 */
static inline uint32_t bb_from_i64(int64_t v) { int64_t m = v % (int64_t)BB_P; return (uint32_t)(m < 0 ? m + BB_P : m); }
/* primitive 2^k-th root of unity: g^((p-1)/2^k) */
static inline uint32_t bb_root_of_unity(unsigned log_n) { return bb_pow(BB_GENERATOR, (uint64_t)(BB_P - 1) >> log_n); }

static inline uint32_t bitrev32(uint32_t x, unsigned bits) {
    uint32_t r = 0;
    for (unsigned i = 0; i < bits; i++) { r = (r << 1) | ((x >> i) & 1); }
    return r;
}

/* ---- degree-4 binomial extension, basis (1, x, x^2, x^3), x^4 = 11 ---- */
typedef struct { uint32_t c[4]; } bb4_t;

static inline bb4_t bb4_from_base(uint32_t a) { bb4_t r = {{a, 0, 0, 0}}; return r; }
static inline bb4_t bb4_add(bb4_t a, bb4_t b) { bb4_t r; for (int i = 0; i < 4; i++) r.c[i] = bb_add(a.c[i], b.c[i]); return r; }
static inline bb4_t bb4_sub(bb4_t a, bb4_t b) { bb4_t r; for (int i = 0; i < 4; i++) r.c[i] = bb_sub(a.c[i], b.c[i]); return r; }
static inline bb4_t bb4_scale(bb4_t a, uint32_t s) { bb4_t r; for (int i = 0; i < 4; i++) r.c[i] = bb_mul(a.c[i], s); return r; }
static inline bb4_t bb4_mul(bb4_t a, bb4_t b) {
    uint32_t t[7] = {0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) t[i + j] = bb_add(t[i + j], bb_mul(a.c[i], b.c[j]));
    bb4_t r;
    for (int i = 0; i < 4; i++) r.c[i] = t[i];
    for (int i = 4; i < 7; i++) r.c[i - 4] = bb_add(r.c[i - 4], bb_mul(t[i], BB_EXT_W));
    return r;
}
static inline bb4_t bb4_pow(bb4_t a, uint64_t e) {
    bb4_t r = bb4_from_base(1);
    while (e) { if (e & 1) r = bb4_mul(r, a); a = bb4_mul(a, a); e >>= 1; }
    return r;
}
/* inverse through the norm to the quadratic subfield then to the base field */
static inline bb4_t bb4_inv(bb4_t a) {
    /* a = A + x B with A = a0 + a2 y, B = a1 + a3 y over y = x^2, y^2 = 11.
       a * conj = A^2 - y B^2 in F_p[y]; then invert there via its norm. */
    uint32_t a0 = a.c[0], a1 = a.c[1], a2 = a.c[2], a3 = a.c[3];
    /* A^2 = (a0^2 + 11 a2^2) + (2 a0 a2) y ;  B^2 = (a1^2 + 11 a3^2) + (2 a1 a3) y ; y*B^2 = 11*(2 a1 a3) + (a1^2 + 11 a3^2) y */
    uint32_t A0 = bb_add(bb_mul(a0, a0), bb_mul(BB_EXT_W, bb_mul(a2, a2)));
    uint32_t A1 = bb_mul(2, bb_mul(a0, a2));
    uint32_t B0 = bb_add(bb_mul(a1, a1), bb_mul(BB_EXT_W, bb_mul(a3, a3)));
    uint32_t B1 = bb_mul(2, bb_mul(a1, a3));
    uint32_t n0 = bb_sub(A0, bb_mul(BB_EXT_W, B1));   /* norm to F_p[y]: n0 + n1 y */
    uint32_t n1 = bb_sub(A1, B0);
    /* (n0 + n1 y)^-1 = (n0 - n1 y) / (n0^2 - 11 n1^2) */
    uint32_t d = bb_inv(bb_sub(bb_mul(n0, n0), bb_mul(BB_EXT_W, bb_mul(n1, n1))));
    uint32_t i0 = bb_mul(n0, d), i1 = bb_neg(bb_mul(n1, d));
    /* a^-1 = conj(a) * (i0 + i1 y), conj(a) = A - x B = (a0, -a1, a2, -a3) */
    bb4_t conj = {{a0, bb_neg(a1), a2, bb_neg(a3)}};
    bb4_t s = {{i0, 0, i1, 0}};
    return bb4_mul(conj, s);
}
/* z lies on shift*H, |H| = 2^log_n: a base-field point with (z/shift)^(2^log_n) = 1 (canonical limbs) */
static inline int bb4_in_coset(const uint32_t z[4], uint32_t shift, unsigned log_n) {
    if (z[1] | z[2] | z[3]) return 0;
    uint32_t y = bb_mul(z[0], bb_inv(shift));
    for (unsigned i = 0; i < log_n; i++) y = bb_mul(y, y);
    return y == 1;
}
#endif
