/*
 * ORACLE / CPU REFERENCE ARM (test infrastructure, not product code): AVX-512 Montgomery implementations of the heavy
 * primitives of the path -- coset LDE, Poseidon2 leaf hashing + Merkle layers, constraint fold / quotient, openings at a point,
 * reduced opening -- with EXACTLY the semantics (canonical u32 in, canonical u32 out, same layouts) of the scalar `%`-based
 * restatement in ntt.c / poseidon2.c / air.c, against which tests/test_oracle_fast.py checks every one of them bit for bit.
 *
 * Why it exists: bench.py's `cpu_baseline` / `--impl reference` arm times the CPU implementation of the path on the GPU
 * box's host cores.  The reference's own CPU prover (Plonky3 behind openvm-stark-backend, un-vendored: SURVEY.md §8c) runs
 * Montgomery arithmetic on packed AVX-512 lanes; timing the scalar `%` port instead made the baseline a strawman
 * (VERDICT r1, weak #4).  This file is the same algorithm at the arithmetic quality of that prover: 16 BabyBear lanes per
 * instruction, signed-free Montgomery product from 6 vpmuludq, one row (leaf hashing, constraints) or one butterfly column
 * position (NTT) per lane, OpenMP over columns / row blocks.
 *
 * Representation trick used throughout: montmul(x_canonical, c*R) = x*c canonical, so data that is only ever multiplied by
 * constants (twiddles, gamma powers, barycentric weights) stays canonical in memory and only the constants are kept in
 * Montgomery form; data*data products (S-box, constraint products) convert on load.
 */
#pragma GCC target("avx512f,avx512dq,avx512bw,avx512vl")
#include <immintrin.h>
#include <stdlib.h>
#include <string.h>
#include "oracle.h"
#include "bb31.h"
#include "../include/pb_poseidon2_constants.h"

#define P BB_P
#define MU 0x88000001u            /* p^-1 mod 2^32 */
#define R1 268435454u             /* 2^32 mod p */
#define R2 1172168163u            /* 2^64 mod p */

int orcf_available(void) { return __builtin_cpu_supports("avx512f") && __builtin_cpu_supports("avx512dq") && __builtin_cpu_supports("avx512bw"); }

/* ---------------- scalar Montgomery ---------------- */
static inline uint32_t m_mul(uint32_t a, uint32_t b) {          /* a*b/R mod p, result in [0,p) when a*b < 2^32 p */
    uint64_t t = (uint64_t)a * b;
    uint32_t q = (uint32_t)t * MU;
    int64_t d = (int64_t)(t >> 32) - (int64_t)(((uint64_t)q * P) >> 32);
    return (uint32_t)(d < 0 ? d + P : d);
}
static inline uint32_t to_m(uint32_t x) { return m_mul(x, R2); }
static inline uint32_t from_m(uint32_t x) { return m_mul(x, 1); }
static inline uint32_t s_add(uint32_t a, uint32_t b) { uint32_t s = a + b; return s >= P ? s - P : s; }
static inline uint32_t s_sub(uint32_t a, uint32_t b) { return a >= b ? a - b : a + P - b; }

/* ---------------- 16-lane Montgomery ---------------- */
typedef __m512i V;
#define VSET(x) _mm512_set1_epi32((int)(x))
static inline V v_add(V a, V b) { V s = _mm512_add_epi32(a, b); return _mm512_min_epu32(s, _mm512_sub_epi32(s, VSET(P))); }
static inline V v_sub(V a, V b) { V d = _mm512_sub_epi32(a, b); return _mm512_min_epu32(d, _mm512_add_epi32(d, VSET(P))); }
static inline V v_neg(V a) { return v_sub(_mm512_setzero_si512(), a); }
static inline V v_mul(V a, V b) {                                /* lane-wise a*b/R mod p in [0,p) */
    const V vp = VSET(P), vmu = VSET(MU);
    V ao = _mm512_srli_epi64(a, 32), bo = _mm512_srli_epi64(b, 32);
    V pe = _mm512_mul_epu32(a, b), po = _mm512_mul_epu32(ao, bo);
    V qe = _mm512_mul_epu32(pe, vmu), qo = _mm512_mul_epu32(po, vmu);
    V qpe = _mm512_mul_epu32(qe, vp), qpo = _mm512_mul_epu32(qo, vp);
    V hp = _mm512_mask_blend_epi32(0xAAAA, _mm512_srli_epi64(pe, 32), po);
    V hq = _mm512_mask_blend_epi32(0xAAAA, _mm512_srli_epi64(qpe, 32), qpo);
    V d = _mm512_sub_epi32(hp, hq);
    return _mm512_min_epu32(d, _mm512_add_epi32(d, vp));
}
static inline V v_halve(V x) {                                    /* x/2 mod p on canonical-range values (any representation) */
    __mmask16 odd = _mm512_test_epi32_mask(x, VSET(1));
    return _mm512_mask_add_epi32(_mm512_srli_epi32(x, 1), odd, _mm512_srli_epi32(x, 1), VSET((P + 1) / 2));
}

/* =====================================================================================================================
 * stage 1: coset LDE.  Per column: bit-reverse gather -> DIT inverse (natural coefficients * N) -> scale by shift^k / N ->
 * zero pad -> DIF forward of size 2^log_m, whose output slot p holds evaluation bitrev(p): the committed bit-reversed order. */
typedef struct { unsigned log_n; int inverse; uint32_t* tw; } twset_t;      /* tw[2^u + k] = (w_{2^(u+1)}^{+-k}) * R */

static uint32_t* make_twiddles(unsigned log_n, int inverse) {
    size_t n = (size_t)1 << log_n;
    uint32_t* tw = (uint32_t*)aligned_alloc(64, (n < 16 ? 16 : n) * sizeof(uint32_t));
    tw[0] = 0;
    for (unsigned u = 0; u < log_n; u++) {
        uint32_t w = bb_root_of_unity(u + 1);
        if (inverse) w = bb_inv(w);
        uint32_t wm = to_m(w), x = R1;
        for (size_t k = 0; k < ((size_t)1 << u); k++) { tw[((size_t)1 << u) + k] = x; x = m_mul(x, wm); }
    }
    return tw;
}

/* one radix-2 stage with half >= 16 */
static inline void stage_big(uint32_t* a, size_t n, size_t half, const uint32_t* tw, int dif) {
    for (size_t blk = 0; blk < n; blk += 2 * half)
        for (size_t j = 0; j < half; j += 16) {
            V u = _mm512_loadu_si512(a + blk + j), v = _mm512_loadu_si512(a + blk + j + half), w = _mm512_loadu_si512(tw + half + j);
            if (dif) {
                _mm512_storeu_si512(a + blk + j, v_add(u, v));
                _mm512_storeu_si512(a + blk + j + half, v_mul(v_sub(u, v), w));
            } else {
                V t = v_mul(v, w);
                _mm512_storeu_si512(a + blk + j, v_add(u, t));
                _mm512_storeu_si512(a + blk + j + half, v_sub(u, t));
            }
        }
}
/* stages with half in {8,4,2,1} on every 16-lane vector: partner through a lane permutation */
static inline void stage_small(uint32_t* a, size_t n, unsigned half, const uint32_t* tw, int dif) {
    uint32_t idx[16], wv[16];
    __mmask16 hi = 0;
    for (unsigned l = 0; l < 16; l++) {
        idx[l] = l ^ half;
        wv[l] = (l & half) ? tw[half + (l & (half - 1))] : R1;
        if (l & half) hi |= (__mmask16)(1u << l);
    }
    const V vi = _mm512_loadu_si512(idx), vw = _mm512_loadu_si512(wv);
    for (size_t i = 0; i < n; i += 16) {
        V x = _mm512_loadu_si512(a + i);
        if (dif) {
            V t = _mm512_permutexvar_epi32(vi, x);
            V r = _mm512_mask_blend_epi32(hi, v_add(x, t), v_mul(v_sub(t, x), vw));
            _mm512_storeu_si512(a + i, r);
        } else {
            V xm = _mm512_mask_blend_epi32(hi, x, v_mul(x, vw));
            V t = _mm512_permutexvar_epi32(vi, xm);
            _mm512_storeu_si512(a + i, _mm512_mask_blend_epi32(hi, v_add(xm, t), v_sub(t, xm)));
        }
    }
}
static void ntt_scalar_stage(uint32_t* a, size_t n, size_t half, const uint32_t* tw, int dif) {
    for (size_t blk = 0; blk < n; blk += 2 * half)
        for (size_t j = 0; j < half; j++) {
            uint32_t u = a[blk + j], v = a[blk + j + half];
            if (dif) { a[blk + j] = s_add(u, v); a[blk + j + half] = m_mul(s_sub(u, v), tw[half + j]); }
            else { uint32_t t = m_mul(v, tw[half + j]); a[blk + j] = s_add(u, t); a[blk + j + half] = s_sub(u, t); }
        }
}
/* DIT: bit-reversed in -> natural out.  DIF: natural in -> bit-reversed out.  Data canonical, twiddles Montgomery.
   Cache blocking: a radix-2 stage of span `half` splits the array into independent blocks of 2*half elements, so all stages
   with 2*half <= 2^BLK_LOG are run block by block (a block = 1 MB stays in L2) and only the few larger stages stream the
   whole column from memory: ~5 passes over a 2^21-point column instead of 21. */
#define BLK_LOG 18
static inline void one_stage(uint32_t* a, size_t n, size_t half, const uint32_t* tw, int dif) {
    if (n < 16) ntt_scalar_stage(a, n, half, tw, dif);
    else if (half < 16) stage_small(a, n, (unsigned)half, tw, dif);
    else stage_big(a, n, half, tw, dif);
}
static void ntt_dit(uint32_t* a, unsigned log_n, const uint32_t* tw) {
    const size_t n = (size_t)1 << log_n;
    const unsigned lb = log_n < BLK_LOG ? log_n : BLK_LOG;
    for (size_t b0 = 0; b0 < n; b0 += (size_t)1 << lb)
        for (unsigned s = 0; s < lb; s++) one_stage(a + b0, (size_t)1 << lb, (size_t)1 << s, tw, 0);
    for (unsigned s = lb; s < log_n; s++) one_stage(a, n, (size_t)1 << s, tw, 0);
}
static void ntt_dif(uint32_t* a, unsigned log_n, const uint32_t* tw) {
    const size_t n = (size_t)1 << log_n;
    const unsigned lb = log_n < BLK_LOG ? log_n : BLK_LOG;
    for (unsigned s = log_n; s-- > lb;) one_stage(a, n, (size_t)1 << s, tw, 1);
    for (size_t b0 = 0; b0 < n; b0 += (size_t)1 << lb)
        for (unsigned s = lb; s-- > 0;) one_stage(a + b0, (size_t)1 << lb, (size_t)1 << s, tw, 1);
}

/* dst[bitrev(i)] = src[i], cache-blocked: index = (a : 5 top bits, b : middle, c : 5 low bits) -> (rev c, rev b, rev a); for a fixed b
   the 32x32 tile {a, c} is read as 32 runs of 128 B and written as 32 runs of 128 B through a 4 KB buffer (a plain gather does one
   cache miss per element: ~100 ms per 2^20-point column) */
static void bitrev_copy(const uint32_t* src, uint32_t* dst, unsigned log_n, const uint32_t* rev_mid /* bitrev over log_n - 10 bits */) {
    if (log_n < 10) {
        for (size_t i = 0; i < ((size_t)1 << log_n); i++) dst[bitrev32((uint32_t)i, log_n)] = src[i];
        return;
    }
    static const uint8_t r5[32] = {0, 16, 8, 24, 4, 20, 12, 28, 2, 18, 10, 26, 6, 22, 14, 30, 1, 17, 9, 25, 5, 21, 13, 29, 3, 19, 11, 27, 7, 23, 15, 31};
    const unsigned mid = log_n - 10;
    uint32_t t[32][32];
    for (size_t b = 0; b < ((size_t)1 << mid); b++) {
        for (unsigned a = 0; a < 32; a++) {
            const uint32_t* p = src + ((size_t)a << (log_n - 5)) + (b << 5);
            for (unsigned c = 0; c < 32; c++) t[r5[c]][r5[a]] = p[c];
        }
        const size_t rb = rev_mid[b];
        for (unsigned rc = 0; rc < 32; rc++) memcpy(dst + ((size_t)rc << (log_n - 5)) + (rb << 5), t[rc], 128);
    }
}

void orcf_lde_batch(const uint32_t* trace, unsigned log_n, size_t width, unsigned log_blowup, uint32_t shift, uint32_t* lde) {
    const size_t n = (size_t)1 << log_n, m = n << log_blowup;
    const unsigned log_m = log_n + log_blowup;
    uint32_t* tw_inv = make_twiddles(log_n, 1);
    uint32_t* tw_fwd = make_twiddles(log_m, 0);
    /* scale[k] = shift^k / N in Montgomery form; rev[i] = bitrev_n(i) */
    uint32_t* scale = (uint32_t*)aligned_alloc(64, (n < 16 ? 16 : n) * sizeof(uint32_t));
    const unsigned mid = log_n >= 10 ? log_n - 10 : 0;
    uint32_t* rev = (uint32_t*)malloc(((size_t)1 << mid) * sizeof(uint32_t));
    {
        uint32_t sm = to_m(shift % P), x = to_m(bb_inv((uint32_t)(n % P)));
        for (size_t k = 0; k < n; k++) { scale[k] = x; x = m_mul(x, sm); }
        for (size_t i = 0; i < ((size_t)1 << mid); i++) rev[i] = bitrev32((uint32_t)i, mid);
    }
#pragma omp parallel
    {
        uint32_t* buf = (uint32_t*)aligned_alloc(64, (m < 16 ? 16 : m) * sizeof(uint32_t));
#pragma omp for schedule(dynamic, 1)
        for (long c = 0; c < (long)width; c++) {
            bitrev_copy(trace + (size_t)c * n, buf, log_n, rev);
            ntt_dit(buf, log_n, tw_inv);
            if (n >= 16)
                for (size_t k = 0; k < n; k += 16) _mm512_storeu_si512(buf + k, v_mul(_mm512_loadu_si512(buf + k), _mm512_loadu_si512(scale + k)));
            else
                for (size_t k = 0; k < n; k++) buf[k] = m_mul(buf[k], scale[k]);
            memset(buf + n, 0, (m - n) * sizeof(uint32_t));
            ntt_dif(buf, log_m, tw_fwd);
            memcpy(lde + (size_t)c * m, buf, m * sizeof(uint32_t));
        }
        free(buf);
    }
    free(tw_inv); free(tw_fwd); free(scale); free(rev);
}

/* =====================================================================================================================
 * stage 3a: Poseidon2 on 16 states at once (lane = row / node), Montgomery form inside the permutation. */
typedef struct {
    uint32_t rc_ext[8][16], rc_int[13], diag[16];      /* Montgomery */
} p2m_t;
static p2m_t g_p2;
static int g_p2_ready = 0;
static void p2_init(void) {
    if (g_p2_ready) return;
    for (int r = 0; r < 8; r++) for (int i = 0; i < 16; i++) g_p2.rc_ext[r][i] = to_m(PB_P2_RC_EXT[r][i]);
    for (int r = 0; r < 13; r++) g_p2.rc_int[r] = to_m(PB_P2_RC_INT[r]);
    for (int i = 0; i < 16; i++) g_p2.diag[i] = to_m(PB_P2_DIAG_M1[i]);
    g_p2_ready = 1;
}
static inline V v_sbox(V x) { V x2 = v_mul(x, x), x3 = v_mul(x2, x), x4 = v_mul(x2, x2); return v_mul(x3, x4); }
static inline void v_external(V s[16]) {
    for (int c = 0; c < 16; c += 4) {
        V x0 = s[c], x1 = s[c + 1], x2 = s[c + 2], x3 = s[c + 3];
        V t01 = v_add(x0, x1), t23 = v_add(x2, x3), t0123 = v_add(t01, t23);
        V t01123 = v_add(t0123, x1), t01233 = v_add(t0123, x3);
        s[c + 3] = v_add(t01233, v_add(x0, x0));      /* 3 x0 +   x1 +   x2 + 2 x3 */
        s[c + 1] = v_add(t01123, v_add(x2, x2));      /* x0 + 2 x1 + 3 x2 + x3 */
        s[c] = v_add(t01123, t01);                     /* 2 x0 + 3 x1 + x2 + x3 */
        s[c + 2] = v_add(t01233, t23);                 /* x0 + x1 + 2 x2 + 3 x3 */
    }
    V q[4];
    for (int i = 0; i < 4; i++) q[i] = v_add(v_add(s[i], s[4 + i]), v_add(s[8 + i], s[12 + i]));
    for (int i = 0; i < 16; i++) s[i] = v_add(s[i], q[i & 3]);
}
static inline void v_permute(V s[16]) {
    v_external(s);
    for (int r = 0; r < 4; r++) {
        for (int i = 0; i < 16; i++) s[i] = v_sbox(v_add(s[i], VSET(g_p2.rc_ext[r][i])));
        v_external(s);
    }
    for (int r = 0; r < 13; r++) {
        s[0] = v_sbox(v_add(s[0], VSET(g_p2.rc_int[r])));
        V a = v_add(v_add(s[0], s[1]), v_add(s[2], s[3])), b = v_add(v_add(s[4], s[5]), v_add(s[6], s[7]));
        V c = v_add(v_add(s[8], s[9]), v_add(s[10], s[11])), d = v_add(v_add(s[12], s[13]), v_add(s[14], s[15]));
        V sum = v_add(v_add(a, b), v_add(c, d));
        for (int i = 0; i < 16; i++) s[i] = v_add(sum, v_mul(s[i], VSET(g_p2.diag[i])));     /* (1 + diag(V)) s, generic in V */
    }
    for (int r = 4; r < 8; r++) {
        for (int i = 0; i < 16; i++) s[i] = v_sbox(v_add(s[i], VSET(g_p2.rc_ext[r][i])));
        v_external(s);
    }
}
/* NB independent permutations interleaved step by step: the 13 internal rounds are one serial S-box chain each (4 dependent
   products of ~20 cycles latency), which a single permutation cannot hide on an out-of-order core */
#define P2_NB 4
static inline __attribute__((always_inline)) void v_permute_nb(V s[P2_NB][16]) {
    for (int b = 0; b < P2_NB; b++) v_external(s[b]);
    for (int r = 0; r < 4; r++) {
        for (int i = 0; i < 16; i++) for (int b = 0; b < P2_NB; b++) s[b][i] = v_sbox(v_add(s[b][i], VSET(g_p2.rc_ext[r][i])));
        for (int b = 0; b < P2_NB; b++) v_external(s[b]);
    }
    for (int r = 0; r < 13; r++) {
        V x[P2_NB], x2[P2_NB], x3[P2_NB], x4[P2_NB];
        for (int b = 0; b < P2_NB; b++) x[b] = v_add(s[b][0], VSET(g_p2.rc_int[r]));
        for (int b = 0; b < P2_NB; b++) x2[b] = v_mul(x[b], x[b]);
        for (int b = 0; b < P2_NB; b++) x3[b] = v_mul(x2[b], x[b]);
        for (int b = 0; b < P2_NB; b++) x4[b] = v_mul(x2[b], x2[b]);
        for (int b = 0; b < P2_NB; b++) s[b][0] = v_mul(x3[b], x4[b]);
        for (int b = 0; b < P2_NB; b++) {
            V* t = s[b];
            V a = v_add(v_add(t[0], t[1]), v_add(t[2], t[3])), bb_ = v_add(v_add(t[4], t[5]), v_add(t[6], t[7]));
            V c = v_add(v_add(t[8], t[9]), v_add(t[10], t[11])), d = v_add(v_add(t[12], t[13]), v_add(t[14], t[15]));
            V sum = v_add(v_add(a, bb_), v_add(c, d));
            for (int i = 0; i < 16; i++) t[i] = v_add(sum, v_mul(t[i], VSET(g_p2.diag[i])));
        }
    }
    for (int r = 4; r < 8; r++) {
        for (int i = 0; i < 16; i++) for (int b = 0; b < P2_NB; b++) s[b][i] = v_sbox(v_add(s[b][i], VSET(g_p2.rc_ext[r][i])));
        for (int b = 0; b < P2_NB; b++) v_external(s[b]);
    }
}

void orcf_merkle_commit(const uint32_t* const* mats, const size_t* widths, size_t n_mats, unsigned log_h, uint32_t* layers) {
    const size_t h = (size_t)1 << log_h;
    if (h < 16) { orc_merkle_commit(mats, widths, n_mats, log_h, layers); return; }
    p2_init();
    size_t total_w = 0;
    for (size_t i = 0; i < n_mats; i++) total_w += widths[i];
    const uint32_t** cols = (const uint32_t**)malloc((total_w ? total_w : 1) * sizeof(*cols));
    {
        size_t k = 0;
        for (size_t i = 0; i < n_mats; i++) for (size_t c = 0; c < widths[i]; c++) cols[k++] = mats[i] + c * h;
    }
    const V vr2 = VSET(R2), one = VSET(1);
    if (h >= 16 * P2_NB) {
        /* 16*P2_NB rows per visit of a column group: P2_NB interleaved sponges, and P2_NB consecutive cache lines per column touched
           (a row block walks total_w columns that are megabytes apart: one TLB miss per column visit) */
#pragma omp parallel for schedule(static)
        for (long r0 = 0; r0 < (long)h; r0 += 16 * P2_NB) {
            V s[P2_NB][16];
            for (int b = 0; b < P2_NB; b++) for (int i = 0; i < 16; i++) s[b][i] = _mm512_setzero_si512();
            for (size_t c0 = 0; c0 < total_w; c0 += 8) {
                const size_t k = total_w - c0 < 8 ? total_w - c0 : 8;
                for (size_t j = 0; j < k; j++)
                    for (int b = 0; b < P2_NB; b++) s[b][j] = v_mul(_mm512_loadu_si512(cols[c0 + j] + r0 + 16 * b), vr2);     /* overwrite-mode absorb */
                v_permute_nb(s);
            }
            for (int b = 0; b < P2_NB; b++) {
                uint32_t tmp[8][16];
                for (int i = 0; i < 8; i++) _mm512_storeu_si512(tmp[i], v_mul(s[b][i], one));
                for (int l = 0; l < 16; l++) for (int i = 0; i < 8; i++) layers[8 * ((size_t)r0 + 16 * b + l) + i] = tmp[i][l];
            }
        }
    } else {
        for (size_t r0 = 0; r0 < h; r0 += 16) {
            V s[16];
            for (int i = 0; i < 16; i++) s[i] = _mm512_setzero_si512();
            for (size_t c0 = 0; c0 < total_w; c0 += 8) {
                const size_t k = total_w - c0 < 8 ? total_w - c0 : 8;
                for (size_t j = 0; j < k; j++) s[j] = v_mul(_mm512_loadu_si512(cols[c0 + j] + r0), vr2);
                v_permute(s);
            }
            uint32_t tmp[8][16];
            for (int i = 0; i < 8; i++) _mm512_storeu_si512(tmp[i], v_mul(s[i], one));
            for (int l = 0; l < 16; l++) for (int i = 0; i < 8; i++) layers[8 * (r0 + l) + i] = tmp[i][l];
        }
    }
    free(cols);
    uint32_t* prev = layers;
    for (size_t n = h >> 1; n >= 1; n >>= 1) {
        uint32_t* cur = prev + 16 * n;
        if (n >= 16) {
            uint32_t ix[16];
            for (int l = 0; l < 16; l++) ix[l] = 16u * (uint32_t)l;
            const V vix = _mm512_loadu_si512(ix);
#pragma omp parallel for schedule(static) if (n >= 1024)
            for (long j0 = 0; j0 < (long)n; j0 += 16) {
                V s[16];
                for (int i = 0; i < 16; i++) s[i] = v_mul(_mm512_i32gather_epi32(vix, prev + 16 * (size_t)j0 + i, 4), vr2);
                v_permute(s);
                uint32_t tmp[8][16];
                for (int i = 0; i < 8; i++) _mm512_storeu_si512(tmp[i], v_mul(s[i], one));
                for (int l = 0; l < 16; l++) for (int i = 0; i < 8; i++) cur[8 * ((size_t)j0 + l) + i] = tmp[i][l];
            }
        } else {
            for (size_t j = 0; j < n; j++) orc_compress(prev + 16 * j, prev + 16 * j + 8, cur + 8 * j);
        }
        prev = cur;
        if (n == 1) break;
    }
}

/* =====================================================================================================================
 * stage 2: constraint fold over 16 rows per vector; program constants pre-converted to Montgomery */
enum { OP_PUSH_APC = 0, OP_PUSH_CONST = 1, OP_ADD = 2, OP_SUB = 3, OP_MUL = 4, OP_NEG = 5, OP_INV_OR_ZERO = 6 };

static V v_inv_or_zero(V x) {            /* rare opcode: per-lane Fermat inverse on Montgomery values */
    uint32_t t[16];
    _mm512_storeu_si512(t, x);
    for (int l = 0; l < 16; l++) {
        uint32_t a = t[l], r = R1, e = P - 2;
        while (e) { if (e & 1) r = m_mul(r, a); a = m_mul(a, a); e >>= 1; }
        t[l] = t[l] ? r : 0;
    }
    return _mm512_loadu_si512(t);
}

/* acc[l] (Montgomery) += sum_k alpha^(C-1-k) c_k(rows r0..r0+15) */
static inline void fold_rows16(const uint32_t* code, const orc_span_t* spans, size_t n_constraints, const uint32_t* mat, size_t height,
                               size_t r0, const uint32_t* apow_m /*[C][4]*/, V acc[4]) {
    const V vr2 = VSET(R2);
    V st[16];
    for (size_t k = 0; k < n_constraints; k++) {
        int sp = 0;
        const uint32_t* bc = code + spans[k].off;
        for (uint32_t ip = 0; ip < spans[k].len;) {
            const uint32_t op = bc[ip++];
            switch (op) {
            case OP_PUSH_APC: st[sp++] = v_mul(_mm512_loadu_si512(mat + (size_t)bc[ip++] * height + r0), vr2); break;
            case OP_PUSH_CONST: st[sp++] = VSET(bc[ip++]); break;           /* already Montgomery */
            case OP_ADD: sp--; st[sp - 1] = v_add(st[sp - 1], st[sp]); break;
            case OP_SUB: sp--; st[sp - 1] = v_sub(st[sp - 1], st[sp]); break;
            case OP_MUL: sp--; st[sp - 1] = v_mul(st[sp - 1], st[sp]); break;
            case OP_NEG: st[sp - 1] = v_neg(st[sp - 1]); break;
            default: st[sp - 1] = v_inv_or_zero(st[sp - 1]); break;
            }
        }
        for (int l = 0; l < 4; l++) acc[l] = v_add(acc[l], v_mul(st[0], VSET(apow_m[4 * k + l])));
    }
}

static uint32_t* pack_code(const uint32_t* bc, const orc_span_t* spans, size_t n_constraints, size_t* n_words) {
    size_t end = 0;
    for (size_t k = 0; k < n_constraints; k++) if (spans[k].off + spans[k].len > end) end = spans[k].off + spans[k].len;
    uint32_t* code = (uint32_t*)malloc((end ? end : 1) * sizeof(uint32_t));
    memcpy(code, bc, end * sizeof(uint32_t));
    for (size_t k = 0; k < n_constraints; k++)
        for (uint32_t ip = spans[k].off; ip < spans[k].off + spans[k].len;) {
            const uint32_t op = code[ip++];
            if (op == OP_PUSH_CONST) { code[ip] = to_m(code[ip] % P); ip++; }
            else if (op == OP_PUSH_APC) ip++;
        }
    *n_words = end;
    return code;
}
static uint32_t* alpha_powers_m(const uint32_t alpha[4], size_t n) {      /* [k] = alpha^(n-1-k), Montgomery limbs */
    uint32_t* ap = (uint32_t*)malloc((n ? n : 1) * 16);
    bb4_t a = {{alpha[0], alpha[1], alpha[2], alpha[3]}}, cur = bb4_from_base(1);
    for (size_t k = n; k-- > 0;) {
        for (int l = 0; l < 4; l++) ap[4 * k + l] = to_m(cur.c[l]);
        cur = bb4_mul(cur, a);
    }
    return ap;
}

void orcf_constraint_fold(const uint32_t* bc, const orc_span_t* spans, size_t n_constraints, const uint32_t* mat, size_t height,
                          const uint32_t alpha[4], uint32_t* out4) {
    if (height < 16 || (height & 15)) { orc_constraint_fold(bc, spans, n_constraints, mat, height, alpha, out4); return; }
    size_t nw;
    uint32_t* code = pack_code(bc, spans, n_constraints, &nw);
    uint32_t* ap = alpha_powers_m(alpha, n_constraints);
    const V one = VSET(1);
#pragma omp parallel for schedule(static)
    for (long r0 = 0; r0 < (long)height; r0 += 16) {
        V acc[4] = {_mm512_setzero_si512(), _mm512_setzero_si512(), _mm512_setzero_si512(), _mm512_setzero_si512()};
        fold_rows16(code, spans, n_constraints, mat, height, (size_t)r0, ap, acc);
        for (int l = 0; l < 4; l++) _mm512_storeu_si512(out4 + (size_t)l * height + (size_t)r0, v_mul(acc[l], one));
    }
    free(code); free(ap);
}

void orcf_quotient(const uint32_t* bc, const orc_span_t* spans, size_t n_constraints, const uint32_t* lde, unsigned log_n,
                   unsigned log_blowup, uint32_t shift, const uint32_t alpha[4], uint32_t* quotient) {
    const size_t n = (size_t)1 << log_n, m = n << 1;
    if (log_blowup != 1 || n < 16) { orc_quotient(bc, spans, n_constraints, lde, log_n, log_blowup, shift, alpha, quotient); return; }
    size_t nw;
    uint32_t* code = pack_code(bc, spans, n_constraints, &nw);
    uint32_t* ap = alpha_powers_m(alpha, n_constraints);
    const uint32_t sn = bb_pow(shift, n);
    const uint32_t zinv[2] = {bb_inv(bb_sub(sn, 1)), bb_inv(bb_sub(bb_neg(sn), 1))};     /* canonical: montmul(acc*R, z) = acc*z */
#pragma omp parallel for schedule(static)
    for (long r0 = 0; r0 < (long)m; r0 += 16) {
        V acc[4] = {_mm512_setzero_si512(), _mm512_setzero_si512(), _mm512_setzero_si512(), _mm512_setzero_si512()};
        fold_rows16(code, spans, n_constraints, lde, m, (size_t)r0, ap, acc);
        const size_t chunk = (size_t)r0 >> log_n, j = (size_t)r0 & (n - 1);
        for (int l = 0; l < 4; l++) _mm512_storeu_si512(quotient + (chunk * 4 + l) * n + j, v_mul(acc[l], VSET(zinv[chunk])));
    }
    free(code); free(ap);
}

/* =====================================================================================================================
 * openings: f(zeta) by the barycentric formula over shift*H:  g(y) = f(shift*y), z = zeta/shift,
 *   g(z) = (z^N - 1)/N * sum_i g_i * w^i / (z - w^i).   Same VALUE as the interpolate-then-Horner restatement in ntt.c. */
static bb4_t e4m_mul(bb4_t a, bb4_t b) {         /* Ext4 product on Montgomery limbs */
    uint32_t t[7] = {0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) t[i + j] = s_add(t[i + j], m_mul(a.c[i], b.c[j]));
    const uint32_t w11 = to_m(BB_EXT_W);
    bb4_t r;
    for (int i = 0; i < 4; i++) r.c[i] = t[i];
    for (int i = 4; i < 7; i++) r.c[i - 4] = s_add(r.c[i - 4], m_mul(t[i], w11));
    return r;
}
static bb4_t e4_to_m(bb4_t a) { for (int i = 0; i < 4; i++) a.c[i] = to_m(a.c[i]); return a; }
static bb4_t e4_from_m(bb4_t a) { for (int i = 0; i < 4; i++) a.c[i] = from_m(a.c[i]); return a; }

/* d[i] <- 1/d[i] for n Ext4 values (Montgomery limbs), Montgomery's trick in blocks (one Ext4 inversion per 64) */
static void e4m_batch_inverse(bb4_t* d, size_t n) {
#pragma omp parallel for schedule(static)
    for (long b0 = 0; b0 < (long)n; b0 += 64) {
        const size_t k = n - (size_t)b0 < 64 ? n - (size_t)b0 : 64;
        bb4_t pre[64], acc = {{R1, 0, 0, 0}};
        for (size_t i = 0; i < k; i++) { pre[i] = acc; acc = e4m_mul(acc, d[b0 + i]); }
        bb4_t inv = e4_to_m(bb4_inv(e4_from_m(acc)));
        for (size_t i = k; i-- > 0;) {
            bb4_t t = e4m_mul(inv, pre[i]);
            inv = e4m_mul(inv, d[b0 + i]);
            d[b0 + i] = t;
        }
    }
}

void orcf_eval_at_point(const uint32_t* mat, unsigned log_n, size_t width, uint32_t shift, const uint32_t zeta[4], uint32_t* out) {
    const size_t n = (size_t)1 << log_n;
    /* below 16 rows, and at a point of the domain, where one weight's denominator is 0: the scalar restatement */
    if (n < 16 || bb4_in_coset(zeta, shift, log_n)) { orc_eval_at_point(mat, log_n, width, shift, zeta, out); return; }
    bb4_t z = {{zeta[0], zeta[1], zeta[2], zeta[3]}};
    z = bb4_scale(z, bb_inv(shift));
    /* weights w^i / (z - w^i), Montgomery limbs, SoA */
    bb4_t* d = (bb4_t*)malloc(n * sizeof(bb4_t));
    uint32_t* wp = (uint32_t*)malloc(n * sizeof(uint32_t));
    const bb4_t zm = e4_to_m(z);
    {
        const uint32_t w = to_m(bb_root_of_unity(log_n));
        /* powers by blocks so the loop parallelises */
#pragma omp parallel for schedule(static)
        for (long b0 = 0; b0 < (long)n; b0 += 4096) {
            uint32_t x = to_m(bb_pow(bb_root_of_unity(log_n), (uint64_t)b0));
            for (size_t i = (size_t)b0; i < (size_t)b0 + 4096 && i < n; i++) {
                wp[i] = x;
                d[i] = zm;
                d[i].c[0] = s_sub(d[i].c[0], x);
                x = m_mul(x, w);
            }
        }
    }
    e4m_batch_inverse(d, n);
    uint32_t* ws = (uint32_t*)aligned_alloc(64, 4 * n * sizeof(uint32_t));
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)n; i++)
        for (int l = 0; l < 4; l++) ws[(size_t)l * n + (size_t)i] = m_mul(d[i].c[l], wp[i]);       /* Montgomery: (d*w)*R */
    free(d); free(wp);
    bb4_t zn = bb4_pow(z, n);
    zn.c[0] = bb_sub(zn.c[0], 1);
    const bb4_t pref = bb4_scale(zn, bb_inv((uint32_t)(n % P)));
#pragma omp parallel for schedule(dynamic, 4)
    for (long c = 0; c < (long)width; c++) {
        const uint32_t* f = mat + (size_t)c * n;
        V acc[4] = {_mm512_setzero_si512(), _mm512_setzero_si512(), _mm512_setzero_si512(), _mm512_setzero_si512()};
        for (size_t i = 0; i < n; i += 16) {
            const V x = _mm512_loadu_si512(f + i);
            for (int l = 0; l < 4; l++) acc[l] = v_add(acc[l], v_mul(x, _mm512_loadu_si512(ws + (size_t)l * n + i)));   /* canonical */
        }
        bb4_t s;
        for (int l = 0; l < 4; l++) {
            uint32_t t[16], a = 0;
            _mm512_storeu_si512(t, acc[l]);
            for (int k = 0; k < 16; k++) a = s_add(a, t[k]);
            s.c[l] = a;
        }
        s = bb4_mul(s, pref);
        memcpy(out + 4 * (size_t)c, s.c, 16);
    }
    free(ws);
}

/* reduced opening, general form used by the prover:
 *   ro[r] = sum_g ( sum_{j in group g} gamma_j * (f_j[r] - y_j) ) / (x_r - z_g),  x_r = shift * w_m^{bitrev(r)}.
 * A group = the columns opened at one point; gamma_j = the column's power of the batching challenge.  out [m][4]. */
void orcf_deep_quotient_groups(const uint32_t* const* cols, const uint32_t* group_of_col, size_t n_cols, const uint32_t* zs /*[G][4]*/,
                               size_t n_groups, unsigned log_m, uint32_t shift, const uint32_t* gamma_pows /*[n_cols][4]*/,
                               const uint32_t* ys /*[n_cols][4]*/, uint32_t* out) {
    const size_t m = (size_t)1 << log_m;
    uint32_t* gp = (uint32_t*)malloc((n_cols ? n_cols : 1) * 16);           /* Montgomery limbs of gamma_j */
    bb4_t* ysum = (bb4_t*)calloc(n_groups, sizeof(bb4_t));
    for (size_t j = 0; j < n_cols; j++) {
        for (int l = 0; l < 4; l++) gp[4 * j + l] = to_m(gamma_pows[4 * j + l]);
        bb4_t gj, y;
        memcpy(gj.c, gamma_pows + 4 * j, 16);
        memcpy(y.c, ys + 4 * j, 16);
        ysum[group_of_col[j]] = bb4_add(ysum[group_of_col[j]], bb4_mul(gj, y));
    }
    const uint32_t w = bb_root_of_unity(log_m);
    bb4_t* acc_all = (bb4_t*)malloc(n_groups * m * sizeof(bb4_t));         /* numerators per group, canonical */
    if (m >= 16) {
#pragma omp parallel for schedule(static)
        for (long r0 = 0; r0 < (long)m; r0 += 16) {
            V acc[8][4];
            for (size_t q = 0; q < n_groups && q < 8; q++) for (int l = 0; l < 4; l++) acc[q][l] = _mm512_setzero_si512();
            for (size_t j = 0; j < n_cols; j++) {
                const V x = _mm512_loadu_si512(cols[j] + r0);
                V* a = acc[group_of_col[j]];
                for (int l = 0; l < 4; l++) a[l] = v_add(a[l], v_mul(x, VSET(gp[4 * j + l])));
            }
            for (size_t q = 0; q < n_groups; q++) {
                uint32_t t[4][16];
                for (int l = 0; l < 4; l++) _mm512_storeu_si512(t[l], acc[q][l]);
                for (int k = 0; k < 16; k++) {
                    bb4_t v = {{t[0][k], t[1][k], t[2][k], t[3][k]}};
                    acc_all[q * m + (size_t)r0 + k] = bb4_sub(v, ysum[q]);
                }
            }
        }
    } else {
        for (size_t r = 0; r < m; r++)
            for (size_t q = 0; q < n_groups; q++) {
                bb4_t a = bb4_from_base(0);
                for (size_t j = 0; j < n_cols; j++)
                    if (group_of_col[j] == q) {
                        bb4_t gj;
                        memcpy(gj.c, gamma_pows + 4 * j, 16);
                        a = bb4_add(a, bb4_scale(gj, cols[j][r]));
                    }
                acc_all[q * m + r] = bb4_sub(a, ysum[q]);
            }
    }
    /* denominators x_r - z_g, batch inverted */
    bb4_t* den = (bb4_t*)malloc(n_groups * m * sizeof(bb4_t));
#pragma omp parallel for schedule(static)
    for (long r = 0; r < (long)m; r++) {
        const uint32_t x = to_m(bb_mul(shift, bb_pow(w, bitrev32((uint32_t)r, log_m))));
        for (size_t q = 0; q < n_groups; q++) {
            bb4_t d = {{to_m(zs[4 * q]), to_m(zs[4 * q + 1]), to_m(zs[4 * q + 2]), to_m(zs[4 * q + 3])}};
            d.c[0] = s_sub(x, d.c[0]);
            for (int l = 1; l < 4; l++) d.c[l] = d.c[l] ? P - d.c[l] : 0;
            den[q * m + (size_t)r] = d;
        }
    }
    e4m_batch_inverse(den, n_groups * m);
#pragma omp parallel for schedule(static)
    for (long r = 0; r < (long)m; r++) {
        bb4_t s = bb4_from_base(0);
        for (size_t q = 0; q < n_groups; q++) {
            /* canonical numerator x Montgomery inverse -> canonical product limb-wise through e4m_mul on (num*1, inv*R) */
            bb4_t t = e4m_mul(acc_all[q * m + (size_t)r], den[q * m + (size_t)r]);
            s = bb4_add(s, t);
        }
        memcpy(out + 4 * (size_t)r, s.c, 16);
    }
    free(gp); free(ysum); free(acc_all); free(den);
}

/* drop-in for orc_deep_quotient (one point, all matrices), with its refusal of a zeta on shift*H' */
int orcf_deep_quotient(const uint32_t* const* mats, const size_t* widths, size_t n_mats, unsigned log_m, uint32_t shift,
                       const uint32_t zeta[4], const uint32_t gamma[4], const uint32_t* ys, uint32_t* out) {
    if (bb4_in_coset(zeta, shift, log_m)) return -1;
    const size_t m = (size_t)1 << log_m;
    size_t total = 0;
    for (size_t i = 0; i < n_mats; i++) total += widths[i];
    const uint32_t** cols = (const uint32_t**)malloc((total ? total : 1) * sizeof(*cols));
    uint32_t* grp = (uint32_t*)calloc(total ? total : 1, sizeof(uint32_t));
    uint32_t* gp = (uint32_t*)malloc((total ? total : 1) * 16);               /* consecutive powers gamma^0, gamma^1, ... */
    size_t k = 0;
    for (size_t i = 0; i < n_mats; i++) for (size_t c = 0; c < widths[i]; c++) cols[k++] = mats[i] + c * m;
    bb4_t cur = bb4_from_base(1);
    const bb4_t g = {{gamma[0], gamma[1], gamma[2], gamma[3]}};
    for (size_t j = 0; j < total; j++) { memcpy(gp + 4 * j, cur.c, 16); cur = bb4_mul(cur, g); }
    orcf_deep_quotient_groups(cols, grp, total, zeta, 1, log_m, shift, gp, ys, out);
    free(cols); free(grp); free(gp);
    return 0;
}

/* =====================================================================================================================
 * LogUp / bus argument, 16 rows per vector (semantics: logup.c).  Montgomery inside, canonical at the edges. */
typedef struct { V c[4]; } V4;
static inline V4 v4_add(V4 a, V4 b) { V4 r; for (int i = 0; i < 4; i++) r.c[i] = v_add(a.c[i], b.c[i]); return r; }
static inline V4 v4_sub(V4 a, V4 b) { V4 r; for (int i = 0; i < 4; i++) r.c[i] = v_sub(a.c[i], b.c[i]); return r; }
static inline V4 v4_scale(V4 a, V s) { V4 r; for (int i = 0; i < 4; i++) r.c[i] = v_mul(a.c[i], s); return r; }
static inline V v_x11(V x) { V x2 = v_add(x, x), x4 = v_add(x2, x2), x8 = v_add(x4, x4); return v_add(v_add(x8, x2), x); }
static inline V4 v4_mul(V4 a, V4 b) {
    const V b1 = v_x11(b.c[1]), b2 = v_x11(b.c[2]), b3 = v_x11(b.c[3]);
    V4 r;
    r.c[0] = v_add(v_add(v_mul(a.c[0], b.c[0]), v_mul(a.c[1], b3)), v_add(v_mul(a.c[2], b2), v_mul(a.c[3], b1)));
    r.c[1] = v_add(v_add(v_mul(a.c[0], b.c[1]), v_mul(a.c[1], b.c[0])), v_add(v_mul(a.c[2], b3), v_mul(a.c[3], b2)));
    r.c[2] = v_add(v_add(v_mul(a.c[0], b.c[2]), v_mul(a.c[1], b.c[1])), v_add(v_mul(a.c[2], b.c[0]), v_mul(a.c[3], b3)));
    r.c[3] = v_add(v_add(v_mul(a.c[0], b.c[3]), v_mul(a.c[1], b.c[2])), v_add(v_mul(a.c[2], b.c[1]), v_mul(a.c[3], b.c[0])));
    return r;
}
static inline V4 v4_bcast(bb4_t m) { V4 r; for (int i = 0; i < 4; i++) r.c[i] = VSET(m.c[i]); return r; }
static V v_inv(V a) {                       /* a^(p-2), lane-wise, Montgomery (0 -> 0) */
    V r = VSET(R1);
    for (uint32_t e = P - 2; e; e >>= 1) { if (e & 1) r = v_mul(r, a); a = v_mul(a, a); }
    return r;
}
static V4 v4_inv(V4 x) {                    /* same tower as bb4_inv */
    const V W = VSET(to_m(BB_EXT_W));
    V A0 = v_add(v_mul(x.c[0], x.c[0]), v_mul(W, v_mul(x.c[2], x.c[2]))), A1 = v_add(v_mul(x.c[0], x.c[2]), v_mul(x.c[0], x.c[2]));
    V B0 = v_add(v_mul(x.c[1], x.c[1]), v_mul(W, v_mul(x.c[3], x.c[3]))), B1 = v_add(v_mul(x.c[1], x.c[3]), v_mul(x.c[1], x.c[3]));
    V n0 = v_sub(A0, v_mul(W, B1)), n1 = v_sub(A1, B0);
    V d = v_inv(v_sub(v_mul(n0, n0), v_mul(W, v_mul(n1, n1))));
    V4 s = {{v_mul(n0, d), _mm512_setzero_si512(), v_neg(v_mul(n1, d)), _mm512_setzero_si512()}};
    V4 cj = {{x.c[0], v_neg(x.c[1]), x.c[2], v_neg(x.c[3])}};
    return v4_mul(cj, s);
}

/* one packed expression (constants already Montgomery) on rows r0..r0+15 of a column-major matrix -> Montgomery vector */
static inline V eval16(const uint32_t* bc, uint32_t len, const uint32_t* mat, size_t height, size_t r0) {
    const V vr2 = VSET(R2);
    V st[16];
    int sp = 0;
    for (uint32_t ip = 0; ip < len;) {
        const uint32_t op = bc[ip++];
        switch (op) {
        case OP_PUSH_APC: st[sp++] = v_mul(_mm512_loadu_si512(mat + (size_t)bc[ip++] * height + r0), vr2); break;
        case OP_PUSH_CONST: st[sp++] = VSET(bc[ip++]); break;
        case OP_ADD: sp--; st[sp - 1] = v_add(st[sp - 1], st[sp]); break;
        case OP_SUB: sp--; st[sp - 1] = v_sub(st[sp - 1], st[sp]); break;
        case OP_MUL: sp--; st[sp - 1] = v_mul(st[sp - 1], st[sp]); break;
        case OP_NEG: st[sp - 1] = v_neg(st[sp - 1]); break;
        default: st[sp - 1] = v_inv_or_zero(st[sp - 1]); break;
        }
    }
    return st[0];
}

typedef struct {
    uint32_t* code;             /* interaction bytecode with Montgomery constants */
    bb4_t alpha_m;              /* alpha_lu, Montgomery limbs */
    bb4_t* kc;                  /* per interaction: alpha_lu + beta^k (bus + 1), Montgomery */
    bb4_t* betas;               /* beta^j, Montgomery */
} lu_ctx_t;

static void lu_ctx_init(lu_ctx_t* L, const uint32_t* ibc, const orc_span_t* isp, const orc_interaction_t* ints, size_t n_ints,
                        const uint32_t alpha_lu[4], const uint32_t beta_lu[4]) {
    size_t n_spans = 0, maxk = 0;
    for (size_t i = 0; i < n_ints; i++) {
        if (ints[i].args_index_off + ints[i].num_args + 1 > n_spans) n_spans = ints[i].args_index_off + ints[i].num_args + 1;
        if (ints[i].num_args > maxk) maxk = ints[i].num_args;
    }
    size_t nw;
    L->code = pack_code(ibc, isp, n_spans, &nw);
    bb4_t al = {{alpha_lu[0], alpha_lu[1], alpha_lu[2], alpha_lu[3]}}, be = {{beta_lu[0], beta_lu[1], beta_lu[2], beta_lu[3]}};
    bb4_t* bc_ = (bb4_t*)malloc((maxk + 1) * sizeof(bb4_t));
    L->betas = (bb4_t*)malloc((maxk + 1) * sizeof(bb4_t));
    bc_[0] = bb4_from_base(1);
    for (size_t j = 1; j <= maxk; j++) bc_[j] = bb4_mul(bc_[j - 1], be);
    for (size_t j = 0; j <= maxk; j++) L->betas[j] = e4_to_m(bc_[j]);
    L->kc = (bb4_t*)malloc((n_ints ? n_ints : 1) * sizeof(bb4_t));
    for (size_t i = 0; i < n_ints; i++) L->kc[i] = e4_to_m(bb4_add(al, bb4_scale(bc_[ints[i].num_args], (ints[i].bus_id + 1) % P)));
    L->alpha_m = e4_to_m(al);
    free(bc_);
}
static void lu_ctx_free(lu_ctx_t* L) { free(L->code); free(L->kc); free(L->betas); }

/* (m_i, d_i) of every interaction on 16 rows, then per chunk (N_c, D_c) */
static void lu_chunks16(const lu_ctx_t* L, const orc_span_t* isp, const orc_interaction_t* ints, const uint32_t* chunk_start, size_t n_chunks,
                        const uint32_t* mat, size_t height, size_t r0, V* mv, V4* dv, V4* Nc, V4* Dc) {
    for (size_t c = 0; c < n_chunks; c++) {
        const uint32_t a = chunk_start[c], e = chunk_start[c + 1];
        for (uint32_t i = a; i < e; i++) {
            const orc_span_t* s = isp + ints[i].args_index_off;
            mv[i - a] = eval16(L->code + s[0].off, s[0].len, mat, height, r0);
            V4 d = v4_bcast(L->kc[i]);
            for (uint32_t j = 0; j < ints[i].num_args; j++) {
                const V x = eval16(L->code + s[1 + j].off, s[1 + j].len, mat, height, r0);
                d = v4_add(d, v4_scale(v4_bcast(L->betas[j]), x));
            }
            dv[i - a] = d;
        }
        /* N = sum_i m_i prod_{j != i} d_j,  D = prod_i d_i  (incrementally) */
        V4 D = dv[0], N = {{mv[0], _mm512_setzero_si512(), _mm512_setzero_si512(), _mm512_setzero_si512()}};
        for (uint32_t i = 1; i < e - a; i++) {
            N = v4_add(v4_mul(N, dv[i]), v4_scale(D, mv[i]));
            D = v4_mul(D, dv[i]);
        }
        Nc[c] = N;
        Dc[c] = D;
    }
}

void orcf_logup_perm_trace(const uint32_t* trace, unsigned log_n, const uint32_t* ibc, const orc_span_t* isp, const orc_interaction_t* ints,
                           size_t n_ints, const uint32_t* chunk_start, size_t n_chunks, const uint32_t alpha_lu[4], const uint32_t beta_lu[4],
                           uint32_t* perm, uint32_t cumsum[4]) {
    const size_t n = (size_t)1 << log_n;
    if (n < 16) { orc_logup_perm_trace(trace, log_n, ibc, isp, ints, n_ints, chunk_start, n_chunks, alpha_lu, beta_lu, perm, cumsum); return; }
    lu_ctx_t L;
    lu_ctx_init(&L, ibc, isp, ints, n_ints, alpha_lu, beta_lu);
    size_t max_chunk = 1;
    for (size_t c = 0; c < n_chunks; c++) if (chunk_start[c + 1] - chunk_start[c] > max_chunk) max_chunk = chunk_start[c + 1] - chunk_start[c];
    uint32_t* rowsum = (uint32_t*)aligned_alloc(64, 4 * n * sizeof(uint32_t));
    const V one = VSET(1);
#pragma omp parallel
    {
        V* mv = (V*)aligned_alloc(64, max_chunk * sizeof(V));
        V4* dv = (V4*)aligned_alloc(64, max_chunk * sizeof(V4));
        V4* Nc = (V4*)aligned_alloc(64, n_chunks * sizeof(V4));
        V4* Dc = (V4*)aligned_alloc(64, n_chunks * sizeof(V4));
        V4* pre = (V4*)aligned_alloc(64, n_chunks * sizeof(V4));
#pragma omp for schedule(static)
        for (long r0 = 0; r0 < (long)n; r0 += 16) {
            lu_chunks16(&L, isp, ints, chunk_start, n_chunks, trace, n, (size_t)r0, mv, dv, Nc, Dc);
            /* Montgomery's trick across the chunks of this row block: one Ext4 inversion per 16 rows */
            V4 acc = v4_bcast((bb4_t){{R1, 0, 0, 0}});
            for (size_t c = 0; c < n_chunks; c++) { pre[c] = acc; acc = v4_mul(acc, Dc[c]); }
            V4 inv = v4_inv(acc), rs = {{_mm512_setzero_si512(), _mm512_setzero_si512(), _mm512_setzero_si512(), _mm512_setzero_si512()}};
            for (size_t c = n_chunks; c-- > 0;) {
                const V4 dinv = v4_mul(inv, pre[c]);
                inv = v4_mul(inv, Dc[c]);
                const V4 v = v4_mul(Nc[c], dinv);
                rs = v4_add(rs, v);
                for (int l = 0; l < 4; l++) _mm512_storeu_si512(perm + (4 * c + l) * n + (size_t)r0, v_mul(v.c[l], one));
            }
            for (int l = 0; l < 4; l++) _mm512_storeu_si512(rowsum + (size_t)l * n + (size_t)r0, v_mul(rs.c[l], one));
        }
        free(mv); free(dv); free(Nc); free(Dc); free(pre);
    }
    uint32_t phi[4] = {0, 0, 0, 0};
    for (size_t r = 0; r < n; r++)
        for (int l = 0; l < 4; l++) { phi[l] = s_add(phi[l], rowsum[(size_t)l * n + r]); perm[(4 * n_chunks + l) * n + r] = phi[l]; }
    memcpy(cumsum, phi, 16);
    free(rowsum);
    lu_ctx_free(&L);
}

void orcf_logup_fold(const uint32_t* lde, const uint32_t* perm_lde, unsigned log_n, uint32_t shift, const uint32_t* ibc, const orc_span_t* isp,
                     const orc_interaction_t* ints, size_t n_ints, const uint32_t* chunk_start, size_t n_chunks, const uint32_t alpha_lu[4],
                     const uint32_t beta_lu[4], const uint32_t cumsum[4], const uint32_t alpha[4], uint32_t* acc4) {
    const size_t n = (size_t)1 << log_n, m = n << 1;
    const unsigned log_m = log_n + 1;
    if (n < 16) { orc_logup_fold(lde, perm_lde, log_n, shift, ibc, isp, ints, n_ints, chunk_start, n_chunks, alpha_lu, beta_lu, cumsum, alpha, acc4); return; }
    lu_ctx_t L;
    lu_ctx_init(&L, ibc, isp, ints, n_ints, alpha_lu, beta_lu);
    size_t max_chunk = 1;
    for (size_t c = 0; c < n_chunks; c++) if (chunk_start[c + 1] - chunk_start[c] > max_chunk) max_chunk = chunk_start[c + 1] - chunk_start[c];
    const bb4_t a_m = e4_to_m((bb4_t){{alpha[0], alpha[1], alpha[2], alpha[3]}});
    const bb4_t cs_m = e4_to_m((bb4_t){{cumsum[0], cumsum[1], cumsum[2], cumsum[3]}});
    const uint32_t w_m = bb_root_of_unity(log_m), w_n_inv = bb_inv(bb_root_of_unity(log_n)), sn = bb_pow(shift, n);
    const V vr2 = VSET(R2), one = VSET(1);
#pragma omp parallel
    {
        V* mv = (V*)aligned_alloc(64, max_chunk * sizeof(V));
        V4* dv = (V4*)aligned_alloc(64, max_chunk * sizeof(V4));
        V4* Nc = (V4*)aligned_alloc(64, n_chunks * sizeof(V4));
        V4* Dc = (V4*)aligned_alloc(64, n_chunks * sizeof(V4));
#pragma omp for schedule(static)
        for (long r0 = 0; r0 < (long)m; r0 += 16) {
            lu_chunks16(&L, isp, ints, chunk_start, n_chunks, lde, m, (size_t)r0, mv, dv, Nc, Dc);
            uint32_t rn[16], sel[3][16];
            int contiguous = 1;
            for (int l = 0; l < 16; l++) {
                const uint32_t i_nat = bitrev32((uint32_t)(r0 + l), log_m);
                rn[l] = bitrev32((uint32_t)((i_nat + 2) & (m - 1)), log_m);
                if (rn[l] != rn[0] + (uint32_t)l) contiguous = 0;
                const uint32_t x = bb_mul(shift, bb_pow(w_m, i_nat));
                const uint32_t zh = bb_sub((i_nat & 1) ? bb_neg(sn) : sn, 1);
                sel[0][l] = to_m(bb_mul(zh, bb_inv(bb_sub(x, 1))));
                sel[1][l] = to_m(bb_sub(x, w_n_inv));
                sel[2][l] = to_m(bb_mul(zh, bb_inv(bb_sub(x, w_n_inv))));
            }
            const V vrn = _mm512_loadu_si512(rn);
#define LDN(col) (contiguous ? _mm512_loadu_si512(perm_lde + (size_t)(col) * m + rn[0]) : _mm512_i32gather_epi32(vrn, perm_lde + (size_t)(col) * m, 4))
            V4 acc, sum = v4_bcast((bb4_t){{0, 0, 0, 0}}), sum_next = sum;
            for (int l = 0; l < 4; l++) acc.c[l] = v_mul(_mm512_loadu_si512(acc4 + (size_t)l * m + (size_t)r0), vr2);
            const V4 va = v4_bcast(a_m);
            for (size_t c = 0; c < n_chunks; c++) {
                V4 pc, pn;
                for (int l = 0; l < 4; l++) {
                    pc.c[l] = v_mul(_mm512_loadu_si512(perm_lde + (4 * c + l) * m + (size_t)r0), vr2);
                    pn.c[l] = v_mul(LDN(4 * c + l), vr2);
                }
                sum = v4_add(sum, pc);
                sum_next = v4_add(sum_next, pn);
                acc = v4_add(v4_mul(acc, va), v4_sub(v4_mul(pc, Dc[c]), Nc[c]));
            }
            V4 phi, phn;
            for (int l = 0; l < 4; l++) {
                phi.c[l] = v_mul(_mm512_loadu_si512(perm_lde + (4 * n_chunks + l) * m + (size_t)r0), vr2);
                phn.c[l] = v_mul(LDN(4 * n_chunks + l), vr2);
            }
#undef LDN
            acc = v4_add(v4_mul(acc, va), v4_scale(v4_sub(phi, sum), _mm512_loadu_si512(sel[0])));
            acc = v4_add(v4_mul(acc, va), v4_scale(v4_sub(v4_sub(phn, phi), sum_next), _mm512_loadu_si512(sel[1])));
            acc = v4_add(v4_mul(acc, va), v4_scale(v4_sub(phi, v4_bcast(cs_m)), _mm512_loadu_si512(sel[2])));
            for (int l = 0; l < 4; l++) _mm512_storeu_si512(acc4 + (size_t)l * m + (size_t)r0, v_mul(acc.c[l], one));
        }
        free(mv); free(dv); free(Nc); free(Dc);
    }
    lu_ctx_free(&L);
}
