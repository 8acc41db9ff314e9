/*
 * ORACLE (test infrastructure, not product code): an independent VERIFIER for the segment proof object of orc_prove_chips
 * (all chips of a segment under one transcript; a single segment is one chip).
 * The reference's own tests pin the prover only by validity -- a proof produced by engine E must verify under the CPU
 * engine (verify_app_proof::<BabyBearPoseidon2CpuEngine>, /root/reference/openvm-riscv/src/lib.rs:337-341; SURVEY.md §4).
 * This file plays that role for the transcript v2 of DESIGN.md §3, §3b: it re-derives every challenge (LogUp, alpha, zeta, gamma,
 * betas), checks the proof of work, checks every mixed-height MMCS opening, recomputes the reduced opening of each LDE height (two
 * opening points) from the opened rows, checks every FRI path and fold with the per-height injection of the reduced openings, that
 * the final polynomial is CONSTANT and matches, and (optionally, for satisfying traces) per chip the constraint identity
 * Horner_alpha(c_k(T(zeta)), LogUp constraints at zeta) = Z_H(zeta) * Q(zeta).
 * It shares no code or state with the prover: inputs are the chip shapes, the proof struct, the cumulative sums, the opened values
 * and the query openings.
 */
#include "oracle.h"
#include "bb31.h"
#include <string.h>
#include <stdlib.h>

static bb4_t ld4(const uint32_t* p) { bb4_t r; memcpy(r.c, p, 16); return r; }
static int eq4(bb4_t a, bb4_t b) { return memcmp(a.c, b.c, 16) == 0; }

static int check_path(const uint32_t leaf[8], size_t idx, const uint32_t* path, unsigned log_h, const uint32_t root[8]) {
    uint32_t node[8], next[8];
    memcpy(node, leaf, 32);
    for (unsigned k = 0; k < log_h; k++) {
        const uint32_t* sib = path + 8 * k;
        if ((idx >> k) & 1) orc_compress(sib, node, next); else orc_compress(node, sib, next);
        memcpy(node, next, 32);
    }
    return memcmp(node, root, 32) == 0;
}

/* bytecode over Ext4 values (column j -> vals[j]); same opcodes as orc_eval_expr */
static bb4_t eval_ext(const uint32_t* bc, uint32_t len, const uint32_t* vals) {
    bb4_t st[16];
    int sp = 0;
    for (uint32_t ip = 0; ip < len;) {
        uint32_t op = bc[ip++];
        switch (op) {
        case 0: st[sp++] = ld4(vals + 4 * bc[ip++]); break;
        case 1: st[sp++] = bb4_from_base(bc[ip++] % BB_P); break;
        case 2: sp--; st[sp - 1] = bb4_add(st[sp - 1], st[sp]); break;
        case 3: sp--; st[sp - 1] = bb4_sub(st[sp - 1], st[sp]); break;
        case 4: sp--; st[sp - 1] = bb4_mul(st[sp - 1], st[sp]); break;
        case 5: st[sp - 1] = bb4_sub(bb4_from_base(0), st[sp - 1]); break;
        default: { bb4_t z = bb4_from_base(0); st[sp - 1] = eq4(st[sp - 1], z) ? z : bb4_inv(st[sp - 1]); break; }
        }
    }
    return st[0];
}

bb4_t orc_logup_fold_at_point(bb4_t acc, bb4_t alpha, const uint32_t* main_ys, const uint32_t* perm_ys, const uint32_t* perm_next_ys,
                              unsigned log_n, bb4_t zeta, const uint32_t* ibc, const orc_span_t* isp, const orc_interaction_t* ints, size_t n_ints,
                              const uint32_t* chunk_start, size_t n_chunks, bb4_t al, const uint32_t beta_lu[4], bb4_t cumsum);

/* one opened row of a matrix of height 2^log_h; a mixed-height MMCS path is checked as prove.c commits it */
typedef struct { const uint32_t* row; size_t width; unsigned log_h; } mv_mat_t;

static void hash_opened(const mv_mat_t* ms, size_t n, unsigned log_h, uint32_t digest[8]) {
    size_t tot = 0;
    for (size_t i = 0; i < n; i++) if (ms[i].log_h == log_h) tot += ms[i].width;
    uint32_t* row = (uint32_t*)malloc((tot ? tot : 1) * 4);
    size_t k = 0;
    for (size_t i = 0; i < n; i++)
        if (ms[i].log_h == log_h) { memcpy(row + k, ms[i].row, ms[i].width * 4); k += ms[i].width; }
    orc_hash_row(row, tot, digest);
    free(row);
}
static int mmcs_verify(const mv_mat_t* ms, size_t n, unsigned h0, size_t idx, const uint32_t* path, const uint32_t root[8]) {
    uint32_t node[8], next[8];
    hash_opened(ms, n, h0, node);
    for (unsigned l = 1; l <= h0; l++) {
        const uint32_t* sib = path + 8 * (l - 1);
        if ((idx >> (l - 1)) & 1) orc_compress(sib, node, next); else orc_compress(node, sib, next);
        memcpy(node, next, 32);
        int inj = 0;
        for (size_t i = 0; i < n; i++) if (ms[i].log_h == h0 - l) inj = 1;
        if (inj) {
            uint32_t d[8];
            hash_opened(ms, n, h0 - l, d);
            orc_compress(node, d, next);
            memcpy(node, next, 32);
        }
    }
    return memcmp(node, root, 32) == 0;
}

int orc_verify_chips(const orc_chip_t* chips, size_t K, const orc_chips_proof_t* proof, const uint32_t* cumsums, const uint32_t* ys,
                     const uint32_t* queries, int check_constraints) {
    unsigned hmax = 0, hperm = 0;
    size_t* wp = (size_t*)calloc(K, sizeof(size_t));
    size_t* nch = (size_t*)calloc(K, sizeof(size_t));
    uint32_t** cstart = (uint32_t**)calloc(K, sizeof(void*));
    size_t* e_main = (size_t*)calloc(K, sizeof(size_t));
    size_t* e_perm = (size_t*)calloc(K, sizeof(size_t));
    size_t* e_q = (size_t*)calloc(K, sizeof(size_t));
    mv_mat_t* mv = (mv_mat_t*)calloc(K, sizeof(mv_mat_t));
    bb4_t* gp = NULL;
    int any_lu = 0, rc = 0;
#define FAILC(code) do { rc = (code); goto done_c; } while (0)
    for (size_t c = 0; c < K; c++) {
        const orc_air_t* a = chips[c].air;
        const unsigned lm = chips[c].log_n + 1;
        if (lm > hmax) hmax = lm;
        if (a->n_ints) {
            cstart[c] = (uint32_t*)malloc((a->n_ints + 1) * sizeof(uint32_t));
            int k = orc_logup_chunks(a->ibc, a->ispans, a->ints, a->n_ints, 3, cstart[c]);
            if (k < 0) FAILC(20);
            nch[c] = (size_t)k;
            wp[c] = 4 * (nch[c] + 1);
            any_lu = 1;
            if (lm > hperm) hperm = lm;
        }
    }
    if (proof->n_chips != K || proof->log_max != hmax || proof->n_fri_layers != hmax - 1 || proof->final_len != 2) FAILC(20);
    size_t n_open = 0;
    for (size_t c = 0; c < K; c++) { e_main[c] = n_open; n_open += chips[c].width; }
    for (size_t c = 0; c < K; c++) if (wp[c]) { e_perm[c] = n_open; n_open += 2 * wp[c]; }
    for (size_t c = 0; c < K; c++) { e_q[c] = n_open; n_open += 8; }

    /* 1. transcript */
    orc_challenger_t ch;
    orc_challenger_init(&ch);
    uint32_t t4[4];
    orc_challenger_observe(&ch, proof->main_root, 8);
    if (any_lu) {
        orc_challenger_sample_ext(&ch, t4);
        if (memcmp(t4, proof->logup_alpha, 16)) FAILC(1);
        orc_challenger_sample_ext(&ch, t4);
        if (memcmp(t4, proof->logup_beta, 16)) FAILC(1);
        orc_challenger_observe(&ch, proof->perm_root, 8);
        for (size_t c = 0; c < K; c++) if (wp[c]) orc_challenger_observe(&ch, cumsums + 4 * c, 4);
    }
    orc_challenger_sample_ext(&ch, t4);
    if (memcmp(t4, proof->alpha, 16)) FAILC(2);
    orc_challenger_observe(&ch, proof->quotient_root, 8);
    orc_challenger_sample_ext(&ch, t4);
    if (memcmp(t4, proof->zeta, 16)) FAILC(3);
    orc_challenger_observe(&ch, ys, 4 * n_open);
    orc_challenger_sample_ext(&ch, t4);
    if (memcmp(t4, proof->gamma, 16)) FAILC(4);
    for (uint32_t i = 0; i < proof->n_fri_layers; i++) {
        orc_challenger_observe(&ch, proof->fri_roots[i], 8);
        orc_challenger_sample_ext(&ch, t4);
        if (memcmp(t4, proof->fri_betas[i], 16)) FAILC(5);
    }
    if (memcmp(proof->final_poly[0], proof->final_poly[1], 16)) FAILC(15);
    orc_challenger_observe(&ch, proof->final_poly[0], 4);
    {
        const uint32_t mask = proof->pow_bits >= 31 ? 0x7fffffffu : ((1u << proof->pow_bits) - 1);
        if (proof->pow_witness >= BB_P) FAILC(6);
        orc_challenger_observe(&ch, &proof->pow_witness, 1);
        if (orc_challenger_sample(&ch) & mask) FAILC(6);
    }
    const bb4_t zeta = ld4(proof->zeta), gamma = ld4(proof->gamma), alpha = ld4(proof->alpha);

    /* 2. per-chip constraint identity at zeta */
    if (check_constraints)
        for (size_t c = 0; c < K; c++) {
            const orc_air_t* a = chips[c].air;
            const size_t n = (size_t)1 << chips[c].log_n;
            const uint32_t* ym = ys + 4 * e_main[c];
            const uint32_t* yq = ys + 4 * e_q[c];
            bb4_t acc = bb4_from_base(0);
            for (size_t k = 0; k < a->n_constraints; k++) {
                acc = bb4_mul(acc, alpha);
                acc = bb4_add(acc, eval_ext(a->bc + a->spans[k].off, a->spans[k].len, ym));
            }
            if (wp[c])
                acc = orc_logup_fold_at_point(acc, alpha, ym, ys + 4 * e_perm[c], ys + 4 * (e_perm[c] + wp[c]), chips[c].log_n, zeta, a->ibc, a->ispans, a->ints,
                                              a->n_ints, cstart[c], nch[c], ld4(proof->logup_alpha), proof->logup_beta, ld4(cumsums + 4 * c));
            bb4_t zn = bb4_pow(zeta, n);
            const uint32_t gn = bb_pow(BB_GENERATOR, n);
            bb4_t q = bb4_from_base(0);
            for (int b = 0; b < 2; b++) {
                uint32_t sgn_b = b ? BB_P - 1 : 1, sgn_nb = b ? 1 : BB_P - 1;
                bb4_t num = zn;
                num.c[0] = bb_sub(num.c[0], bb_mul(gn, sgn_nb));
                uint32_t den = bb_inv(bb_mul(2, bb_mul(gn, sgn_b)));
                bb4_t qb = bb4_from_base(0);
                for (int l = 0; l < 4; l++) {
                    bb4_t e = bb4_from_base(0);
                    e.c[l] = 1;
                    qb = bb4_add(qb, bb4_mul(e, ld4(yq + 4 * (4 * b + l))));
                }
                q = bb4_add(q, bb4_mul(bb4_scale(num, den), qb));
            }
            bb4_t zh = zn;
            zh.c[0] = bb_sub(zh.c[0], 1);
            if (!eq4(acc, bb4_mul(zh, q))) FAILC(16);
        }

    /* 3. queries */
    size_t wm = 0, wpt = 0;
    for (size_t c = 0; c < K; c++) { wm += chips[c].width; wpt += wp[c]; }
    size_t wpq = 1 + wm + 8 * hmax + (wpt ? wpt + 8 * hperm : 0) + 8 * K + 8 * hmax;
    for (unsigned i = 0; i + 1 < hmax; i++) wpq += 8 + 8 * (hmax - 1 - i);
    gp = (bb4_t*)malloc(n_open * sizeof(bb4_t));
    {
        bb4_t cur = bb4_from_base(1);
        for (size_t j = 0; j < n_open; j++) { gp[j] = cur; cur = bb4_mul(cur, gamma); }
    }
    const uint32_t two_inv = bb_inv(2);
    for (size_t qi = 0; qi < proof->n_queries && !rc; qi++) {
        const uint32_t* o = queries + qi * wpq;
        const size_t r = o[0];
        if (r != (orc_challenger_sample(&ch) & (((size_t)1 << hmax) - 1))) { rc = 7; break; }
        const uint32_t* mrows = o + 1;
        const uint32_t* mpath = mrows + wm;
        const uint32_t* prows = mpath + 8 * hmax;
        const uint32_t* ppath = prows + wpt;
        const uint32_t* qrows = wpt ? ppath + 8 * hperm : prows;
        const uint32_t* qpath = qrows + 8 * K;
        const uint32_t* fr = qpath + 8 * hmax;
        /* MMCS openings */
        {
            size_t off = 0;
            for (size_t c = 0; c < K; c++) { mv[c] = (mv_mat_t){mrows + off, chips[c].width, chips[c].log_n + 1}; off += chips[c].width; }
            if (!mmcs_verify(mv, K, hmax, r, mpath, proof->main_root)) { rc = 8; break; }
            if (wpt) {
                size_t np = 0;
                off = 0;
                for (size_t c = 0; c < K; c++) if (wp[c]) { mv[np++] = (mv_mat_t){prows + off, wp[c], chips[c].log_n + 1}; off += wp[c]; }
                if (!mmcs_verify(mv, np, hperm, r >> (hmax - hperm), ppath, proof->perm_root)) { rc = 9; break; }
            }
            for (size_t c = 0; c < K; c++) mv[c] = (mv_mat_t){qrows + 8 * c, 8, chips[c].log_n + 1};
            if (!mmcs_verify(mv, K, hmax, r, qpath, proof->quotient_root)) { rc = 10; break; }
        }
        /* reduced opening per height from the opened rows */
        bb4_t val_h[32];
        int have_h[32] = {0};
        for (int h = 0; h < 32; h++) val_h[h] = bb4_from_base(0);
        size_t moff = 0, poff = 0;
        for (size_t c = 0; c < K; c++) {
            const unsigned lm = chips[c].log_n + 1;
            const size_t rr = r >> (hmax - lm);
            const uint32_t* trow = mrows + moff;
            const uint32_t* prow = prows + poff;
            const uint32_t* qrow = qrows + 8 * c;
            bb4_t a0 = bb4_from_base(0), a1 = bb4_from_base(0);
            for (size_t j = 0; j < chips[c].width; j++) {
                const size_t e = e_main[c] + j;
                a0 = bb4_add(a0, bb4_sub(bb4_scale(gp[e], trow[j]), bb4_mul(gp[e], ld4(ys + 4 * e))));
            }
            for (size_t j = 0; j < wp[c]; j++) {
                const size_t e = e_perm[c] + j, e2 = e_perm[c] + wp[c] + j;
                a0 = bb4_add(a0, bb4_sub(bb4_scale(gp[e], prow[j]), bb4_mul(gp[e], ld4(ys + 4 * e))));
                a1 = bb4_add(a1, bb4_sub(bb4_scale(gp[e2], prow[j]), bb4_mul(gp[e2], ld4(ys + 4 * e2))));
            }
            for (size_t j = 0; j < 8; j++) {
                const size_t e = e_q[c] + j;
                a0 = bb4_add(a0, bb4_sub(bb4_scale(gp[e], qrow[j]), bb4_mul(gp[e], ld4(ys + 4 * e))));
            }
            const uint32_t x = bb_mul(BB_GENERATOR, bb_pow(bb_root_of_unity(lm), bitrev32((uint32_t)rr, lm)));
            const bb4_t zeta_next = bb4_scale(zeta, bb_root_of_unity(chips[c].log_n));
            bb4_t v = bb4_mul(a0, bb4_inv(bb4_sub(bb4_from_base(x), zeta)));
            if (wp[c]) v = bb4_add(v, bb4_mul(a1, bb4_inv(bb4_sub(bb4_from_base(x), zeta_next))));
            val_h[lm] = bb4_add(val_h[lm], v);
            have_h[lm] = 1;
            moff += chips[c].width;
            poff += wp[c];
        }
        bb4_t val = val_h[hmax];
        size_t idx = r;
        uint32_t shift = BB_GENERATOR;
        for (unsigned i = 0; i + 1 < hmax; i++) {
            const unsigned log_len = hmax - i, log_h = log_len - 1;
            const uint32_t* pair = fr;
            const uint32_t* path = fr + 8;
            fr += 8 + 8 * log_h;
            bb4_t lo = ld4(pair), hi = ld4(pair + 4);
            if (!eq4((idx & 1) ? hi : lo, val)) { rc = i == 0 ? 11 : 13; break; }
            const size_t j = idx >> 1;
            uint32_t leaf[8];
            orc_hash_row(pair, 8, leaf);
            if (!check_path(leaf, j, path, log_h, proof->fri_roots[i])) { rc = 12; break; }
            uint32_t xj = bb_mul(shift, bb_pow(bb_root_of_unity(log_len), bitrev32((uint32_t)j, log_h)));
            bb4_t beta = ld4(proof->fri_betas[i]);
            bb4_t s = bb4_scale(bb4_add(lo, hi), two_inv);
            bb4_t df = bb4_scale(bb4_sub(lo, hi), bb_mul(two_inv, bb_inv(xj)));
            val = bb4_add(s, bb4_mul(beta, df));
            idx = j;
            shift = bb_mul(shift, shift);
            if (log_h > 1 && have_h[log_h]) val = bb4_add(val, val_h[log_h]);        /* this height's codeword joins here */
        }
        if (!rc && !eq4(val, ld4(proof->final_poly[idx]))) rc = 14;
    }
done_c:
    free(gp);
    for (size_t c = 0; c < K; c++) free(cstart[c]);
    free(cstart); free(wp); free(nch); free(e_main); free(e_perm); free(e_q); free(mv);
    return rc;
#undef FAILC
}
