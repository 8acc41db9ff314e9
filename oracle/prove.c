/*
 * ORACLE (test infrastructure, not product code): all chips of one APC segment under ONE transcript, through the whole path in
 * the order the V1-shaped FRI prover runs it (metric names from /root/reference/openvm/metrics-viewer/CLAUDE.md:52-78:
 * main_trace_commit, perm_trace_commit, quotient_poly_compute, quotient_poly_commit, pcs_opening).  Call site being restated:
 * engine.prove(pk, ProvingContext) behind sdk.app_prover(exe)?.prove(stdin) (/root/reference/openvm-riscv/src/lib.rs:327-332), with
 * ONE proving context for all chips of a segment (/root/reference/openvm/src/trace_generation.rs:113-140; SURVEY.md App. C.3); the
 * engine itself is un-vendored => parity unpinned (oracle.h).  A single segment is the proof of one chip.
 *
 * Transcript v2 (DuplexChallenger; DESIGN.md §3, §3b):
 *   observe(main_root)
 *   [some chip has interactions]  alpha_lu, beta_lu <- sample_ext x2;  observe(perm_root);  observe(cumulative sum of each such chip)
 *   alpha <- sample_ext;  observe(quotient_root);  zeta <- sample_ext
 *   observe every opened value: main at zeta (chip order) | per chip with interactions perm at zeta, perm at zeta*w_chip |
 *     quotient chunks at zeta (chip order);  gamma <- sample_ext
 *   per FRI layer: observe(root_i), beta_i <- sample_ext;  observe(final polynomial constant)
 *   proof of work: observe(witness), sample_bits(pow_bits) == 0;  n_queries x sample_bits(log of the tallest LDE)
 * Chips of different heights share every challenge, three mixed-height MMCS commitments (main, permutation, quotient) and one FRI
 * instance: one reduced-opening codeword per distinct LDE height; folding starts from the tallest, and after the fold that reaches a
 * height with its own codeword that codeword is added index-wise.  Each phase runs for every chip before the next one starts.
 * The heavy primitives run either on the scalar `%` restatement or (prm->fast) on the AVX-512 Montgomery ones of fast.c,
 * which are checked bit for bit against the former -- the proof is the same either way.
 */
#include "oracle.h"
#include "bb31.h"
#include <stdlib.h>
#include <string.h>
#include <time.h>

/* big working buffers: 2 MB aligned and advised to transparent huge pages -- the per-row kernels walk thousands of columns that are
   megabytes apart, which thrashes the TLB with 4 KB pages */
#include <sys/mman.h>
void* orc_big_alloc(size_t bytes) {
    const size_t al = (size_t)2 << 20;
    bytes = (bytes + al - 1) / al * al;
    void* p = aligned_alloc(al, bytes ? bytes : al);
#ifdef MADV_HUGEPAGE
    if (p) madvise(p, bytes ? bytes : al, MADV_HUGEPAGE);
#endif
    return p;
}
void orc_big_free(void* p) { free(p); }
#define BIG(n_words) ((uint32_t*)orc_big_alloc((size_t)(n_words) * sizeof(uint32_t)))

static double now_s(void) { struct timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t.tv_sec + 1e-9 * t.tv_nsec; }

typedef struct {
    void (*lde_batch)(const uint32_t*, unsigned, size_t, unsigned, uint32_t, uint32_t*);
    void (*merkle_commit)(const uint32_t* const*, const size_t*, size_t, unsigned, uint32_t*);
    void (*constraint_fold)(const uint32_t*, const orc_span_t*, size_t, const uint32_t*, size_t, const uint32_t[4], uint32_t*);
    void (*eval_at_point)(const uint32_t*, unsigned, size_t, uint32_t, const uint32_t[4], uint32_t*);
    void (*deep_groups)(const uint32_t* const*, const uint32_t*, size_t, const uint32_t*, size_t, unsigned, uint32_t, const uint32_t*,
                        const uint32_t*, uint32_t*);
    void (*logup_perm_trace)(const uint32_t*, unsigned, const uint32_t*, const orc_span_t*, const orc_interaction_t*, size_t, const uint32_t*, size_t,
                             const uint32_t[4], const uint32_t[4], uint32_t*, uint32_t[4]);
    void (*logup_fold)(const uint32_t*, const uint32_t*, unsigned, uint32_t, const uint32_t*, const orc_span_t*, const orc_interaction_t*, size_t,
                       const uint32_t*, size_t, const uint32_t[4], const uint32_t[4], const uint32_t[4], const uint32_t[4], uint32_t*);
} ops_t;
static const ops_t OPS_SLOW = {orc_lde_batch, orc_merkle_commit, orc_constraint_fold, orc_eval_at_point, orc_deep_quotient_groups,
                               orc_logup_perm_trace, orc_logup_fold};
static const ops_t OPS_FAST = {orcf_lde_batch, orcf_merkle_commit, orcf_constraint_fold, orcf_eval_at_point, orcf_deep_quotient_groups,
                               orcf_logup_perm_trace, orcf_logup_fold};

/* Merkle tree (all layers, node-major) of a row-major matrix; returns malloc'ed [2h-1][8] */
static uint32_t* merkle_tree_rowmajor(const uint32_t* mat, size_t width, unsigned log_h) {
    size_t h = (size_t)1 << log_h;
    uint32_t* t = (uint32_t*)malloc(8 * (2 * h) * sizeof(uint32_t));
#pragma omp parallel for schedule(static) if (h >= 2048)
    for (long r = 0; r < (long)h; r++) orc_hash_row(mat + (size_t)r * width, width, t + 8 * (size_t)r);
    uint32_t* prev = t;
    for (size_t n = h >> 1; n >= 1; n >>= 1) {
        uint32_t* cur = prev + 16 * n;
#pragma omp parallel for schedule(static) if (n >= 2048)
        for (long j = 0; j < (long)n; j++) orc_compress(prev + 16 * (size_t)j, prev + 16 * (size_t)j + 8, cur + 8 * (size_t)j);
        prev = cur;
        if (n == 1) break;
    }
    return t;
}

static void copy_path(const uint32_t* tree, unsigned log_h, size_t idx, uint32_t* out) {
    for (unsigned k = 0; k < log_h; k++) {
        size_t level_off = ((size_t)2 << log_h) - ((size_t)2 << (log_h - k));
        memcpy(out + 8 * k, tree + 8 * (level_off + ((idx >> k) ^ 1)), 32);
    }
}

size_t orc_perm_width(const orc_air_t* air) {
    if (!air->n_ints) return 0;
    uint32_t* cs = (uint32_t*)malloc((air->n_ints + 1) * sizeof(uint32_t));
    int nc = orc_logup_chunks(air->ibc, air->ispans, air->ints, air->n_ints, 3, cs);
    free(cs);
    return nc < 0 ? 0 : 4 * ((size_t)nc + 1);
}

uint32_t orc_grind(const orc_challenger_t* c, unsigned bits) {
    const uint32_t mask = bits >= 31 ? 0x7fffffffu : ((1u << bits) - 1);
    for (uint32_t base = 0;; base += 4096) {
        uint32_t found = 0xffffffffu;
#pragma omp parallel for schedule(static)
        for (long i = 0; i < 4096; i++) {
            const uint32_t w = base + (uint32_t)i;
            if (w >= BB_P) continue;
            orc_challenger_t t = *c;
            orc_challenger_observe(&t, &w, 1);
            if ((orc_challenger_sample(&t) & mask) == 0) {
#pragma omp critical
                if (w < found) found = w;
            }
        }
        if (found != 0xffffffffu) return found;
    }
}

/* MMCS (Plonky3 MerkleTreeMmcs): matrices sorted by height (descending, stable); leaves = sponge of the concatenated rows of the
   tallest matrices; going up, a level whose size equals the height of further matrices gets them injected:
   node = compress(compress(left, right), sponge(rows of those matrices)).  Opening index r: matrix of height 2^h opens row r >> (h0 - h). */
typedef struct { const uint32_t* mat; size_t width; unsigned log_h; } mc_mat_t;

/* mixed-height tree, node-major layers back to back (2^(h0+1) - 1 nodes); returns BIG()-allocated, *log_h0 = tallest.  The rows of
   each height are hashed by ops->merkle_commit over that height's matrices: with one height its tree is the whole tree, otherwise the
   levels from the tallest injection upward are rebuilt from the leaf digests of the injected heights. */
static uint32_t* mmcs_commit(const ops_t* ops, const mc_mat_t* ms, size_t n, unsigned* log_h0) {
    unsigned h0 = 0;
    for (size_t i = 0; i < n; i++) if (ms[i].log_h > h0) h0 = ms[i].log_h;
    *log_h0 = h0;
    uint32_t* t = BIG(8 * ((size_t)2 << h0));
    uint32_t* leaves[32] = {0};                           /* leaves[h]: the tree of the height-2^h matrices, layer 0 used */
    const uint32_t** mats = (const uint32_t**)malloc(n * sizeof(*mats));
    size_t* widths = (size_t*)malloc(n * sizeof(size_t));
    for (unsigned h = 0; h <= h0; h++) {
        size_t k = 0;
        for (size_t i = 0; i < n; i++) if (ms[i].log_h == h) { mats[k] = ms[i].mat; widths[k++] = ms[i].width; }
        if (!k) continue;
        if (h < h0) leaves[h] = BIG(8 * ((size_t)2 << h));
        ops->merkle_commit(mats, widths, k, h, h < h0 ? leaves[h] : t);
    }
    uint32_t* prev = t;
    int injected = 0;
    for (unsigned h = h0; h-- > 0;) {
        uint32_t* cur = prev + 8 * ((size_t)2 << h);      /* the level below has 2^(h+1) nodes */
        const size_t cnt = (size_t)1 << h;
        const uint32_t* d = leaves[h];
        injected |= d != NULL;
        if (injected) {
#pragma omp parallel for schedule(static) if (cnt >= 1024)
            for (long j = 0; j < (long)cnt; j++) {
                uint32_t* node = cur + 8 * (size_t)j;
                orc_compress(prev + 16 * (size_t)j, prev + 16 * (size_t)j + 8, node);
                if (d) {
                    uint32_t o[8];
                    orc_compress(node, d + 8 * (size_t)j, o);
                    memcpy(node, o, 32);
                }
            }
        }
        prev = cur;
    }
    for (unsigned h = 0; h < h0; h++) free(leaves[h]);
    free(mats); free(widths);
    return t;
}

size_t orc_chips_num_opened(const orc_chip_t* chips, size_t K) {
    size_t n = 0;
    for (size_t c = 0; c < K; c++) n += chips[c].width + 2 * orc_perm_width(chips[c].air) + 8;
    return n;
}
size_t orc_chips_query_words(const orc_chip_t* chips, size_t K) {
    unsigned hmax = 0, hperm = 0;
    size_t wm = 0, wp = 0;
    for (size_t c = 0; c < K; c++) {
        const unsigned lm = chips[c].log_n + 1;
        const size_t p = orc_perm_width(chips[c].air);
        if (lm > hmax) hmax = lm;
        if (p && lm > hperm) hperm = lm;
        wm += chips[c].width;
        wp += p;
    }
    size_t w = 1 + wm + 8 * hmax + (wp ? wp + 8 * hperm : 0) + 8 * K + 8 * hmax;
    for (unsigned i = 0; i + 1 < hmax; i++) w += 8 + 8 * (hmax - 1 - i);
    return w;
}

static double lap(double* t) { const double n = now_s(), d = n - *t; *t = n; return d; }

/* the LDE columns behind opened values: column j of `lde` (height 2^log_m) opened at point 0 (zeta) or 1 (zeta*w) */
typedef struct { const uint32_t* col; uint32_t point; unsigned log_m; } opened_col_t;
static size_t opened_cols(opened_col_t* o, const uint32_t* lde, size_t width, unsigned log_m, uint32_t point) {
    for (size_t j = 0; j < width; j++) o[j] = (opened_col_t){lde + (j << log_m), point, log_m};
    return width;
}

void orc_prove_chips(const orc_chip_t* chips, size_t K, const orc_params_t* prm, orc_chips_proof_t* proof, uint32_t* cumsums, uint32_t* ys_out,
                     uint32_t* queries_out, double stage_seconds[10]) {
    const ops_t* ops = (prm->fast && orcf_available()) ? &OPS_FAST : &OPS_SLOW;
    double st[10] = {0};
    memset(proof, 0, sizeof *proof);
    proof->pow_bits = prm->pow_bits;
    proof->n_queries = prm->n_queries;
    proof->n_chips = (uint32_t)K;
    orc_challenger_t ch;
    orc_challenger_init(&ch);
    uint32_t** lde = (uint32_t**)calloc(K, sizeof(void*));
    uint32_t** perm = (uint32_t**)calloc(K, sizeof(void*));
    uint32_t** plde = (uint32_t**)calloc(K, sizeof(void*));
    uint32_t** qlde = (uint32_t**)calloc(K, sizeof(void*));
    uint32_t** nat = (uint32_t**)calloc(K, sizeof(void*));
    uint32_t** cstart = (uint32_t**)calloc(K, sizeof(void*));
    size_t* wp = (size_t*)calloc(K, sizeof(size_t));
    size_t* nch = (size_t*)calloc(K, sizeof(size_t));
    mc_mat_t* mm = (mc_mat_t*)calloc(K, sizeof(mc_mat_t));
    unsigned hmax = 0, hperm = 0, hq = 0;
    int any_lu = 0;

    /* main trace: LDE of every chip, one commitment */
    double t = now_s();
    for (size_t c = 0; c < K; c++) {
        const size_t m = (size_t)2 << chips[c].log_n;
        lde[c] = BIG(chips[c].width * m);
        ops->lde_batch(chips[c].trace, chips[c].log_n, chips[c].width, 1, BB_GENERATOR, lde[c]);
        mm[c] = (mc_mat_t){lde[c], chips[c].width, chips[c].log_n + 1};
    }
    st[0] = lap(&t);
    uint32_t* tree_m = mmcs_commit(ops, mm, K, &hmax);
    memcpy(proof->main_root, tree_m + 8 * (((size_t)2 << hmax) - 2), 32);
    orc_challenger_observe(&ch, proof->main_root, 8);
    proof->log_max = hmax;
    st[1] = lap(&t);

    /* LogUp: shared challenges, one permutation trace per chip with interactions, one commitment, every chip's cumulative sum */
    for (size_t c = 0; c < K; c++) if (chips[c].air->n_ints) any_lu = 1;
    uint32_t* tree_p = NULL;
    if (any_lu) {
        orc_challenger_sample_ext(&ch, proof->logup_alpha);
        orc_challenger_sample_ext(&ch, proof->logup_beta);
        for (size_t c = 0; c < K; c++) {
            const orc_air_t* a = chips[c].air;
            if (!a->n_ints) continue;
            cstart[c] = (uint32_t*)malloc((a->n_ints + 1) * sizeof(uint32_t));
            int k = orc_logup_chunks(a->ibc, a->ispans, a->ints, a->n_ints, 3, cstart[c]);
            if (k < 0) abort();
            nch[c] = (size_t)k;
            wp[c] = 4 * (nch[c] + 1);
            perm[c] = BIG(wp[c] << chips[c].log_n);
            ops->logup_perm_trace(chips[c].trace, chips[c].log_n, a->ibc, a->ispans, a->ints, a->n_ints, cstart[c], nch[c], proof->logup_alpha, proof->logup_beta,
                                  perm[c], cumsums + 4 * c);
        }
        st[2] = lap(&t);
        size_t np = 0;
        for (size_t c = 0; c < K; c++) {
            if (!wp[c]) continue;
            plde[c] = BIG(wp[c] << (chips[c].log_n + 1));
            ops->lde_batch(perm[c], chips[c].log_n, wp[c], 1, BB_GENERATOR, plde[c]);
            mm[np++] = (mc_mat_t){plde[c], wp[c], chips[c].log_n + 1};
        }
        tree_p = mmcs_commit(ops, mm, np, &hperm);
        memcpy(proof->perm_root, tree_p + 8 * (((size_t)2 << hperm) - 2), 32);
        orc_challenger_observe(&ch, proof->perm_root, 8);
        for (size_t c = 0; c < K; c++) if (wp[c]) orc_challenger_observe(&ch, cumsums + 4 * c, 4);
        st[3] = lap(&t);
    }
    for (size_t c = 0; c < K; c++) if (!wp[c]) memset(cumsums + 4 * c, 0, 16);
    orc_challenger_sample_ext(&ch, proof->alpha);

    /* quotients, the same alpha for every chip: (Horner fold of the AIR's constraints, then of the LogUp constraints) / Z_H, split by
       natural-index parity into two chunks of natural-order evaluations over g*w_{2N}^b*H */
    for (size_t c = 0; c < K; c++) {
        const orc_air_t* a = chips[c].air;
        const unsigned ln = chips[c].log_n;
        const size_t n = (size_t)1 << ln, m = n << 1;
        uint32_t* acc4 = BIG(4 * m);
        ops->constraint_fold(a->bc, a->spans, a->n_constraints, lde[c], m, proof->alpha, acc4);
        if (wp[c]) ops->logup_fold(lde[c], plde[c], ln, BB_GENERATOR, a->ibc, a->ispans, a->ints, a->n_ints, cstart[c], nch[c], proof->logup_alpha, proof->logup_beta,
                                   cumsums + 4 * c, proof->alpha, acc4);
        const uint32_t sn = bb_pow(BB_GENERATOR, n);
        const uint32_t zinv[2] = {bb_inv(bb_sub(sn, 1)), bb_inv(bb_sub(bb_neg(sn), 1))};
        uint32_t* q = nat[c] = BIG(8 * n);
#pragma omp parallel for schedule(static)
        for (long r = 0; r < (long)m; r++) {
            const size_t chunk = (size_t)r >> ln, j = bitrev32((uint32_t)r & (uint32_t)(n - 1), ln);
            for (int l = 0; l < 4; l++) q[(chunk * 4 + l) * n + j] = bb_mul(acc4[(size_t)l * m + r], zinv[chunk]);
        }
        free(acc4);
    }
    st[4] = lap(&t);

    /* quotient commit: chunk b LDE'd with shift g/s_b, one commitment */
    for (size_t c = 0; c < K; c++) {
        const unsigned ln = chips[c].log_n;
        const size_t n = (size_t)1 << ln, m = n << 1;
        qlde[c] = BIG(8 * m);
        ops->lde_batch(nat[c], ln, 4, 1, 1, qlde[c]);
        ops->lde_batch(nat[c] + 4 * n, ln, 4, 1, bb_inv(bb_root_of_unity(ln + 1)), qlde[c] + 4 * m);
        mm[c] = (mc_mat_t){qlde[c], 8, ln + 1};
    }
    uint32_t* tree_q = mmcs_commit(ops, mm, K, &hq);
    memcpy(proof->quotient_root, tree_q + 8 * (((size_t)2 << hq) - 2), 32);
    orc_challenger_observe(&ch, proof->quotient_root, 8);
    orc_challenger_sample_ext(&ch, proof->zeta);
    st[5] = lap(&t);

    /* openings, in observation order: main at zeta (chip order) | per chip with interactions perm at zeta, perm at zeta*w_chip (the
       transition constraint reads the next row) | quotient chunks at zeta (chip order) */
    size_t n_open = 0;
    for (size_t c = 0; c < K; c++) n_open += chips[c].width + 2 * wp[c] + 8;
    uint32_t* ys = (uint32_t*)calloc(4 * n_open, sizeof(uint32_t));
    opened_col_t* oc = (opened_col_t*)malloc(n_open * sizeof(opened_col_t));
    size_t pos = 0;
    for (size_t c = 0; c < K; c++) {
        ops->eval_at_point(chips[c].trace, chips[c].log_n, chips[c].width, 1, proof->zeta, ys + 4 * pos);
        pos += opened_cols(oc + pos, lde[c], chips[c].width, chips[c].log_n + 1, 0);
    }
    for (size_t c = 0; c < K; c++) {
        if (!wp[c]) continue;
        const bb4_t zn = bb4_scale((bb4_t){{proof->zeta[0], proof->zeta[1], proof->zeta[2], proof->zeta[3]}}, bb_root_of_unity(chips[c].log_n));
        ops->eval_at_point(perm[c], chips[c].log_n, wp[c], 1, proof->zeta, ys + 4 * pos);
        ops->eval_at_point(perm[c], chips[c].log_n, wp[c], 1, zn.c, ys + 4 * (pos + wp[c]));
        pos += opened_cols(oc + pos, plde[c], wp[c], chips[c].log_n + 1, 0);
        pos += opened_cols(oc + pos, plde[c], wp[c], chips[c].log_n + 1, 1);
    }
    for (size_t c = 0; c < K; c++) {
        const size_t n = (size_t)1 << chips[c].log_n;
        const uint32_t w2n = bb_root_of_unity(chips[c].log_n + 1);
        ops->eval_at_point(nat[c], chips[c].log_n, 4, BB_GENERATOR, proof->zeta, ys + 4 * pos);
        ops->eval_at_point(nat[c] + 4 * n, chips[c].log_n, 4, bb_mul(BB_GENERATOR, w2n), proof->zeta, ys + 4 * (pos + 4));
        pos += opened_cols(oc + pos, qlde[c], 8, chips[c].log_n + 1, 0);
    }
    if (prm->cheat_opening) ys[0] = bb_add(ys[0], 1);
    orc_challenger_observe(&ch, ys, 4 * n_open);
    orc_challenger_sample_ext(&ch, proof->gamma);

    /* one reduced-opening codeword per LDE height, over the columns of that height: opened value e weighs gamma^e */
    uint32_t* ro[32] = {0};
    {
        uint32_t* gp = (uint32_t*)malloc(16 * n_open);
        bb4_t cur = bb4_from_base(1);
        const bb4_t g = {{proof->gamma[0], proof->gamma[1], proof->gamma[2], proof->gamma[3]}};
        for (size_t e = 0; e < n_open; e++) { memcpy(gp + 4 * e, cur.c, 16); cur = bb4_mul(cur, g); }
        const uint32_t** cols = (const uint32_t**)malloc(n_open * sizeof(*cols));
        uint32_t* grp = (uint32_t*)malloc(n_open * sizeof(uint32_t));
        uint32_t* gk = (uint32_t*)malloc(16 * n_open);
        uint32_t* yk = (uint32_t*)malloc(16 * n_open);
        for (unsigned lm = 2; lm <= hmax; lm++) {
            size_t k = 0;
            uint32_t n_points = 1;
            for (size_t e = 0; e < n_open; e++) {
                if (oc[e].log_m != lm) continue;
                cols[k] = oc[e].col;
                grp[k] = oc[e].point;
                if (oc[e].point) n_points = 2;
                memcpy(gk + 4 * k, gp + 4 * e, 16);
                memcpy(yk + 4 * k, ys + 4 * e, 16);
                k++;
            }
            if (!k) continue;
            const bb4_t zn = bb4_scale((bb4_t){{proof->zeta[0], proof->zeta[1], proof->zeta[2], proof->zeta[3]}}, bb_root_of_unity(lm - 1));
            uint32_t zs[8];
            memcpy(zs, proof->zeta, 16);
            memcpy(zs + 4, zn.c, 16);
            ro[lm] = BIG((size_t)4 << lm);
            ops->deep_groups(cols, grp, k, zs, n_points, lm, BB_GENERATOR, gk, yk, ro[lm]);
        }
        free(gp); free(cols); free(grp); free(gk); free(yk);
    }
    if (ys_out) memcpy(ys_out, ys, 16 * n_open);
    st[6] = lap(&t);

    /* FRI: fold from the tallest codeword, adding the codeword of each height when the fold reaches it */
    uint32_t* f = ro[hmax];
    ro[hmax] = NULL;
    unsigned log_len = hmax;
    uint32_t shift = BB_GENERATOR;
    uint32_t layer_i = 0;
    uint32_t* words[32];
    uint32_t* trees[32];
    while (log_len > 1) {                                /* log_blowup = 1, final_poly_len = 1 */
        words[layer_i] = f;
        trees[layer_i] = merkle_tree_rowmajor(f, 8, log_len - 1);
        memcpy(proof->fri_roots[layer_i], trees[layer_i] + 8 * (((size_t)2 << (log_len - 1)) - 2), 32);
        orc_challenger_observe(&ch, proof->fri_roots[layer_i], 8);
        orc_challenger_sample_ext(&ch, proof->fri_betas[layer_i]);
        uint32_t* nf = (uint32_t*)malloc(4 * ((size_t)1 << (log_len - 1)) * sizeof(uint32_t));
        orc_fri_fold(f, log_len, shift, proof->fri_betas[layer_i], nf);
        f = nf;
        shift = bb_mul(shift, shift);
        log_len--;
        layer_i++;
        if (log_len > 1 && ro[log_len]) {
            for (size_t i = 0; i < ((size_t)4 << log_len); i++) f[i] = bb_add(f[i], ro[log_len][i]);
            free(ro[log_len]);
            ro[log_len] = NULL;
        }
    }
    proof->n_fri_layers = layer_i;
    proof->final_len = 2;
    memcpy(proof->final_poly, f, 32);
    free(f);
    orc_challenger_observe(&ch, proof->final_poly[0], 4);
    st[7] = lap(&t);

    /* proof of work, then the query phase */
    proof->pow_witness = orc_grind(&ch, prm->pow_bits);
    orc_challenger_observe(&ch, &proof->pow_witness, 1);
    (void)orc_challenger_sample(&ch);
    st[8] = lap(&t);
    if (prm->n_queries && queries_out) {
        const size_t wpq = orc_chips_query_words(chips, K);
        for (size_t qi = 0; qi < prm->n_queries; qi++) {
            uint32_t* o = queries_out + qi * wpq;
            const size_t r = orc_challenger_sample(&ch) & (((size_t)1 << hmax) - 1);
            *o++ = (uint32_t)r;
            for (size_t c = 0; c < K; c++) {
                const unsigned lm = chips[c].log_n + 1;
                const size_t m = (size_t)1 << lm, rr = r >> (hmax - lm);
                for (size_t j = 0; j < chips[c].width; j++) *o++ = lde[c][j * m + rr];
            }
            copy_path(tree_m, hmax, r, o);
            o += 8 * hmax;
            if (any_lu) {
                for (size_t c = 0; c < K; c++) {
                    if (!wp[c]) continue;
                    const unsigned lm = chips[c].log_n + 1;
                    const size_t m = (size_t)1 << lm, rr = r >> (hmax - lm);
                    for (size_t j = 0; j < wp[c]; j++) *o++ = plde[c][j * m + rr];
                }
                copy_path(tree_p, hperm, r >> (hmax - hperm), o);
                o += 8 * hperm;
            }
            for (size_t c = 0; c < K; c++) {
                const unsigned lm = chips[c].log_n + 1;
                const size_t m = (size_t)1 << lm, rr = r >> (hmax - lm);
                for (size_t j = 0; j < 8; j++) *o++ = qlde[c][j * m + rr];
            }
            copy_path(tree_q, hq, r, o);
            o += 8 * hq;
            for (unsigned i = 0; i < layer_i; i++) {
                const unsigned lh = hmax - 1 - i;
                const size_t j = r >> (i + 1);
                memcpy(o, words[i] + 8 * j, 32);
                o += 8;
                copy_path(trees[i], lh, j, o);
                o += 8 * lh;
            }
        }
    }
    st[9] = lap(&t);
    if (stage_seconds) memcpy(stage_seconds, st, sizeof st);
    for (unsigned i = 0; i < layer_i; i++) { free(words[i]); free(trees[i]); }
    for (unsigned h = 0; h < 32; h++) free(ro[h]);
    for (size_t c = 0; c < K; c++) { free(lde[c]); free(perm[c]); free(plde[c]); free(qlde[c]); free(nat[c]); free(cstart[c]); }
    free(lde); free(perm); free(plde); free(qlde); free(nat); free(cstart); free(wp); free(nch); free(mm);
    free(tree_m); free(tree_p); free(tree_q); free(ys); free(oc);
}
