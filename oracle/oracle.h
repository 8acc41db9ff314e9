/*
 * ORACLE (test infrastructure, not product code) -- public entry points of the CPU restatement.
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may call this.
 * All field values crossing this API are CANONICAL u32 in [0, p).  Matrices are COLUMN-MAJOR
 * (element (row r, col c) at c*height + r), the layout of the reference's DeviceMatrix
 * (/root/reference/openvm/cuda/src/apc_tracegen.cu:13,36).
 *
 * PARITY STATUS: stage 0 (tracegen) and the expression/bytecode semantics of stage 2 are pinned by
 * in-tree reference sources and fixtures.  Stages 1 and 3 (LDE, Poseidon2/Merkle, FRI) restate the
 * published Plonky3 algorithms; the reference tree holds no source, golden vector or KAT for them
 * => "parity unpinned" against the reference for those stages (SURVEY.md §8c).
 */
#ifndef PB_ORACLE_H
#define PB_ORACLE_H
#include <stdint.h>
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

/* ---- stage 1: NTT / coset LDE ---- */
void orc_dft_naive(const uint32_t* in, uint32_t* out, unsigned log_n, uint32_t shift);      /* O(n^2), out[k] = f(shift*w^k) from coeffs */
void orc_ntt(uint32_t* a, unsigned log_n);            /* in-place, natural in -> natural out, evaluations of coeffs on <w_n> */
void orc_intt(uint32_t* a, unsigned log_n);           /* inverse of orc_ntt */
/* evals of W columns over the subgroup H (natural order) -> evals over shift*H' (|H'| = 2^log_blowup |H|),
   rows in BIT-REVERSED order (Plonky3 TwoAdicFriPcs::commit convention, SURVEY.md App. C.1). */
void orc_lde_batch(const uint32_t* trace, unsigned log_n, size_t width, unsigned log_blowup, uint32_t shift, uint32_t* lde);

/* ---- Poseidon2 (width 16, x^7, 8 full + 13 partial) ---- */
void orc_poseidon2_permute(uint32_t state[16]);
void orc_poseidon2_permute_with(uint32_t state[16], const uint32_t* rc_ext, const uint32_t* rc_int, const uint32_t* diag);
/* install the instantiation (canonical rc_ext [8][16], rc_int [13], diag [16]) that orc_poseidon2_permute and everything built on it
   uses; reset: back to the default.  Process-wide: not to be changed while another thread hashes.  fast.c keeps the default. */
void orc_set_poseidon2(const uint32_t* rc_ext, const uint32_t* rc_int, const uint32_t* diag);
void orc_reset_poseidon2(void);
void orc_hash_row(const uint32_t* row, size_t len, uint32_t digest[8]);     /* PaddingFreeSponge<16,8,8>: overwrite-mode absorb */
void orc_compress(const uint32_t l[8], const uint32_t r[8], uint32_t out[8]); /* TruncatedPermutation<2,8,16> */

/* ---- stage 3a: Merkle tree (MerkleTreeMmcs over matrices of equal height) ----
   mats[i] column-major, height 2^log_h, width widths[i]; leaf r = sponge(row r of mat0 || row r of mat1 ...).
   digest_layers: node-major, 8 words per node; layer 0 = 2^log_h leaves, then 2^(log_h-1) ... root.
   Total nodes = 2^(log_h+1) - 1. */
void orc_merkle_commit(const uint32_t* const* mats, const size_t* widths, size_t n_mats, unsigned log_h, uint32_t* digest_layers);

/* ---- stage 2: constraint evaluation ----
   Stack-machine bytecode with the reference opcode set (/root/reference/openvm/cuda/src/expr_eval.cuh:12-20):
   0 PUSH_APC idx, 1 PUSH_CONST c, 2 ADD, 3 SUB, 4 MUL, 5 NEG, 6 INV_OR_ZERO.  For orc_eval_expr the PUSH_APC
   operand is an absolute element offset (col*H, as the reference encodes it: cuda/mod.rs:61) and `r` is added. */
typedef struct { uint32_t off, len; } orc_span_t;
uint32_t orc_eval_expr(const uint32_t* bc, uint32_t len, const uint32_t* mat, size_t r);
/* quotient over the LDE domain (log_blowup = 1: quotient domain == LDE domain g*H', bit-reversed rows).
   PUSH_APC operand here is a COLUMN INDEX (height independent).  For each lde row: acc = sum_k alpha^(C-1-k) c_k(row)
   (Horner in declaration order, SURVEY.md App. C.2), q = acc * Z_H(x)^-1, Z_H(x)=x^N-1.  Output: quotient[(chunk*4+limb)*N + j]
   where chunk = top bit of the bit-reversed row (= natural index parity) and j = low bits (bit-reversed order within chunk). */
void orc_quotient(const uint32_t* bc, const orc_span_t* spans, size_t n_constraints, const uint32_t* lde, unsigned log_n,
                  unsigned log_blowup, uint32_t shift, const uint32_t alpha[4], uint32_t* quotient);
/* raw folded constraint value per row, no vanishing division (used for parity on random traces) */
void orc_constraint_fold(const uint32_t* bc, const orc_span_t* spans, size_t n_constraints, const uint32_t* mat, size_t height,
                         const uint32_t alpha[4], uint32_t* out4 /* [4][height] */);

/* ---- stage 3b: FRI fold (arity 2, bit-reversed evaluations over shift*<w_len>) ----
   in: len=2^log_len ext elements as [len][4]; out [len/2][4].  out[j] = (lo+hi)/2 + beta*(lo-hi)/(2 x_j). */
void orc_fri_fold(const uint32_t* in, unsigned log_len, uint32_t shift, const uint32_t beta[4], uint32_t* out);

/* ---- openings + DEEP reduced opening (row f-4 of SURVEY.md §8, widened in round 1) ---- */
void orc_eval_at_point(const uint32_t* mat, unsigned log_n, size_t width, uint32_t shift, const uint32_t zeta[4], uint32_t* out);
/* -1 (nothing written) when zeta lies on the LDE domain shift*H' */
int orc_deep_quotient(const uint32_t* const* mats, const size_t* widths, size_t n_mats, unsigned log_m, uint32_t shift,
                      const uint32_t zeta[4], const uint32_t gamma[4], const uint32_t* ys, uint32_t* out);

/* ---- DuplexChallenger<BabyBear, Perm16, 16, 8> ---- */
typedef struct { uint32_t sponge[16]; uint32_t in_buf[8]; int n_in; uint32_t out_buf[8]; int n_out; } orc_challenger_t;
void orc_challenger_init(orc_challenger_t* c);
void orc_challenger_observe(orc_challenger_t* c, const uint32_t* vals, size_t n);
uint32_t orc_challenger_sample(orc_challenger_t* c);
void orc_challenger_sample_ext(orc_challenger_t* c, uint32_t out[4]);

/* ---- stage 0: APC trace generation (CPU mirror of the three reference kernels) ---- */
typedef struct { int32_t width, height; const uint32_t* buffer; int32_t row_block_size; } orc_original_air_t;
typedef struct { int32_t air_index, col, row, apc_col; } orc_subst_t;
typedef struct { uint64_t col_base; orc_span_t span; } orc_derived_spec_t;
typedef struct { uint32_t bus_id, num_args, args_index_off; } orc_interaction_t;
void orc_apc_tracegen(uint32_t* out, size_t H, const orc_original_air_t* airs, const orc_subst_t* subs, size_t n_subs, int num_apc_calls);
void orc_apc_apply_derived_expr(uint32_t* out, size_t H, int num_apc_calls, const orc_derived_spec_t* specs, size_t n_cols, const uint32_t* bc);
void orc_apc_apply_bus(const uint32_t* out, int num_apc_calls, const uint32_t* bc, const orc_interaction_t* ints, size_t n_ints,
                       const orc_span_t* arg_spans, uint32_t var_range_bus_id, uint32_t* var_hist, size_t var_num_bins,
                       uint32_t tuple2_bus_id, uint32_t* tuple2_hist, uint32_t sz0, uint32_t sz1,
                       uint32_t bitwise_bus_id, uint32_t* bitwise_hist);

/* ---- LogUp / bus-interaction argument (logup.c) ---- */
int orc_logup_chunks(const uint32_t* ibc, const orc_span_t* isp, const orc_interaction_t* ints, size_t n_ints, unsigned max_degree,
                     uint32_t* chunk_start /* n_ints + 1 entries */);
void orc_logup_perm_trace(const uint32_t* trace, unsigned log_n, const uint32_t* ibc, const orc_span_t* isp, const orc_interaction_t* ints,
                          size_t n_ints, const uint32_t* chunk_start, size_t n_chunks, const uint32_t alpha_lu[4], const uint32_t beta_lu[4],
                          uint32_t* perm /* [4*(n_chunks+1)][N] */, uint32_t cumsum[4]);
void orc_logup_fold(const uint32_t* lde, const uint32_t* perm_lde, unsigned log_n, uint32_t shift, const uint32_t* ibc, const orc_span_t* isp,
                    const orc_interaction_t* ints, size_t n_ints, const uint32_t* chunk_start, size_t n_chunks, const uint32_t alpha_lu[4],
                    const uint32_t beta_lu[4], const uint32_t cumsum[4], const uint32_t alpha[4], uint32_t* acc4 /* [4][2N] in/out */);
/* reduced opening over several (column group, point) pairs, column j weighted by gamma_pows[j] -- see ntt.c */
void orc_deep_quotient_groups(const uint32_t* const* cols, const uint32_t* group_of_col, size_t n_cols, const uint32_t* zs, size_t n_groups,
                              unsigned log_m, uint32_t shift, const uint32_t* gamma_pows, const uint32_t* ys, uint32_t* out);

/* ---- all chips of a segment (the metric's unit of work) under ONE transcript, v2 (DESIGN.md §3, §3b; prove.c, verify.c) ----
   main commit -> [LogUp challenges, permutation trace commit, cumulative sums] -> alpha -> quotient commit -> zeta ->
   openings (every opened value observed) -> gamma -> FRI commit phase -> final polynomial observed -> proof-of-work -> queries.
   Mixed-height MMCS commitments, shared challenges, one FRI instance.  A single segment is a one-chip proof. */
typedef struct {
    const uint32_t* bc; const orc_span_t* spans; size_t n_constraints;                              /* polynomial identities */
    const uint32_t* ibc; const orc_span_t* ispans; const orc_interaction_t* ints; size_t n_ints;   /* bus interactions (may be 0) */
} orc_air_t;
typedef struct {
    uint32_t n_queries, pow_bits;
    int fast;             /* 1: AVX-512 primitives of fast.c where available */
    int cheat_opening;    /* test hook: a dishonest prover that claims main_col0(zeta) + 1 -- its reduced opening is not a polynomial */
} orc_params_t;
size_t orc_perm_width(const orc_air_t* air);
/* proof-of-work grinding on a challenger state: smallest witness w with (observe(w); sample() & (2^bits - 1)) == 0 */
uint32_t orc_grind(const orc_challenger_t* c, unsigned bits);
typedef struct { const orc_air_t* air; const uint32_t* trace; unsigned log_n; size_t width; } orc_chip_t;
typedef struct {
    uint32_t main_root[8], perm_root[8], quotient_root[8];
    uint32_t logup_alpha[4], logup_beta[4];        /* zero when no chip has interactions */
    uint32_t alpha[4], zeta[4] /* out-of-domain opening point */, gamma[4] /* batching challenge of the reduced opening */;
    uint32_t n_fri_layers;
    uint32_t fri_roots[32][8];
    uint32_t fri_betas[32][4];
    uint32_t final_poly[8][4];     /* last layer (length 2^log_blowup): evaluations of the constant final polynomial */
    uint32_t final_len;
    uint32_t pow_witness;
    uint32_t pow_bits, n_queries, n_chips, log_max;       /* log_max: log2 of the tallest LDE */
} orc_chips_proof_t;
size_t orc_chips_num_opened(const orc_chip_t* chips, size_t n_chips);
size_t orc_chips_query_words(const orc_chip_t* chips, size_t n_chips);
/* cumsums: [n_chips][4] (zero for chips without interactions); ys_out: [orc_chips_num_opened][4] = main at zeta (chip order) | per chip with
   interactions perm at zeta, perm at zeta*w_chip | quotient chunks at zeta (chip order); queries_out: [n_queries][orc_chips_query_words].
   query layout: [ r | main rows of all chips (row r >> (log_max - log_m_chip)) | main path (log_max x 8) | perm rows of the chips with
   interactions | perm path (both absent when no chip has interactions) | quotient rows (8 per chip) | quotient path | per FRI layer: pair (8), path ]
   stage_seconds[10] (NULL: not clocked): lde, merkle, logup_gen, logup_commit, quotient, quotient_commit, openings, fri_commit, pow, query */
void orc_prove_chips(const orc_chip_t* chips, size_t n_chips, const orc_params_t* prm, orc_chips_proof_t* proof, uint32_t* cumsums, uint32_t* ys_out,
                     uint32_t* queries_out, double stage_seconds[10]);
/* independent verifier (only the shapes of the chips are read, not their traces); 0 = accept, else the failed check:
   1 logup challenges 2 alpha 3 zeta 4 gamma 5 beta 6 proof of work 7 query index 8 main path 9 perm path 10 quotient path
   (8/9/10: MMCS openings) 11 reduced opening != FRI layer 0 12 FRI path 13 fold consistency 14 final polynomial value
   15 final polynomial not constant 16 constraint identity at zeta 20 malformed */
int orc_verify_chips(const orc_chip_t* chips_without_traces, size_t n_chips, const orc_chips_proof_t* proof, const uint32_t* cumsums, const uint32_t* ys,
                     const uint32_t* queries, int check_constraints);

/* ---- AVX-512 Montgomery implementations of the heavy primitives (fast.c), same semantics ---- */
int orcf_available(void);
void orcf_lde_batch(const uint32_t* trace, unsigned log_n, size_t width, unsigned log_blowup, uint32_t shift, uint32_t* lde);
void orcf_merkle_commit(const uint32_t* const* mats, const size_t* widths, size_t n_mats, unsigned log_h, uint32_t* digest_layers);
void orcf_constraint_fold(const uint32_t* bc, const orc_span_t* spans, size_t n_constraints, const uint32_t* mat, size_t height,
                          const uint32_t alpha[4], uint32_t* out4);
void orcf_quotient(const uint32_t* bc, const orc_span_t* spans, size_t n_constraints, const uint32_t* lde, unsigned log_n,
                   unsigned log_blowup, uint32_t shift, const uint32_t alpha[4], uint32_t* quotient);
void orcf_eval_at_point(const uint32_t* mat, unsigned log_n, size_t width, uint32_t shift, const uint32_t zeta[4], uint32_t* out);
int orcf_deep_quotient(const uint32_t* const* mats, const size_t* widths, size_t n_mats, unsigned log_m, uint32_t shift,
                       const uint32_t zeta[4], const uint32_t gamma[4], const uint32_t* ys, uint32_t* out);
void orcf_logup_perm_trace(const uint32_t* trace, unsigned log_n, const uint32_t* ibc, const orc_span_t* isp, const orc_interaction_t* ints,
                           size_t n_ints, const uint32_t* chunk_start, size_t n_chunks, const uint32_t alpha_lu[4], const uint32_t beta_lu[4],
                           uint32_t* perm, uint32_t cumsum[4]);
void orcf_logup_fold(const uint32_t* lde, const uint32_t* perm_lde, unsigned log_n, uint32_t shift, const uint32_t* ibc, const orc_span_t* isp,
                     const orc_interaction_t* ints, size_t n_ints, const uint32_t* chunk_start, size_t n_chunks, const uint32_t alpha_lu[4],
                     const uint32_t beta_lu[4], const uint32_t cumsum[4], const uint32_t alpha[4], uint32_t* acc4);
void orcf_deep_quotient_groups(const uint32_t* const* cols, const uint32_t* group_of_col, size_t n_cols, const uint32_t* zs, size_t n_groups,
                               unsigned log_m, uint32_t shift, const uint32_t* gamma_pows, const uint32_t* ys, uint32_t* out);
int orc_num_threads(void);
void* orc_big_alloc(size_t bytes);   /* 2 MB aligned, MADV_HUGEPAGE */
void orc_big_free(void* p);
#ifdef __cplusplus
}
#endif
#endif
