/*
 * powdr_b200 -- C ABI of the H100-native STARK proving hot path for powdr autoprecompile (APC) chips over BabyBear.
 *
 * Conventions (copied from the reference's only in-tree FFI, /root/reference/openvm/src/cuda_abi.rs:8-64):
 *   - every entry point returns int: 0 = ok, a positive cudaError_t, or a negative PB_ERR_* code; nothing aborts;
 *   - device buffers are raw pointers + explicit sizes, allocated and owned by the caller;
 *   - kernels are enqueued on the context's stream and NOT synchronised (except where a host result is returned);
 *   - matrices are COLUMN-MAJOR (element (row r, col c) at c*height + r) -- DeviceMatrix<BabyBear>
 *     (/root/reference/openvm/cuda/src/apc_tracegen.cu:13,36);
 *   - field elements in device/host data buffers are u32 in MONTGOMERY form (R = 2^32), the in-memory form of
 *     p3_baby_bear::BabyBear / the device Fp.  Scalars passed by value in arguments (shift, alpha, beta, constants)
 *     are CANONICAL u32 in [0,p), like `PushConst` operands (/root/reference/openvm/src/powdr_extension/trace_generator/cuda/mod.rs:57-58).
 *
 * Reference interfaces each group replaces are cited per function; the Rust-side bindings are in INTEGRATION.md.
 */
#ifndef POWDR_B200_H
#define POWDR_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define PB_ERR_INVALID_ARG (-1)
#define PB_ERR_UNSUPPORTED (-2)
#define PB_ERR_STACK_DEPTH (-3)   /* expression needs more than 16 stack slots (STACK_CAPACITY, expr_eval.cuh:22) */
#define PB_ERR_BAD_BYTECODE (-4)
#define PB_ERR_NO_DEVICE (-5)
#define PB_ERR_COMM (-6)          /* a caller-supplied collective (pb_comm_t) reported failure */
#define PB_ERR_INTERNAL (-7)      /* a self-check failed (the host replay of the device-driven FRI transcript disagreed): a bug */
#define PB_ERR_REJECTED (-8)      /* pb_verify_*: the proof is not accepted; *reason says which check failed */

#define PB_BABYBEAR_P 2013265921u
#define PB_DIGEST_WORDS 8

typedef struct pb_ctx pb_ctx_t;   /* device + stream + twiddle/constant caches + scratch */
typedef struct pb_air pb_air_t;   /* compiled constraint program of one APC AIR */

/* ---- context -------------------------------------------------------------------------------------------------
 * Replaces the implicit "default stream + global device state" of the reference launchers (apc_tracegen.cu:139-145).
 * `cuda_stream` is a cudaStream_t (NULL = default stream). */
int pb_ctx_create(pb_ctx_t** out, int device, void* cuda_stream);
int pb_ctx_destroy(pb_ctx_t* ctx);
int pb_ctx_synchronize(pb_ctx_t* ctx);
/* Poseidon2 instantiation as data (canonical values): 8x16 external round constants (4 initial then 4 terminal),
 * 13 internal, 16-entry internal diagonal V (matrix 1 + diag(V)).  Default = include/pb_poseidon2_constants.h (Plonky3's
 * default BabyBear width-16 instance).  The DEVICE copy is one __constant__ bank per process and GPU: setting it on one context
 * changes the hashing of every context of this process on that GPU -- use one instantiation per process.  pb_ctx_create puts
 * the default back in that bank: a context that set other constants before then proves with a device that disagrees with its
 * transcript, and its proofs end in PB_ERR_INTERNAL. */
int pb_ctx_set_poseidon2(pb_ctx_t* ctx, const uint32_t rc_ext[8][16], const uint32_t rc_int[13], const uint32_t diag_m1[16]);

/* pinned host memory + representation helpers */
int pb_host_alloc(void** out, size_t bytes);
int pb_host_free(void* p);
int pb_device_alloc(void** out, size_t bytes);
int pb_device_free(void* p);
/* stream-ordered copies, the MemCopyH2D::to_device / to_host of openvm-cuda-common (use-sites cuda/mod.rs:331-355) */
int pb_copy_h2d(pb_ctx_t* ctx, void* d_dst, const void* h_src, size_t bytes);
int pb_copy_d2h(pb_ctx_t* ctx, void* h_dst, const void* d_src, size_t bytes);   /* synchronises the stream */
int pb_memset_zero(pb_ctx_t* ctx, void* d_dst, size_t bytes);                    /* DeviceBuffer::fill_zero */
int pb_to_monty(pb_ctx_t* ctx, uint32_t* d_buf, size_t n);     /* in place, canonical -> Montgomery */
int pb_from_monty(pb_ctx_t* ctx, uint32_t* d_buf, size_t n);   /* in place, Montgomery -> canonical */

/* ---- stage 1: coset LDE (replaces the backend's main_trace_commit LDE; SURVEY.md §8 a6) -------------------------
 * d_trace: width columns of 2^log_n evaluations over the subgroup H, natural row order.
 * d_lde:   width columns of 2^(log_n+log_blowup) evaluations over shift*H', rows BIT-REVERSED. */
int pb_lde_batch(pb_ctx_t* ctx, const uint32_t* d_trace, size_t log_n, size_t width, uint32_t log_blowup, uint32_t shift,
                 uint32_t* d_lde);

/* ---- stage 2: constraint evaluation / quotient (replaces quotient_poly_compute over PowdrAir::eval,
 *      /root/reference/openvm/src/powdr_extension/chip.rs:94-130) --------------------------------------------------
 * Bytecode = the reference stack machine (/root/reference/openvm/cuda/src/expr_eval.cuh:12-20) with the PUSH_APC operand
 * being the COLUMN INDEX (height independent) and PUSH_CONST a canonical u32. */
typedef struct { uint32_t off; uint32_t len; } pb_expr_span_t;   /* == ExprSpan, cuda_abi.rs:162-169 */
int pb_air_compile(pb_ctx_t* ctx, const uint32_t* bytecode, size_t n_words, const pb_expr_span_t* constraints,
                   size_t n_constraints, uint32_t width, pb_air_t** out);
int pb_air_free(pb_air_t* air);
/* NOTE: a pb_air_t owns small per-proof device buffers (alpha powers, LogUp constants): one proof at a time per handle -- concurrent
 * provers (e.g. one per GPU) compile their own handle, which is also what binds the kernels to their device's CUDA context. */
/* 1 when the AIR runs on its NVRTC-generated straight-line kernel, 0 when on the bytecode interpreter kernel */
int pb_air_is_jit(const pb_air_t* air);
/* host-only check of the code generator: packs the program, generates CUDA C and compiles it for sm_90a (no device needed) */
int pb_air_jit_compile_only(const uint32_t* bytecode, size_t n_words, const pb_expr_span_t* constraints, size_t n_constraints,
                            uint32_t width, size_t* cubin_bytes);
/* d_quotient: [2 chunks][4 limbs][2^log_n], chunk = parity of the natural LDE index (= top bit of the bit-reversed row),
 * rows inside a chunk in bit-reversed order.  log_blowup must be 1 (constraint degree <= 3, openvm/src/lib.rs:97-101). */
int pb_quotient(pb_ctx_t* ctx, const pb_air_t* air, const uint32_t* d_lde, size_t log_n, uint32_t log_blowup, uint32_t shift,
                const uint32_t alpha[4], uint32_t* d_quotient);
/* raw alpha-fold of all constraints on every row of any column-major matrix: d_out [4][height] */
int pb_constraint_fold(pb_ctx_t* ctx, const pb_air_t* air, const uint32_t* d_mat, size_t height, const uint32_t alpha[4],
                       uint32_t* d_out);

/* ---- stage 3a: Poseidon2 Merkle tree (replaces MerkleTreeMmcs::commit of the backend; SURVEY.md §8 a8) -------------
 * d_mats[i]: column-major, height 2^log_height, width widths[i]; leaf r = sponge(row r of mat 0 || row r of mat 1 ...).
 * d_digest_layers: (2^(log_height+1) - 1) * 8 words, node-major: 2^log_height leaves, then each parent layer, root last.
 * root_out (host, canonical, may be NULL): synchronises the stream when given. */
int pb_merkle_commit(pb_ctx_t* ctx, const uint32_t* const* d_mats, const size_t* widths, size_t n_mats, size_t log_height,
                     uint32_t* d_digest_layers, uint32_t root_out[8]);
/* same tree over ONE row-major matrix of width 8 (a FRI layer: row j = the fold pair (f[2j], f[2j+1])) */
int pb_merkle_commit_rows8(pb_ctx_t* ctx, const uint32_t* d_rows, size_t log_height, uint32_t* d_digest_layers, uint32_t root_out[8]);
/* n independent permutations of [n][16] states, in place (tests, micro-benchmarks) */
int pb_poseidon2_permute(pb_ctx_t* ctx, uint32_t* d_states, size_t n, int reps);
/* the same on the 16-lanes-per-permutation form that Merkle tops, short leaf sponges and the FRI challenges run on (tests,
 * micro-benchmarks) */
int pb_poseidon2_permute_coop(pb_ctx_t* ctx, uint32_t* d_states, size_t n);

/* ---- stage 3b: FRI fold (replaces the commit-phase fold of pcs_opening; SURVEY.md §8 a9) -----------------------------
 * d_in: 2^log_len Ext4 elements [len][4], bit-reversed evaluations over shift*<w_len>; d_out: [len/2][4]. */
int pb_fri_fold(pb_ctx_t* ctx, const uint32_t* d_in, size_t log_len, uint32_t shift, const uint32_t beta[4], uint32_t* d_out);

/* ---- openings + reduced opening (the opening phase of pcs_opening; SURVEY.md §8f-4, widened in round 1) -------------------
 * pb_eval_at_point: y_k = f_k(zeta) for `width` columns given as 2^log_n evaluations over shift*H (natural order), f_k the
 *   polynomial of degree < 2^log_n through them; any zeta, including a point shift*w^i of shift*H, where y_k is row i of column k.
 *   d_ys: [width][4] Ext4 values (Montgomery limbs).
 * pb_deep_quotient: ro[r] = (sum_j gamma^j (f_j[r] - y_j)) / (x_r - zeta) over the LDE domain shift*H' (bit-reversed rows),
 *   j over all columns of d_mats in order; d_ys as produced by pb_eval_at_point; d_out: [2^log_m][4]. Synchronises (reads d_ys).
 *   zeta on shift*H' (a base-field zeta with (zeta/shift)^(2^log_m) = 1), where x_r - zeta = 0 at one row, is PB_ERR_UNSUPPORTED,
 *   returned before any kernel is launched. */
int pb_eval_at_point(pb_ctx_t* ctx, const uint32_t* d_mat, size_t log_n, size_t width, uint32_t shift, const uint32_t zeta[4],
                     uint32_t* d_ys);
int pb_deep_quotient(pb_ctx_t* ctx, const uint32_t* const* d_mats, const size_t* widths, size_t n_mats, size_t log_m, uint32_t shift,
                     const uint32_t zeta[4], const uint32_t gamma[4], const uint32_t* d_ys, uint32_t* d_out);

/* ---- whole segment: the metric's unit of work ------------------------------------------------------------------------
 * Replaces engine.prove(pk, ProvingContext{common_main}) for one APC chip behind sdk.app_prover(exe)?.prove(stdin)
 * (/root/reference/openvm-riscv/src/lib.rs:327-332; AirProvingContext built at
 * /root/reference/openvm/src/powdr_extension/trace_generator/cuda/mod.rs:415-419).  Stages, in the V1 metric names of
 * /root/reference/openvm/metrics-viewer/CLAUDE.md:52-78: main_trace_commit (LDE + Merkle), perm_trace_commit (the LogUp
 * permutation trace of the AIR's bus interactions: generated, LDE'd, committed), quotient_poly_compute, quotient_poly_commit,
 * pcs_opening (openings at zeta / zeta*w, reduced opening, FRI commit phase, proof of work, queries).
 * Transcript v2 is documented in DESIGN.md §3 (CPU restatement and independent verifier live in the test tree). */
typedef struct {
    uint32_t trace_root[8];
    uint32_t logup_alpha[4], logup_beta[4];   /* LogUp challenges; zero when the AIR has no interactions */
    uint32_t perm_root[8];
    uint32_t cumulative_sum[4];               /* exposed value phi(N-1) of the running sum */
    uint32_t alpha[4];
    uint32_t quotient_root[8];
    uint32_t zeta[4];              /* out-of-domain opening point */
    uint32_t gamma[4];             /* batching challenge of the reduced opening */
    uint32_t n_fri_layers;
    uint32_t fri_roots[32][8];
    uint32_t fri_betas[32][4];
    uint32_t final_poly[8][4];     /* last FRI layer (2^log_blowup evaluations of the constant final polynomial) */
    uint32_t final_len;
    uint32_t pow_witness;
    uint32_t pow_bits, n_queries, perm_width;
} pb_segment_proof_t;               /* all values canonical */
#define PB_TRACE_ON_DEVICE 1u       /* `trace` is a device pointer (value-only timing); else host memory, copied in */
/* FRI parameters of the context; default 100 queries, 16 proof-of-work bits (the reference's app configuration for
 * log_blowup 1: standard_fri_params_with_100_bits_conjectured_security in the un-vendored SDK -- recollection) */
int pb_ctx_set_fri_params(pb_ctx_t* ctx, uint32_t n_queries, uint32_t pow_bits);
int pb_prove_segment(pb_ctx_t* ctx, const pb_air_t* air, const uint32_t* trace, size_t log_n, size_t width, uint32_t flags,
                     pb_segment_proof_t* proof);
/* ---- query phase: the state of the last pb_prove_segment stays on the device ----------------------------------------------
 * pb_query_segment samples n_queries indices from the transcript (sample_bits(log_m) each, continuing after the proof of work)
 * and gathers, per query (canonical words, pb_query_words of them):
 *   [ r | trace LDE row (width) | trace path (log_m x 8) | perm LDE row (perm_width) | perm path (log_m x 8)  (both absent
 *     when perm_width = 0) | quotient row (8) | quotient path (log_m x 8) | per FRI layer i: opened pair row (8), path ((log_m-1-i) x 8) ]
 * pb_last_openings: the opened values, [(width + 2*perm_width + 8)][4] canonical:
 *   main at zeta | perm at zeta | perm at zeta*w | quotient chunks at zeta. */
/* ONE proof state per context: pb_prove_segment, pb_prove_segment_sharded, pb_prove_chips and pb_prove_chips_sharded share workspaces, so
 * each of them, even when it fails, invalidates the query state of any earlier proof of the context; each pb_query_* answers only for a
 * proof of its own prover, pb_last_openings for pb_prove_segment and pb_prove_segment_sharded (otherwise they return PB_ERR_INVALID_ARG). */
int pb_query_words(size_t log_n, size_t width, size_t perm_width, size_t* words_per_query);
int pb_query_segment(pb_ctx_t* ctx, uint32_t* h_out, size_t out_capacity_words);
int pb_last_openings(pb_ctx_t* ctx, uint32_t* h_ys, size_t capacity_words);

/* ---- all chips of a segment under ONE transcript -----------------------------------------------------------------------
 * Replaces engine.prove(pk, ProvingContext{per_air}) with SEVERAL AIRs: the reference collects one AirProvingContext per chip of
 * the segment (/root/reference/openvm/src/powdr_extension/trace_generator/cuda/mod.rs:415-419 for the APC chip, the VM's other
 * chips beside it) and proves them in one call (/root/reference/openvm-riscv/src/lib.rs:327-332).  Chips have different heights:
 *   - three commitments (main, permutation, quotient), each a mixed-height MMCS (Plonky3 MerkleTreeMmcs): leaves hash the rows of
 *     the tallest matrices; at the level whose size equals a shorter height, node = compress(compress(l, r), hash(rows there));
 *   - LogUp challenges, alpha, zeta, gamma are shared; every chip with interactions exposes its own cumulative sum (the verifier
 *     checks that they add up to zero over the segment);
 *   - opened values in observation order: main at zeta (chip order) | per chip with interactions: perm at zeta, perm at zeta*w_chip |
 *     quotient chunks at zeta (chip order); column j of that list is batched with gamma^j;
 *   - ONE FRI: a reduced-opening codeword per distinct LDE height; folding starts from the tallest, and the codeword of a shorter
 *     height is added to the folded codeword when the fold reaches that height; final polynomial, proof of work and queries as in
 *     pb_prove_segment.  A query index r has log_max bits; the matrix of a chip with LDE height 2^h opens row r >> (log_max - h).
 * With one chip the proof equals pb_prove_segment's.  Traces are device-resident (Montgomery, column-major) and must stay valid
 * until the last pb_query_chips. */
typedef struct { const pb_air_t* air; const uint32_t* d_trace; size_t log_n; size_t width; } pb_chip_t;
typedef struct {
    uint32_t main_root[8], perm_root[8], quotient_root[8];
    uint32_t logup_alpha[4], logup_beta[4], alpha[4], zeta[4], gamma[4];
    uint32_t n_fri_layers;
    uint32_t fri_roots[32][8];
    uint32_t fri_betas[32][4];
    uint32_t final_poly[8][4];
    uint32_t final_len;
    uint32_t pow_witness;
    uint32_t pow_bits, n_queries, n_chips, log_max;   /* log_max: log2 of the tallest LDE */
} pb_chips_proof_t;                  /* all values canonical */
/* h_cumsums: [n_chips][4] canonical (zero for chips without interactions) */
int pb_prove_chips(pb_ctx_t* ctx, const pb_chip_t* chips, size_t n_chips, pb_chips_proof_t* proof, uint32_t* h_cumsums);
/* pb_prove_chips with every chips[c].d_trace in HOST memory, in the same layout (Montgomery, column-major, width x 2^log_n): the same
 * proof and cumulative sums, and pb_query_chips then returns the same opened values and query words, word for word.  The traces are
 * copied to the device behind the work on them: their columns stream over PCIe in chunks, grouped by LDE height (tallest first), and
 * the copy of a chunk overlaps the LDE and the leaf hashing of the one before (DESIGN.md §3b).  Pinned memory (pb_host_alloc) gives
 * that overlap; pageable memory gives the same proof without it.  The library keeps its own device copy, counted in the footprint: the
 * host buffers may be freed or overwritten as soon as the call returns.  Argument checks, error codes and the proof state as
 * pb_prove_chips's (pb_query_chips answers for it).  pb_prove_segment without PB_TRACE_ON_DEVICE is the one-chip case. */
int pb_prove_chips_host(pb_ctx_t* ctx, const pb_chip_t* chips, size_t n_chips, pb_chips_proof_t* proof, uint32_t* h_cumsums);
/* n_opened Ext4 values; words per query of the layout
 *   [ r | main rows of all chips | main path (log_max x 8) | perm rows of the chips with interactions | perm path (tallest such chip) |
 *     quotient rows (8 per chip) | quotient path | per FRI layer i: pair (8), path ((log_max-1-i) x 8) ] */
int pb_chips_sizes(const pb_chip_t* chips, size_t n_chips, size_t* n_opened, size_t* words_per_query);
/* queries ([n_queries][words_per_query], may be NULL) and opened values ([n_opened][4], may be NULL) of the last pb_prove_chips or
 * pb_prove_chips_host */
int pb_query_chips(pb_ctx_t* ctx, uint32_t* h_queries, size_t queries_capacity_words, uint32_t* h_ys, size_t ys_capacity_words);

/* ---- device memory of the single-GPU provers (pb_prove_segment, pb_prove_chips) ---------------------------------------------
 * A proof whose footprint fits the budget keeps every committed matrix resident (the LDEs of the traces and permutation traces).  One
 * that does not is proved in B = 2^log_blocks row blocks, 2 <= B <= 16: the chips of its tallest LDE heights keep their coefficients
 * (the permutation trace becomes its coefficients in place) and one row block of each LDE, which every phase that reads the LDE (the
 * main and permutation commitments, the quotient, the reduced opening, the query phase) recomputes block by block.  The proof is the
 * same, word for word.  A height is blocked for all of its chips or none, and only if log_n >= log_blocks + 3.  The prover takes the
 * resident path when it fits, else the smallest B and, at that B, the fewest blocked heights (tallest first) that fit; if nothing fits
 * it returns cudaErrorMemoryAllocation (2) before launching anything.  Host-resident traces (pb_prove_chips_host, pb_prove_segment
 * without PB_TRACE_ON_DEVICE) count in the footprint as their device copies, plus on the resident path 16 x 2^(log_n + 1) words of
 * sponge state per distinct height; on the row-blocked path they are copied whole to the device first. */
/* the budget: by default the device's free memory at the call plus what the context's proof workspaces hold; `bytes` lowers it, 0
 * restores the default */
int pb_ctx_set_memory_budget(pb_ctx_t* ctx, size_t bytes);
/* log2 of the row blocks of the last pb_prove_segment / pb_prove_chips of the context, or of the sub-blocks of each rank block of the
 * last sharded proof: 0 for the resident path */
int pb_last_row_blocks(pb_ctx_t* ctx, uint32_t* log_blocks);
/* the bytes the choice above counts for chips of these heights, widths and permutation widths (pb_air_perm_width) with device-resident
 * traces (not counted), every height with log_n >= log_blocks + 3 in 2^log_blocks row blocks (0: resident); needs no device */
int pb_footprint_bytes(const size_t* log_n, const size_t* width, const size_t* perm_width, size_t n_chips, uint32_t log_blocks, size_t* bytes);

/* ---- one segment across G = 2^g GPUs, one process (and one pb_ctx) per GPU: SURVEY.md §8e ----
 * The trace is column-sharded on input (rank r holds columns pb_shard_columns(width, G, r)), the LDE and everything after it
 * is row-sharded (rank r holds rows [r*2N/G, (r+1)*2N/G) of the bit-reversed LDE for ALL columns); one all-to-all of folded
 * coefficients connects the two (the distributed-FFT transpose), after which only digests, the quotient columns, the opened
 * values and the tail of the FRI codeword are exchanged.  Collectives are supplied by the caller (NCCL, MPI, a test harness):
 * both take DEVICE pointers, are called with the context's stream idle, and must return once d_recv is complete.
 * The resulting proof is bit-identical to pb_prove_segment's on the gathered trace.  (Reference: the stark backend proves a
 * segment on one device -- /root/reference/openvm/src/lib.rs:69-95 selects one engine per process; this is the north_star's
 * "trace-column shards partitioned across the GPUs, one all-gather of Merkle caps and FRI fold outputs".) */
typedef int (*pb_collective_fn)(void* user, const void* d_send, void* d_recv, size_t bytes_per_rank);
typedef struct pb_comm {
    int rank, world;                  /* world: 2, 4, 8 or 16 */
    pb_collective_fn all_gather;      /* d_recv[r * bytes ..] = rank r's d_send[0 .. bytes) */
    pb_collective_fn all_to_all;      /* d_recv[r * bytes ..] = rank r's d_send[rank * bytes ..) */
    void* user;
    uint32_t flags;                   /* PB_COMM_STREAM_ORDERED or 0 */
} pb_comm_t;
/* the collectives are enqueued on (or ordered after) the context's CUDA stream and complete in stream order, like ncclAllGather /
 * ncclSend+ncclRecv on that stream: the library then neither drains the stream before a collective nor waits after it (it still
 * synchronises where the HOST needs a result: roots, opened values).  Without the flag the contract is the conservative one:
 * called with the stream idle, returns once d_recv is complete. */
#define PB_COMM_STREAM_ORDERED 1u
/* the column block of `rank`: first = min(width, rank*ceil(width/world)), count = min(ceil(width/world), width - first) */
int pb_shard_columns(size_t width, int world, int rank, size_t* first, size_t* count);
/* rows [blk*2N/world, (blk+1)*2N/world) of pb_lde_batch(.., log_blowup 1, shift)'s result for every column, computed without
 * the other rows (sub-coset evaluation); d_out column-major [width][2N/world] */
int pb_lde_shard(pb_ctx_t* ctx, const uint32_t* d_trace, size_t log_n, size_t width, uint32_t shift, int world, int blk, uint32_t* d_out);
/* trace_cols: this rank's column block [count][2^log_n] (device if PB_TRACE_ON_DEVICE, else host); width: the whole trace's.
 * Bus interactions attached to the AIR are proved here too (the LogUp phase runs on row / column shards, DESIGN.md §6); the query
 * phase is pb_query_segment_sharded.  FAILURE SEMANTICS: arguments and workspace sizes are checked before the first collective, but a rank that
 * fails later (a CUDA error, a collective reporting failure) returns at once while its peers are still inside a collective -- the
 * caller's collectives must carry the abort (NCCL: a communicator timeout / ncclCommAbort on the failing rank's error path). */
int pb_prove_segment_sharded(pb_ctx_t* ctx, const pb_air_t* air, const uint32_t* trace_cols, size_t log_n, size_t width, uint32_t flags,
                             const pb_comm_t* comm, pb_segment_proof_t* proof);
/* query phase of the last pb_prove_segment_sharded, collective over the same ranks: the same indices, layout (pb_query_words) and
 * words as pb_query_segment after pb_prove_segment on the gathered trace, on every rank.  A row and the bottom of its Merkle path come
 * from the rank that holds that row block, the top log2(world) levels from the subtree roots kept at commit time; one all-gather.
 * After a row-blocked proof (pb_last_row_blocks > 0) each sub-step that holds a queried row is exchanged again first: one all-to-all
 * per blocked height and sub-step (two with a permutation trace), so comm->all_to_all is then required (else PB_ERR_INVALID_ARG). */
int pb_query_segment_sharded(pb_ctx_t* ctx, const pb_comm_t* comm, uint32_t* h_out, size_t out_capacity_words);
/* ALL chips of a segment under one transcript across the same ranks: the proof, cumulative sums, opened values and query words of
 * pb_prove_chips + pb_query_chips on the gathered traces, word for word, on every rank.  Every rank passes all chips in the same order;
 * chips[c].d_trace = this rank's column block pb_shard_columns(chips[c].width, world, rank) (device, Montgomery; NULL when the block is
 * empty), chips[c].width = the whole width.  Rank r holds rows [r*2^h/G, (r+1)*2^h/G) of the bit-reversed LDE of every chip of LDE height
 * 2^h, so the mixed-height commitments, reduced openings and FRI injections are local to a rank (DESIGN.md §6); every exchange is one
 * collective for all chips, so their number does not depend on n_chips.  A chip shorter than 2^(g+3) rows on G = 2^g ranks, or a world
 * other than 2, 4, 8, 16, is PB_ERR_UNSUPPORTED.  Failure semantics as pb_prove_segment_sharded's: arguments are checked before the first
 * collective.  pb_prove_segment_sharded is the one-chip case. */
int pb_prove_chips_sharded(pb_ctx_t* ctx, const pb_chip_t* chips, size_t n_chips, const pb_comm_t* comm, pb_chips_proof_t* proof,
                           uint32_t* h_cumsums);
/* collective over the same ranks, on every rank: the queries and opened values pb_query_chips returns after pb_prove_chips on the gathered
 * traces (layout: pb_chips_sizes); h_queries / h_ys may be NULL (no queries: no collective).  One all-gather; after a row-blocked proof
 * also the all-to-alls of pb_query_segment_sharded's note, so comm->all_to_all is then required (else PB_ERR_INVALID_ARG). */
int pb_query_chips_sharded(pb_ctx_t* ctx, const pb_comm_t* comm, uint32_t* h_queries, size_t queries_capacity_words, uint32_t* h_ys,
                           size_t ys_capacity_words);
/* ---- device memory of the sharded provers (pb_prove_chips_sharded, pb_prove_segment_sharded) ----------------------------------
 * Without a budget (pb_ctx_set_memory_budget 0, the default) every rank keeps its row block of every LDE resident.  With a nonzero
 * budget, which EVERY RANK MUST BE GIVEN ALIKE (the ranks choose the same path from the chip shapes, the world and that number alone, with
 * no collective and without reading free memory), a proof whose per-rank footprint does not fit is proved with each rank block in
 * B = 2^log_blocks sub-blocks, G * B <= 16: the chips of the tallest heights keep the coefficients of the rank's columns and of its
 * permutation columns and one sub-block of each LDE; each phase that reads an LDE runs sub-step k = 0..B-1 as one all-to-all that
 * brings every rank its sub-block k, so the proof and every answer stay word for word those of the resident path.  The choice is the
 * single-GPU rule: a height is blocked for all its chips or none and only if log_n >= log2(G) + log_blocks + 3; the smallest B first,
 * then the fewest heights, tallest first.  If nothing fits, every rank returns cudaErrorMemoryAllocation (2) before any collective.
 * A row-blocked proof first frees the workspaces an earlier proof of the context left.  pb_last_row_blocks reports log_blocks. */
/* one rank's bytes of that choice for chips of these heights, widths and permutation widths on `world` ranks, every height with
 * log_n >= log2(world) + log_blocks + 3 in 2^log_blocks sub-blocks (0: resident).  The caller's column share of the traces is not
 * counted.  PB_ERR_INVALID_ARG: world not 2..16 and a power of two, world * 2^log_blocks > 16, a chip below 2^(log2(world) + 3) rows.
 * Needs no device. */
int pb_footprint_bytes_sharded(const size_t* log_n, const size_t* width, const size_t* perm_width, size_t n_chips, int world, uint32_t log_blocks,
                               size_t* bytes);

/* ---- the sharded provers on the ranks of ONE process: a group of contexts -----------------------------------------------------
 * One call proves all chips of a segment on `world` contexts (one per GPU, or several on one device), the way the reference proves a
 * segment in one process (engine.prove on one host thread per VM instance).  The library owns the rank threads: each call starts one
 * per rank, which runs pb_prove_chips_sharded (pb_query_chips_sharded) on its context with the group's collectives.  Those are
 * stream-ordered device-to-device copies (cudaMemcpyPeerAsync, over NVLink between GPUs with peer access) behind the kernels that
 * produce them: no communication library, no host staging, no callbacks to write.
 * pb_group_create: world = 2, 4, 8 or 16 (else PB_ERR_UNSUPPORTED, checked before any context is read) distinct contexts (else
 * PB_ERR_INVALID_ARG), rank r = ctxs[r]; contexts may share a device.  It enables peer access between every pair of their distinct
 * devices that supports it.  The contexts stay the caller's: destroy the group first.  One call at a time per group, and no other use
 * of its contexts while a call runs. */
typedef struct pb_group pb_group_t;
int pb_group_create(pb_ctx_t* const* ctxs, int world, pb_group_t** out);
int pb_group_destroy(pb_group_t* group);
/* chips[r]: rank r's n_chips entries, each with an AIR compiled on ctxs[r] and d_trace = rank r's column block
 * pb_shard_columns(width, world, r) on ctxs[r]'s device (NULL when empty).  proof and h_cumsums are pb_prove_chips' output on the
 * gathered traces.
 *   Inputs: pb_prove_chips_sharded's contract, per rank.  Where the column blocks come from stays with the caller (each rank's
 *     tracegen, or its own copies); they must stay valid until the last pb_query_chips_group.
 *   Checked before any rank starts (no kernel, no collective) -> PB_ERR_INVALID_ARG: NULL arguments; every rank has the same
 *     (log_n, width) and AIR permutation width per chip; every context has the same memory budget, n_queries and pow_bits.  Per-rank
 *     arguments (a NULL d_trace where the rank holds columns, a NULL AIR) are each rank's own check, as in pb_prove_chips_sharded.
 *   Output: from rank 0; every rank's proof struct and cumulative sums are compared with rank 0's, a difference is PB_ERR_INTERNAL.
 *   Errors: the first error in rank order that is not PB_ERR_COMM, PB_ERR_COMM only if nothing else failed.  A rank that fails aborts
 *     the call: every other rank leaves its pending or next collective with PB_ERR_COMM, so no rank is left waiting.  On return every
 *     context's stream is idle and the group can be used again.
 *   Results on each context: its rank's proof state, exactly as after pb_prove_chips_sharded (pb_last_row_blocks, pb_last_stage_ms
 *     per context).  Any other prover run on one of the contexts invalidates the group's proof. */
int pb_prove_chips_group(pb_group_t* group, const pb_chip_t* const* chips, size_t n_chips, pb_chips_proof_t* proof,
                         uint32_t* h_cumsums);
/* pb_query_chips' queries and opened values for the group's last proof (layout: pb_chips_sizes; h_queries / h_ys may be NULL), every
 * rank's compared with rank 0's (PB_ERR_INTERNAL if they differ).  PB_ERR_INVALID_ARG without a proof of this group, or after another
 * prover ran on one of its contexts. */
int pb_query_chips_group(pb_group_t* group, uint32_t* h_queries, size_t queries_capacity_words, uint32_t* h_ys,
                         size_t ys_capacity_words);

/* The Fiat-Shamir transcript (DuplexChallenger over Poseidon2, width 16, rate 8) runs on the HOST: absorbing the opened values is a
 * serial sponge (4363 dependent permutations for the keccak shape), so it uses an AVX-512 permutation with the whole state in one
 * register when the CPU has it (scalar otherwise; PB_HOST_P2_SCALAR=1 forces scalar).  This entry applies that permutation `reps`
 * times with the default constants, canonical words in and out, without a device: a known-answer / cross-check hook. */
int pb_host_poseidon2_permute(uint32_t state[16], int reps, int force_scalar, int* used_avx512);

/* per-stage device milliseconds of the last pb_prove_segment, pb_prove_chips, pb_prove_segment_sharded or pb_prove_chips_sharded:
 * [h2d, lde, merkle, logup_gen, logup_commit, quotient, qlde, qmerkle, open, fri, pow, total]; for several chips a stage spans that
 * phase of every chip (pb_prove_chips runs each phase for all chips before the next). */
#define PB_N_STAGES 12
int pb_last_stage_ms(pb_ctx_t* ctx, float ms[PB_N_STAGES]);
/* kernels launched by this context since creation (bench.py's gpu_launches) */
uint64_t pb_launch_count(pb_ctx_t* ctx);
/* CUDA-event timing of the dominant kernel (Poseidon2 leaf hashing of column-major matrices) since the last call:
 * number of launches (first 16 kept), summed device ms and summed algorithmic bytes (4*h*w in + 32*h out). Synchronises. */
int pb_leaf_kernel_profile(pb_ctx_t* ctx, int* n_launches, double* total_ms, double* total_bytes);

/* ---- stage 0: drop-in replacements with the reference's exact symbols and layouts (cuda_abi.rs:8-64) ------------------- */
typedef struct { int width; int height; const uint32_t* buffer; int row_block_size; } OriginalAir;   /* cuda_abi.rs:66-73 */
typedef struct { int air_index; int col; int row; int apc_col; } Subst;                               /* cuda_abi.rs:75-86 */
typedef struct { uint32_t off; uint32_t len; } ExprSpan;                                               /* cuda_abi.rs:162-169 */
typedef struct { uint64_t col_base; ExprSpan span; } DerivedExprSpec;                                  /* cuda_abi.rs:88-95 */
typedef struct { uint32_t bus_id; uint32_t num_args; uint32_t args_index_off; } DevInteraction;        /* cuda_abi.rs:150-160 */
/* ---- LogUp / bus interactions of an AIR (SURVEY.md §8 f1) -------------------------------------------------------------------
 * Attaches the bus interactions PowdrAir::eval pushes (/root/reference/openvm/src/powdr_extension/chip.rs:117-128) to a compiled
 * AIR, in the layout compile_bus_to_gpu produces (cuda/mod.rs:143-177: per interaction the spans [mult, arg_0 .. arg_{k-1}]
 * from args_index_off) with the PUSH_APC operand being the COLUMN INDEX.  Generates and compiles the AIR's LogUp kernels
 * (NVRTC, sm_90a); pb_prove_segment then runs the permutation-trace phase for this AIR.  HOST pointers. */
int pb_air_set_interactions(pb_ctx_t* ctx, pb_air_t* air, const uint32_t* bytecode, size_t n_words, const ExprSpan* arg_spans,
                            size_t n_arg_spans, const DevInteraction* interactions, size_t n_interactions);
/* host-only check of the LogUp code generator (no device needed): generates and compiles the kernels, reports their size */
int pb_air_logup_compile_only(const uint32_t* bytecode, size_t n_words, const ExprSpan* arg_spans, size_t n_arg_spans,
                              const DevInteraction* interactions, size_t n_interactions, uint32_t width, size_t* cubin_bytes,
                              size_t* perm_width);
/* width of the permutation trace in base columns: 4 * (number of LogUp chunks + 1), 0 without interactions */
int pb_air_perm_width(const pb_air_t* air, size_t* perm_width);
/* the one collective of the per-chip / per-segment sharding (SURVEY.md §8b, north_star "single NCCL all-gather of Merkle caps"):
 * all_caps[r*8 .. r*8+8) = rank r's local_cap, through the caller's pb_comm_t (device pointers; no NCCL is linked here, which is
 * also why pb_ctx_create takes no ncclComm_t: the collectives are callbacks so that the same library serves NCCL, MPI or tests) */
int pb_allgather_caps(pb_ctx_t* ctx, const pb_comm_t* comm, const uint32_t* d_local_cap, uint32_t* d_all_caps);

/* ---- verifying a proof on the host: no device, no CUDA context, no NVRTC ----------------------------------------------------------
 * Where the reference checks its own prover, verify_app_proof on the CPU engine (the reference's openvm-riscv/src/lib.rs:337-341), and
 * what a prover service calls before it publishes a proof.  The key of an AIR holds what the verifier reads of it: the constraints and
 * the bus interactions in the arrays pb_air_compile and pb_air_set_interactions take, validated by the same code (PB_ERR_BAD_BYTECODE,
 * PB_ERR_STACK_DEPTH, PB_ERR_UNSUPPORTED for an interaction above the degree bound, exactly where those return them).  n_interactions = 0:
 * an AIR without interactions (the bus arrays are then not read). */
typedef struct pb_vk pb_vk_t;
int pb_vk_create(const uint32_t* bytecode, size_t n_words, const pb_expr_span_t* constraints, size_t n_constraints, uint32_t width,
                 const uint32_t* bus_bytecode, size_t bus_words, const ExprSpan* arg_spans, size_t n_arg_spans,
                 const DevInteraction* interactions, size_t n_interactions, pb_vk_t** out);
int pb_vk_free(pb_vk_t* vk);
/* one chip of the proof: its key and log2 of its trace height (1..24) */
typedef struct { const pb_vk_t* vk; size_t log_n; } pb_verify_chip_t;
/* the verifier's security parameters, which the proof must match (n_queries 1..65536, pow_bits 0..30), and its Poseidon2 instance
 * (canonical values as for pb_ctx_set_poseidon2; all three NULL: the default of include/pb_poseidon2_constants.h) */
typedef struct {
    uint32_t n_queries, pow_bits;
    const uint32_t (*rc_ext)[16];
    const uint32_t* rc_int;
    const uint32_t* diag_m1;
} pb_verify_params_t;
/* pb_verify_chips checks a proof of pb_prove_chips / pb_prove_chips_sharded, given what those and pb_query_chips(_sharded) return:
 * h_cumsums [n_chips][4], h_ys [n_opened][4] and h_queries [n_queries][words_per_query], ys_words and queries_words being the lengths
 * of the last two.  It checks, in this order, with *reason (may be NULL) set to the first failure:
 *   20 proof shape: a chip height outside 1..24, or n_chips, log_max, n_fri_layers, final_len not following from the chip heights;
 *   21 the proof's n_queries or pow_bits differ from params;
 *   then the lengths, which must be what pb_chips_sizes gives for these chips (else PB_ERR_INVALID_ARG): no buffer is read before;
 *   20 also: a nonzero cumulative sum for a chip without interactions (it has none, and a caller's bus balance sums every slot);
 *   22 a word of h_ys, h_cumsums, the query openings (index aside), a digest, final_poly or pow_witness is not canonical (>= p);
 *   then it replays the transcript of DESIGN.md §3 / §3b:
 *   1 LogUp challenges, 2 alpha, 3 zeta, 4 gamma, 5 a FRI beta, 15 final polynomial not constant, 6 proof of work;
 *   16 per chip the constraint identity at zeta: Horner_alpha(AIR constraints, LogUp chunk and phi constraints) = Z_H(zeta) * Q(zeta);
 *   per query: 7 index, 8 / 9 / 10 main / permutation / quotient MMCS opening, 11 reduced opening != FRI layer 0, 12 FRI path,
 *   13 fold, 14 final value.
 * -> 0 accepted, PB_ERR_REJECTED, or PB_ERR_INVALID_ARG (NULL pointers, a chip without a key, n_chips = 0, mismatched lengths, bad
 * params).  The bus balance (the cumulative sums of ALL chips of a segment add up to zero) is the caller's check: a proof of the APC
 * chips alone does not contain the chips that balance their buses.  Pure host code: thread-safe, no CUDA call. */
int pb_verify_chips(const pb_verify_chip_t* chips, size_t n_chips, const pb_verify_params_t* params, const pb_chips_proof_t* proof,
                    const uint32_t* h_cumsums, const uint32_t* h_ys, size_t ys_words, const uint32_t* h_queries, size_t queries_words,
                    int* reason);
/* a proof of pb_prove_segment / pb_prove_segment_sharded with pb_query_segment(_sharded) and pb_last_openings: the one-chip case of
 * pb_verify_chips, its cumulative_sum being h_cumsums (a perm_width other than the key's is reason 20, after the argument checks) */
int pb_verify_segment(const pb_vk_t* vk, size_t log_n, const pb_verify_params_t* params, const pb_segment_proof_t* proof,
                      const uint32_t* h_ys, size_t ys_words, const uint32_t* h_queries, size_t queries_words, int* reason);

/* ---- a proof as bytes: what a prover publishes and a verifier on another machine reads (host code, no device, thread-safe) ----------
 * One format for both provers: a segment proof is written as the one-chip multi-chip proof, so the blob of pb_prove_segment on a trace
 * is byte for byte the blob of pb_prove_chips on that one chip.  The blob is a sequence of little-endian u32 words, field words canonical
 * as in the proof structs, in this order (K = n_chips, L = n_fri_layers, F = final_len):
 *   header       PB_PROOF_MAGIC, PB_PROOF_VERSION, K, n_queries, pow_bits, log_max, L, F, 0 (reserved)
 *                per chip: log_n, width, perm_width                                                               9 + 3K words
 *   proof        main_root, perm_root, quotient_root (8 each), logup_alpha, logup_beta, alpha, zeta, gamma (4 each),
 *                fri_roots [L][8], fri_betas [L][4], final_poly [F][4], pow_witness                    44 + 12L + 4F + 1 words
 *   cumsums      [K][4]
 *   opened       [n_opened][4]                 n_opened = sum width + 2 * sum perm_width + 8K (pb_chips_sizes)
 *   queries      [n_queries][words_per_query]  the layout of pb_chips_sizes / pb_query_chips for these chips
 * so the blob's length follows from the header alone.  The blob carries the chips' widths and heights because its receiver holds only
 * the verifying keys.  A blob is MALFORMED (PB_ERR_REJECTED, reason 23) if its magic or version differs, its length is not exactly the
 * one its header gives (no trailing bytes), K is 0 or above PB_PROOF_MAX_CHIPS, a log_n is outside 1..24, a perm_width is neither 0 nor
 * 4 * (chunks + 1) (a multiple of 4, at least 8), L is above 32 or F above 8 (the proof struct's arrays), the length computation
 * overflows, or the reserved word is not zero.  The decoder checks all of that before it reads past the header. */
#define PB_PROOF_MAGIC 0x46504250u     /* the bytes "PBPF" */
#define PB_PROOF_VERSION 1u
#define PB_PROOF_MAX_CHIPS 4096u
typedef struct { uint32_t log_n, width, perm_width; } pb_proof_chip_t;
/* The blob of a proof of pb_prove_chips / pb_prove_chips_sharded with the cumulative sums, opened values and queries of pb_query_chips:
 * chips[c] = (log_n, width, pb_air_perm_width) of chip c.  out = NULL: only *len (bytes) is set.  PB_ERR_INVALID_ARG: NULL pointers,
 * n_chips other than proof->n_chips, a shape the format cannot hold (see MALFORMED), ys_words / queries_words other than pb_chips_sizes
 * gives (n_opened * 4, proof->n_queries * words_per_query), or capacity < *len.  Words are written as given: the verifier checks them. */
int pb_chips_proof_encode(const pb_chips_proof_t* proof, const pb_proof_chip_t* chips, size_t n_chips, const uint32_t* h_cumsums,
                          const uint32_t* h_ys, size_t ys_words, const uint32_t* h_queries, size_t queries_words, void* out, size_t capacity,
                          size_t* len);
/* the same blob for a proof of pb_prove_segment / pb_prove_segment_sharded with pb_last_openings and pb_query_segment(_sharded) */
int pb_segment_proof_encode(const pb_segment_proof_t* proof, size_t log_n, size_t width, const uint32_t* h_ys, size_t ys_words,
                            const uint32_t* h_queries, size_t queries_words, void* out, size_t capacity, size_t* len);
/* decoding in two calls: pb_proof_bytes_sizes gives the blob's chip count and the lengths in words of its opened values and queries (the
 * cumulative sums are 4 * n_chips words); the decoder then fills the struct, the chips' shapes and the three arrays, whose lengths must
 * be exactly those (else PB_ERR_INVALID_ARG).  Both return PB_ERR_REJECTED with *reason 23 for a malformed blob.  pb_segment_proof_decode
 * gives a one-chip blob back as a segment proof (its cumulative_sum, perm_width, log_n and width from the blob); another chip count, or
 * a log_max other than log_n + 1, which the segment struct cannot hold, is reason 20. */
int pb_proof_bytes_sizes(const void* bytes, size_t len, size_t* n_chips, size_t* ys_words, size_t* queries_words, int* reason);
int pb_chips_proof_decode(const void* bytes, size_t len, pb_chips_proof_t* proof, pb_proof_chip_t* chips, size_t n_chips, uint32_t* h_cumsums,
                          uint32_t* h_ys, size_t ys_words, uint32_t* h_queries, size_t queries_words, int* reason);
int pb_segment_proof_decode(const void* bytes, size_t len, pb_segment_proof_t* proof, size_t* log_n, size_t* width, uint32_t* h_ys, size_t ys_words,
                            uint32_t* h_queries, size_t queries_words, int* reason);
/* decodes the blob and runs the checks of pb_verify_chips on it, chip c's key being vks[c] and its height the blob's: 23 a malformed blob;
 * 20 also: a chip count other than n_vks, or a width or perm_width other than the key's; then every check and reason of pb_verify_chips,
 * so a blob and the struct it encodes get the same verdict.  PB_ERR_INVALID_ARG: NULL pointers, n_vks = 0, bad params. */
int pb_verify_proof_bytes(const pb_vk_t* const* vks, size_t n_vks, const pb_verify_params_t* params, const void* bytes, size_t len, int* reason);

int _apc_tracegen(uint32_t* d_output, size_t output_height, const OriginalAir* d_original_airs, const Subst* d_subs,
                  size_t n_subs, int num_apc_calls);
int _apc_apply_derived_expr(uint32_t* d_output, size_t output_height, int num_apc_calls, const DerivedExprSpec* d_specs,
                            size_t n_cols, const uint32_t* d_bytecode);
int _apc_apply_bus(const uint32_t* d_output, int num_apc_calls, const uint32_t* d_bytecode, size_t bytecode_len,
                   const DevInteraction* d_interactions, size_t n_interactions, const ExprSpan* d_arg_spans, size_t n_arg_spans,
                   uint32_t var_range_bus_id, uint32_t* d_var_hist, size_t var_num_bins,
                   uint32_t tuple2_bus_id, uint32_t* d_tuple2_hist, uint32_t tuple2_sz0, uint32_t tuple2_sz1,
                   uint32_t bitwise_bus_id, uint32_t* d_bitwise_hist);

/* ---- stage 0, periphery histograms with a per-AIR GENERATED kernel: same result as _apc_apply_bus (which stays the drop-in with the
 * reference's shape), built at key-generation time from the same interaction table with COLUMN-INDEX operands (host pointers);
 * pb_bus_apply enqueues on the context's stream.  d_trace: the APC trace, column-major, height H, Montgomery words. */
typedef struct pb_bus pb_bus_t;
int pb_bus_compile(pb_ctx_t* ctx, const uint32_t* bytecode, size_t n_words, const ExprSpan* arg_spans, size_t n_arg_spans,
                   const DevInteraction* interactions, size_t n_interactions, uint32_t width, uint32_t var_range_bus_id, uint32_t tuple2_bus_id,
                   uint32_t bitwise_bus_id, pb_bus_t** out);
int pb_bus_free(pb_bus_t* bus);
int pb_bus_apply(pb_ctx_t* ctx, const pb_bus_t* bus, const uint32_t* d_trace, size_t H, int num_apc_calls, uint32_t* d_var_hist, size_t var_num_bins,
                 uint32_t* d_tuple2_hist, uint32_t tuple2_sz0, uint32_t tuple2_sz1, uint32_t* d_bitwise_hist);

#ifdef __cplusplus
}
#endif
#endif
