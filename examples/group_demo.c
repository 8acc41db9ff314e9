/* All chips of a segment on several ranks of ONE process, from plain C: nothing but include/powdr_b200.h and libpowdr_b200.so, no
 * communication library, no threads of the caller's.
 *
 *   gcc -std=c99 -O2 -I include examples/group_demo.c -L powdr_b200/_lib -lpowdr_b200 -Wl,-rpath,$PWD/powdr_b200/_lib -o group_demo
 *   ./group_demo [log_n] [world]
 *
 * Proves a two-chip segment (a 3-column AIR of 2^log_n rows with  a*b - c = 0  and  a*(a - 1)*(a - 2) = 0, and a 5-column AIR of
 * 2^(log_n - 2) rows with  x0 + x1 - x2 = 0  and  x3*x4 - x0 = 0) with pb_prove_chips_group, asks for its queries and opened values
 * with pb_query_chips_group and checks the proof with pb_verify_chips.  The ranks are one context per visible GPU (world: the largest
 * power of two of them, at most 16), or `world` (default 2) contexts on device 0 when there is one.  Each rank holds only its column
 * block (pb_shard_columns) of each trace, on its context's device.  tests/test_gpu_group.py builds and runs it and compares the printed
 * proof with the Python binding's on the same traces. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "powdr_b200.h"

#define P 2013265921u
#define MAX_RANKS 16
enum { OP_PUSH_APC = 0, OP_PUSH_CONST = 1, OP_ADD = 2, OP_SUB = 3, OP_MUL = 4 };

static uint32_t to_monty(uint32_t x) { return (uint32_t)((((uint64_t)x) << 32) % P); }

static uint64_t rng_state = 88172645463325252ull;
static uint64_t next_rand(void) {
    rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17;
    return rng_state;
}

#define CHECK(call)                                                          \
    do {                                                                     \
        int rc_ = (call);                                                    \
        if (rc_ != 0) { fprintf(stderr, "%s -> %d\n", #call, rc_); return 1; } \
    } while (0)

static void print_words(const char* name, const uint32_t* w, size_t n) {
    printf("%s", name);
    for (size_t i = 0; i < n; i++) printf(" %u", w[i]);
    printf("\n");
}

int main(int argc, char** argv) {
    const size_t log_n = argc > 1 ? (size_t)atoi(argv[1]) : 10;
    const uint32_t bc0[] = {
        OP_PUSH_APC, 0, OP_PUSH_APC, 1, OP_MUL, OP_PUSH_APC, 2, OP_SUB,                                   /* a*b - c          */
        OP_PUSH_APC, 0, OP_PUSH_APC, 0, OP_PUSH_CONST, 1, OP_SUB, OP_MUL, OP_PUSH_APC, 0, OP_PUSH_CONST, 2, OP_SUB, OP_MUL,   /* a(a-1)(a-2) */
    };
    const uint32_t bc1[] = {
        OP_PUSH_APC, 0, OP_PUSH_APC, 1, OP_ADD, OP_PUSH_APC, 2, OP_SUB,                                   /* x0 + x1 - x2     */
        OP_PUSH_APC, 3, OP_PUSH_APC, 4, OP_MUL, OP_PUSH_APC, 0, OP_SUB,                                   /* x3*x4 - x0       */
    };
    const pb_expr_span_t cons0[2] = {{0, 8}, {8, 14}}, cons1[2] = {{0, 8}, {8, 8}};
    const uint32_t* bcs[2] = {bc0, bc1};
    const size_t bc_words[2] = {sizeof bc0 / sizeof bc0[0], sizeof bc1 / sizeof bc1[0]};
    const pb_expr_span_t* cons[2] = {cons0, cons1};
    const size_t widths[2] = {3, 5}, log_ns[2] = {log_n, log_n - 2};

    /* the visible GPUs: a context on each device until one cannot be created (the first failing is PB_ERR_NO_DEVICE without a GPU) */
    pb_ctx_t* probe = NULL;
    CHECK(pb_ctx_create(&probe, 0, NULL));
    CHECK(pb_ctx_destroy(probe));
    int n_dev = 1;
    while (n_dev < MAX_RANKS && pb_ctx_create(&probe, n_dev, NULL) == 0) {
        pb_ctx_destroy(probe);
        n_dev++;
    }
    int world = 2;
    if (n_dev >= 2) while (world * 2 <= n_dev) world *= 2;
    if (argc > 2) world = atoi(argv[2]);
    if (world < 2 || world > MAX_RANKS) { fprintf(stderr, "world %d: 2, 4, 8 or 16\n", world); return 1; }

    /* canonical traces, column-major, satisfying both AIRs */
    uint32_t* traces[2];
    for (int c = 0; c < 2; c++) {
        const size_t n = (size_t)1 << log_ns[c];
        traces[c] = (uint32_t*)malloc(4 * widths[c] * n);
        for (size_t r = 0; r < n; r++) {
            uint32_t* t = traces[c];
            const uint64_t s = next_rand();
            if (c == 0) {
                const uint32_t a = (uint32_t)(s % 3), b = (uint32_t)((s >> 8) % P);
                t[r] = a; t[n + r] = b; t[2 * n + r] = (uint32_t)(((uint64_t)a * b) % P);
            } else {
                const uint32_t x3 = (uint32_t)(s % P), x4 = (uint32_t)((s >> 31) % P), x1 = (uint32_t)((s >> 17) % P);
                const uint32_t x0 = (uint32_t)(((uint64_t)x3 * x4) % P);
                t[r] = x0; t[n + r] = x1; t[2 * n + r] = (uint32_t)(((uint64_t)x0 + x1) % P); t[3 * n + r] = x3; t[4 * n + r] = x4;
            }
        }
    }

    /* per rank: its context, its AIRs and its column blocks.  pb_device_alloc allocates on the current device, which pb_ctx_create
     * has just made the rank's */
    pb_ctx_t* ctxs[MAX_RANKS];
    pb_air_t* airs[MAX_RANKS][2];
    uint32_t* blocks[MAX_RANKS][2];
    pb_chip_t chips[MAX_RANKS][2];
    const pb_chip_t* chip_ptrs[MAX_RANKS];
    for (int r = 0; r < world; r++) {
        CHECK(pb_ctx_create(&ctxs[r], r % n_dev, NULL));
        CHECK(pb_ctx_set_fri_params(ctxs[r], 4, 8));        /* 4 queries, 8 proof-of-work bits: the same on every rank */
        for (int c = 0; c < 2; c++) {
            const size_t n = (size_t)1 << log_ns[c];
            size_t first = 0, count = 0;
            CHECK(pb_air_compile(ctxs[r], bcs[c], bc_words[c], cons[c], 2, (uint32_t)widths[c], &airs[r][c]));
            CHECK(pb_shard_columns(widths[c], world, r, &first, &count));
            blocks[r][c] = NULL;
            if (count) {
                uint32_t* h = (uint32_t*)malloc(4 * count * n);
                for (size_t i = 0; i < count * n; i++) h[i] = to_monty(traces[c][first * n + i]);
                CHECK(pb_device_alloc((void**)&blocks[r][c], 4 * count * n));
                CHECK(pb_copy_h2d(ctxs[r], blocks[r][c], h, 4 * count * n));
                CHECK(pb_ctx_synchronize(ctxs[r]));
                free(h);
            }
            chips[r][c].air = airs[r][c];
            chips[r][c].d_trace = blocks[r][c];
            chips[r][c].log_n = log_ns[c];
            chips[r][c].width = widths[c];
        }
        chip_ptrs[r] = chips[r];
    }

    pb_group_t* group = NULL;
    CHECK(pb_group_create(ctxs, world, &group));
    pb_chips_proof_t proof;
    uint32_t cums[2][4];
    CHECK(pb_prove_chips_group(group, chip_ptrs, 2, &proof, &cums[0][0]));
    size_t n_open = 0, wpq = 0;
    CHECK(pb_chips_sizes(chips[0], 2, &n_open, &wpq));
    uint32_t* ys = (uint32_t*)malloc(4 * 4 * n_open);
    uint32_t* q = (uint32_t*)malloc(4 * wpq * proof.n_queries);
    CHECK(pb_query_chips_group(group, q, wpq * proof.n_queries, ys, 4 * n_open));

    printf("world %d devices %d\n", world, n_dev);
    print_words("main_root", proof.main_root, 8);
    print_words("quotient_root", proof.quotient_root, 8);
    print_words("zeta", proof.zeta, 4);
    print_words("final_poly", &proof.final_poly[0][0], 4 * (size_t)proof.final_len);
    printf("pow_witness %u\n", proof.pow_witness);
    printf("query_rows");
    for (uint32_t i = 0; i < proof.n_queries; i++) printf(" %u", q[i * wpq]);
    printf("\n");

    /* the library's host verifier, with the constraint identity */
    pb_vk_t* vks[2];
    pb_verify_chip_t vchips[2];
    for (int c = 0; c < 2; c++) {
        CHECK(pb_vk_create(bcs[c], bc_words[c], cons[c], 2, (uint32_t)widths[c], NULL, 0, NULL, 0, NULL, 0, &vks[c]));
        vchips[c].vk = vks[c];
        vchips[c].log_n = log_ns[c];
    }
    const pb_verify_params_t params = {4, 8, NULL, NULL, NULL};
    int reason = 0;
    const int vrc = pb_verify_chips(vchips, 2, &params, &proof, &cums[0][0], ys, 4 * n_open, q, wpq * proof.n_queries, &reason);
    printf("verify %d reason %d\n", vrc, reason);
    for (int r = 0; r < world; r++) {
        float ms[PB_N_STAGES];
        CHECK(pb_last_stage_ms(ctxs[r], ms));
        printf("rank %d total_ms %.3f\n", r, ms[PB_N_STAGES - 1]);
    }

    CHECK(pb_group_destroy(group));
    for (int c = 0; c < 2; c++) { CHECK(pb_vk_free(vks[c])); free(traces[c]); }
    for (int r = 0; r < world; r++) {
        for (int c = 0; c < 2; c++) {
            if (blocks[r][c]) CHECK(pb_device_free(blocks[r][c]));
            CHECK(pb_air_free(airs[r][c]));
        }
        CHECK(pb_ctx_destroy(ctxs[r]));
    }
    free(ys);
    free(q);
    return vrc == 0 ? 0 : 1;
}
