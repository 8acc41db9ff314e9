/* A proof that leaves the process: the prover writes its byte form to a file, and a verifier reads the file back, with nothing but
 * include/powdr_b200.h and libpowdr_b200.so, from plain C99.
 *
 *   gcc -std=c99 -O2 -I include examples/proof_bytes_demo.c -L powdr_b200/_lib -lpowdr_b200 -Wl,-rpath,$PWD/powdr_b200/_lib -o proof_bytes_demo
 *   ./proof_bytes_demo prove proof.bin [log_n]     (needs a GPU)
 *   ./proof_bytes_demo verify proof.bin            (needs none: it never calls pb_ctx_create)
 *
 * The AIR is abi_demo.c's: 3 columns with the constraints  a*b - c = 0  and  a*(a - 1)*(a - 2) = 0.  `prove` proves one segment of a
 * satisfying trace held in pinned host memory, gathers the query openings and the opened values and writes the blob of
 * pb_segment_proof_encode.  `verify` builds the AIR's verifying key and runs pb_verify_proof_bytes on the file's bytes; it prints
 * "accepted" and exits 0, or prints the reason and exits 2.  The security parameters are fixed on both sides: 4 queries, 16 bits of
 * proof of work. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "powdr_b200.h"

#define P 2013265921u
#define N_QUERIES 4u
#define POW_BITS 16u
enum { OP_PUSH_APC = 0, OP_PUSH_CONST = 1, OP_ADD = 2, OP_SUB = 3, OP_MUL = 4 };

static const uint32_t bytecode[] = {
    OP_PUSH_APC, 0, OP_PUSH_APC, 1, OP_MUL, OP_PUSH_APC, 2, OP_SUB,                                   /* a*b - c          */
    OP_PUSH_APC, 0, OP_PUSH_APC, 0, OP_PUSH_CONST, 1, OP_SUB, OP_MUL, OP_PUSH_APC, 0, OP_PUSH_CONST, 2, OP_SUB, OP_MUL,   /* a(a-1)(a-2) */
};
static const pb_expr_span_t constraints[2] = {{0, 8}, {8, 14}};
static const size_t width = 3;

static uint32_t to_monty(uint32_t x) { return (uint32_t)((((uint64_t)x) << 32) % P); }

#define CHECK(call)                                                          \
    do {                                                                     \
        int rc_ = (call);                                                    \
        if (rc_ != 0) { fprintf(stderr, "%s -> %d\n", #call, rc_); return 1; } \
    } while (0)

static int prove(const char* path, size_t log_n) {
    const size_t n = (size_t)1 << log_n;
    pb_ctx_t* ctx = NULL;
    CHECK(pb_ctx_create(&ctx, 0, NULL));            /* PB_ERR_NO_DEVICE without a GPU: there is no CPU prover */
    CHECK(pb_ctx_set_fri_params(ctx, N_QUERIES, POW_BITS));
    pb_air_t* air = NULL;
    CHECK(pb_air_compile(ctx, bytecode, sizeof bytecode / sizeof bytecode[0], constraints, 2, (uint32_t)width, &air));

    uint32_t* trace = NULL;                          /* column-major [3][n], Montgomery words, pinned */
    CHECK(pb_host_alloc((void**)&trace, 4 * width * n));
    uint64_t s = 88172645463325252ull;
    for (size_t r = 0; r < n; r++) {
        s ^= s << 13; s ^= s >> 7; s ^= s << 17;
        const uint32_t a = (uint32_t)(s % 3), b = (uint32_t)((s >> 8) % P), c = (uint32_t)(((uint64_t)a * b) % P);
        trace[0 * n + r] = to_monty(a);
        trace[1 * n + r] = to_monty(b);
        trace[2 * n + r] = to_monty(c);
    }
    pb_segment_proof_t proof;
    CHECK(pb_prove_segment(ctx, air, trace, log_n, width, 0u /* host trace */, &proof));

    size_t wpq = 0, len = 0;
    CHECK(pb_query_words(log_n, width, proof.perm_width, &wpq));
    const size_t q_words = N_QUERIES * wpq, ys_words = 4 * (width + 2 * proof.perm_width + 8);
    uint32_t* q = (uint32_t*)malloc(4 * q_words);
    uint32_t* ys = (uint32_t*)malloc(4 * ys_words);
    CHECK(q && ys ? 0 : -1);
    CHECK(pb_query_segment(ctx, q, q_words));
    CHECK(pb_last_openings(ctx, ys, ys_words));
    CHECK(pb_segment_proof_encode(&proof, log_n, width, ys, ys_words, q, q_words, NULL, 0, &len));      /* the size */
    unsigned char* blob = (unsigned char*)malloc(len);
    CHECK(blob ? 0 : -1);
    CHECK(pb_segment_proof_encode(&proof, log_n, width, ys, ys_words, q, q_words, blob, len, &len));
    FILE* f = fopen(path, "wb");
    CHECK(f && fwrite(blob, 1, len, f) == len && fclose(f) == 0 ? 0 : -1);
    printf("wrote %zu bytes, log_n %zu\n", len, log_n);

    free(blob);
    free(ys);
    free(q);
    CHECK(pb_host_free(trace));
    CHECK(pb_air_free(air));
    CHECK(pb_ctx_destroy(ctx));
    return 0;
}

static int verify(const char* path) {
    FILE* f = fopen(path, "rb");
    CHECK(f ? 0 : -1);
    CHECK(fseek(f, 0, SEEK_END));
    const long size = ftell(f);
    CHECK(size >= 0 && fseek(f, 0, SEEK_SET) == 0 ? 0 : -1);
    unsigned char* blob = (unsigned char*)malloc(size ? (size_t)size : 1);
    CHECK(blob && fread(blob, 1, (size_t)size, f) == (size_t)size ? 0 : -1);
    fclose(f);

    pb_vk_t* vk = NULL;                              /* host only: no device, no CUDA context */
    CHECK(pb_vk_create(bytecode, sizeof bytecode / sizeof bytecode[0], constraints, 2, (uint32_t)width, NULL, 0, NULL, 0, NULL, 0, &vk));
    const pb_vk_t* vks[1] = {vk};
    const pb_verify_params_t params = {N_QUERIES, POW_BITS, NULL, NULL, NULL};
    int reason = 0;
    const int rc = pb_verify_proof_bytes(vks, 1, &params, blob, (size_t)size, &reason);
    CHECK(pb_vk_free(vk));
    free(blob);
    if (rc == PB_ERR_REJECTED) {
        printf("rejected reason %d\n", reason);
        return 2;
    }
    CHECK(rc);
    printf("accepted %ld bytes\n", size);
    return 0;
}

int main(int argc, char** argv) {
    if (argc >= 3 && !strcmp(argv[1], "prove")) return prove(argv[2], argc > 3 ? (size_t)atoi(argv[3]) : 10);
    if (argc == 3 && !strcmp(argv[1], "verify")) return verify(argv[2]);
    fprintf(stderr, "usage: %s prove FILE [log_n] | verify FILE\n", argv[0]);
    return 1;
}
