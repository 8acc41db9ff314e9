/*
 * ORACLE (test infrastructure, not product code): expression bytecode evaluation, constraint folding /
 * quotient, and the CPU mirror of the reference's three APC trace-generation kernels.
 *
 * Pinned by in-tree reference sources:
 *   stack machine + opcodes        /root/reference/openvm/cuda/src/expr_eval.cuh:12-89
 *   host bytecode compiler         /root/reference/openvm/src/powdr_extension/trace_generator/cuda/mod.rs:49-177
 *   expression semantics           /root/reference/expression/src/lib.rs:179-207
 *   PowdrAir::eval (assert_zero on each constraint of row_slice(0))   /root/reference/openvm/src/powdr_extension/chip.rs:94-130
 *   tracegen gather                /root/reference/openvm/cuda/src/apc_tracegen.cu:35-66
 *   derived columns                /root/reference/openvm/cuda/src/apc_tracegen.cu:72-100, cpu/mod.rs:181-200
 *   periphery histograms           /root/reference/openvm/cuda/src/apc_apply_bus.cu:52-112, cpu/periphery.rs:179-236
 * The quotient's alpha-folding order, vanishing polynomial and chunk split follow Plonky3 (SURVEY.md App. C.2);
 * that part has no in-tree source => unpinned.
 */
#include "oracle.h"
#include "bb31.h"
#include <assert.h>
#include <stdlib.h>
#include <string.h>

enum { OP_PUSH_APC = 0, OP_PUSH_CONST = 1, OP_ADD = 2, OP_SUB = 3, OP_MUL = 4, OP_NEG = 5, OP_INV_OR_ZERO = 6 };
#define ORC_STACK 16   /* STACK_CAPACITY, expr_eval.cuh:22 */

static inline uint32_t eval_generic(const uint32_t* bc, uint32_t len, const uint32_t* mat, size_t r, size_t col_stride) {
    uint32_t st[ORC_STACK];
    int sp = 0;
    for (uint32_t ip = 0; ip < len;) {
        uint32_t op = bc[ip++];
        switch (op) {
        case OP_PUSH_APC: { uint32_t b = bc[ip++]; assert(sp < ORC_STACK); st[sp++] = mat[(size_t)b * col_stride + r]; break; }
        case OP_PUSH_CONST: { uint32_t u = bc[ip++]; assert(sp < ORC_STACK); st[sp++] = u % BB_P; break; }
        case OP_ADD: { uint32_t b = st[--sp], a = st[--sp]; st[sp++] = bb_add(a, b); break; }
        case OP_SUB: { uint32_t b = st[--sp], a = st[--sp]; st[sp++] = bb_sub(a, b); break; }
        case OP_MUL: { uint32_t b = st[--sp], a = st[--sp]; st[sp++] = bb_mul(a, b); break; }
        case OP_NEG: { uint32_t a = st[--sp]; st[sp++] = bb_neg(a); break; }
        case OP_INV_OR_ZERO: { uint32_t a = st[--sp]; st[sp++] = bb_inv(a); break; }
        default: assert(0 && "unknown opcode");
        }
    }
    assert(sp == 1);
    return st[0];
}

uint32_t orc_eval_expr(const uint32_t* bc, uint32_t len, const uint32_t* mat, size_t r) { return eval_generic(bc, len, mat, r, 1); }

void orc_constraint_fold(const uint32_t* bc, const orc_span_t* spans, size_t n_constraints, const uint32_t* mat, size_t height,
                         const uint32_t alpha[4], uint32_t* out4) {
    bb4_t a = {{alpha[0], alpha[1], alpha[2], alpha[3]}};
#pragma omp parallel for schedule(static)
    for (long r = 0; r < (long)height; r++) {
        bb4_t acc = bb4_from_base(0);
        for (size_t k = 0; k < n_constraints; k++) {
            uint32_t c = eval_generic(bc + spans[k].off, spans[k].len, mat, (size_t)r, height);
            acc = bb4_mul(acc, a);
            acc.c[0] = bb_add(acc.c[0], c);
        }
        for (int l = 0; l < 4; l++) out4[(size_t)l * height + (size_t)r] = acc.c[l];
    }
}

void orc_quotient(const uint32_t* bc, const orc_span_t* spans, size_t n_constraints, const uint32_t* lde, unsigned log_n,
                  unsigned log_blowup, uint32_t shift, const uint32_t alpha[4], uint32_t* quotient) {
    assert(log_blowup == 1);
    size_t n = (size_t)1 << log_n, m = n << 1;
    uint32_t* folded = (uint32_t*)malloc(4 * m * sizeof(uint32_t));
    orc_constraint_fold(bc, spans, n_constraints, lde, m, alpha, folded);
    /* Z_H(x) = x^N - 1 on x = shift * w_{2N}^i takes two values: shift^N * (+1 | -1) - 1 */
    uint32_t sn = bb_pow(shift, n);
    uint32_t zinv[2] = {bb_inv(bb_sub(sn, 1)), bb_inv(bb_sub(bb_neg(sn), 1))};
#pragma omp parallel for schedule(static)
    for (long r = 0; r < (long)m; r++) {
        size_t chunk = (size_t)r >> log_n;            /* = parity of the natural index bitrev(r) */
        size_t j = (size_t)r & (n - 1);
        for (int l = 0; l < 4; l++) quotient[(chunk * 4 + l) * n + j] = bb_mul(folded[(size_t)l * m + r], zinv[chunk]);
    }
    free(folded);
}

/* ---------------- stage 0 ---------------- */
void orc_apc_tracegen(uint32_t* out, size_t H, const orc_original_air_t* airs, const orc_subst_t* subs, size_t n_subs, int num_apc_calls) {
    for (size_t r = 0; r < H; r++)
        for (size_t i = 0; i < n_subs; i++) {
            orc_subst_t s = subs[i];
            size_t dst = (size_t)s.apc_col * H + r;
            if (r >= (size_t)num_apc_calls) { out[dst] = 0; continue; }
            const orc_original_air_t* a = &airs[s.air_index];
            out[dst] = a->buffer[(size_t)s.col * (size_t)a->height + (size_t)s.row + r * (size_t)a->row_block_size];
        }
}

void orc_apc_apply_derived_expr(uint32_t* out, size_t H, int num_apc_calls, const orc_derived_spec_t* specs, size_t n_cols, const uint32_t* bc) {
    for (size_t r = 0; r < H; r++)
        for (size_t i = 0; i < n_cols; i++)
            out[specs[i].col_base + r] = r < (size_t)num_apc_calls ? orc_eval_expr(bc + specs[i].span.off, specs[i].span.len, out, r) : 0;
}

void orc_apc_apply_bus(const uint32_t* out, int num_apc_calls, const uint32_t* bc, const orc_interaction_t* ints, size_t n_ints,
                       const orc_span_t* sp, uint32_t var_range_bus_id, uint32_t* var_hist, size_t var_num_bins,
                       uint32_t tuple2_bus_id, uint32_t* tuple2_hist, uint32_t sz0, uint32_t sz1,
                       uint32_t bitwise_bus_id, uint32_t* bitwise_hist) {
    /* an interaction whose arguments are outside its table is counted nowhere (periphery.rs:179-236 refuses it); each component
     * is bounded on its own, so an out-of-table argument never aliases into another entry's bin */
    for (int r = 0; r < num_apc_calls; r++)
        for (size_t i = 0; i < n_ints; i++) {
            orc_interaction_t it = ints[i];
#define ARG(k) orc_eval_expr(bc + sp[it.args_index_off + (k)].off, sp[it.args_index_off + (k)].len, out, (size_t)r)
            uint32_t m = ARG(0);
            if (m == 0) continue;
            if (it.bus_id == var_range_bus_id) {
                uint32_t value = ARG(1), max_bits = ARG(2);
                /* bin (1 << max_bits) + value - 1; all 2^max_bits bins of max_bits must fit in the table */
                if (max_bits < 32 && (2ull << max_bits) - 1 <= var_num_bins && value < (1ull << max_bits))
                    var_hist[(1u << max_bits) + value - 1u] += m;
            } else if (it.bus_id == tuple2_bus_id) {
                uint32_t v0 = ARG(1), v1 = ARG(2);
                if (v0 < sz0 && v1 < sz1) tuple2_hist[(size_t)v0 * sz1 + v1] += m;
            } else if (it.bus_id == bitwise_bus_id) {
                uint32_t x = ARG(1), y = ARG(2), sel = ARG(4);
                /* BitwiseOperationLookup<8> count layout [range 2^16 | xor 2^16] (dependency header, not in tree) */
                if (x < 256 && y < 256 && sel <= 1) bitwise_hist[sel * 65536u + ((x << 8) | y)] += m;
            }
#undef ARG
        }
}
