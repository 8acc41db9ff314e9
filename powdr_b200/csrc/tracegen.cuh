// Stage 0: sm_90a re-designs of the reference's three APC trace-generation kernels, behind the SAME extern "C" entry
// points and #[repr(C)] descriptors (/root/reference/openvm/src/cuda_abi.rs:8-95,150-169):
//   _apc_tracegen            replaces apc_tracegen_kernel            (/root/reference/openvm/cuda/src/apc_tracegen.cu:35-66)
//   _apc_apply_derived_expr  replaces apc_apply_derived_expr_kernel  (apc_tracegen.cu:72-100)
//   _apc_apply_bus           replaces apc_apply_bus_kernel           (/root/reference/openvm/cuda/src/apc_apply_bus.cu:23-113)
//
// Re-design notes
//  * gather: the reference runs one thread per ROW with a serial loop over all ~W substitutions, re-reading the Subst and
//    OriginalAir descriptors from global memory on every iteration.  Here the grid is (row tiles) x (substitutions): each
//    CTA copies one column segment, descriptors are read once per CTA, four rows per thread are in flight, and both sides
//    are unit-stride (row_block_size == 1) or fixed-stride coalesced streams -- a pure HBM copy.
//  * bus: multiplicities are added with ONE atomic per (warp, distinct bin) through __match_any_sync aggregation instead
//    of `mult` single increments per lane.
#pragma once
#include "bb31.cuh"

namespace tg {

struct OriginalAir { int width; int height; const uint32_t* buffer; int row_block_size; };
struct Subst { int air_index; int col; int row; int apc_col; };
struct ExprSpan { uint32_t off; uint32_t len; };
struct DerivedExprSpec { uint64_t col_base; ExprSpan span; };
struct DevInteraction { uint32_t bus_id; uint32_t num_args; uint32_t args_index_off; };

enum : uint32_t { OP_PUSH_APC = 0, OP_PUSH_CONST = 1, OP_ADD = 2, OP_SUB = 3, OP_MUL = 4, OP_NEG = 5, OP_INV_OR_ZERO = 6 };
constexpr int STACK_CAPACITY = 16;

// the reference's bytecode verbatim: PUSH_APC operand is an absolute element offset (col*H), PUSH_CONST a canonical u32
__device__ __forceinline__ uint32_t eval_expr(const uint32_t* __restrict__ bc, uint32_t len, const uint32_t* __restrict__ trace, size_t r) {
    uint32_t st[STACK_CAPACITY];
    int sp = 0;
    for (uint32_t ip = 0; ip < len;) {
        const uint32_t op = __ldg(bc + ip++);
        switch (op) {
        case OP_PUSH_APC: { uint32_t base = __ldg(bc + ip++); st[sp++] = trace[base + r]; break; }
        case OP_PUSH_CONST: { uint32_t u = __ldg(bc + ip++); st[sp++] = bb::to_monty(u); break; }
        case OP_ADD: { uint32_t b = st[--sp], a = st[--sp]; st[sp++] = bb::add(a, b); break; }
        case OP_SUB: { uint32_t b = st[--sp], a = st[--sp]; st[sp++] = bb::sub(a, b); break; }
        case OP_MUL: { uint32_t b = st[--sp], a = st[--sp]; st[sp++] = bb::mul(a, b); break; }
        case OP_NEG: { st[sp - 1] = bb::neg(st[sp - 1]); break; }
        default: { st[sp - 1] = bb::inv(st[sp - 1]); break; }
        }
    }
    return st[0];
}

constexpr int GATHER_THREADS = 256;
constexpr int GATHER_ROWS_PER_THREAD = 4;

__global__ void __launch_bounds__(GATHER_THREADS) apc_tracegen_kernel(uint32_t* __restrict__ out, size_t H,
                                                                      const OriginalAir* __restrict__ airs,
                                                                      const Subst* __restrict__ subs, int num_apc_calls) {
    const Subst sub = subs[blockIdx.y];
    const OriginalAir air = airs[sub.air_index];
    const uint32_t* __restrict__ src = air.buffer + (size_t)sub.col * (size_t)air.height + (size_t)sub.row;
    uint32_t* __restrict__ dst = out + (size_t)sub.apc_col * H;
    const size_t base = (size_t)blockIdx.x * (GATHER_THREADS * GATHER_ROWS_PER_THREAD) + threadIdx.x;
    uint32_t v[GATHER_ROWS_PER_THREAD];
#pragma unroll
    for (int i = 0; i < GATHER_ROWS_PER_THREAD; i++) {
        size_t r = base + (size_t)i * GATHER_THREADS;
        v[i] = (r < (size_t)num_apc_calls) ? __ldg(src + r * (size_t)air.row_block_size) : 0u;
    }
#pragma unroll
    for (int i = 0; i < GATHER_ROWS_PER_THREAD; i++) {
        size_t r = base + (size_t)i * GATHER_THREADS;
        if (r < H) dst[r] = v[i];
    }
}

__global__ void __launch_bounds__(256) apc_apply_derived_expr_kernel(uint32_t* __restrict__ out, size_t H, int num_apc_calls,
                                                                     const DerivedExprSpec* __restrict__ specs, size_t n_cols,
                                                                     const uint32_t* __restrict__ bc) {
    const size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= H) return;
    const bool live = r < (size_t)num_apc_calls;
    for (size_t i = 0; i < n_cols; i++) {           // in order: a derived column may read an earlier one of the same row
        const DerivedExprSpec spec = specs[i];
        out[spec.col_base + r] = live ? eval_expr(bc + spec.span.off, spec.span.len, out, r) : 0u;
    }
}

// warp-aggregated histogram increment: lanes with the same bin elect a leader that adds the summed multiplicity
__device__ __forceinline__ void hist_add(uint32_t* hist, uint32_t idx, uint32_t mult) {
    const unsigned active = __activemask();
    const unsigned peers = __match_any_sync(active, idx);
    const int leader = __ffs(peers) - 1;
    uint32_t total = 0;
    for (unsigned rem = peers; rem;) {              // sum multiplicities over the peer group
        int l = __ffs(rem) - 1;
        rem &= rem - 1;
        total += __shfl_sync(peers, mult, l);
    }
    if ((int)(threadIdx.x & 31) == leader) atomicAdd(hist + idx, total);
}

constexpr uint32_t BITWISE_NUM_BITS = 8u;

__global__ void __launch_bounds__(128) apc_apply_bus_kernel(const uint32_t* __restrict__ trace, int num_apc_calls,
                                                            const uint32_t* __restrict__ bc,
                                                            const DevInteraction* __restrict__ ints, size_t n_ints,
                                                            const ExprSpan* __restrict__ spans,
                                                            uint32_t var_range_bus_id, uint32_t* __restrict__ var_hist, size_t var_num_bins,
                                                            uint32_t tuple2_bus_id, uint32_t* __restrict__ tuple2_hist, uint32_t sz0, uint32_t sz1,
                                                            uint32_t bitwise_bus_id, uint32_t* __restrict__ bitwise_hist) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= num_apc_calls) return;
    for (size_t i = 0; i < n_ints; i++) {
        const DevInteraction it = ints[i];
        if (it.bus_id != var_range_bus_id && it.bus_id != tuple2_bus_id && it.bus_id != bitwise_bus_id) continue;   // uniform
#define PB_ARG(k) bb::from_monty(eval_expr(bc + spans[it.args_index_off + (k)].off, spans[it.args_index_off + (k)].len, trace, (size_t)r))
        const uint32_t m = PB_ARG(0);
        if (m == 0u) continue;
        if (it.bus_id == var_range_bus_id) {
            const uint32_t value = PB_ARG(1), max_bits = PB_ARG(2);
            const uint32_t idx = (1u << max_bits) + value - 1u;     // VariableRangeChecker::add_count indexing (apc_apply_bus.cu:74)
            if (idx < var_num_bins) hist_add(var_hist, idx, m);
        } else if (it.bus_id == tuple2_bus_id) {
            const uint32_t v0 = PB_ARG(1), v1 = PB_ARG(2);
            const uint32_t idx = v0 * sz1 + v1;                     // apc_apply_bus.cu:89
            if (idx < sz0 * sz1) hist_add(tuple2_hist, idx, m);
        } else {
            const uint32_t x = PB_ARG(1), y = PB_ARG(2), sel = PB_ARG(4);
            const uint32_t idx = ((x << BITWISE_NUM_BITS) | y) + (sel == 1u ? (1u << (2 * BITWISE_NUM_BITS)) : 0u);   // [range | xor]
            if (sel <= 1u && idx < (2u << (2 * BITWISE_NUM_BITS))) hist_add(bitwise_hist, idx, m);
        }
#undef PB_ARG
    }
}

}  // namespace tg
