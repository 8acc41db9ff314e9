// TMA-staged shared-memory butterflies for the low-bit LDE passes at n_lo = 10 (n = 19, 20: the 2^20-row headline and its
// permutation trace), replacing nttf::transposed_kernel there:
//   * transposed_tma_kernel: K2a alone (inverse low bits), for the callers that want the coefficients (coefficients(), the sharded
//     inverse-and-fold);
//   * lde_low_bits_kernel: K2a and K2b of pb_lde_batch in one pass.  The inverse ends with the low bits (DIF) and the forward
//     starts with them (DIT), on the same 2^10-position blocks, so the coefficients never leave the SM: the pass reads the block
//     once and writes it once per coset, 1 + 2^b words per element instead of 2 + 1 + 2^b (9 instead of 11 for the whole LDE at
//     b = 1).  Forward-only callers at n_lo = 10 (the sharded forward block) run nttf::transposed_kernel<10, false>.
//
// Why these passes: a K2 tile is 16 consecutive blocks of 2^10 positions of one column = ONE contiguous 64 KB span of global
// memory, so the whole tile moves with two `cp.async.bulk.tensor.2d` boxes (32 words x 256 rows each) in and two out; no thread
// computes a global address, issues an LDG/STG or runs a transpose loop (the per-thread tile movement and swizzled staging of
// the LDG/STS version were 25-30 % of these kernels' instructions).
//
// Layout: the tensor map views the buffer as rows of 32 words (128 B) with CU_TENSOR_MAP_SWIZZLE_128B, i.e. the 16-byte chunk index
// of a word is XORed with (row mod 8) on the way into shared memory (and back on the way out).  Block-local position t (10 bits)
// lives in row t >> 5, so physical word = t ^ (((t >> 5) & 7) << 2).  One WARP owns one block (lane i):
//   round A (stage bits 5..9): lane i holds t = i + 32 e, e < 32  -> word 32 e + (i ^ ((e & 7) << 2)): 32 distinct banks per access;
//   round B (stage bits 0..4): lane i holds t = 32 i + e          -> row i, 16-byte chunk c at physical chunk c ^ (i & 7): LDS.128 /
//                                                                    STS.128, 8 distinct chunk slots per quarter warp.
// Both rounds are bank-conflict free on the layout the TMA delivers, so no re-staging is needed; the rounds are separated by
// __syncwarp() only (a block is private to its warp).  Inverse = A then B (DIF, high bits first), forward = B then A (DIT).
// Completion: one mbarrier per CTA armed with the tile's byte count; the stores are bulk groups the issuing thread waits on.
#pragma once
#include <cuda.h>
#include <dlfcn.h>

#include "bb31.cuh"
#include "ntt_fast.cuh"

namespace ntttma {

constexpr int RB = 10;                    // block = 2^10 positions
constexpr int BLOCKS_PER_TILE = 16;       // 64 KB
constexpr int THREADS = 256;              // 8 warps x 2 blocks
constexpr uint32_t TILE_BYTES = BLOCKS_PER_TILE * (4u << RB);
constexpr uint32_t BLOCK_BYTES = 4u << RB;
constexpr int SMEM_BYTES = TILE_BYTES + 1024;   // dynamic shared memory: the tile, aligned up to 1024 B in the kernel
// lde_low_bits_kernel: the tile (the block's coefficients once the inverse rounds ran) and one output block per warp
constexpr int LOW_BITS_SMEM_BYTES = TILE_BYTES + (THREADS / 32) * BLOCK_BYTES + 1024;
// ... whose output is K3's source with its rows in groups of 2^LOG_ROW_GROUP (nttf::strided_kernel): K3's tile of 16 lanes reads
// 2^LOG_ROW_GROUP x 64 B contiguous instead of 64 B pieces 4 KB apart
constexpr int K3_LANES = 16;
constexpr int LOG_ROW_GROUP = 1;
static_assert((1 << nttf::log_lc_of(9)) == K3_LANES && (1 << nttf::log_lc_of(10)) == K3_LANES, "K3 lanes at n_lo = 10");

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem_dst)),
                 "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* tm, const void* smem_src, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %2, %3, %4}], [%1];" ::"l"(tm), "r"(smem_u32(smem_src)), "r"(0), "r"(c2),
                 "r"(c3)
                 : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tm, const void* smem_src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(tm), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
                 : "memory");
}

// round A: stage bits [5, 10); lane i holds t = i + 32 e
template <bool INV>
__device__ __forceinline__ void round_a(uint32_t* blk, uint32_t lane, const uint2* __restrict__ tw, uint2 ninv) {
    uint32_t x[32];
#pragma unroll
    for (int e = 0; e < 32; e++) x[e] = blk[32 * e + (lane ^ ((e & 7) << 2))];
    nttf::stages<5, INV, 32, false>(x, tw, 5, lane, ninv);
#pragma unroll
    for (int e = 0; e < 32; e++) blk[32 * e + (lane ^ ((e & 7) << 2))] = x[e];
}
// round B's layout: lane i holds t = 32 i + e, as 8 swizzled 16-byte chunks of row i
__device__ __forceinline__ void load_b(uint32_t (&x)[32], const uint32_t* blk, uint32_t lane) {
    const uint4* row = reinterpret_cast<const uint4*>(blk + 32 * lane);
#pragma unroll
    for (int c = 0; c < 8; c++) {
        const uint4 v = row[c ^ (lane & 7)];
        x[4 * c] = v.x; x[4 * c + 1] = v.y; x[4 * c + 2] = v.z; x[4 * c + 3] = v.w;
    }
}
__device__ __forceinline__ void store_b(uint32_t* blk, uint32_t lane, const uint32_t (&x)[32]) {
    uint4* row = reinterpret_cast<uint4*>(blk + 32 * lane);
#pragma unroll
    for (int c = 0; c < 8; c++) row[c ^ (lane & 7)] = make_uint4(x[4 * c], x[4 * c + 1], x[4 * c + 2], x[4 * c + 3]);
}

// the inverse rounds of one block in place (A then B); lane i ends with row i
__device__ __forceinline__ void inverse_block(uint32_t* blk, uint32_t lane, const uint2* __restrict__ tw, uint2 ninv) {
    round_a<true>(blk, lane, tw, ninv);
    __syncwarp();
    uint32_t x[32];
    load_b(x, blk, lane);
    nttf::stages<5, true, 1, true>(x, tw, 0, 0u, ninv);
    store_b(blk, lane, x);
}

// forward round A on an output block that round B left in the swizzled layout; the result in natural order (word t = position t)
__device__ __forceinline__ void round_a_out(uint32_t* blk, uint32_t lane, const uint2* __restrict__ tw) {
    uint32_t x[32];
#pragma unroll
    for (int e = 0; e < 32; e++) x[e] = blk[32 * e + (lane ^ ((e & 7) << 2))];
    nttf::stages<5, false, 32, false>(x, tw, 5, lane, make_uint2(0u, 0u));
    __syncwarp();
#pragma unroll
    for (int e = 0; e < 32; e++) blk[32 * e + lane] = x[e];
}

// the tile of CTA x: blocks [16 x, 16 x + 16) of the src tensor map (rows [x * 512, (x + 1) * 512)), into sm once the mbarrier completes
__device__ __forceinline__ void load_tile(uint32_t* sm, uint64_t* bar, const CUtensorMap* tm_src) {
    if (threadIdx.x == 0) {
        mbar_init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(bar, TILE_BYTES);
        const int row0 = (int)((size_t)blockIdx.x * BLOCKS_PER_TILE << (RB - 5));
        tma_load_2d(sm, tm_src, bar, 0, row0);
        tma_load_2d(sm + 8192, tm_src, bar, 0, row0 + 256);
    }
    mbar_wait(bar, 0);
}

// K2a.  tm_src / tm_dst: 2-D tensor maps {32 words, rows} with 128 B swizzle and a {32, 256} box over the source / destination
// buffers (stride N).  The pass is capped at 2 CTAs per SM instead of 3: under the 80-register cap of 3 CTAs, ptxas spills 124
// bytes of it (round B's warp-uniform twiddles and the 1/N pair on top of x[32]).  At 2^20 x 2022 on the H100 the 121-register
// version takes 6.8 ms against 8.7 ms with the spill (DESIGN.md §4).
__global__ void __launch_bounds__(THREADS, 2) transposed_tma_kernel(const __grid_constant__ CUtensorMap tm_src, const __grid_constant__ CUtensorMap tm_dst,
                                                                    const uint2* __restrict__ tw, uint2 ninv) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t bar;
    uint32_t* sm = reinterpret_cast<uint32_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);      // SWIZZLE_128B: 1024 B alignment
    load_tile(sm, &bar, &tm_src);
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll 1
    for (uint32_t l = warp; l < BLOCKS_PER_TILE; l += THREADS / 32) {
        inverse_block(sm + (l << RB), lane, tw, ninv);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");       // generic-proxy smem writes -> visible to the TMA (async proxy)
    __syncthreads();
    if (threadIdx.x == 0) {
        const int drow0 = (int)((size_t)blockIdx.x * BLOCKS_PER_TILE << (RB - 5));
        tma_store_2d(&tm_dst, sm, 0, drow0);
        tma_store_2d(&tm_dst, sm + 8192, 0, drow0 + 256);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // shared memory must outlive the bulk read
    }
}

// K2a + K2b of pb_lde_batch.  tm_src: as above, over K1's output (stride N).  tm_dst: make_group_map over the [col][coset][N]
// scratch K3 reads, box = one block.  Each warp runs the inverse rounds of its two blocks in place, so the tile holds their
// coefficients.  Then, per block and coset, it runs forward round B from the coefficients into its own output block, round A on
// that block, and stores it with one TMA box; the output block is reused once the previous store has read it (waited on after
// round B's butterflies, so the two overlap).  Inverse first, forward second: interleaved per block, ptxas spills at the
// 128-register cap of 2 CTAs per SM (2 x 97 KB of shared memory).
__global__ void __launch_bounds__(THREADS, 2) lde_low_bits_kernel(const __grid_constant__ CUtensorMap tm_src, const __grid_constant__ CUtensorMap tm_dst,
                                                                  int n, int log_blowup, const uint2* __restrict__ tw_inv, uint2 ninv,
                                                                  const uint2* __restrict__ tw_fwd) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t bar;
    uint32_t* sm = reinterpret_cast<uint32_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);      // SWIZZLE_128B: 1024 B alignment
    load_tile(sm, &bar, &tm_src);
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll 1
    for (uint32_t l = warp; l < BLOCKS_PER_TILE; l += THREADS / 32) {
        inverse_block(sm + (l << RB), lane, tw_inv, ninv);      // lane i's row of coefficients: only lane i reads it below
    }
    uint32_t* out = sm + (BLOCKS_PER_TILE << RB) + (warp << RB);
    const int log_bpc = n - RB;                                   // blocks per column
    const size_t b_first = (size_t)blockIdx.x * BLOCKS_PER_TILE;
    const size_t col = b_first >> log_bpc, blk0 = b_first & (((size_t)1 << log_bpc) - 1);
    const int blk_c0 = (int)(((col << log_blowup) << log_bpc) + blk0);       // int32: checked by the host
#pragma unroll 1
    for (uint32_t l = warp; l < BLOCKS_PER_TILE; l += THREADS / 32) {
        const uint32_t* blk = sm + (l << RB);
#pragma unroll 1
        for (int c = 0; c < (1 << log_blowup); c++) {
            const uint2* tw = tw_fwd + ((size_t)c << n);
            uint32_t x[32];
            load_b(x, blk, lane);
            nttf::stages<5, false, 1, false>(x, tw, 0, 0u, ninv);
            if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");       // the previous store has read out
            __syncwarp();
            store_b(out, lane, x);
            __syncwarp();
            round_a_out(out, lane, tw);
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) {
                const int t = blk_c0 + (c << log_bpc) + (int)l;              // block index in the scratch
                tma_store_4d(&tm_dst, out, t & ((1 << LOG_ROW_GROUP) - 1), t >> LOG_ROW_GROUP);
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
        }
    }
    if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

// ---------------- host side ----------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = [] {
        void* h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
        return h ? (EncodeTiledFn)dlsym(h, "cuTensorMapEncodeTiled") : (EncodeTiledFn) nullptr;
    }();
    return fn;
}

// rows of 32 words over `words` u32 starting at base (16-byte aligned), box {32, box_rows}, 128 B swizzle
inline bool make_map(CUtensorMap* tm, const uint32_t* base, size_t words, uint32_t box_rows) {
    const cuuint64_t dims[2] = {32, (cuuint64_t)(words / 32)};
    const cuuint64_t strides[1] = {128};
    const cuuint32_t box[2] = {32, box_rows};
    const cuuint32_t estr[2] = {1, 1};
    return encode_fn()(tm, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                       CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// the [col][coset][N] scratch as {16 lanes, 64 lane groups, 2^LOG_ROW_GROUP rows, row groups}: word
// ((t >> g) << (10 + g)) + ((j >> 4) << (4 + g)) + ((t mod 2^g) << 4) + (j mod 16) holds position j of block t (nttf::strided_kernel's
// grouped rows at n_lo = 10); box {16, 64, 1, 1} = one block in natural order, no swizzle
inline bool make_group_map(CUtensorMap* tm, const uint32_t* base, size_t words) {
    constexpr uint32_t G = 1u << LOG_ROW_GROUP;
    const cuuint64_t dims[4] = {K3_LANES, (1u << RB) / K3_LANES, G, (cuuint64_t)(words >> (RB + LOG_ROW_GROUP))};
    const cuuint64_t strides[3] = {4ull * K3_LANES * G, 4ull * K3_LANES, (4ull << RB) * G};
    const cuuint32_t box[4] = {K3_LANES, (1u << RB) / K3_LANES, 1, 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    return encode_fn()(tm, CU_TENSOR_MAP_DATA_TYPE_UINT32, 4, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                       CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// whether the TMA passes run nb columns of 2^n points split at n_lo, writing dst_words (row coordinates are int32)
inline bool applies(int n, int n_lo, unsigned nb, size_t dst_words) {
    return getenv("PB_LDE_NO_TMA") == nullptr && encode_fn() != nullptr && n_lo == RB && (n - RB) >= 4 && (dst_words >> 5) <= 0x7fffffffull
        && ((size_t)nb << n) % (BLOCKS_PER_TILE << RB) == 0;
}

// K2a on nb columns (stride 2^n) of src into dst; false when it does not apply (caller launches nttf::transposed_kernel instead).
// The caller's context has opted the kernel in to SMEM_BYTES of dynamic shared memory.
inline bool launch_inverse(int n, int n_lo, cudaStream_t st, const uint32_t* src, uint32_t* dst, unsigned nb, const uint2* tw, uint2 ninv) {
    const size_t words = (size_t)nb << n;
    if (!applies(n, n_lo, nb, words)) return false;
    CUtensorMap ts, td;
    if (!make_map(&ts, src, words, 256) || !make_map(&td, dst, words, 256)) return false;
    transposed_tma_kernel<<<(unsigned)(words / (TILE_BYTES / 4)), THREADS, SMEM_BYTES, st>>>(ts, td, tw, ninv);
    return true;
}

// K2a + K2b on nb columns (stride 2^n) of src into dst[col][coset][2^n], rows grouped for K3 (make_group_map); false when it does not apply (caller launches K2a and K2b).
// The caller's context has opted the kernel in to LOW_BITS_SMEM_BYTES of dynamic shared memory.
inline bool launch_low_bits(int n, int n_lo, cudaStream_t st, const uint32_t* src, uint32_t* dst, unsigned nb, int log_blowup, const uint2* tw_inv,
                            uint2 ninv, const uint2* tw_fwd) {
    const size_t words = (size_t)nb << n;
    if (!applies(n, n_lo, nb, words << log_blowup)) return false;
    CUtensorMap ts, td;
    if (!make_map(&ts, src, words, 256) || !make_group_map(&td, dst, words << log_blowup)) return false;
    lde_low_bits_kernel<<<(unsigned)(words / (TILE_BYTES / 4)), THREADS, LOW_BITS_SMEM_BYTES, st>>>(ts, td, n, log_blowup, tw_inv, ninv, tw_fwd);
    return true;
}

}  // namespace ntttma
