// TMA-staged shared-memory butterflies for the two "transposed" LDE passes (K2a inverse low bits, K2b forward low bits) -- the
// north-star's "TMA-staged shared-memory butterflies for the NTT" (BASELINE.json), replacing nttf::transposed_kernel for n_lo = 10
// (n = 19, 20: the 2^20-row headline and its permutation trace).
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
// Completion: one mbarrier per CTA armed with the tile's byte count; the stores are a bulk group the issuing thread waits on.
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
constexpr int SMEM_BYTES = TILE_BYTES + 1024;   // dynamic shared memory: the tile, aligned up to 1024 B in the kernel

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
// round B: stage bits [0, 5); lane i holds t = 32 i + e, as 8 swizzled 16-byte chunks of row i
template <bool INV>
__device__ __forceinline__ void round_b(uint32_t* blk, uint32_t lane, const uint2* __restrict__ tw, uint2 ninv) {
    uint32_t x[32];
    uint4* row = reinterpret_cast<uint4*>(blk + 32 * lane);
#pragma unroll
    for (int c = 0; c < 8; c++) {
        const uint4 v = row[c ^ (lane & 7)];
        x[4 * c] = v.x; x[4 * c + 1] = v.y; x[4 * c + 2] = v.z; x[4 * c + 3] = v.w;
    }
    nttf::stages<5, INV, 1, INV>(x, tw, 0, 0u, ninv);
#pragma unroll
    for (int c = 0; c < 8; c++) row[c ^ (lane & 7)] = make_uint4(x[4 * c], x[4 * c + 1], x[4 * c + 2], x[4 * c + 3]);
}

// tm_src / tm_dst: 2-D tensor maps {32 words, rows} with 128 B swizzle and a {32, 256} box over the source / destination buffers.
// src tile of CTA x = rows [x * 512, (x + 1) * 512); dst rows = ((col * cosets + c) << (n - 5)) + (blk_in_col << 5).
// The inverse pass is capped at 2 CTAs per SM instead of 3: under the 80-register cap of 3 CTAs, ptxas spills 124 bytes of it
// (round B's warp-uniform twiddles and the 1/N pair on top of x[32]).  At 2^20 x 2022 on the H100 the 121-register version
// takes 6.8 ms against 8.7 ms with the spill (DESIGN.md §4).
template <bool INV>
__global__ void __launch_bounds__(THREADS, INV ? 2 : 3) transposed_tma_kernel(const __grid_constant__ CUtensorMap tm_src, const __grid_constant__ CUtensorMap tm_dst, int n,
                                                                 int log_blowup, const uint2* __restrict__ tw_all, uint2 ninv) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t bar;
    uint32_t* sm = reinterpret_cast<uint32_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);      // SWIZZLE_128B: 1024 B alignment
    const int c = INV ? 0 : (int)blockIdx.z;
    const int cosets = INV ? 1 : (1 << log_blowup);
    const size_t b_first = (size_t)blockIdx.x * BLOCKS_PER_TILE;
    const int log_bpc = n - RB;                                   // blocks per column
    const size_t col = b_first >> log_bpc, blk0 = b_first & (((size_t)1 << log_bpc) - 1);
    if (threadIdx.x == 0) {
        mbar_init(&bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(&bar, TILE_BYTES);
        const int row0 = (int)(b_first << (RB - 5));
        tma_load_2d(sm, &tm_src, &bar, 0, row0);
        tma_load_2d(sm + 8192, &tm_src, &bar, 0, row0 + 256);
    }
    mbar_wait(&bar, 0);
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint2* tw = tw_all + ((size_t)c << n);
#pragma unroll 1
    for (uint32_t l = warp; l < BLOCKS_PER_TILE; l += THREADS / 32) {
        uint32_t* blk = sm + (l << RB);
        if (INV) {
            round_a<true>(blk, lane, tw, ninv);
            __syncwarp();
            round_b<true>(blk, lane, tw, ninv);
        } else {
            round_b<false>(blk, lane, tw, ninv);
            __syncwarp();
            round_a<false>(blk, lane, tw, ninv);
        }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");       // generic-proxy smem writes -> visible to the TMA (async proxy)
    __syncthreads();
    if (threadIdx.x == 0) {
        const int drow0 = (int)((((col * cosets + (size_t)c) << log_bpc) + blk0) << (RB - 5));
        tma_store_2d(&tm_dst, sm, 0, drow0);
        tma_store_2d(&tm_dst, sm + 8192, 0, drow0 + 256);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // shared memory must outlive the bulk read
    }
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
inline bool available() { return getenv("PB_LDE_NO_TMA") == nullptr && encode_fn() != nullptr; }
inline bool supported(int n_lo) { return n_lo == RB; }

// rows of 32 words over `words` u32 starting at base (16-byte aligned), box {32, 256}, 128 B swizzle
inline bool make_map(CUtensorMap* tm, const uint32_t* base, size_t words) {
    const cuuint64_t dims[2] = {32, (cuuint64_t)(words / 32)};
    const cuuint64_t strides[1] = {128};
    const cuuint32_t box[2] = {32, 256};
    const cuuint32_t estr[2] = {1, 1};
    return encode_fn()(tm, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                       CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// launches the TMA version of K2a / K2b; false when it does not apply (caller launches nttf::transposed_kernel instead).
// The caller's context has opted both kernels in to SMEM_BYTES of dynamic shared memory.
inline bool launch_transposed(bool inv, int n, int n_lo, cudaStream_t st, const uint32_t* src, uint32_t* dst, int log_blowup, size_t total_blocks,
                              size_t src_words, size_t dst_words, const uint2* tw, uint2 ninv) {
    if (!available() || !supported(n_lo) || (total_blocks % BLOCKS_PER_TILE) != 0 || (n - RB) < 4) return false;
    if ((src_words >> 5) > 0x7fffffffull || (dst_words >> 5) > 0x7fffffffull) return false;      // row coordinates are int32
    CUtensorMap ts, td;
    if (!make_map(&ts, src, src_words) || !make_map(&td, dst, dst_words)) return false;
    const dim3 grid((unsigned)(total_blocks / BLOCKS_PER_TILE), 1, inv ? 1u : (1u << log_blowup));
    if (inv) transposed_tma_kernel<true><<<grid, THREADS, SMEM_BYTES, st>>>(ts, td, n, log_blowup, tw, ninv);
    else transposed_tma_kernel<false><<<grid, THREADS, SMEM_BYTES, st>>>(ts, td, n, log_blowup, tw, ninv);
    return true;
}

}  // namespace ntttma
