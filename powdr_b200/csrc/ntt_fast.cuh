// The LDE passes K1, K2a, K2b, K3 (algorithm: see the header of ntt.cuh), one specialisation per pass geometry.
// The row-bit count RB, the low split NLO, the round plan (Q, B0) and the lane count are template parameters, so shared/global
// addressing folds into immediates and each kernel carries only its own two or three register rounds.  Kernels that read
// their geometry at run time spent more than half of their instructions on shifts/masks for it (ncu r01: 20-30 instructions
// per butterfly, ALU pipe 55 % busy with address math).
#pragma once
#include "bb31.cuh"
#include "ntt.cuh"

namespace nttf {

using ntt::brev;
// 256-thread CTAs on 64 KB tiles: two or three CTAs are co-resident per SM, so the load phase of one overlaps the butterfly
// phase of another (ncu r01b: one 512-thread / 128 KB CTA per SM kept issue utilisation at 40-60 % -- all 16 warps wait on the
// same barrier-separated phases).  Rows of 16 lanes are still 64-byte coalesced segments.
constexpr int THREADS = 256;
constexpr int LOG_TILE = 14;

__host__ __device__ constexpr int log_lc_of(int rb) { return rb <= LOG_TILE - 4 ? 4 : LOG_TILE - rb; }
__host__ __device__ constexpr int n_rounds(int rb) { return (rb + 4) / 5; }
__host__ __device__ constexpr int q_of(int rb, int i) { return rb / n_rounds(rb) + (i < rb % n_rounds(rb) ? 1 : 0); }
__host__ __device__ constexpr int b0_of(int rb, int i) { return i == 0 ? 0 : b0_of(rb, i - 1) + q_of(rb, i - 1); }

enum { SWZ_NONE = 0, SWZ_TOP = 1, SWZ_LOW = 2 };

template <int RB, int LLC, int SWZ>
__device__ __forceinline__ uint32_t sidx(uint32_t t, uint32_t j) {
    constexpr uint32_t M = (1u << LLC) - 1;
    if (SWZ == SWZ_TOP) return (t << LLC) + (j ^ ((t >> (RB >= LLC ? RB - LLC : 0)) & M));
    if (SWZ == SWZ_LOW) return (t << LLC) + (j ^ (t & M));
    return (t << LLC) + j;
}

// Q radix-2 stages in registers.  Twiddles are (w, w') pairs for Shoup's constant product (w canonical, w' = floor(w 2^32/p)):
// IMAD.HI + 2 IMAD = 8 FMA-pipe cycles instead of 10, lazy [0,2p) operands accepted, data stays in Montgomery form.
// KS = twiddle-index stride of local bit 0.
//
// Every loop below has a compile-time trip count (the stage index S is a template parameter, stages recurse over it), so x[]
// stays in registers.  With the stage index a run-time loop variable, the inner trip count 1 << s depends on it and NVVM for
// sm_90 leaves the Q = 5 stage loops rolled: x[32] then lives in a 128-byte stack frame and every stage round-trips it through
// local memory.
template <int Q, int S, bool INV, int KS>
__device__ __forceinline__ void stage(uint32_t (&x)[1 << Q], const uint2* __restrict__ t) {
#pragma unroll
    for (int el = 0; el < (1 << S); el++) {
        const uint2 w = __ldg(t + (size_t)el * KS);
#pragma unroll
        for (int eh = 0; eh < (1 << (Q - 1 - S)); eh++) {
            const int e = (eh << (S + 1)) | el;
            if constexpr (INV) {
                uint32_t a = x[e], b = x[e | (1 << S)];
                x[e] = bb::add(a, b);
                x[e | (1 << S)] = bb::mul_shoup(a - b + bb::P, w);      // lazy difference in (0, 2p)
            } else {
                uint32_t a = x[e], m = bb::mul_shoup(x[e | (1 << S)], w);
                x[e] = bb::add(a, m);
                x[e | (1 << S)] = bb::sub(a, m);
            }
        }
    }
}

// Inverse: stages Q-1 .. 0 (DIF); forward: stages 0 .. Q-1 (DIT).  LAST_INV: stage 0 is the last of the whole inverse
// transform, whose twiddle is 1, and folds in the 1/N scale instead.
template <int Q, bool INV, int KS, bool LAST_INV, int I = 0>
__device__ __forceinline__ void stages(uint32_t (&x)[1 << Q], const uint2* __restrict__ tw, int u0, uint32_t koff, uint2 ninv) {
    if constexpr (I < Q) {
        constexpr int S = INV ? Q - 1 - I : I;
        if constexpr (INV && LAST_INV && S == 0) {
#pragma unroll
            for (int e = 0; e < (1 << Q); e += 2) {
                uint32_t a = x[e], b = x[e + 1];
                x[e] = bb::mul_shoup(a + b, ninv);
                x[e + 1] = bb::mul_shoup(a - b + bb::P, ninv);
            }
        } else {
            stage<Q, S, INV, KS>(x, tw + ((size_t)1 << (u0 + S)) + koff);
        }
        stages<Q, INV, KS, LAST_INV, I + 1>(x, tw, u0, koff, ninv);
    }
}

// one register round over a [2^RB rows][2^LLC lanes] tile; UB = global bit index of row bit 0 (NLO strided, 0 transposed).
// G_IN reads row t of the tile at gsrc + ((t >> lg) << (UB + lg)) + ((t mod 2^lg) << LLC): lg = 0 natural order, else the rows of
// the tile's lanes come in contiguous groups of 2^lg (K3 after ntttma::lde_low_bits_kernel).
template <int RB, int LLC, int Q, int B0, int UB, bool INV, int SWZ, bool LANE_K, bool G_IN, bool G_OUT>
__device__ __forceinline__ void round_dev(uint32_t* __restrict__ sm, const uint2* __restrict__ tw, uint2 ninv,
                                          const uint32_t* __restrict__ gsrc, uint32_t lg, uint32_t* __restrict__ gdst, uint32_t live) {
    constexpr uint32_t LC = 1u << LLC;
    constexpr uint32_t TASKS = (1u << (RB - Q)) << LLC;
    constexpr int KS = 1 << (B0 + UB);
#pragma unroll 1
    for (uint32_t id = threadIdx.x; id < TASKS; id += THREADS) {
        const uint32_t j = id & (LC - 1), g = id >> LLC;
        const uint32_t tl = g & ((1u << B0) - 1);
        const uint32_t tbase = ((g >> B0) << (B0 + Q)) | tl;
        if (j >= live) continue;
        uint32_t x[1 << Q];
#pragma unroll
        for (int e = 0; e < (1 << Q); e++) {
            const uint32_t t = tbase + ((uint32_t)e << B0);
            x[e] = G_IN ? __ldg(gsrc + ((size_t)(t >> lg) << (UB + lg)) + ((t & ((1u << lg) - 1)) << LLC) + j) : sm[sidx<RB, LLC, SWZ>(t, j)];
        }
        const uint32_t koff = (LANE_K ? j : 0u) + (tl << UB);
        stages<Q, INV, KS, INV && UB == 0 && B0 == 0>(x, tw, UB + B0, koff, ninv);
#pragma unroll
        for (int e = 0; e < (1 << Q); e++) {
            const uint32_t t = tbase + ((uint32_t)e << B0);
            if (G_OUT) gdst[((size_t)t << UB) + j] = x[e];
            else sm[sidx<RB, LLC, SWZ>(t, j)] = x[e];
        }
    }
}

// all rounds of a pass, unrolled at compile time in processing order (inverse: high bits first; forward: low bits first)
template <int RB, int LLC, int UB, bool INV, int SWZ, bool LANE_K, bool G_FIRST, bool G_LAST, int I = 0>
__device__ __forceinline__ void pass_rounds(uint32_t* sm, const uint2* tw, uint2 ninv, const uint32_t* gsrc, uint32_t lg, uint32_t* gdst,
                                            uint32_t live) {
    constexpr int NR = n_rounds(RB);
    if constexpr (I < NR) {
        constexpr int R = INV ? NR - 1 - I : I;
        constexpr bool gi = G_FIRST && I == 0, go = G_LAST && I == NR - 1;
        round_dev<RB, LLC, q_of(RB, R), b0_of(RB, R), UB, INV, SWZ, LANE_K, gi, go>(sm, tw, ninv, gsrc, lg, gdst, live);
        if constexpr (I + 1 < NR) __syncthreads();
        pass_rounds<RB, LLC, UB, INV, SWZ, LANE_K, G_FIRST, G_LAST, I + 1>(sm, tw, ninv, gsrc, lg, gdst, live);
    }
}

// K1 (INV) / K3 (!INV): strided tile, rows <-> position bits [NLO, NLO+RB), lane j <-> position j0 + j.
// K3's source rows come in groups of 2^lg (0 for natural order; K1 ignores lg and reads natural order): position k = j + (t << NLO) of a coset is at word
// ((t >> lg) << (NLO + lg)) + ((j >> LLC) << (LLC + lg)) + ((t mod 2^lg) << LLC) + (j mod 2^LLC), so a tile reads 2^lg rows of its
// lanes as one contiguous piece instead of 2^lg pieces of 2^LLC words
template <int RB, int NLO, bool INV>
__global__ void __launch_bounds__(THREADS) strided_kernel(const uint32_t* __restrict__ src, size_t src_col_stride, uint32_t lg,
                                                          uint32_t* __restrict__ dst, size_t dst_col_stride, int log_blowup,
                                                          const uint2* __restrict__ tw_all) {
    extern __shared__ uint32_t sm[];
    constexpr int LLC = log_lc_of(RB);
    constexpr int n = RB + NLO;
    const uint32_t j0 = blockIdx.x << LLC;
    const int c = INV ? 0 : (int)blockIdx.z;
    const int cosets = INV ? 1 : (1 << log_blowup);
    const uint32_t* s = INV ? src + (size_t)blockIdx.y * src_col_stride + j0 : src + (((size_t)blockIdx.y * cosets + c) << n) + ((size_t)j0 << lg);
    const uint2* tw = tw_all + ((size_t)c << n) + j0;         // lane part of the twiddle index is the position j0 + j
    uint32_t* d1 = dst + (size_t)blockIdx.y * dst_col_stride + j0;
    pass_rounds<RB, LLC, NLO, INV, INV ? SWZ_NONE : SWZ_TOP, true, true, INV>(sm, tw, make_uint2(0u, 0u), s, INV ? 0u : lg, d1, 1u << LLC);
    if (!INV) {
        __syncthreads();
        // natural evaluation index k = j0 + j + (t << NLO) of coset c lands at row  bitrev_b(c)*N + bitrev_n(k)
        constexpr uint32_t ROWS = 1u << RB, TILE = ROWS << LLC;
        uint32_t* dcol = dst + (size_t)blockIdx.y * dst_col_stride + ((size_t)brev((uint32_t)c, log_blowup) << n);
#pragma unroll 4
        for (uint32_t e = threadIdx.x; e < TILE; e += THREADS) {
            const uint32_t p = e & (ROWS - 1), j = e >> RB;
            const uint32_t t = __brev(p) >> (32 - RB);
            dcol[((size_t)(__brev(j0 + j) >> (32 - NLO)) << RB) + p] = sm[sidx<RB, LLC, SWZ_TOP>(t, j)];
        }
    }
}

// K2a (INV) / K2b (!INV): transposed tile, lane l <-> one contiguous block of 2^RB positions (RB == n_lo)
template <int RB, bool INV>
__global__ void __launch_bounds__(THREADS) transposed_kernel(const uint32_t* __restrict__ src, size_t src_col_stride,
                                                             uint32_t* __restrict__ dst, int n, int log_blowup, size_t total_blocks,
                                                             const uint2* __restrict__ tw_all, uint2 ninv) {
    extern __shared__ uint32_t sm[];
    constexpr int LLC = log_lc_of(RB);
    constexpr uint32_t LC = 1u << LLC, ROWS = 1u << RB;
    const int c = INV ? 0 : (int)blockIdx.z;
    const int cosets = INV ? 1 : (1 << log_blowup);
    const size_t b_first = (size_t)blockIdx.x << LLC;
    const uint32_t live = (uint32_t)min((size_t)LC, total_blocks - b_first);
    const int log_bpc = n - RB;
    const uint2* tw = tw_all + ((size_t)c << n);
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (uint32_t l = warp; l < live; l += THREADS / 32) {
        const size_t b = b_first + l, col = b >> log_bpc, blk = b & (((size_t)1 << log_bpc) - 1);
        const uint32_t* p = src + col * src_col_stride + (blk << RB);
#pragma unroll 8
        for (uint32_t t = lane; t < ROWS; t += 32) sm[sidx<RB, LLC, SWZ_LOW>(t, l)] = __ldg(p + t);
    }
    __syncthreads();
    pass_rounds<RB, LLC, 0, INV, SWZ_LOW, false, false, false>(sm, tw, ninv, nullptr, 0u, nullptr, live);
    __syncthreads();
    for (uint32_t l = warp; l < live; l += THREADS / 32) {
        const size_t b = b_first + l, col = b >> log_bpc, blk = b & (((size_t)1 << log_bpc) - 1);
        uint32_t* p = dst + ((col * cosets + c) << n) + (blk << RB);
#pragma unroll 8
        for (uint32_t t = lane; t < ROWS; t += 32) p[t] = sm[sidx<RB, LLC, SWZ_LOW>(t, l)];
    }
}

// Pass plan of a 2^n-point transform: n = n_hi + n_lo, K1/K3 = strided_kernel<n_hi, n_lo>, K2a/K2b = transposed_kernel<n_lo>.
// Up to 2^10 points n_hi = 0: one transposed pass each way, then ntt::bitrev_store_kernel.
constexpr int n_lo_of(int n) { return n <= 10 ? n : (n + 1) / 2; }
// dynamic shared memory of a pass over 2^rb rows: at most 2^LOG_TILE words
constexpr size_t tile_bytes(int rb) { return (size_t)4 << (rb + log_lc_of(rb)); }

}  // namespace nttf
