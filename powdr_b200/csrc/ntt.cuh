// Stage 1 of the north-star path: batched coset low-degree extension of column-major trace columns
// (SURVEY.md §8 a6; call site main_trace_commit behind /root/reference/openvm-riscv/src/lib.rs:332).
//
// Per column:  evals over H (natural order)  --iNTT-->  coefficients  --coset NTT x 2^b-->  evals over shift*H',
// rows bit-reversed.  H100 mapping:
//   * inverse = decimation-in-frequency (natural in, bit-reversed coefficient slots out), forward = decimation-in-time
//     on those slots (natural out): no standalone permutation pass; the one bit reversal is folded into the last store.
//   * the coset shift is folded into the forward twiddles (w_u[k] = shift^(2^(n-1-u)) * omega^k), the 1/N into the last
//     inverse stage: no scaling passes.
//   * index bits are split n = n_hi + n_lo.  Four passes per column batch:
//       K1  inverse, bits [n_lo,n)   strided tiles   [2^n_hi rows x 32 lanes], lane = consecutive position (128 B rows)
//       K2a inverse, bits [0,n_lo)   transposed tiles [2^n_lo rows x 32 lanes], lane = one contiguous 2^n_lo block
//       K2b forward, bits [0,n_lo)   per coset, same geometry
//       K3  forward, bits [n_lo,n)   per coset, strided tiles, then the bit-reversed store
//     Each pass reads and writes its column batch through HBM (11 words per element at b = 1); the batch is sized to fill the
//     SMs, not to keep the intermediates in the 50 MB L2 (smaller, L2-sized batches measured no faster, capi.cu).
//   * inside a pass the butterfly network never crosses lanes: a thread owns 2^q (q<=5) rows of one lane in REGISTERS and
//     runs q radix-2 stages on them (80 butterflies per 32 loads + 32 stores for q=5); shared memory is touched once per
//     round, conflict-free (lane = bank, XOR swizzle for the two transposed accesses).
// Integer-pipe bound: a Montgomery product costs 10 FMA-pipe cycles per warp on sm_90 (IMAD.WIDE and IMAD.HI are half rate).
#pragma once
#include "bb31.cuh"

namespace ntt {

constexpr int THREADS = 512;
constexpr int LOG_TILE_MAX = 15;   // 2^15 elements = 128 KB of shared memory per CTA
constexpr int MAX_ROUNDS = 4;

struct Rounds {              // processing order of the register rounds of one pass
    int n;                   // number of rounds
    int q[MAX_ROUNDS];       // bits handled by round i (1..5)
    int b0[MAX_ROUNDS];      // lowest row bit handled by round i
};

__device__ __forceinline__ uint32_t brev(uint32_t x, int bits) { return bits ? (__brev(x) >> (32 - bits)) : 0u; }

// Q radix-2 stages on 2^Q register-resident elements whose row indices differ in bits [b0, b0+Q).
// tw        : stage tables, tw[2^u + k]
// u0        : global index bit of local bit 0
// koff      : lane-dependent part of the twiddle index (position mod 2^u0, pre-shifted)
// kstride   : twiddle-index stride of local bit 0
template <int Q, bool INV>
__device__ __forceinline__ void reg_stages(uint32_t (&x)[1 << Q], const uint2* __restrict__ tw, int u0, uint32_t koff,
                                           uint32_t kstride, uint2 ninv) {
    if (INV) {
#pragma unroll
        for (int s = Q - 1; s >= 0; s--) {
            if (s == 0 && u0 == 0) {          // last inverse stage of the whole transform: twiddle 1, fold in 1/N
#pragma unroll
                for (int e = 0; e < (1 << Q); e += 2) {
                    uint32_t a = x[e], b = x[e + 1];
                    x[e] = bb::mul_shoup(a + b, ninv);
                    x[e + 1] = bb::mul_shoup(a - b + bb::P, ninv);
                }
            } else {
                const uint2* t = tw + ((size_t)1 << (u0 + s)) + koff;
#pragma unroll
                for (int el = 0; el < (1 << s); el++) {
                    const uint2 w = __ldg(t + (size_t)el * kstride);
#pragma unroll
                    for (int eh = 0; eh < (1 << (Q - 1 - s)); eh++) {
                        const int e = (eh << (s + 1)) | el;
                        uint32_t a = x[e], b = x[e | (1 << s)];
                        x[e] = bb::add(a, b);
                        x[e | (1 << s)] = bb::mul_shoup(a - b + bb::P, w);
                    }
                }
            }
        }
    } else {
#pragma unroll
        for (int s = 0; s < Q; s++) {
            const uint2* t = tw + ((size_t)1 << (u0 + s)) + koff;
#pragma unroll
            for (int el = 0; el < (1 << s); el++) {
                const uint2 w = __ldg(t + (size_t)el * kstride);
#pragma unroll
                for (int eh = 0; eh < (1 << (Q - 1 - s)); eh++) {
                    const int e = (eh << (s + 1)) | el;
                    uint32_t a = x[e], m = bb::mul_shoup(x[e | (1 << s)], w);
                    x[e] = bb::add(a, m);
                    x[e | (1 << s)] = bb::sub(a, m);
                }
            }
        }
    }
}

// shared-memory index of (row t, lane j): XOR swizzle so that both "fixed row, lanes = j" and the transposed
// "fixed j, lanes = rows that differ in the swizzled bits" accesses are conflict-free
__device__ __forceinline__ uint32_t sidx(uint32_t t, uint32_t j, int log_lc, int sshift) {
    return (t << log_lc) + (j ^ ((t >> sshift) & ((1u << log_lc) - 1)));
}

// One register round over the whole tile.  SRC/DST: 0 = shared memory, 1 = global memory through the address functor.
template <int Q, bool INV, bool G_IN, bool G_OUT, typename AddrIn, typename AddrOut>
__device__ __forceinline__ void tile_round(uint32_t* sm, int log_rows, int log_lc, int sshift, int b0, const uint2* __restrict__ tw,
                                           int ubase, uint32_t lane_koff_mul, uint2 ninv, AddrIn gin, AddrOut gout, uint32_t lanes_live) {
    const uint32_t lc = 1u << log_lc;
    const uint32_t tasks = (1u << (log_rows - Q)) << log_lc;
    const uint32_t lowmask = (1u << b0) - 1;
    for (uint32_t id = threadIdx.x; id < tasks; id += THREADS) {
        const uint32_t j = id & (lc - 1), g = id >> log_lc;
        const uint32_t tl = g & lowmask;
        const uint32_t tbase = ((g >> b0) << (b0 + Q)) | tl;
        if (j >= lanes_live) continue;
        uint32_t x[1 << Q];
#pragma unroll
        for (int e = 0; e < (1 << Q); e++) {
            const uint32_t t = tbase | ((uint32_t)e << b0);
            x[e] = G_IN ? gin(t, j) : sm[sidx(t, j, log_lc, sshift)];
        }
        // twiddle index of a pair = (position mod 2^u): lane part (strided passes only) + low row bits + el << b0
        const uint32_t koff = j * lane_koff_mul + (tl << ubase);
        reg_stages<Q, INV>(x, tw, ubase + b0, koff, 1u << (b0 + ubase), ninv);
#pragma unroll
        for (int e = 0; e < (1 << Q); e++) {
            const uint32_t t = tbase | ((uint32_t)e << b0);
            if (G_OUT) gout(t, j, x[e]);
            else sm[sidx(t, j, log_lc, sshift)] = x[e];
        }
    }
}

template <bool INV, bool G_IN, bool G_OUT, typename AddrIn, typename AddrOut>
__device__ __forceinline__ void tile_round_q(int q, uint32_t* sm, int log_rows, int log_lc, int sshift, int b0, const uint2* tw,
                                             int ubase, uint32_t lane_koff_mul, uint2 ninv, AddrIn gin, AddrOut gout, uint32_t lanes_live) {
    switch (q) {
    case 5: tile_round<5, INV, G_IN, G_OUT>(sm, log_rows, log_lc, sshift, b0, tw, ubase, lane_koff_mul, ninv, gin, gout, lanes_live); break;
    case 4: tile_round<4, INV, G_IN, G_OUT>(sm, log_rows, log_lc, sshift, b0, tw, ubase, lane_koff_mul, ninv, gin, gout, lanes_live); break;
    case 3: tile_round<3, INV, G_IN, G_OUT>(sm, log_rows, log_lc, sshift, b0, tw, ubase, lane_koff_mul, ninv, gin, gout, lanes_live); break;
    case 2: tile_round<2, INV, G_IN, G_OUT>(sm, log_rows, log_lc, sshift, b0, tw, ubase, lane_koff_mul, ninv, gin, gout, lanes_live); break;
    default: tile_round<1, INV, G_IN, G_OUT>(sm, log_rows, log_lc, sshift, b0, tw, ubase, lane_koff_mul, ninv, gin, gout, lanes_live); break;
    }
}

struct NoAddr {
    __device__ __forceinline__ uint32_t operator()(uint32_t, uint32_t) const { return 0; }
    __device__ __forceinline__ void operator()(uint32_t, uint32_t, uint32_t) const {}
};

// ---------------------------------------------------------------------------------------------------------------------
// K1 (INV) / K3 (!INV): strided tile of one column.  Rows t <-> position bits [n_lo, n), lane j <-> position j0 + j.
// K1: src = input column, dst = tmp (same layout).  K3: src = tmp2[col][coset], dst = LDE column, bit-reversed store.
template <bool INV>
__global__ void __launch_bounds__(THREADS) strided_pass_kernel(const uint32_t* __restrict__ src, size_t src_col_stride,
                                                               uint32_t* __restrict__ dst, size_t dst_col_stride, int n, int n_lo,
                                                               int log_lc, int log_blowup, const uint2* __restrict__ tw_all,
                                                               Rounds rounds) {
    extern __shared__ uint32_t sm[];
    const int n_hi = n - n_lo;
    const uint32_t j0 = blockIdx.x << log_lc;
    const int c = INV ? 0 : (int)blockIdx.z;
    const int cosets = INV ? 1 : (1 << log_blowup);
    const uint32_t* s = INV ? src + (size_t)blockIdx.y * src_col_stride : src + (((size_t)blockIdx.y * cosets + c) << n);
    // the lane part of a twiddle index is the position itself, j0 + j: fold j0 into the table pointer
    const uint2* tw = tw_all + ((size_t)c << n) + j0;
    const int sshift = n_hi >= log_lc ? n_hi - log_lc : 0;
    auto gin = [&](uint32_t t, uint32_t j) -> uint32_t { return __ldg(s + ((size_t)t << n_lo) + j0 + j); };
    uint32_t* d1 = dst + (size_t)blockIdx.y * dst_col_stride;
    auto gout = [&](uint32_t t, uint32_t j, uint32_t v) { d1[((size_t)t << n_lo) + j0 + j] = v; };
    for (int r = 0; r < rounds.n; r++) {
        const bool first = r == 0, last = r == rounds.n - 1;
        const bool g_out = last && INV;               // K3 always finishes through shared memory (transposed store)
        if (first && g_out) tile_round_q<INV, true, true>(rounds.q[r], sm, n_hi, log_lc, sshift, rounds.b0[r], tw, n_lo, 1u, make_uint2(0u, 0u), gin, gout, 1u << log_lc);
        else if (first) tile_round_q<INV, true, false>(rounds.q[r], sm, n_hi, log_lc, sshift, rounds.b0[r], tw, n_lo, 1u, make_uint2(0u, 0u), gin, gout, 1u << log_lc);
        else if (g_out) tile_round_q<INV, false, true>(rounds.q[r], sm, n_hi, log_lc, sshift, rounds.b0[r], tw, n_lo, 1u, make_uint2(0u, 0u), gin, gout, 1u << log_lc);
        else tile_round_q<INV, false, false>(rounds.q[r], sm, n_hi, log_lc, sshift, rounds.b0[r], tw, n_lo, 1u, make_uint2(0u, 0u), gin, gout, 1u << log_lc);
        __syncthreads();
    }
    if (!INV) {
        // natural evaluation index k = j0 + j + (t << n_lo) of coset c lands at row  bitrev_b(c)*N + bitrev_n(k)
        const uint32_t rows = 1u << n_hi, tile = rows << log_lc;
        uint32_t* dcol = dst + (size_t)blockIdx.y * dst_col_stride + ((size_t)brev((uint32_t)c, log_blowup) << n);
        for (uint32_t e = threadIdx.x; e < tile; e += THREADS) {
            const uint32_t p = e & (rows - 1), j = e >> n_hi;       // consecutive threads -> consecutive output rows
            const uint32_t t = brev(p, n_hi);
            dcol[((size_t)brev(j0 + j, n_lo) << n_hi) + p] = sm[sidx(t, j, log_lc, sshift)];
        }
    }
}

// K2a (INV) / K2b (!INV): transposed tile.  Lane l <-> one contiguous block of 2^n_lo positions, rows t <-> bits [0, n_lo).
// Blocks are numbered across the whole column batch (block id = col * blocks_per_col + blk) so narrow/short inputs still
// fill the 32 lanes.  K2a: src -> coefficients (bit-reversed slots) in `dst`, both [col][N].  K2b: dst is [col][coset][N].
template <bool INV>
__global__ void __launch_bounds__(THREADS) transposed_pass_kernel(const uint32_t* __restrict__ src, size_t src_col_stride,
                                                                  uint32_t* __restrict__ dst, int n, int n_lo, int log_lc,
                                                                  int log_blowup, size_t total_blocks, const uint2* __restrict__ tw_all,
                                                                  uint2 ninv, Rounds rounds) {
    extern __shared__ uint32_t sm[];
    const int c = INV ? 0 : (int)blockIdx.z;
    const int cosets = INV ? 1 : (1 << log_blowup);
    const uint32_t lc = 1u << log_lc, rows = 1u << n_lo, tile = rows << log_lc;
    const size_t b_first = (size_t)blockIdx.x << log_lc;
    const uint32_t live = (uint32_t)min((size_t)lc, total_blocks - b_first);
    const int log_bpc = n - n_lo;                                   // blocks per column
    const uint2* tw = tw_all + ((size_t)c << n);
    // fill: consecutive threads read consecutive positions of one block (coalesced), scatter into [t][l] with the swizzle
    for (uint32_t e = threadIdx.x; e < tile; e += THREADS) {
        const uint32_t t = e & (rows - 1), l = e >> n_lo;
        if (l < live) {
            const size_t b = b_first + l, col = b >> log_bpc, blk = b & (((size_t)1 << log_bpc) - 1);
            sm[sidx(t, l, log_lc, 0)] = __ldg(src + col * src_col_stride + (blk << n_lo) + t);
        }
    }
    __syncthreads();
    NoAddr na;
    for (int r = 0; r < rounds.n; r++) {
        tile_round_q<INV, false, false>(rounds.q[r], sm, n_lo, log_lc, 0, rounds.b0[r], tw, 0, 0u, ninv, na, na, live);
        __syncthreads();
    }
    for (uint32_t e = threadIdx.x; e < tile; e += THREADS) {
        const uint32_t t = e & (rows - 1), l = e >> n_lo;
        if (l < live) {
            const size_t b = b_first + l, col = b >> log_bpc, blk = b & (((size_t)1 << log_bpc) - 1);
            dst[((col * cosets + c) << n) + (blk << n_lo) + t] = sm[sidx(t, l, log_lc, 0)];
        }
    }
}

// n_hi == 0 only: scatter the natural-order evaluations of tmp2[col][coset][N] to bit-reversed rows of the LDE
__global__ void bitrev_store_kernel(const uint32_t* __restrict__ tmp2, uint32_t* __restrict__ out, size_t out_col_stride, int n,
                                    int log_blowup, size_t n_cols) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int cosets = 1 << log_blowup;
    if (i >= ((n_cols * cosets) << n)) return;
    const uint32_t k = (uint32_t)(i & (((size_t)1 << n) - 1));
    const size_t cc = i >> n, col = cc / cosets, c = cc % cosets;
    out[col * out_col_stride + ((size_t)brev((uint32_t)c, log_blowup) << n) + brev(k, n)] = tmp2[i];
}

// bit-reversal of rows inside each column (used to feed bit-reversed quotient chunks back into the LDE)
__global__ void bitrev_rows_kernel(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, int n, size_t n_cols) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (n_cols << n)) return;
    size_t col = i >> n;
    uint32_t r = (uint32_t)(i & (((size_t)1 << n) - 1));
    out[(col << n) + brev(r, n)] = in[i];
}

}  // namespace ntt
