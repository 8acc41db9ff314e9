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
//       K1  inverse, bits [n_lo,n)   strided tiles   [2^n_hi rows x 2^log_lc lanes], lane = consecutive position
//       K2a inverse, bits [0,n_lo)   transposed tiles [2^n_lo rows x 2^log_lc lanes], lane = one contiguous 2^n_lo block
//       K2b forward, bits [0,n_lo)   per coset, same geometry
//       K3  forward, bits [n_lo,n)   per coset, strided tiles, then the bit-reversed store
//     Each pass reads and writes its column batch through HBM (11 words per element at b = 1); the batch is sized to fill the
//     SMs, not to keep the intermediates in the 50 MB L2 (smaller, L2-sized batches measured no faster, capi.cu).  At n_lo = 10
//     pb_lde_batch runs K2a and K2b as one pass that keeps the coefficients on chip (ntt_tma.cuh): 9 words per element.
//   * inside a pass the butterfly network never crosses lanes: a thread owns 2^q (q<=5) rows of one lane in REGISTERS and
//     runs q radix-2 stages on them (80 butterflies per 32 loads + 32 stores for q=5); shared memory is touched once per
//     round, conflict-free (lane = bank, XOR swizzle for the two transposed accesses).
// The passes are compile-time specialisations per (n_hi, n_lo) (ntt_fast.cuh, ntt_tma.cuh).  Measured on the H100 they are
// bound by neither pipe alone: 40-75 % of HBM bandwidth at 3-6 butterflies/clk/SM (lde_column_batch in capi.cu, DESIGN.md §4).
#pragma once
#include "bb31.cuh"

namespace ntt {

__device__ __forceinline__ uint32_t brev(uint32_t x, int bits) { return bits ? (__brev(x) >> (32 - bits)) : 0u; }

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
