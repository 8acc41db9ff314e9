// Stage 3b of the north-star path: arity-2 FRI folding on bit-reversed Ext4 evaluations (SURVEY.md §8 a9, App. C.5):
//   f'[j] = (lo + hi)/2 + beta * (lo - hi) / (2 x_j),   lo = f[2j], hi = f[2j+1],  x_j = shift * w_len^{bitrev(j)}.
// Codewords are [len][4] (16 B per Ext4 element, fold partners adjacent => two 128-bit loads per output).
// inv_tw[j] = w_len^{-bitrev(j)}; the table of the first layer serves every later layer (its prefix is the next
// layer's table), and the per-layer scalar (2*shift)^-1 is folded into beta on the host.
#pragma once
#include "bb31.cuh"

namespace fri {

__global__ void __launch_bounds__(256) fold_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, size_t half,
                                                   const uint32_t* __restrict__ inv_tw, bb::E4 beta_c, uint32_t half_inv) {
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= half) return;
    uint4 l = __ldg(in + 2 * j), h = __ldg(in + 2 * j + 1);
    bb::E4 lo = {{l.x, l.y, l.z, l.w}}, hi = {{h.x, h.y, h.z, h.w}};
    bb::E4 s = bb::e4_scale(bb::e4_add(lo, hi), half_inv);
    bb::E4 d = bb::e4_scale(bb::e4_sub(lo, hi), __ldg(inv_tw + j));
    bb::E4 r = bb::e4_add(s, bb::e4_mul(beta_c, d));
    out[j] = make_uint4(r.c[0], r.c[1], r.c[2], r.c[3]);
}

// same fold with the challenge read from device memory (Montgomery Ext4, written by p2::fri_challenge_kernel); c = (2*shift)^-1
__global__ void __launch_bounds__(256) fold_dev_beta_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, size_t half,
                                                            const uint32_t* __restrict__ inv_tw, const uint32_t* __restrict__ beta4, uint32_t c,
                                                            uint32_t half_inv) {
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= half) return;
    const bb::E4 beta_c = {{bb::mul(__ldg(beta4), c), bb::mul(__ldg(beta4 + 1), c), bb::mul(__ldg(beta4 + 2), c), bb::mul(__ldg(beta4 + 3), c)}};
    uint4 l = __ldg(in + 2 * j), h = __ldg(in + 2 * j + 1);
    bb::E4 lo = {{l.x, l.y, l.z, l.w}}, hi = {{h.x, h.y, h.z, h.w}};
    bb::E4 s = bb::e4_scale(bb::e4_add(lo, hi), half_inv);
    bb::E4 d = bb::e4_scale(bb::e4_sub(lo, hi), __ldg(inv_tw + j));
    bb::E4 r = bb::e4_add(s, bb::e4_mul(beta_c, d));
    out[j] = make_uint4(r.c[0], r.c[1], r.c[2], r.c[3]);
}

// f[i] += g[i] over n words (multi-chip FRI: the reduced-opening codeword of a shorter height joins the folded codeword)
__global__ void __launch_bounds__(256) add_words_kernel(uint32_t* __restrict__ f, const uint32_t* __restrict__ g, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) f[i] = bb::add(f[i], g[i]);
}

}  // namespace fri

// ---------------- query phase: gather the openings a verifier needs for each sampled index (SURVEY.md §8f-4) ----------------
// One CTA per query and one launch per piece of the layout (include/powdr_b200.h): the index; per commitment the row of each of its
// matrices, then the Merkle path; per FRI layer i the opened pair and its path ((log_max-1-i) x 8).  All words canonical.
// Merkle trees are node-major with level k at node offset 2^(h+1) - 2^(h-k+1); the sibling of leaf idx at level k is (idx>>k)^1.
// A context gathers what it holds: a window of rows [row0, row0 + rows) of each matrix (stored with stride rows) and the subtree over
// them, which gives the bottom log2(rows) levels of the path.  A query whose row lies outside the window writes nothing.
namespace fri {

__device__ __forceinline__ void copy_path(const uint32_t* tree, int log_h, size_t idx, uint32_t* out) {
    for (int k = 0; k < log_h; k++) {
        const size_t level_off = ((size_t)2 << log_h) - ((size_t)2 << (log_h - k));
        const uint32_t* node = tree + 8 * (level_off + ((idx >> k) ^ 1));
        for (int e = threadIdx.x; e < 8; e += blockDim.x) out[8 * k + e] = bb::from_monty(node[e]);
    }
}

// out[q * wpq + off + c] = canonical(mat[c * rows + (idx[q] >> shift) - row0])
__global__ void gather_rows_kernel(const uint32_t* __restrict__ mat, size_t row0, size_t rows, uint32_t width, int shift, const uint32_t* __restrict__ idx,
                                   uint32_t* __restrict__ out, size_t wpq, size_t off) {
    const size_t r = (idx[blockIdx.x] >> shift) - row0;
    if (r >= rows) return;
    uint32_t* o = out + (size_t)blockIdx.x * wpq + off;
    for (uint32_t c = threadIdx.x; c < width; c += blockDim.x) o[c] = bb::from_monty(mat[(size_t)c * rows + r]);
}
// the window is [row0, row0 + 2^log_h), `tree` the subtree over it
__global__ void gather_path_kernel(const uint32_t* __restrict__ tree, size_t row0, int log_h, int shift, const uint32_t* __restrict__ idx, uint32_t* __restrict__ out,
                                   size_t wpq, size_t off) {
    const size_t r = (idx[blockIdx.x] >> shift) - row0;
    if (r >> log_h) return;
    copy_path(tree, log_h, r, out + (size_t)blockIdx.x * wpq + off);
}
__global__ void gather_index_kernel(const uint32_t* __restrict__ idx, uint32_t* __restrict__ out, size_t wpq) {
    if (threadIdx.x == 0) out[(size_t)blockIdx.x * wpq] = idx[blockIdx.x];
}
// layer i: pair rows [row0[i], row0[i] + rows[i]) (a power of two, or 0: nothing held) at word_off[i], their subtree at tree_off[i]
struct FriDesc {
    const uint32_t* fri_words; const uint32_t* fri_trees; int log_m; int n_layers;
    size_t word_off[32]; size_t tree_off[32]; size_t row0[32]; size_t rows[32];
};
__global__ void gather_fri_kernel(FriDesc d, const uint32_t* __restrict__ idx, uint32_t* __restrict__ out, size_t wpq, size_t off) {
    const size_t r = idx[blockIdx.x];
    uint32_t* o = out + (size_t)blockIdx.x * wpq + off;
    for (int i = 0; i < d.n_layers; i++) {
        const size_t j = (r >> (i + 1)) - d.row0[i];
        if (j < d.rows[i]) {
            const uint32_t* row = d.fri_words + d.word_off[i] + 8 * j;
            for (uint32_t e = threadIdx.x; e < 8; e += blockDim.x) o[e] = bb::from_monty(row[e]);
            copy_path(d.fri_trees + d.tree_off[i], __ffsll((long long)d.rows[i]) - 1, j, o + 8);
        }
        o += 8 + 8 * (d.log_m - 1 - i);
    }
}
}  // namespace fri
