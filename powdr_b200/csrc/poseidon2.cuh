// Poseidon2 over BabyBear, width 16, x^7, 8 external + 13 internal rounds -- one permutation state per thread,
// 16 registers, Montgomery form.  Stage 3a of the north-star path (SURVEY.md §8 a8); the reference holds only the
// type names (BabyBearPoseidon2Config, /root/reference/openvm/src/lib.rs:26-28) and the S-box degree
// (/root/reference/openvm/src/powdr_extension/trace_generator/cpu/periphery.rs:80).
//
// Integer-pipe bound (≈22 mulmod per hashed byte): the design goal is instruction count, not bytes.
//  * S-box runs in SIGNED Montgomery form: x = s + (rc - p) in [-p,p) costs one IADD, the four products need no
//    correction (3 IMAD-class ops each), one 2-op fix-up returns to [0,p).
//  * linear layers are add chains on canonical values (IADD3 + IADD3 + UMIN per modular add).
#pragma once
#include "bb31.cuh"

namespace p2 {

struct Consts {
    uint32_t rc_ext_mp[8][16];   // Montgomery(rc) - p   (as two's-complement u32)
    uint32_t rc_int_mp[13];      // Montgomery(rc) - p
    uint32_t diag_w[16];         // V_i canonical, internal matrix = 1 + diag(V): multiplying a Montgomery value by a CANONICAL
    uint32_t diag_wp[16];        // constant keeps it in Montgomery form -> Shoup's method, wp = floor(w * 2^32 / p)
    uint32_t p3_diag;            // 1 when V is the Plonky3 vector [-2,1,2,1/2,3,4,-1/2,-3,-4,2^-8,1/4,1/8,2^-27,-2^-8,-1/16,-2^-27]
};
__constant__ Consts c_p2;

__device__ __forceinline__ uint32_t sbox_rc(uint32_t s, uint32_t rc_minus_p) {
    int32_t x = (int32_t)(s + rc_minus_p);          // [-p, p)
    int32_t x2 = bb::smul(x, x);
    int32_t x3 = bb::smul(x2, x);
    int32_t x4 = bb::smul(x2, x2);
    return bb::from_signed(bb::smul(x3, x4));
}

// M4 = [[2,3,1,1],[1,2,3,1],[1,1,2,3],[3,1,1,2]] on each 4-chunk, then add the column sums: circ(2*M4, M4, M4, M4)
__device__ __forceinline__ void external_linear(uint32_t (&s)[16]) {
#pragma unroll
    for (int c = 0; c < 16; c += 4) {
        uint32_t x0 = s[c], x1 = s[c + 1], x2 = s[c + 2], x3 = s[c + 3];
        uint32_t t01 = bb::add(x0, x1), t23 = bb::add(x2, x3);
        uint32_t t0123 = bb::add(t01, t23);
        uint32_t t01123 = bb::add(t0123, x1), t01233 = bb::add(t0123, x3);
        s[c + 3] = bb::add(t01233, bb::add(x0, x0));
        s[c + 1] = bb::add(t01123, bb::add(x2, x2));
        s[c] = bb::add(t01123, t01);
        s[c + 2] = bb::add(t01233, t23);
    }
    uint32_t q0 = bb::add(bb::add(s[0], s[4]), bb::add(s[8], s[12]));
    uint32_t q1 = bb::add(bb::add(s[1], s[5]), bb::add(s[9], s[13]));
    uint32_t q2 = bb::add(bb::add(s[2], s[6]), bb::add(s[10], s[14]));
    uint32_t q3 = bb::add(bb::add(s[3], s[7]), bb::add(s[11], s[15]));
#pragma unroll
    for (int c = 0; c < 16; c += 4) {
        s[c] = bb::add(s[c], q0);
        s[c + 1] = bb::add(s[c + 1], q1);
        s[c + 2] = bb::add(s[c + 2], q2);
        s[c + 3] = bb::add(s[c + 3], q3);
    }
}

// a * w mod p for a fixed w (Shoup): q = hi(a*w'), r = a*w - q*p in [0,2p), one correction.  IMAD.HI + 2 IMAD = 8 FMA-pipe
// cycles per warp against 10 for a Montgomery product (IMAD.WIDE and IMAD.HI are half rate on sm_90), and no fix-up adds.
__device__ __forceinline__ uint32_t mul_const(uint32_t a, uint32_t w, uint32_t wp) {
    const uint32_t q = __umulhi(a, wp);
    return bb::reduce_2p(a * w - q * bb::P);
}
__device__ __forceinline__ uint32_t halve(uint32_t x) { return (x >> 1) + (x & 1u) * ((bb::P + 1) / 2); }
// x * 2^-K mod p for x in [0,p), K <= 27, WITHOUT a modular product: p = 15*2^27 + 1 is 1 mod 2^K, so the Montgomery-style
// quotient digit is m = (-x) mod 2^K and (x + m p) / 2^K = ((x + m) >> K) + m * 15 * 2^(27-K) < p.  One IMAD (2 FMA-pipe cycles)
// and three ALU instructions instead of a Shoup product (IMAD.HI + 2 IMAD = 8 cycles) and its correction.
template <int K>
__device__ __forceinline__ uint32_t div_2k(uint32_t x) {
    const uint32_t m = (0u - x) & ((1u << K) - 1u);
    return ((x + m) >> K) + m * (15u << (27 - K));
}

__device__ __forceinline__ void internal_round(uint32_t (&s)[16], int r) {
    s[0] = sbox_rc(s[0], c_p2.rc_int_mp[r]);
    uint32_t a = bb::add(bb::add(s[0], s[1]), bb::add(s[2], s[3]));
    uint32_t b = bb::add(bb::add(s[4], s[5]), bb::add(s[6], s[7]));
    uint32_t c = bb::add(bb::add(s[8], s[9]), bb::add(s[10], s[11]));
    uint32_t d = bb::add(bb::add(s[12], s[13]), bb::add(s[14], s[15]));
    uint32_t sum = bb::add(bb::add(a, b), bb::add(c, d));
    if (c_p2.p3_diag) {
        // every entry of the Plonky3 diagonal [-2,1,2,1/2,3,4,-1/2,-3,-4,2^-8,1/4,1/8,2^-27,-2^-8,-1/16,-2^-27] without a modular
        // product: small multiples as add chains, the 2^-K entries through div_2k -- the multiplier pipe is the binding one
        const uint32_t x4 = bb::dbl(s[4]), x5 = bb::dbl(bb::dbl(s[5])), x7 = bb::dbl(s[7]), x8 = bb::dbl(bb::dbl(s[8]));
        s[0] = bb::sub(bb::sub(sum, s[0]), s[0]);          // -2
        s[1] = bb::add(sum, s[1]);                         //  1
        s[2] = bb::add(sum, bb::dbl(s[2]));                //  2
        s[3] = bb::add(sum, halve(s[3]));                  //  1/2
        s[4] = bb::add(sum, bb::add(x4, s[4]));            //  3
        s[5] = bb::add(sum, x5);                           //  4
        s[6] = bb::sub(sum, halve(s[6]));                  // -1/2
        s[7] = bb::sub(sum, bb::add(x7, s[7]));            // -3
        s[8] = bb::sub(sum, x8);                           // -4
        s[9] = bb::add(sum, div_2k<8>(s[9]));              //  2^-8
        s[10] = bb::add(sum, div_2k<2>(s[10]));            //  1/4
        s[11] = bb::add(sum, div_2k<3>(s[11]));            //  1/8
        s[12] = bb::add(sum, div_2k<27>(s[12]));           //  2^-27
        s[13] = bb::sub(sum, div_2k<8>(s[13]));            // -2^-8
        s[14] = bb::sub(sum, div_2k<4>(s[14]));            // -1/16
        s[15] = bb::sub(sum, div_2k<27>(s[15]));           // -2^-27
    } else {
#pragma unroll
        for (int i = 0; i < 16; i++) s[i] = bb::add(sum, mul_const(s[i], c_p2.diag_w[i], c_p2.diag_wp[i]));
    }
}

__device__ __forceinline__ void permute(uint32_t (&s)[16]) {
    external_linear(s);
#pragma unroll 1
    for (int r = 0; r < 4; r++) {
#pragma unroll
        for (int i = 0; i < 16; i++) s[i] = sbox_rc(s[i], c_p2.rc_ext_mp[r][i]);
        external_linear(s);
    }
#pragma unroll 1
    for (int r = 0; r < 13; r++) internal_round(s, r);
#pragma unroll 1
    for (int r = 4; r < 8; r++) {
#pragma unroll
        for (int i = 0; i < 16; i++) s[i] = sbox_rc(s[i], c_p2.rc_ext_mp[r][i]);
        external_linear(s);
    }
}

// ---------------- kernels ----------------

// Leaf kernels: __launch_bounds__(256, 1) lets ptxas take 64 registers (it stops at 40 with the default bound); the extra
// registers buy instruction-level parallelism across the 16 independent S-boxes and measured +8.6 % permutations/s
// (4.07 vs 3.75 G/s) even though resident warps drop from 48 to 32 per SM.  Forcing 32 registers (64 warps) is slower (3.8).
constexpr int LEAF_THREADS = 128;

// leaf r = sponge(row r of the concatenation of all committed matrices); `cols` holds one base pointer per column.
// Overwrite-mode absorb, rate 8, no padding (PaddingFreeSponge<16,8,8>).  One thread per row; consecutive threads read
// consecutive rows of a column-major matrix => every load is a fully coalesced 128 B warp transaction.
__global__ void __launch_bounds__(256, 1) leaf_hash_cols_kernel(const uint32_t* const* __restrict__ cols, uint32_t n_cols,
                                                 size_t height, uint32_t* __restrict__ digests) {
    size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= height) return;
    uint32_t s[16];
#pragma unroll
    for (int i = 0; i < 16; i++) s[i] = 0;
    uint32_t full = n_cols / 8;
    uint32_t nxt[8];
    if (full) {
#pragma unroll
        for (int k = 0; k < 8; k++) nxt[k] = __ldg(cols[k] + r);
    }
    for (uint32_t c = 0; c < full; c++) {
#pragma unroll
        for (int k = 0; k < 8; k++) s[k] = nxt[k];
        if (c + 1 < full) {
#pragma unroll
            for (int k = 0; k < 8; k++) nxt[k] = __ldg(cols[(c + 1) * 8 + k] + r);
        }
        permute(s);
    }
    uint32_t rem = n_cols - full * 8;
    if (rem) {
#pragma unroll
        for (int k = 0; k < 8; k++)
            if ((uint32_t)k < rem) s[k] = __ldg(cols[full * 8 + k] + r);
        permute(s);
    }
    uint4* out = reinterpret_cast<uint4*>(digests + 8 * r);
    out[0] = make_uint4(s[0], s[1], s[2], s[3]);
    out[1] = make_uint4(s[4], s[5], s[6], s[7]);
}

// Streaming variant of the leaf sponge for the host-input pipeline: absorbs one CHUNK of columns (a multiple of 8 unless
// it is the last chunk) into per-row sponge states kept in HBM as [16][height] (word-major => coalesced), so hashing of
// chunk k overlaps the PCIe copy and the LDE of chunk k+1.  first: start from the zero state; last: emit the digest.
__global__ void __launch_bounds__(256, 1) leaf_absorb_cols_kernel(const uint32_t* const* __restrict__ cols, uint32_t n_cols, size_t height,
                                                   uint32_t* __restrict__ state, uint32_t* __restrict__ digests,
                                                   int first, int last) {
    size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= height) return;
    uint32_t s[16];
    if (first) {
#pragma unroll
        for (int i = 0; i < 16; i++) s[i] = 0;
    } else {
#pragma unroll
        for (int i = 0; i < 16; i++) s[i] = state[(size_t)i * height + r];
    }
    uint32_t full = n_cols / 8;
    uint32_t nxt[8];
    if (full) {
#pragma unroll
        for (int k = 0; k < 8; k++) nxt[k] = __ldg(cols[k] + r);
    }
    for (uint32_t c = 0; c < full; c++) {
#pragma unroll
        for (int k = 0; k < 8; k++) s[k] = nxt[k];
        if (c + 1 < full) {
#pragma unroll
            for (int k = 0; k < 8; k++) nxt[k] = __ldg(cols[(c + 1) * 8 + k] + r);
        }
        permute(s);
    }
    uint32_t rem = n_cols - full * 8;
    if (rem) {
#pragma unroll
        for (int k = 0; k < 8; k++)
            if ((uint32_t)k < rem) s[k] = __ldg(cols[full * 8 + k] + r);
        permute(s);
    }
    if (last) {
        uint4* out = reinterpret_cast<uint4*>(digests + 8 * r);
        out[0] = make_uint4(s[0], s[1], s[2], s[3]);
        out[1] = make_uint4(s[4], s[5], s[6], s[7]);
    } else {
#pragma unroll
        for (int i = 0; i < 16; i++) state[(size_t)i * height + r] = s[i];
    }
}

// leaves of a row-major width-8 matrix (FRI layer: row = (f[2j], f[2j+1]) as 8 base elements): one permutation each
__global__ void __launch_bounds__(256, 1) leaf_hash_rows8_kernel(const uint4* __restrict__ rows, size_t height, uint32_t* __restrict__ digests) {
    size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= height) return;
    uint4 a = __ldg(rows + 2 * r), b = __ldg(rows + 2 * r + 1);
    uint32_t s[16] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, 0, 0, 0, 0, 0, 0, 0, 0};
    permute(s);
    uint4* out = reinterpret_cast<uint4*>(digests + 8 * r);
    out[0] = make_uint4(s[0], s[1], s[2], s[3]);
    out[1] = make_uint4(s[4], s[5], s[6], s[7]);
}

// one Merkle layer: parent j = TruncatedPermutation(left || right)
__global__ void __launch_bounds__(256, 1) compress_layer_kernel(const uint4* __restrict__ prev, uint4* __restrict__ next, size_t n_parents) {
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_parents) return;
    uint4 a = prev[4 * j], b = prev[4 * j + 1], c = prev[4 * j + 2], d = prev[4 * j + 3];
    uint32_t s[16] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, c.x, c.y, c.z, c.w, d.x, d.y, d.z, d.w};
    permute(s);
    next[2 * j] = make_uint4(s[0], s[1], s[2], s[3]);
    next[2 * j + 1] = make_uint4(s[4], s[5], s[6], s[7]);
}

// mixed-height MMCS (Plonky3 MerkleTreeMmcs): a level whose size equals the height of further matrices gets the digest of their rows
// injected: node[j] = compress(node[j], injected[j])
__global__ void __launch_bounds__(256, 1) inject_layer_kernel(uint4* __restrict__ nodes, const uint4* __restrict__ injected, size_t n) {
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    uint4 a = nodes[2 * j], b = nodes[2 * j + 1], c = injected[2 * j], d = injected[2 * j + 1];
    uint32_t s[16] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, c.x, c.y, c.z, c.w, d.x, d.y, d.z, d.w};
    permute(s);
    nodes[2 * j] = make_uint4(s[0], s[1], s[2], s[3]);
    nodes[2 * j + 1] = make_uint4(s[4], s[5], s[6], s[7]);
}

// kb tree levels per launch: CTA b reduces nodes [b << kb, (b + 1) << kb) of the level at `level` (n nodes) to one node,
// writing every intermediate level at its place in the node-major layer array (level l+1 follows level l).  A thread reads
// back only what its own CTA wrote, so __syncthreads() orders the global traffic.  Cuts the launches of a 2^21-leaf tree
// from 12 to 3 (FRI commits 20 trees per segment, so launch latency was most of that phase).
__global__ void __launch_bounds__(256) compress_block_kernel(uint4* level, size_t n, int kb) {
    uint4* lvl = level;
    size_t nn = n, off = (size_t)blockIdx.x << kb;
    uint32_t cnt = 1u << kb;
    for (int l = 0; l < kb; l++) {
        uint4* next = lvl + 2 * nn;
        const uint32_t m = cnt >> 1;
        const size_t q0 = off >> 1;
        for (uint32_t j = threadIdx.x; j < m; j += blockDim.x) {
            const uint4* pr = lvl + 4 * (q0 + j);
            uint4 a = pr[0], b = pr[1], c = pr[2], d = pr[3];
            uint32_t s[16] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, c.x, c.y, c.z, c.w, d.x, d.y, d.z, d.w};
            permute(s);
            next[2 * (q0 + j)] = make_uint4(s[0], s[1], s[2], s[3]);
            next[2 * (q0 + j) + 1] = make_uint4(s[4], s[5], s[6], s[7]);
        }
        __syncthreads();
        lvl = next;
        nn >>= 1;
        cnt = m;
        off = q0;
    }
}

// proof-of-work grinding (Plonky3 `grind`): candidate w = base + thread; the challenger's duplex state with the pending inputs
// already written in is `st`, the witness goes to slot `pos`, ONE permutation, the sampled word is output slot 7; accept when
// its canonical value has the `mask` bits clear.  found <- min accepted witness (atomicMin), 0xffffffff when none in this batch.
struct GrindState { uint32_t s[16]; };
__global__ void __launch_bounds__(256, 1) grind_kernel(GrindState st, int pos, uint32_t mask, uint32_t base, uint32_t count, uint32_t* found) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const uint32_t w = base + i;
    if (w >= bb::P) return;
    uint32_t s[16];
#pragma unroll
    for (int k = 0; k < 16; k++) s[k] = st.s[k];
#pragma unroll
    for (int k = 0; k < 8; k++)
        if (k == pos) s[k] = bb::to_monty(w);
    permute(s);
    if ((bb::from_monty(s[7]) & mask) == 0) atomicMin(found, w);
}

// ---------------- 16 lanes per permutation: the latency-bound end of the path ----------------
// One thread per permutation is the throughput shape, but a single permutation then takes ~8 us (5 k dependent-issue instructions
// in one warp), and the top of every Merkle tree, every small FRI layer and the transcript itself are CHAINS of single
// permutations: 210 dependent levels in the FRI commit phase of a 2^21 codeword.  Here lane i of a 16-lane group holds state
// word i: the S-box layer is one x^7 per lane, the external layer is two in-group rotations + two xor-shuffles
// (y_i = S + x_i + 2 x_(i+1) inside a 4-lane chunk, then the column sums), the internal layer a 4-step xor-shuffle sum plus one
// Shoup product by the lane's diagonal entry.  ~4x shorter latency per permutation, ~4x more issue slots: used where a level has
// at most a few thousand permutations.
struct CoopConsts { uint32_t rc[8], dw, dwp; };
__device__ __forceinline__ CoopConsts coop_load(int lane) {
    CoopConsts k;
#pragma unroll
    for (int r = 0; r < 8; r++) k.rc[r] = c_p2.rc_ext_mp[r][lane];
    k.dw = c_p2.diag_w[lane];
    k.dwp = c_p2.diag_wp[lane];
    return k;
}
__device__ __forceinline__ uint32_t coop_external(uint32_t x, int lane) {
    const int base = lane & ~3;
    const uint32_t x1 = __shfl_sync(0xffffffffu, x, base | ((lane + 1) & 3), 16);
    const uint32_t t = bb::add(x, x1);
    const uint32_t S = bb::add(t, __shfl_sync(0xffffffffu, t, base | ((lane + 2) & 3), 16));
    const uint32_t y = bb::add(bb::add(S, x), bb::dbl(x1));
    const uint32_t a = bb::add(y, __shfl_xor_sync(0xffffffffu, y, 4, 16));
    const uint32_t q = bb::add(a, __shfl_xor_sync(0xffffffffu, a, 8, 16));
    return bb::add(y, q);
}
// every lane of the warp must call this (full-mask shuffles); lane = threadIdx.x & 15
__device__ __forceinline__ uint32_t permute_coop16(uint32_t x, int lane, const CoopConsts& k) {
    x = coop_external(x, lane);
#pragma unroll
    for (int r = 0; r < 4; r++) x = coop_external(sbox_rc(x, k.rc[r]), lane);
#pragma unroll 1
    for (int r = 0; r < 13; r++) {
        const uint32_t xs = sbox_rc(x, c_p2.rc_int_mp[r]);
        x = lane == 0 ? xs : x;
        uint32_t sum = x;
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) sum = bb::add(sum, __shfl_xor_sync(0xffffffffu, sum, o, 16));
        x = bb::add(sum, mul_const(x, k.dw, k.dwp));
    }
#pragma unroll
    for (int r = 4; r < 8; r++) x = coop_external(sbox_rc(x, k.rc[r]), lane);
    return x;
}

// kb tree levels, CTA b reduces nodes [b << kb, (b + 1) << kb) of the level at `level` (n nodes) to one node -- the 16-lane
// counterpart of compress_block_kernel (grid 1, kb = log2 n: the whole top of a tree).  blockDim.x = 16 * groups.
__global__ void __launch_bounds__(1024) compress_coop_kernel(uint32_t* level, size_t n, int kb) {
    const int lane = threadIdx.x & 15;
    const uint32_t grp = threadIdx.x >> 4, ngrp = blockDim.x >> 4;
    const CoopConsts k = coop_load(lane);
    uint32_t* lvl = level;
    size_t nn = n, off = (size_t)blockIdx.x << kb;
    uint32_t cnt = 1u << kb;
    for (int l = 0; l < kb; l++) {
        uint32_t* next = lvl + 8 * nn;
        const uint32_t m = cnt >> 1;
        const size_t q0 = off >> 1;
        for (uint32_t j0 = 0; j0 < m; j0 += ngrp) {          // the same trip count for every thread: the shuffles need whole warps
            const uint32_t j = j0 + grp;
            const bool live = j < m;
            uint32_t x = live ? lvl[16 * (q0 + j) + lane] : 0u;
            x = permute_coop16(x, lane, k);
            if (live && lane < 8) next[8 * (q0 + j) + lane] = x;
        }
        __syncthreads();
        lvl = next;
        nn >>= 1;
        cnt = m;
        off = q0;
    }
}

// leaves of a row-major width-8 matrix, one 16-lane group per row (small FRI layers)
__global__ void __launch_bounds__(256) leaf_hash_rows8_coop_kernel(const uint32_t* __restrict__ rows, size_t height, uint32_t* __restrict__ digests) {
    const int lane = threadIdx.x & 15;
    const size_t r = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 4;
    const bool live = r < height;
    const CoopConsts k = coop_load(lane);
    uint32_t x = (live && lane < 8) ? __ldg(rows + 8 * r + lane) : 0u;
    x = permute_coop16(x, lane, k);
    if (live && lane < 8) digests[8 * r + lane] = x;
}

// leaf sponge over column-major matrices, one 16-lane group per row (short chips: the sponge is width/8 DEPENDENT permutations per row)
__global__ void __launch_bounds__(256) leaf_hash_cols_coop_kernel(const uint32_t* const* __restrict__ cols, uint32_t n_cols, size_t height,
                                                                  uint32_t* __restrict__ digests) {
    const int lane = threadIdx.x & 15;
    const size_t r = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 4;
    const bool live = r < height;
    const CoopConsts k = coop_load(lane);
    uint32_t x = 0u;
    for (uint32_t c0 = 0; c0 < n_cols; c0 += 8) {            // uniform trip count
        const uint32_t c = c0 + lane;
        if (live && lane < 8 && c < n_cols) x = __ldg(cols[c] + r);      // overwrite mode: a partial last block leaves the other words
        x = permute_coop16(x, lane, k);
    }
    if (live && lane < 8) digests[8 * r + lane] = x;
}

// The FRI commit phase without a host round trip per layer: the duplex sponge lives in device memory, one 16-lane group absorbs
// the layer's root (8 words, overwrite mode, exactly one permutation: the challenger has no pending input between layers) and the
// folding challenge is output words 7..4.  Root and challenge are logged so that the host can replay the transcript afterwards
// (it stays the authority: a mismatch is an internal error) and fill the proof.
__global__ void __launch_bounds__(32) fri_challenge_kernel(uint32_t* sponge16, const uint32_t* __restrict__ root, uint32_t* __restrict__ log12) {
    const int lane = threadIdx.x & 15;
    const bool first = threadIdx.x < 16;
    const CoopConsts k = coop_load(lane);
    uint32_t x = lane < 8 ? root[lane] : sponge16[lane];
    if (first && lane < 8) log12[lane] = x;
    x = permute_coop16(x, lane, k);
    if (first) {
        sponge16[lane] = x;
        if (lane >= 4 && lane < 8) log12[8 + (7 - lane)] = x;
    }
}

// single permutation per thread on [n][16] states -- used by tests and the throughput micro-benchmark
__global__ void __launch_bounds__(256, 1) permute_states_kernel(uint32_t* states, size_t n, int reps) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t s[16];
#pragma unroll
    for (int k = 0; k < 16; k++) s[k] = states[16 * i + k];
    for (int r = 0; r < reps; r++) permute(s);
#pragma unroll
    for (int k = 0; k < 16; k++) states[16 * i + k] = s[k];
}

}  // namespace p2
