// Openings and the DEEP reduced opening (SURVEY.md §8f-4, the first "next" row widened in round 1): what turns the committed
// trace / quotient LDEs into the single Ext4 codeword FRI folds.  Backend counterpart: the opening phase of pcs_opening behind
// sdk.app_prover(exe)?.prove(stdin) (/root/reference/openvm-riscv/src/lib.rs:327-332); APC AIRs are single-row
// (/root/reference/openvm/src/powdr_extension/chip.rs:99-108), so every column is opened at ONE point zeta.
//
//   y_k      = f_k(zeta)                      barycentric over the N trace-domain evaluations:  4 unreduced MACs per element, one pass
//   ro(x_r)  = (sum_j gamma^j f_j(x_r) - sum_j gamma^j y_j) / (x_r - zeta)   over the 2N LDE rows: 4 unreduced 32x32->96-bit MACs per element
// Both stream column-major matrices with lane = row (coalesced), like the leaf and quotient kernels.
#pragma once
#include "bb31.cuh"

namespace deep {

__device__ __forceinline__ bb::E4 e4_inv(bb::E4 a) {
    // norm to F_p[y]/(y^2-11) (y = x^2), then to F_p; all limbs Montgomery
    const uint32_t a0 = a.c[0], a1 = a.c[1], a2 = a.c[2], a3 = a.c[3];
    const uint32_t W = bb::W11_M;
    uint32_t A0 = bb::add(bb::mul(a0, a0), bb::mul(W, bb::mul(a2, a2)));
    uint32_t A1 = bb::dbl(bb::mul(a0, a2));
    uint32_t B0 = bb::add(bb::mul(a1, a1), bb::mul(W, bb::mul(a3, a3)));
    uint32_t B1 = bb::dbl(bb::mul(a1, a3));
    uint32_t n0 = bb::sub(A0, bb::mul(W, B1)), n1 = bb::sub(A1, B0);
    uint32_t d = bb::inv(bb::sub(bb::mul(n0, n0), bb::mul(W, bb::mul(n1, n1))));
    uint32_t i0 = bb::mul(n0, d), i1 = bb::neg(bb::mul(n1, d));
    bb::E4 conj = {{a0, bb::neg(a1), a2, bb::neg(a3)}};
    bb::E4 s = {{i0, 0u, i1, 0u}};
    return bb::e4_mul(conj, s);
}

// barycentric weights over the subgroup H of size 2^log_n at the point z:  w_i = omega^i / (z - omega^i).
// one_hot (z is a point of H, where one denominator is 0 and the prefactor (z^N - 1)/N too): w_i = [omega^i == z], so that
// with prefactor 1 the weighted sum is the value at that row.
__global__ void __launch_bounds__(256) bary_weights_kernel(uint4* __restrict__ w, int log_n, uint32_t omega_m, bb::E4 z, int one_hot) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ((size_t)1 << log_n)) return;
    const uint32_t x = bb::pow(omega_m, i);
    if (one_hot) {
        w[i] = make_uint4(x == z.c[0] ? bb::R1 : 0u, 0u, 0u, 0u);
        return;
    }
    bb::E4 d = z;
    d.c[0] = bb::sub(d.c[0], x);
    bb::E4 r = bb::e4_scale(e4_inv(d), x);
    w[i] = make_uint4(r.c[0], r.c[1], r.c[2], r.c[3]);
}

// monomial weights for coefficients in bit-reversed slots (what the inverse LDE passes leave):  w_j = z^bitrev(j), so that
// sum_j coef_j * w_j = f(z).  zp[k] = z^(2^k); bit i of j contributes zp[log_n - 1 - i].
struct ZPow2 { bb::E4 p[24]; };
__global__ void __launch_bounds__(256) monomial_weights_kernel(uint4* __restrict__ w, int log_n, ZPow2 zp) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= ((size_t)1 << log_n)) return;
    bb::E4 r = {{bb::R1, 0u, 0u, 0u}};
#pragma unroll
    for (int k = 0; k < 24; k++)          // unrolled: zp stays in the parameter space
        if (k < log_n && ((j >> (log_n - 1 - k)) & 1)) r = bb::e4_mul(r, zp.p[k]);
    w[j] = make_uint4(r.c[0], r.c[1], r.c[2], r.c[3]);
}

// 96-bit accumulator a += f * g.  ptxas turns the carry chain into IMAD.WIDE.U32 with a carry-out predicate and folds two
// carries into one IADD3.X, i.e. 1 multiplier-pipe + 0.5 ALU instruction per MAC.
struct Acc96 { uint32_t w0, w1, w2; };
__device__ __forceinline__ void mac96(Acc96& a, uint32_t f, uint32_t g) {
    asm("mad.lo.cc.u32 %0, %3, %4, %0;\n\tmadc.hi.cc.u32 %1, %3, %4, %1;\n\taddc.u32 %2, %2, 0;" : "+r"(a.w0), "+r"(a.w1), "+r"(a.w2) : "r"(f), "r"(g));
}
// (hi*2^64 + lo) mod p of a 96-bit accumulator, canonical result
__device__ __forceinline__ uint32_t acc96_mod(const Acc96& a) {
    constexpr uint64_t R1_ = 0x100000000ull % bb::P, R2_ = (R1_ * R1_) % bb::P;      // 2^32, 2^64 mod p
    const uint64_t lo = ((uint64_t)a.w1 << 32) | a.w0;
    return (uint32_t)(((uint64_t)(a.w2 % bb::P) * R2_ % bb::P + lo % bb::P) % bb::P);
}

constexpr int EV_COLS = 4;       // columns per CTA (each weight load is reused 4 times; 48 accumulator registers)
constexpr int EV_THREADS = 256;
constexpr int EV_UNROLL = 4;    // rows per thread and step

// partial[k][split] = sum over this CTA's rows of mat[k][i] * w_i.  Both factors are Montgomery words < p, so the products are
// accumulated unreduced in 96 bits (1 IMAD.WIDE + half a carry add per limb instead of a 3-instruction Montgomery product and
// a 2-instruction modular add); the sum is R^2 * (true sum), one Montgomery reduction at the end brings it back to R * sum.
__global__ void __launch_bounds__(EV_THREADS, 2) eval_partial_kernel(const uint32_t* __restrict__ mat, size_t n, uint32_t width,
                                                                  const uint4* __restrict__ w, uint4* __restrict__ partial,
                                                                  uint32_t rows_per_cta) {
    const uint32_t k0 = blockIdx.x * EV_COLS;
    const size_t r0 = (size_t)blockIdx.y * rows_per_cta, r1 = min(n, r0 + rows_per_cta);
    Acc96 acc[EV_COLS][4];
#pragma unroll
    for (int c = 0; c < EV_COLS; c++)
#pragma unroll
        for (int l = 0; l < 4; l++) acc[c][l] = Acc96{0u, 0u, 0u};
    // software-pipelined, EV_UNROLL rows per step: the 20 loads of the next step are in flight while this step's 64 MACs issue
    // (at ~110 registers only 16 warps are resident per SM, so the memory-level parallelism has to come from each thread)
    const uint32_t* col[EV_COLS];
#pragma unroll
    for (int c = 0; c < EV_COLS; c++) col[c] = mat + (size_t)min(k0 + c, width - 1) * n;      // out-of-range columns: results discarded
    size_t i = r0 + threadIdx.x;
    uint4 wi[EV_UNROLL];
    uint32_t f[EV_UNROLL][EV_COLS];
#pragma unroll
    for (int u = 0; u < EV_UNROLL; u++) {
        const size_t iu = i + (size_t)u * EV_THREADS;
        const bool ok = iu < r1;
        wi[u] = ok ? __ldg(w + iu) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
        for (int c = 0; c < EV_COLS; c++) f[u][c] = ok ? __ldg(col[c] + iu) : 0u;
    }
    while (i < r1) {
        const size_t in = i + (size_t)EV_UNROLL * EV_THREADS;
        uint4 wn[EV_UNROLL];
        uint32_t fn[EV_UNROLL][EV_COLS];
#pragma unroll
        for (int u = 0; u < EV_UNROLL; u++) {
            const size_t iu = in + (size_t)u * EV_THREADS;
            const bool ok = iu < r1;
            wn[u] = ok ? __ldg(w + iu) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
            for (int c = 0; c < EV_COLS; c++) fn[u][c] = ok ? __ldg(col[c] + iu) : 0u;
        }
#pragma unroll
        for (int u = 0; u < EV_UNROLL; u++)
#pragma unroll
            for (int c = 0; c < EV_COLS; c++) {
                mac96(acc[c][0], f[u][c], wi[u].x); mac96(acc[c][1], f[u][c], wi[u].y);
                mac96(acc[c][2], f[u][c], wi[u].z); mac96(acc[c][3], f[u][c], wi[u].w);
            }
#pragma unroll
        for (int u = 0; u < EV_UNROLL; u++) {
            wi[u] = wn[u];
#pragma unroll
            for (int c = 0; c < EV_COLS; c++) f[u][c] = fn[u][c];
        }
        i = in;
    }
    __shared__ uint32_t red[EV_THREADS / 32][EV_COLS * 4];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int c = 0; c < EV_COLS; c++)
#pragma unroll
        for (int l = 0; l < 4; l++) {
            uint32_t v = bb::mul(acc96_mod(acc[c][l]), 1u);          // R^2 * sum  ->  R * sum
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v = bb::add(v, __shfl_xor_sync(0xffffffffu, v, o));
            if (lane == 0) red[warp][c * 4 + l] = v;
        }
    __syncthreads();
    if (threadIdx.x < EV_COLS * 4) {
        uint32_t v = 0;
#pragma unroll
        for (int q = 0; q < EV_THREADS / 32; q++) v = bb::add(v, red[q][threadIdx.x]);
        const uint32_t c = threadIdx.x >> 2, l = threadIdx.x & 3;
        if (k0 + c < width) reinterpret_cast<uint32_t*>(partial + ((size_t)(k0 + c) * gridDim.y + blockIdx.y))[l] = v;
    }
}

// y_k = pref * sum_splits partial[k][split]
__global__ void eval_finalize_kernel(const uint4* __restrict__ partial, uint32_t width, uint32_t splits, bb::E4 pref, uint4* __restrict__ ys) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= width) return;
    bb::E4 s = {{0u, 0u, 0u, 0u}};
    for (uint32_t q = 0; q < splits; q++) {
        const uint4 p = partial[(size_t)k * splits + q];
        s.c[0] = bb::add(s.c[0], p.x); s.c[1] = bb::add(s.c[1], p.y); s.c[2] = bb::add(s.c[2], p.z); s.c[3] = bb::add(s.c[3], p.w);
    }
    const bb::E4 y = bb::e4_mul(s, pref);
    ys[k] = make_uint4(y.c[0], y.c[1], y.c[2], y.c[3]);
}

// reduced opening over the LDE domain (bit-reversed rows).
// sum_j gamma^j f_j(x_r) is accumulated WITHOUT modular reduction, in 96-bit integers: one IMAD.WIDE with carry-out plus one
// carry add per limb of gamma^j (canonical, < 2^31) and column -- half the multiplier-pipe work of four reduced products and
// no reductions; f is in Montgomery form, so the sum reduced mod p at the end is the Montgomery form of the result.
// The gamma powers are staged through shared memory in chunks (every thread of the CTA needs the same ones); the opened
// columns come as up to MAX_SEGS runs of equal stride so there is no dependent pointer load, and the 8 loads of the next
// step are issued before the 32 MACs of the current one (ncu r01c: the previous per-column-pointer version with Shoup
// products stalled 75 % on long_scoreboard at 39 % of HBM).
// The m rows passed are rows [row0, row0 + m) of the 2^log_m-row domain (row0 = 0, m = 2^log_m for the whole domain).
constexpr int DQ_MAX_SEGS = 8;
constexpr int DQ_CHUNK = 256;
struct DeepSegs {
    const uint32_t* base[DQ_MAX_SEGS];     // first column of the run, already offset to the row block
    size_t stride[DQ_MAX_SEGS];            // words between consecutive columns
    uint32_t count[DQ_MAX_SEGS];
    uint32_t gp_off[DQ_MAX_SEGS];          // gamma exponent of the run's first column
    uint32_t gp_off2[DQ_MAX_SEGS];         // DQ_NO_SECOND, or the exponent under which the same columns are ALSO opened at the second point
    int n;
};
constexpr uint32_t DQ_NO_SECOND = 0xffffffffu;

__device__ __forceinline__ void dq_mac(Acc96 (&acc)[4], uint32_t f, const uint4 g) {
    mac96(acc[0], f, g.x); mac96(acc[1], f, g.y); mac96(acc[2], f, g.z); mac96(acc[3], f, g.w);
}

__global__ void __launch_bounds__(256) deep_quotient_kernel(DeepSegs segs, size_t m, int log_m, size_t row0, uint32_t shift_m, uint32_t omega_m,
                                                            const uint4* __restrict__ gpow, bb::E4 ysum, bb::E4 zeta, bb::E4 ysum2, bb::E4 zeta2,
                                                            int two_points, uint4* __restrict__ out, int accumulate) {
    __shared__ uint4 sg[DQ_CHUNK];
    const size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = r < m;
    const size_t rr = live ? r : m - 1;           // dead threads of the last CTA still take part in the staging barriers
    Acc96 acc[4] = {{0u, 0u, 0u}, {0u, 0u, 0u}, {0u, 0u, 0u}, {0u, 0u, 0u}};
    Acc96 acc2[4] = {{0u, 0u, 0u}, {0u, 0u, 0u}, {0u, 0u, 0u}, {0u, 0u, 0u}};      // columns opened at the second point (read once, used twice)
    for (int sgi = 0; sgi < segs.n; sgi++) {
        const size_t jglob = segs.gp_off[sgi];
        if (segs.gp_off2[sgi] != DQ_NO_SECOND) {
            // run opened at both points: one load feeds both accumulators
            const size_t stride2 = segs.stride[sgi], jglob2 = segs.gp_off2[sgi];
            const uint32_t count2 = segs.count[sgi];
            const uint32_t* p2 = segs.base[sgi] + rr;
            for (uint32_t c0 = 0; c0 < count2; c0 += DQ_CHUNK / 2) {
                const uint32_t nc = min((uint32_t)(DQ_CHUNK / 2), count2 - c0);
                __syncthreads();
                for (uint32_t i = threadIdx.x; i < nc; i += blockDim.x) { sg[i] = __ldg(gpow + jglob + c0 + i); sg[DQ_CHUNK / 2 + i] = __ldg(gpow + jglob2 + c0 + i); }
                __syncthreads();
                // software-pipelined like the single-point path: the 8 loads of the next step are in flight during the 64 MACs of this one
                uint32_t j = 0;
                if (nc >= 8) {
                    uint32_t f[8], fn[8];
#pragma unroll
                    for (int u = 0; u < 8; u++) f[u] = __ldg(p2 + (size_t)(c0 + u) * stride2);
                    for (; j + 16 <= nc; j += 8) {
#pragma unroll
                        for (int u = 0; u < 8; u++) fn[u] = __ldg(p2 + (size_t)(c0 + j + 8 + u) * stride2);
#pragma unroll
                        for (int u = 0; u < 8; u++) { dq_mac(acc, f[u], sg[j + u]); dq_mac(acc2, f[u], sg[DQ_CHUNK / 2 + j + u]); }
#pragma unroll
                        for (int u = 0; u < 8; u++) f[u] = fn[u];
                    }
#pragma unroll
                    for (int u = 0; u < 8; u++) { dq_mac(acc, f[u], sg[j + u]); dq_mac(acc2, f[u], sg[DQ_CHUNK / 2 + j + u]); }
                    j += 8;
                }
                for (; j < nc; j++) { const uint32_t f1 = __ldg(p2 + (size_t)(c0 + j) * stride2); dq_mac(acc, f1, sg[j]); dq_mac(acc2, f1, sg[DQ_CHUNK / 2 + j]); }
            }
            continue;
        }
        const size_t stride = segs.stride[sgi];
        const uint32_t count = segs.count[sgi];
        for (uint32_t c0 = 0; c0 < count; c0 += DQ_CHUNK) {
            const uint32_t nc = min((uint32_t)DQ_CHUNK, count - c0);
            __syncthreads();
            for (uint32_t i = threadIdx.x; i < nc; i += blockDim.x) sg[i] = __ldg(gpow + jglob + c0 + i);
            __syncthreads();
            const uint32_t* p = segs.base[sgi] + (size_t)c0 * stride + rr;
            uint32_t f[8], fn[8];
            uint32_t j = 0;
            if (nc >= 8) {
#pragma unroll
                for (int u = 0; u < 8; u++) f[u] = __ldg(p + (size_t)u * stride);
                for (; j + 16 <= nc; j += 8) {
#pragma unroll
                    for (int u = 0; u < 8; u++) fn[u] = __ldg(p + (size_t)(j + 8 + u) * stride);
#pragma unroll
                    for (int u = 0; u < 8; u++) dq_mac(acc, f[u], sg[j + u]);
#pragma unroll
                    for (int u = 0; u < 8; u++) f[u] = fn[u];
                }
#pragma unroll
                for (int u = 0; u < 8; u++) dq_mac(acc, f[u], sg[j + u]);
                j += 8;
            }
            for (; j < nc; j++) dq_mac(acc, __ldg(p + (size_t)j * stride), sg[j]);
        }
    }
    if (!live) return;
    bb::E4 a;
#pragma unroll
    for (int l = 0; l < 4; l++) {
        a.c[l] = bb::sub(acc96_mod(acc[l]), ysum.c[l]);
    }
    const uint32_t x = bb::mul(shift_m, bb::pow(omega_m, (uint64_t)(__brev((uint32_t)(row0 + r)) >> (32 - log_m))));
    bb::E4 d = {{bb::sub(x, zeta.c[0]), bb::neg(zeta.c[1]), bb::neg(zeta.c[2]), bb::neg(zeta.c[3])}};
    bb::E4 v = bb::e4_mul(a, e4_inv(d));
    if (two_points) {
        bb::E4 a2;
#pragma unroll
        for (int l = 0; l < 4; l++) a2.c[l] = bb::sub(acc96_mod(acc2[l]), ysum2.c[l]);
        bb::E4 d2 = {{bb::sub(x, zeta2.c[0]), bb::neg(zeta2.c[1]), bb::neg(zeta2.c[2]), bb::neg(zeta2.c[3])}};
        v = bb::e4_add(v, bb::e4_mul(a2, e4_inv(d2)));
    }
    if (accumulate) {
        const uint4 o = out[r];
        v.c[0] = bb::add(v.c[0], o.x); v.c[1] = bb::add(v.c[1], o.y); v.c[2] = bb::add(v.c[2], o.z); v.c[3] = bb::add(v.c[3], o.w);
    }
    out[r] = make_uint4(v.c[0], v.c[1], v.c[2], v.c[3]);
}

}  // namespace deep
