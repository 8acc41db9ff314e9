// BabyBear (p = 15*2^27 + 1) in Montgomery form, R = 2^32 -- the in-memory representation of
// p3_baby_bear::BabyBear and of the device `Fp` the reference's kernels operate on
// (/root/reference/openvm/cuda/src/expr_eval.cuh:49-50: PUSH_CONST passes a canonical u32 through Fp(u)).
// Everything on the device stays in this form; conversions happen only at the C-ABI edge.
//
// Montgomery product as two wide multiply-adds (sm_90a: IMAD.WIDE x2 + IMAD):
//   t = a*b;  m = lo(t) * (-p^-1 mod 2^32);  d = m*p + t  (low word == 0);  r = hi(d) in [0, 2p)
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

namespace bb {

constexpr uint32_t P = 0x78000001u;         // 2013265921
constexpr uint32_t NEG_PINV = 0x77ffffffu;  // -p^-1 mod 2^32
constexpr uint32_t PINV = 0x88000001u;      //  p^-1 mod 2^32
constexpr uint32_t R1 = 0x0ffffffeu;        // R mod p   (Montgomery form of 1)
constexpr uint32_t R2 = 1172168163u;        // R^2 mod p
constexpr uint32_t GEN = 31u;               // multiplicative generator (canonical)
constexpr uint32_t W11_M = 939524073u;      // 11 * R mod p (extension non-residue, Montgomery form)

#define BB_HD __host__ __device__ __forceinline__

BB_HD uint32_t reduce_2p(uint32_t x) {      // [0,2p) -> [0,p)
    uint32_t y = x - P;
    return y < x ? y : x;                   // unsigned min: x-P wraps above x when x < P
}
BB_HD uint32_t add(uint32_t a, uint32_t b) { return reduce_2p(a + b); }
BB_HD uint32_t sub(uint32_t a, uint32_t b) {
    uint32_t d = a - b, e = d + P;
    return e < d ? e : d;                   // a>=b: d<p<=e (no wrap) -> d ; a<b: d wraps high, e = d+P wraps low -> e
}
BB_HD uint32_t neg(uint32_t a) { return a ? P - a : 0u; }
BB_HD uint32_t dbl(uint32_t a) { return reduce_2p(a + a); }

BB_HD uint32_t mul_lazy(uint32_t a, uint32_t b) {   // a*b < 2^32 * p  ->  result in [0, 2p)
    // plain C on purpose: ptxas folds this into IMAD.WIDE.U32 + IMAD + IMAD.HI.U32 (64-bit addend), 3 instructions
    uint64_t t = (uint64_t)a * b;
    uint32_t m = (uint32_t)t * NEG_PINV;
    uint64_t d = (uint64_t)m * P + t;
    return (uint32_t)(d >> 32);
}
BB_HD uint32_t mul(uint32_t a, uint32_t b) { return reduce_2p(mul_lazy(a, b)); }

// signed Montgomery: |a*b| < 2^31 * p  ->  result in (-p, p), no correction step
BB_HD int32_t smul(int32_t a, int32_t b) {
    // t - m*p has a zero low word when m = lo(t) * p^-1, so the quotient is hi(t) - hi(m*p): no carry to track
#ifdef __CUDA_ARCH__
    int64_t t;
    int32_t lo, hi;
    asm("mul.wide.s32 %0, %1, %2;" : "=l"(t) : "r"(a), "r"(b));
    asm("mov.b64 {%0, %1}, %2;" : "=r"(lo), "=r"(hi) : "l"(t));
    int32_t m = (int32_t)((uint32_t)lo * PINV);
    return hi - __mulhi(m, (int32_t)P);
#else
    int64_t t = (int64_t)a * (int64_t)b;
    int32_t m = (int32_t)((uint32_t)t * PINV);
    int64_t u = ((int64_t)m * (int64_t)P) >> 32;
    return (int32_t)((t >> 32) - u);
#endif
}
BB_HD uint32_t from_signed(int32_t x) {     // (-p,p) -> [0,p)
    uint32_t u = (uint32_t)x, v = u + P;
    return v < u ? v : u;
}

// Shoup product with a fixed multiplier: w.x = w (canonical), w.y = floor(w * 2^32 / p); a may be any u32 (lazy operands ok).
// r = a*w - hi(a*w')*p lies in [0, 2p); one correction makes it canonical.  A Montgomery-form `a` stays in Montgomery form.
BB_HD uint32_t mul_shoup(uint32_t a, uint2 w) {
#ifdef __CUDA_ARCH__
    const uint32_t q = __umulhi(a, w.y);
#else
    const uint32_t q = (uint32_t)(((uint64_t)a * w.y) >> 32);
#endif
    return reduce_2p(a * w.x - q * P);
}
BB_HD uint2 shoup_pair(uint32_t w_canonical) {
    uint2 r;
    r.x = w_canonical;
    r.y = (uint32_t)(((uint64_t)w_canonical << 32) / P);
    return r;
}

BB_HD uint32_t to_monty(uint32_t canonical) { return mul(canonical, R2); }
BB_HD uint32_t from_monty(uint32_t m) { return reduce_2p(mul_lazy(m, 1u)); }

BB_HD uint32_t pow(uint32_t a_m, uint64_t e) {
    uint32_t r = R1;
    while (e) { if (e & 1) r = mul(r, a_m); a_m = mul(a_m, a_m); e >>= 1; }
    return r;
}
BB_HD uint32_t inv(uint32_t a_m) { return pow(a_m, (uint64_t)P - 2); }   // inv(0) = 0

// ---- Ext4 = F_p[x]/(x^4 - 11), Montgomery limbs ----
struct E4 { uint32_t c[4]; };
BB_HD E4 e4_add(E4 a, E4 b) { E4 r; for (int i = 0; i < 4; i++) r.c[i] = add(a.c[i], b.c[i]); return r; }
BB_HD E4 e4_sub(E4 a, E4 b) { E4 r; for (int i = 0; i < 4; i++) r.c[i] = sub(a.c[i], b.c[i]); return r; }
BB_HD E4 e4_scale(E4 a, uint32_t s) { E4 r; for (int i = 0; i < 4; i++) r.c[i] = mul(a.c[i], s); return r; }
BB_HD E4 e4_mul(E4 a, E4 b) {
    // schoolbook; the x^4..x^6 coefficients are folded back through x^4 = 11
    uint32_t hi0 = add(add(mul(a.c[1], b.c[3]), mul(a.c[2], b.c[2])), mul(a.c[3], b.c[1]));   // x^4 coefficient
    uint32_t hi1 = add(mul(a.c[2], b.c[3]), mul(a.c[3], b.c[2]));                               // x^5
    uint32_t hi2 = mul(a.c[3], b.c[3]);                                                         // x^6
    E4 r;
    r.c[0] = add(mul(a.c[0], b.c[0]), mul(hi0, W11_M));
    r.c[1] = add(add(mul(a.c[0], b.c[1]), mul(a.c[1], b.c[0])), mul(hi1, W11_M));
    r.c[2] = add(add(add(mul(a.c[0], b.c[2]), mul(a.c[1], b.c[1])), mul(a.c[2], b.c[0])), mul(hi2, W11_M));
    r.c[3] = add(add(mul(a.c[0], b.c[3]), mul(a.c[1], b.c[2])), add(mul(a.c[2], b.c[1]), mul(a.c[3], b.c[0])));
    return r;
}

}  // namespace bb
