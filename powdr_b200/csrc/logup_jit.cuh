// LogUp / bus-interaction argument on the GPU (SURVEY.md §8 f1): per-AIR code generation, like air_jit.cuh for the constraints.
// What is evaluated is pinned by the reference -- PowdrAir::eval pushes every SymbolicBusInteraction {id, mult, args} on
// row_slice(0) (/root/reference/openvm/src/powdr_extension/chip.rs:117-128), bytecode layout = compile_bus_to_gpu
// (/root/reference/openvm/src/powdr_extension/trace_generator/cuda/mod.rs:143-177) -- the argument built from it restates the
// FRI-LogUp phase of stark-backend v1 (formulas in DESIGN.md §3; parity unpinned).
//
// Two generated kernels per AIR, both one thread per row with lane = row (coalesced column-major loads), interactions in
// straight-line code (one SSA value per expression node, constant operands as Shoup products, literal arguments folded into a
// per-interaction Ext4 constant on the host), grouped 16 interactions (<= 8 chunks) per __noinline__ function:
//   pbl_perm  trace domain (N rows):  d_i = kc_i + sum_j beta^j arg_j,  per chunk (N_c, D_c) = (sum_i m_i prod_{j!=i} d_j, prod_i d_i),
//             ONE Ext4 inversion per group (Montgomery's trick across its chunks), perm_c = N_c / D_c -> 4 base columns; row sum out
//   pbl_fold  LDE domain (2N rows):   same (N_c, D_c) from the LDE row, L_c = perm_c * D_c - N_c, acc += alpha^e_c * L_c, S += perm_c
// The running sum phi (a prefix scan over rows), the three phi constraints and the division by Z_H are generic kernels below.
#pragma once
#include <string>
#include <vector>

#include "air.cuh"
#include "air_jit.cuh"
#include "bb31.cuh"
#include "deep.cuh"

namespace logup {

struct Interaction { uint32_t bus_id, num_args, span0; };     // spans[span0] = mult, spans[span0 + 1 + j] = arg j
struct LitArg { uint32_t interaction, j, value_m; };          // literal argument folded into the interaction's Ext4 constant

struct Program {
    std::vector<Interaction> ints;
    std::vector<uint32_t> chunk_start;          // n_chunks + 1
    std::vector<LitArg> lits;
    size_t max_args = 0;
    size_t n_chunks() const { return chunk_start.empty() ? 0 : chunk_start.size() - 1; }
    size_t perm_width() const { return ints.empty() ? 0 : 4 * (n_chunks() + 1); }
};

struct Kernels {
    std::vector<CUmodule> mods;
    std::vector<CUfunction> perm_fns, fold_fns;
};

// degree of a packed expression (air.cuh encoding)
inline unsigned expr_degree(const std::vector<uint32_t>& code, air::Span sp) {
    unsigned st[air::STACK_CAPACITY];
    int n = 0;
    for (uint32_t ip = sp.off; ip < sp.off + sp.len; ip++) {
        const uint32_t op = code[ip] >> 28;
        if (op == air::OP_PUSH_APC) st[n++] = 1;
        else if (op == air::OP_PUSH_CONST) st[n++] = 0;
        else if (op == air::OP_ADD || op == air::OP_SUB) { n--; st[n - 1] = std::max(st[n - 1], st[n]); }
        else if (op == air::OP_MUL) { n--; st[n - 1] += st[n]; }
        else if (op == air::OP_INV_OR_ZERO) st[n - 1] = 99;
    }
    return st[0];
}

// greedy chunking, same rule as the CPU restatement (DESIGN.md §3).  false when one interaction alone exceeds the bound.
inline bool make_chunks(const std::vector<uint32_t>& code, const std::vector<air::Span>& spans, Program& p, unsigned max_degree = 3) {
    p.chunk_start.clear();
    size_t i = 0;
    const size_t n = p.ints.size();
    while (i < n) {
        p.chunk_start.push_back((uint32_t)i);
        unsigned sum_dd = 0, max_extra = 0;
        size_t cnt = 0;
        for (; i < n; i++, cnt++) {
            const Interaction& it = p.ints[i];
            unsigned md = expr_degree(code, spans[it.span0]), dd = 0;
            for (uint32_t j = 0; j < it.num_args; j++) dd = std::max(dd, expr_degree(code, spans[it.span0 + 1 + j]));
            const unsigned extra = md > dd ? md - dd : 0, nsum = sum_dd + dd, nextra = std::max(extra, max_extra);
            if (std::max(1u, nextra) + nsum > max_degree) {
                if (cnt == 0) return false;
                break;
            }
            sum_dd = nsum;
            max_extra = nextra;
        }
    }
    p.chunk_start.push_back((uint32_t)n);
    return true;
}

static const char* LU_PRELUDE = R"(
struct E4 { u32 a, b, c, d; };
__device__ __forceinline__ E4 ld4(const uint4* p) { uint4 v = __ldg(p); E4 r; r.a = v.x; r.b = v.y; r.c = v.z; r.d = v.w; return r; }
// t < 2.4 p^2 (two products of values < p, plus a word): Montgomery reduction to [0, p)
__device__ __forceinline__ u32 mred(u64 t) { u32 m = (u32)t * 0x77ffffffu; u64 d = (u64)m * P + t; return red((u32)(d >> 32)); }
__device__ __forceinline__ u32 x11(u32 x) { u32 x2 = add(x, x), x4 = add(x2, x2), x8 = add(x4, x4); return add(add(x8, x2), x); }
__device__ __forceinline__ E4 e_add(E4 x, E4 y) { E4 r; r.a = add(x.a, y.a); r.b = add(x.b, y.b); r.c = add(x.c, y.c); r.d = add(x.d, y.d); return r; }
__device__ __forceinline__ E4 e_sub(E4 x, E4 y) { E4 r; r.a = sub(x.a, y.a); r.b = sub(x.b, y.b); r.c = sub(x.c, y.c); r.d = sub(x.d, y.d); return r; }
__device__ __forceinline__ E4 e_scale(E4 x, u32 s) { E4 r; r.a = mul(x.a, s); r.b = mul(x.b, s); r.c = mul(x.c, s); r.d = mul(x.d, s); return r; }
// Ext4 product, x^4 = 11: 16 wide products accumulated in pairs (8 reductions instead of 19 Montgomery products)
__device__ __forceinline__ E4 e_mul(E4 x, E4 y) {
    const u32 yb = x11(y.b), yc = x11(y.c), yd = x11(y.d);
    E4 r;
    r.a = add(mred((u64)x.a * y.a + (u64)x.b * yd), mred((u64)x.c * yc + (u64)x.d * yb));
    r.b = add(mred((u64)x.a * y.b + (u64)x.b * y.a), mred((u64)x.c * yd + (u64)x.d * yc));
    r.c = add(mred((u64)x.a * y.c + (u64)x.b * y.b), mred((u64)x.c * y.a + (u64)x.d * yd));
    r.d = add(mred((u64)x.a * y.d + (u64)x.b * y.c), mred((u64)x.c * y.b + (u64)x.d * y.a));
    return r;
}
// d + bt * s  (bt Ext4 constant, s base)
__device__ __forceinline__ E4 e_mac(E4 d, E4 bt, u32 s) { d.a = add(d.a, mul(bt.a, s)); d.b = add(d.b, mul(bt.b, s)); d.c = add(d.c, mul(bt.c, s)); d.d = add(d.d, mul(bt.d, s)); return d; }
// d + bt0 * s0 + bt1 * s1: one reduction per limb for the two products
__device__ __forceinline__ E4 e_mac2(E4 d, E4 b0, u32 s0, E4 b1, u32 s1) {
    d.a = add(d.a, mred((u64)b0.a * s0 + (u64)b1.a * s1)); d.b = add(d.b, mred((u64)b0.b * s0 + (u64)b1.b * s1));
    d.c = add(d.c, mred((u64)b0.c * s0 + (u64)b1.c * s1)); d.d = add(d.d, mred((u64)b0.d * s0 + (u64)b1.d * s1)); return d; }
// x * m0 + y * m1  (numerator of a two-interaction chunk)
__device__ __forceinline__ E4 e_lin2(E4 x, u32 m0, E4 y, u32 m1) {
    E4 r; r.a = mred((u64)x.a * m0 + (u64)y.a * m1); r.b = mred((u64)x.b * m0 + (u64)y.b * m1);
    r.c = mred((u64)x.c * m0 + (u64)y.c * m1); r.d = mred((u64)x.d * m0 + (u64)y.d * m1); return r; }
__device__ __noinline__ E4 e_inv(E4 x) {
    // norm to F_p[y]/(y^2 - 11) (y = x^2), then to F_p
    const u32 W = 939524073u;      // 11 * R mod p (bb::W11_M)
    u32 A0 = add(mul(x.a, x.a), mul(W, mul(x.c, x.c))), A1 = add(mul(x.a, x.c), mul(x.a, x.c));
    u32 B0 = add(mul(x.b, x.b), mul(W, mul(x.d, x.d))), B1 = add(mul(x.b, x.d), mul(x.b, x.d));
    u32 n0 = sub(A0, mul(W, B1)), n1 = sub(A1, B0);
    u32 dd = inv(sub(mul(n0, n0), mul(W, mul(n1, n1))));
    E4 s; s.a = mul(n0, dd); s.b = 0u; s.c = neg(mul(n1, dd)); s.d = 0u;
    E4 cj; cj.a = x.a; cj.b = neg(x.b); cj.c = x.c; cj.d = neg(x.d);
    return e_mul(cj, s);
}
__device__ __forceinline__ E4 ldp(const u32* __restrict__ p, u64 c, u64 h) { E4 r; r.a = __ldg(p + (4 * c) * h); r.b = __ldg(p + (4 * c + 1) * h); r.c = __ldg(p + (4 * c + 2) * h); r.d = __ldg(p + (4 * c + 3) * h); return r; }
)";

// emits SSA code for one packed expression; returns the name (or literal) of its value
struct Val { bool lit; uint32_t mont; std::string name; };
inline Val emit_expr(std::string& src, const std::vector<uint32_t>& code, air::Span sp, const std::vector<uint32_t>& pool, size_t& vid,
                     std::unordered_map<uint32_t, std::string>& cols, std::string& loads) {
    char buf[256];
    std::vector<Val> st;
    auto lit_str = [&](const Val& v) { snprintf(buf, sizeof buf, "0x%08xu", v.mont); return std::string(buf); };
    auto as_str = [&](const Val& v) { return v.lit ? lit_str(v) : v.name; };
    auto fresh = [&]() { snprintf(buf, sizeof buf, "v%zu", vid++); return std::string(buf); };
    for (uint32_t ip = sp.off; ip < sp.off + sp.len; ip++) {
        const uint32_t w = code[ip], op = w >> 28, arg = w & 0x0fffffffu;
        if (op == air::OP_PUSH_APC) {
            auto h = cols.find(arg);
            if (h == cols.end()) {
                snprintf(buf, sizeof buf, "c%zu", cols.size());
                const std::string nm = buf;
                snprintf(buf, sizeof buf, " u32 %s; asm volatile(\"ld.global.nc.u32 %%0, [%%1];\" : \"=r\"(%s) : \"l\"(b + %uull * h));\n", nm.c_str(), nm.c_str(), arg);
                loads += buf;
                h = cols.emplace(arg, nm).first;
            }
            st.push_back(Val{false, 0, h->second});
        } else if (op == air::OP_PUSH_CONST) {
            st.push_back(Val{true, pool[arg], ""});
        } else if (op == air::OP_ADD || op == air::OP_SUB || op == air::OP_MUL) {
            Val y = st.back(); st.pop_back();
            Val x = st.back(); st.pop_back();
            if (x.lit && y.lit) {
                st.push_back(Val{true, op == air::OP_ADD ? bb::add(x.mont, y.mont) : op == air::OP_SUB ? bb::sub(x.mont, y.mont) : bb::mul(x.mont, y.mont), ""});
            } else {
                Val v{false, 0, fresh()};
                if (op == air::OP_MUL && (x.lit || y.lit)) {
                    const Val& c = x.lit ? x : y;
                    const Val& z = x.lit ? y : x;
                    const uint32_t wc = bb::from_monty(c.mont);
                    snprintf(buf, sizeof buf, " u32 %s = mulc(%s, 0x%08xu, 0x%08xu);\n", v.name.c_str(), z.name.c_str(), wc, (uint32_t)(((uint64_t)wc << 32) / bb::P));
                } else {
                    snprintf(buf, sizeof buf, " u32 %s = %s(%s, %s);\n", v.name.c_str(), op == air::OP_ADD ? "add" : op == air::OP_SUB ? "sub" : "mul",
                             as_str(x).c_str(), as_str(y).c_str());
                }
                src += buf;
                st.push_back(v);
            }
        } else {
            Val x = st.back(); st.pop_back();
            if (x.lit) st.push_back(Val{true, op == air::OP_NEG ? bb::neg(x.mont) : bb::inv(x.mont), ""});
            else {
                Val v{false, 0, fresh()};
                snprintf(buf, sizeof buf, " u32 %s = %s(%s);\n", v.name.c_str(), op == air::OP_NEG ? "neg" : "inv", x.name.c_str());
                src += buf;
                st.push_back(v);
            }
        }
    }
    return st.back();
}

// chunks per generated function: permutation kernel 2 (one inversion per 2 chunks), fold kernel 1 -- fewer live Ext4 values beat
// the amortised inversion
constexpr size_t PERM_GROUP_CHUNKS = 2, FOLD_GROUP_CHUNKS = 1;
constexpr unsigned BLOCK_THREADS = 128;     // threads per CTA of both generated kernels

// source of one module covering chunks [c_begin, c_end): both kernels.  lits_out: literal arguments found (recorded once per interaction).
inline std::string generate(const std::vector<uint32_t>& code, const std::vector<air::Span>& spans, const std::vector<uint32_t>& pool, const Program& p,
                            size_t c_begin, size_t c_end, std::vector<LitArg>* lits_out) {
    std::string src = airjit::PRELUDE;
    src += LU_PRELUDE;
    char buf[512];
    std::string perm_calls, fold_calls;
    // one __noinline__ function per group of chunks; the two kernels use their own group size (the permutation kernel amortises one
    // Ext4 inversion over the group, the fold kernel has nothing to share between chunks and runs best with the fewest live values)
    for (int kind = 0; kind < 2; kind++) {
        const bool for_perm = kind == 0;
        const size_t GROUP = for_perm ? PERM_GROUP_CHUNKS : FOLD_GROUP_CHUNKS;
        size_t n_groups = 0;
        for (size_t cb = c_begin; cb < c_end; cb += GROUP, n_groups++) {
            const size_t ce = std::min(c_end, cb + GROUP);
            // ---- (m_i, d_i) of the group's interactions ----
            std::string body, loads;
            std::unordered_map<uint32_t, std::string> cols;
            size_t vid = 0;
            std::vector<std::string> m_name(p.chunk_start[ce] - p.chunk_start[cb]);
            const uint32_t i0 = p.chunk_start[cb];
            for (uint32_t i = i0; i < p.chunk_start[ce]; i++) {
                const Interaction& it = p.ints[i];
                Val mv = emit_expr(body, code, spans[it.span0], pool, vid, cols, loads);
                snprintf(buf, sizeof buf, "0x%08xu", mv.mont);
                m_name[i - i0] = mv.lit ? std::string(buf) : mv.name;
                snprintf(buf, sizeof buf, " E4 d%u = ld4(kc + %u);\n", i, i);
                body += buf;
                std::vector<std::pair<uint32_t, std::string>> dyn;       // (j, value name)
                for (uint32_t j = 0; j < it.num_args; j++) {
                    Val av = emit_expr(body, code, spans[it.span0 + 1 + j], pool, vid, cols, loads);
                    if (av.lit) { if (lits_out && for_perm) lits_out->push_back(LitArg{i, j, av.mont}); }
                    else dyn.emplace_back(j, av.name);
                }
                size_t q = 0;
                for (; q + 2 <= dyn.size(); q += 2) {
                    snprintf(buf, sizeof buf, " d%u = e_mac2(d%u, ld4(bt + %u), %s, ld4(bt + %u), %s);\n", i, i, dyn[q].first, dyn[q].second.c_str(),
                             dyn[q + 1].first, dyn[q + 1].second.c_str());
                    body += buf;
                }
                if (q < dyn.size()) {
                    snprintf(buf, sizeof buf, " d%u = e_mac(d%u, ld4(bt + %u), %s);\n", i, i, dyn[q].first, dyn[q].second.c_str());
                    body += buf;
                }
            }
            // per chunk: D<c>, N<c> (N is Ext4; for a one-interaction chunk the numerator is the base value m)
            std::string chunks;
            std::vector<bool> single(ce - cb);
            for (size_t c = cb; c < ce; c++) {
                const uint32_t a = p.chunk_start[c], e = p.chunk_start[c + 1];
                single[c - cb] = e - a == 1;
                if (e - a == 1) {
                    snprintf(buf, sizeof buf, " const E4 D%zu = d%u;\n", c, a);
                    chunks += buf;
                } else {
                    snprintf(buf, sizeof buf, " E4 D%zu = e_mul(d%u, d%u); E4 N%zu = e_lin2(d%u, %s, d%u, %s);\n", c, a, a + 1, c, a + 1, m_name[a - i0].c_str(), a,
                             m_name[a + 1 - i0].c_str());
                    chunks += buf;
                    for (uint32_t i = a + 2; i < e; i++) {
                        snprintf(buf, sizeof buf, " N%zu = e_add(e_mul(N%zu, d%u), e_scale(D%zu, %s)); D%zu = e_mul(D%zu, d%u);\n", c, c, i, c, m_name[i - i0].c_str(), c, c, i);
                        chunks += buf;
                    }
                }
            }
            if (for_perm) {
                // ---- perm kernel group: batch inversion of D over the group's chunks ----
                snprintf(buf, sizeof buf, "__device__ __noinline__ E4 pg%zu(const u32* __restrict__ b, u64 h, const uint4* __restrict__ kc, const uint4* __restrict__ bt, u32* __restrict__ perm) {\n", n_groups);
                src += buf;
                src += loads + body + chunks;
                const size_t G = ce - cb;
                for (size_t k = 1; k < G; k++) {
                    if (k == 1) snprintf(buf, sizeof buf, " E4 p1 = e_mul(D%zu, D%zu);\n", cb, cb + 1);
                    else snprintf(buf, sizeof buf, " E4 p%zu = e_mul(p%zu, D%zu);\n", k, k - 1, cb + k);
                    src += buf;
                }
                if (G == 1) snprintf(buf, sizeof buf, " E4 iv = e_inv(D%zu);\n", cb);
                else snprintf(buf, sizeof buf, " E4 iv = e_inv(p%zu);\n", G - 1);
                src += buf;
                src += " E4 sum; sum.a = 0u; sum.b = 0u; sum.c = 0u; sum.d = 0u; E4 t;\n";
                for (size_t k = G; k-- > 0;) {
                    const size_t c = cb + k;
                    // inverse of D_c = iv * prefix_{k-1};  then iv *= D_c
                    std::string invname;
                    if (k == 0) invname = "iv";
                    else {
                        if (k == 1) snprintf(buf, sizeof buf, " t = e_mul(iv, D%zu); iv = e_mul(iv, D%zu);\n", cb, c);
                        else snprintf(buf, sizeof buf, " t = e_mul(iv, p%zu); iv = e_mul(iv, D%zu);\n", k - 1, c);
                        src += buf;
                        invname = "t";
                    }
                    if (single[k]) snprintf(buf, sizeof buf, " t = e_scale(%s, %s);\n", invname.c_str(), m_name[p.chunk_start[c] - i0].c_str());
                    else snprintf(buf, sizeof buf, " t = e_mul(N%zu, %s);\n", c, invname.c_str());
                    src += buf;
                    snprintf(buf, sizeof buf, " perm[%zuull * h] = t.a; perm[%zuull * h] = t.b; perm[%zuull * h] = t.c; perm[%zuull * h] = t.d; sum = e_add(sum, t);\n",
                             4 * c, 4 * c + 1, 4 * c + 2, 4 * c + 3);
                    src += buf;
                }
                src += " return sum;\n}\n";
                snprintf(buf, sizeof buf, "    rs = e_add(rs, pg%zu(b, n, kc, bt, pr));\n", n_groups);
                perm_calls += buf;
            } else {
                // ---- fold kernel group ----
                snprintf(buf, sizeof buf, "__device__ __noinline__ void fg%zu(const u32* __restrict__ b, u64 h, const u32* __restrict__ pl, const uint4* __restrict__ kc, const uint4* __restrict__ bt, const uint4* __restrict__ apl, E4& acc, E4& S) {\n", n_groups);
                src += buf;
                src += loads + body + chunks;
                for (size_t c = cb; c < ce; c++) {
                    if (single[c - cb])
                        snprintf(buf, sizeof buf, " { E4 pc = ldp(pl, %zuull, h); S = e_add(S, pc); E4 L = e_mul(pc, D%zu); L.a = sub(L.a, %s); acc = e_add(acc, e_mul(ld4(apl + %zu), L)); }\n",
                                 c, c, m_name[p.chunk_start[c] - i0].c_str(), c);
                    else
                        snprintf(buf, sizeof buf, " { E4 pc = ldp(pl, %zuull, h); S = e_add(S, pc); E4 L = e_sub(e_mul(pc, D%zu), N%zu); acc = e_add(acc, e_mul(ld4(apl + %zu), L)); }\n", c, c, c, c);
                    src += buf;
                }
                src += "}\n";
                snprintf(buf, sizeof buf, "    fg%zu(b, m, pl, kc, bt, apl, acc, S);\n", n_groups);
                fold_calls += buf;
            }
        }
    }
    char lb[64];
    snprintf(lb, sizeof lb, "__launch_bounds__(%u)", BLOCK_THREADS);
    src += std::string("\nextern \"C\" __global__ void ") + lb + R"( pbl_perm(const u32* __restrict__ mat, u64 n, const uint4* __restrict__ kc, const uint4* __restrict__ bt,
                                                            u32* __restrict__ perm, u32* __restrict__ rowsum, int first) {
    const u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const u32* b = mat + r;
    u32* pr = perm + r;
    E4 rs; rs.a = 0u; rs.b = 0u; rs.c = 0u; rs.d = 0u;
    if (!first) { rs.a = rowsum[r]; rs.b = rowsum[n + r]; rs.c = rowsum[2 * n + r]; rs.d = rowsum[3 * n + r]; }
)";
    src += perm_calls;
    src += R"(    rowsum[r] = rs.a; rowsum[n + r] = rs.b; rowsum[2 * n + r] = rs.c; rowsum[3 * n + r] = rs.d;
}
)";
    src += std::string("extern \"C\" __global__ void ") + lb + R"( pbl_fold(const u32* __restrict__ lde, const u32* __restrict__ plde, u64 m, const uint4* __restrict__ kc,
                                                            const uint4* __restrict__ bt, const uint4* __restrict__ apl, u32* __restrict__ raw,
                                                            u32* __restrict__ Ssum, int first) {
    const u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= m) return;
    const u32* b = lde + r;
    const u32* pl = plde + r;
    E4 acc; acc.a = raw[r]; acc.b = raw[m + r]; acc.c = raw[2 * m + r]; acc.d = raw[3 * m + r];
    E4 S; S.a = 0u; S.b = 0u; S.c = 0u; S.d = 0u;
    if (!first) { S.a = Ssum[r]; S.b = Ssum[m + r]; S.c = Ssum[2 * m + r]; S.d = Ssum[3 * m + r]; }
)";
    src += fold_calls;
    src += R"(    raw[r] = acc.a; raw[m + r] = acc.b; raw[2 * m + r] = acc.c; raw[3 * m + r] = acc.d;
    Ssum[r] = S.a; Ssum[m + r] = S.b; Ssum[2 * m + r] = S.c; Ssum[3 * m + r] = S.d;
}
)";
    return src;
}

// compile every module (in parallel on the host threads) and load them; 0 on success
inline int build(const std::vector<uint32_t>& code, const std::vector<air::Span>& spans, const std::vector<uint32_t>& pool, Program& p, Kernels* out,
                 size_t* cubin_bytes = nullptr) {
    airjit::Api& a = airjit::api();
    if (!a.nvrtc_ok || (out && !a.ok)) return 3;
    // chunks per module = per kernel launch: the generated code is straight-line, every warp streams through all of it once, so a
    // module must fit the instruction cache (ncu: `no_instruction` was the top stall with 64-chunk modules = 460 KB of SASS)
    const size_t mod_chunks = 16;
    const size_t nc = p.n_chunks(), n_mods = (nc + mod_chunks - 1) / mod_chunks;
    std::vector<std::vector<char>> cubins(n_mods);
    std::vector<std::vector<LitArg>> lits(n_mods);
    std::vector<int> rcs(n_mods, 0);
    std::atomic<size_t> next{0};
    auto worker = [&]() {
        for (size_t k = next.fetch_add(1); k < n_mods; k = next.fetch_add(1)) {
            const std::string src = generate(code, spans, pool, p, k * mod_chunks, std::min(nc, (k + 1) * mod_chunks), &lits[k]);
            rcs[k] = airjit::compile_chunk(src, cubins[k]);
            if (const char* dump = getenv("PB_LOGUP_JIT_DUMP")) {
                const std::string base = std::string(dump) + "." + std::to_string(k);
                if (FILE* f = fopen((base + ".cu").c_str(), "w")) { fwrite(src.data(), 1, src.size(), f); fclose(f); }
                if (FILE* f = fopen((base + ".cubin").c_str(), "wb")) { fwrite(cubins[k].data(), 1, cubins[k].size(), f); fclose(f); }
            }
        }
    };
    const size_t n_threads = std::min<size_t>(n_mods, std::max(1u, std::thread::hardware_concurrency()));
    std::vector<std::thread> ths;
    for (size_t t = 1; t < n_threads; t++) ths.emplace_back(worker);
    worker();
    for (auto& t : ths) t.join();
    size_t total = 0;
    p.lits.clear();
    for (size_t k = 0; k < n_mods; k++) {
        if (rcs[k]) return rcs[k];
        total += cubins[k].size();
        p.lits.insert(p.lits.end(), lits[k].begin(), lits[k].end());
    }
    if (cubin_bytes) *cubin_bytes = total;
    if (!out) return 0;
    for (size_t k = 0; k < n_mods; k++) {
        CUmodule mod = nullptr;
        CUfunction f1 = nullptr, f2 = nullptr;
        if (a.ModuleLoadData(&mod, cubins[k].data()) != CUDA_SUCCESS || a.ModuleGetFunction(&f1, mod, "pbl_perm") != CUDA_SUCCESS ||
            a.ModuleGetFunction(&f2, mod, "pbl_fold") != CUDA_SUCCESS) {
            if (mod) a.ModuleUnload(mod);
            for (CUmodule m2 : out->mods) a.ModuleUnload(m2);
            out->mods.clear(); out->perm_fns.clear(); out->fold_fns.clear();
            return 6;
        }
        out->mods.push_back(mod);
        out->perm_fns.push_back(f1);
        out->fold_fns.push_back(f2);
    }
    return 0;
}

inline void destroy(Kernels& k) {
    for (CUmodule m : k.mods) airjit::api().ModuleUnload(m);
    k.mods.clear(); k.perm_fns.clear(); k.fold_fns.clear();
}

inline int launch_perm(const Kernels& k, cudaStream_t st, const uint32_t* mat, unsigned long long n, const uint4* kc, const uint4* bt, uint32_t* perm,
                       uint32_t* rowsum) {
    for (size_t c = 0; c < k.perm_fns.size(); c++) {
        int first = c == 0;
        void* args[] = {(void*)&mat, (void*)&n, (void*)&kc, (void*)&bt, (void*)&perm, (void*)&rowsum, (void*)&first};
        CUresult rc = airjit::api().LaunchKernel(k.perm_fns[c], (unsigned)((n + BLOCK_THREADS - 1) / BLOCK_THREADS), 1, 1, BLOCK_THREADS, 1, 1, 0,
                                                 (CUstream)st, args, nullptr);
        if (rc != CUDA_SUCCESS) return 700 + (int)rc;
    }
    return 0;
}
inline int launch_fold(const Kernels& k, cudaStream_t st, const uint32_t* lde, const uint32_t* plde, unsigned long long m, const uint4* kc, const uint4* bt,
                       const uint4* apl, uint32_t* raw, uint32_t* ssum) {
    for (size_t c = 0; c < k.fold_fns.size(); c++) {
        int first = c == 0;
        void* args[] = {(void*)&lde, (void*)&plde, (void*)&m, (void*)&kc, (void*)&bt, (void*)&apl, (void*)&raw, (void*)&ssum, (void*)&first};
        CUresult rc = airjit::api().LaunchKernel(k.fold_fns[c], (unsigned)((m + BLOCK_THREADS - 1) / BLOCK_THREADS), 1, 1, BLOCK_THREADS, 1, 1, 0,
                                                 (CUstream)st, args, nullptr);
        if (rc != CUDA_SUCCESS) return 700 + (int)rc;
    }
    return 0;
}

// ---------------- generic kernels ----------------
// inclusive prefix sums over rows of 4 independent base-field sequences (the limbs of the Ext4 row sums): [4][n] -> phi columns.
// Three phases: per-CTA scan + CTA totals; one CTA scans the totals; add the offsets.
constexpr int SCAN_THREADS = 256, SCAN_ITEMS = 8;       // 2048 rows per CTA
__global__ void __launch_bounds__(SCAN_THREADS) scan_local_kernel(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, size_t n, uint32_t* __restrict__ totals) {
    __shared__ uint32_t sh[SCAN_THREADS];
    const int limb = blockIdx.y;
    const uint32_t* src = in + (size_t)limb * n;
    uint32_t* dst = out + (size_t)limb * n;
    const size_t base = ((size_t)blockIdx.x * SCAN_THREADS + threadIdx.x) * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS], run = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) { const size_t i = base + k; run = bb::add(run, i < n ? src[i] : 0u); v[k] = run; }
    sh[threadIdx.x] = run;
    __syncthreads();
    for (int off = 1; off < SCAN_THREADS; off <<= 1) {
        uint32_t t = threadIdx.x >= off ? sh[threadIdx.x - off] : 0u;
        __syncthreads();
        sh[threadIdx.x] = bb::add(sh[threadIdx.x], t);
        __syncthreads();
    }
    const uint32_t prev = threadIdx.x ? sh[threadIdx.x - 1] : 0u;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) { const size_t i = base + k; if (i < n) dst[i] = bb::add(v[k], prev); }
    if (threadIdx.x == SCAN_THREADS - 1) totals[(size_t)limb * gridDim.x + blockIdx.x] = sh[threadIdx.x];
}
__global__ void scan_totals_kernel(uint32_t* totals, uint32_t n_blocks) {       // 4 threads: exclusive scan of each limb's CTA totals
    if (threadIdx.x >= 4) return;
    uint32_t* t = totals + (size_t)threadIdx.x * n_blocks;
    uint32_t run = 0;
    for (uint32_t i = 0; i < n_blocks; i++) { const uint32_t x = t[i]; t[i] = run; run = bb::add(run, x); }
}
__global__ void __launch_bounds__(256) scan_add_kernel(uint32_t* __restrict__ out, size_t n, const uint32_t* __restrict__ totals, uint32_t n_blocks) {
    const int limb = blockIdx.y;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t off = totals[(size_t)limb * n_blocks + i / (SCAN_THREADS * SCAN_ITEMS)];
    out[(size_t)limb * n + i] = bb::add(out[(size_t)limb * n + i], off);
}

// the three phi constraints, then the division by Z_H and the chunk split (the tail of the quotient when the AIR has interactions).
//   acc = raw + alpha^2 * is_first * (phi - S) + alpha * is_trans * (phi' - phi - S') + is_last * (phi - cumsum)
// rows are LDE rows in bit-reversed order; ' = the LDE point 2 steps on in natural order (the next trace row).
// The kernel does rows [row0, row0 + 2^log_ms) of the 2N: raw is [4][2^log_ms] over them.  ssum and phi are given as row blocks of
// 2^log_ms rows, block b's [4][2^log_ms] at b * blk_stride, because the next row may lie in another block (the whole matrix: one block,
// log_ms = log_n + 1).  out: the quotient of these rows split at the coset boundary, [rows / N][4][min(rows, N)].
__global__ void __launch_bounds__(256) finish_kernel(const uint32_t* __restrict__ raw, const uint32_t* __restrict__ ssum, const uint32_t* __restrict__ phi,
                                                     size_t blk_stride, int log_ms, size_t row0, int log_n, uint32_t shift_m, uint32_t omega_m_m,
                                                     uint32_t w_n_inv_m, uint32_t sn_m, bb::E4 alpha, bb::E4 alpha2, bb::E4 cumsum, uint32_t zinv0,
                                                     uint32_t zinv1, uint32_t* __restrict__ out) {
    const size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x, m = (size_t)1 << log_ms;
    if (r >= m) return;
    const int log_m = log_n + 1;
    const size_t R = row0 + r;
    const uint32_t i_nat = __brev((uint32_t)R) >> (32 - log_m);
    const size_t Rn = __brev((i_nat + 2) & (uint32_t)(((size_t)1 << log_m) - 1)) >> (32 - log_m);
    const size_t here = (R >> log_ms) * blk_stride + r, next = (Rn >> log_ms) * blk_stride + (Rn & (m - 1));
    const uint32_t x = bb::mul(shift_m, bb::pow(omega_m_m, (uint64_t)i_nat));
    const uint32_t zh = bb::sub((i_nat & 1) ? bb::neg(sn_m) : sn_m, bb::R1);
    const uint32_t is_first = bb::mul(zh, bb::inv(bb::sub(x, bb::R1)));
    const uint32_t is_last = bb::mul(zh, bb::inv(bb::sub(x, w_n_inv_m)));
    const uint32_t is_trans = bb::sub(x, w_n_inv_m);
    bb::E4 acc, S, Sn, ph, phn;
#pragma unroll
    for (int l = 0; l < 4; l++) {
        acc.c[l] = raw[(size_t)l * m + r];
        S.c[l] = ssum[(size_t)l * m + here];
        Sn.c[l] = ssum[(size_t)l * m + next];
        ph.c[l] = phi[(size_t)l * m + here];
        phn.c[l] = phi[(size_t)l * m + next];
    }
    acc = bb::e4_add(acc, bb::e4_mul(alpha2, bb::e4_scale(bb::e4_sub(ph, S), is_first)));
    acc = bb::e4_add(acc, bb::e4_mul(alpha, bb::e4_scale(bb::e4_sub(bb::e4_sub(phn, ph), Sn), is_trans)));
    acc = bb::e4_add(acc, bb::e4_scale(bb::e4_sub(ph, cumsum), is_last));
    const int log_ld = min(log_ms, log_n);
    const size_t ld = (size_t)1 << log_ld, chunk = r >> log_ld, j = r & (ld - 1);
    const uint32_t z = (R >> log_n) ? zinv1 : zinv0;
#pragma unroll
    for (int l = 0; l < 4; l++) out[(chunk * 4 + l) * ld + j] = bb::mul(acc.c[l], z);
}

}  // namespace logup
