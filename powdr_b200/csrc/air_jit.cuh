// Per-AIR code generation for stage 2.  The bytecode interpreter (air.cuh) spends ~28 instructions per expression node
// (ncu r01: 143 k instructions per LDE row for the keccak-shaped AIR, 20 % of the HBM roof).  An autoprecompile's constraint
// set is fixed at key-generation time, so pb_air_compile turns the packed program into straight-line CUDA C -- one SSA value
// per node, constants folded into Shoup products, constraints grouped into small __noinline__ functions to keep ptxas
// basic blocks short -- and compiles it with NVRTC for sm_90a.  NVRTC and the driver API are dlopen'ed lazily so the
// library itself links against nothing but cudart; when either is missing, or PB_AIR_NO_JIT is set, the interpreter
// kernel (still CUDA) is used instead.
#pragma once
#include <algorithm>
#include <atomic>
#include <mutex>
#include <thread>
#include <unordered_map>
#include <cuda.h>
#include <dlfcn.h>
#include <nvrtc.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <sys/stat.h>
#include <unistd.h>
#include <string>
#include <vector>

#include "air.cuh"
#include "bb31.cuh"

namespace airjit {

struct Api {
    bool tried = false, ok = false /* nvrtc + driver */, nvrtc_ok = false;
    nvrtcResult (*CreateProgram)(nvrtcProgram*, const char*, const char*, int, const char* const*, const char* const*) = nullptr;
    nvrtcResult (*CompileProgram)(nvrtcProgram, int, const char* const*) = nullptr;
    nvrtcResult (*GetCUBINSize)(nvrtcProgram, size_t*) = nullptr;
    nvrtcResult (*GetCUBIN)(nvrtcProgram, char*) = nullptr;
    nvrtcResult (*GetProgramLogSize)(nvrtcProgram, size_t*) = nullptr;
    nvrtcResult (*GetProgramLog)(nvrtcProgram, char*) = nullptr;
    nvrtcResult (*DestroyProgram)(nvrtcProgram*) = nullptr;
    CUresult (*ModuleLoadData)(CUmodule*, const void*) = nullptr;
    CUresult (*ModuleGetFunction)(CUfunction*, CUmodule, const char*) = nullptr;
    CUresult (*ModuleUnload)(CUmodule) = nullptr;
    CUresult (*LaunchKernel)(CUfunction, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, CUstream, void**, void**) = nullptr;
};

inline void api_init(Api& a);
inline Api& api() {
    static Api a;
    static std::once_flag once;           // pb_air_compile may be called from several host threads
    std::call_once(once, [] { api_init(a); });
    return a;
}
inline void api_init(Api& a) {
    a.tried = true;
    void* hn = nullptr;
    for (const char* n : {"libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so"})
        if ((hn = dlopen(n, RTLD_NOW | RTLD_GLOBAL))) break;
    void* hc = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
    if (!hn) return;
#define PB_SYM(field, handle, name) *(void**)(&a.field) = dlsym(handle, name); if (!a.field) return;
    PB_SYM(CreateProgram, hn, "nvrtcCreateProgram") PB_SYM(CompileProgram, hn, "nvrtcCompileProgram")
    PB_SYM(GetCUBINSize, hn, "nvrtcGetCUBINSize") PB_SYM(GetCUBIN, hn, "nvrtcGetCUBIN")
    PB_SYM(GetProgramLogSize, hn, "nvrtcGetProgramLogSize") PB_SYM(GetProgramLog, hn, "nvrtcGetProgramLog")
    PB_SYM(DestroyProgram, hn, "nvrtcDestroyProgram")
    a.nvrtc_ok = true;
    if (!hc) return;
    PB_SYM(ModuleLoadData, hc, "cuModuleLoadData") PB_SYM(ModuleGetFunction, hc, "cuModuleGetFunction")
    PB_SYM(ModuleUnload, hc, "cuModuleUnload") PB_SYM(LaunchKernel, hc, "cuLaunchKernel")
#undef PB_SYM
    a.ok = true;
}

struct Kernel {
    // the AIR's constraints are split into chunks, one module each (compiled in parallel: ptxas time grows faster than linearly
    // with the size of a module); chunk c adds its constraints' contribution to the running fold
    std::vector<CUmodule> mods;
    std::vector<CUfunction> fns;
};

static const char* PRELUDE = R"(
typedef unsigned int u32; typedef unsigned long long u64;
#define P 0x78000001u
__device__ __forceinline__ u32 red(u32 x) { u32 y = x - P; return y < x ? y : x; }
__device__ __forceinline__ u32 add(u32 a, u32 b) { return red(a + b); }
__device__ __forceinline__ u32 sub(u32 a, u32 b) { u32 d = a - b, e = d + P; return e < d ? e : d; }
__device__ __forceinline__ u32 neg(u32 a) { return a ? P - a : 0u; }
__device__ __forceinline__ u32 mul(u32 a, u32 b) { u64 t = (u64)a * b; u32 m = (u32)t * 0x77ffffffu; u64 d = (u64)m * P + t; return red((u32)(d >> 32)); }
__device__ __forceinline__ u32 mulc(u32 a, u32 w, u32 wp) { u32 q = __umulhi(a, wp); return red(a * w - q * P); }
// x^(p-2), p - 2 = 0b111_0_1^27, by an addition chain: 30 squarings + 7 products (square-and-multiply: 31 + 30) -- the LogUp
// permutation kernel inverts once per two chunks, which was a fifth of its modular products
__device__ __forceinline__ u32 sqn(u32 a, int n) { for (int i = 0; i < n; i++) a = mul(a, a); return a; }
__device__ __noinline__ u32 inv(u32 x) {
    const u32 a = sqn(x, 8), b = mul(a, x), c = sqn(a, 8), d = mul(c, b), e = sqn(d, 3), f = sqn(e, 5), g = mul(f, x), h = mul(g, e);
    const u32 i = mul(g, g), j = mul(i, h), k = mul(i, i), l = mul(k, j);
    return mul(sqn(l, 4), l);
}
__device__ __forceinline__ uint4 fold(uint4 acc, u32 c, uint4 w) {
    acc.x = add(acc.x, mul(c, w.x)); acc.y = add(acc.y, mul(c, w.y)); acc.z = add(acc.z, mul(c, w.z)); acc.w = add(acc.w, mul(c, w.w)); return acc; }
)";

// packed program (air.cuh encoding) -> CUDA C.  Literals stay symbolic so constant operands become Shoup products.
inline std::string generate(const std::vector<uint32_t>& code, const std::vector<air::Span>& spans_all, const std::vector<uint32_t>& pool,
                            size_t k_begin, size_t k_end) {
    // constraints [k_begin, k_end) only; alpha-power indices stay global
    struct SpanView {
        const std::vector<air::Span>& v; size_t e;
        size_t size() const { return e; }
        const air::Span& operator[](size_t i) const { return v[i]; }
    } spans{spans_all, k_end};
    std::string src = PRELUDE;
    struct Val { bool lit; uint32_t mont; std::string name; };
    char buf[256];
    const size_t GROUP_OPS = 600, GROUP_COLS = 32;
    size_t k = k_begin, n_groups = 0, vid = 0, group_end = 0;
    while (k < spans.size()) {
        snprintf(buf, sizeof buf, "__device__ __noinline__ uint4 g%zu(const u32* __restrict__ b, u64 m, const uint4* __restrict__ ap, uint4 acc) {\n", n_groups);
        src += buf;
        // A group = consecutive constraints that together read at most GROUP_COLS distinct columns.  Their loads are hoisted to
        // the top of the function as volatile asm (kept in order, nothing to wait for), so one thread has that many loads in
        // flight before the first use: ncu r01c showed the load-at-use version 90 % stalled on long_scoreboard at 54 % of HBM.
        std::unordered_map<uint32_t, size_t> hoisted;
        {
            size_t ops_la = 0, k1 = k;
            while (k1 < spans.size()) {
                std::vector<uint32_t> fresh_cols;
                for (uint32_t ip = spans[k1].off; ip < spans[k1].off + spans[k1].len; ip++) {
                    const uint32_t w = code[ip];
                    if ((w >> 28) == air::OP_PUSH_APC && !hoisted.count(w & 0x0fffffffu) &&
                        std::find(fresh_cols.begin(), fresh_cols.end(), w & 0x0fffffffu) == fresh_cols.end())
                        fresh_cols.push_back(w & 0x0fffffffu);
                }
                if (k1 > k && (ops_la + spans[k1].len > GROUP_OPS || hoisted.size() + fresh_cols.size() > GROUP_COLS)) break;
                for (uint32_t c : fresh_cols)
                    if (hoisted.size() < GROUP_COLS) {
                        const size_t id = hoisted.size();
                        hoisted[c] = id;
                        snprintf(buf, sizeof buf, " u32 c%zu; asm volatile(\"ld.global.nc.u32 %%0, [%%1];\" : \"=r\"(c%zu) : \"l\"(b + %uull * m));\n", id, id, c);
                        src += buf;
                    }
                ops_la += spans[k1].len;
                k1++;
            }
            group_end = k1;
        }
        size_t ops = 0;
        while (k < group_end) {
            std::vector<Val> st;
            for (uint32_t ip = spans[k].off; ip < spans[k].off + spans[k].len; ip++) {
                const uint32_t w = code[ip], op = w >> 28, arg = w & 0x0fffffffu;
                auto lit_str = [&](const Val& v) { snprintf(buf, sizeof buf, "0x%08xu", v.mont); return std::string(buf); };
                auto as_str = [&](const Val& v) { return v.lit ? lit_str(v) : v.name; };
                auto fresh = [&]() { snprintf(buf, sizeof buf, "v%zu", vid++); return std::string(buf); };
                if (op == air::OP_PUSH_APC) {
                    auto h = hoisted.find(arg);
                    if (h != hoisted.end()) {
                        snprintf(buf, sizeof buf, "c%zu", h->second);
                        st.push_back(Val{false, 0, buf});
                    } else {
                        Val v{false, 0, fresh()};
                        snprintf(buf, sizeof buf, " u32 %s = __ldg(b + %uull * m);\n", v.name.c_str(), arg);
                        src += buf;
                        st.push_back(v);
                    }
                } else if (op == air::OP_PUSH_CONST) {
                    st.push_back(Val{true, pool[arg], ""});
                } else if (op == air::OP_ADD || op == air::OP_SUB || op == air::OP_MUL) {
                    Val bb_ = st.back(); st.pop_back();
                    Val aa = st.back(); st.pop_back();
                    if (aa.lit && bb_.lit) {
                        uint32_t r = op == air::OP_ADD ? bb::add(aa.mont, bb_.mont) : op == air::OP_SUB ? bb::sub(aa.mont, bb_.mont) : bb::mul(aa.mont, bb_.mont);
                        st.push_back(Val{true, r, ""});
                    } else {
                        Val v{false, 0, fresh()};
                        if (op == air::OP_MUL && (aa.lit || bb_.lit)) {
                            const Val& c = aa.lit ? aa : bb_;
                            const Val& x = aa.lit ? bb_ : aa;
                            const uint32_t wc = bb::from_monty(c.mont);
                            snprintf(buf, sizeof buf, " u32 %s = mulc(%s, 0x%08xu, 0x%08xu);\n", v.name.c_str(), x.name.c_str(), wc,
                                     (uint32_t)(((uint64_t)wc << 32) / bb::P));
                        } else {
                            snprintf(buf, sizeof buf, " u32 %s = %s(%s, %s);\n", v.name.c_str(), op == air::OP_ADD ? "add" : op == air::OP_SUB ? "sub" : "mul",
                                     as_str(aa).c_str(), as_str(bb_).c_str());
                        }
                        src += buf;
                        st.push_back(v);
                    }
                } else {
                    Val aa = st.back(); st.pop_back();
                    if (aa.lit) {
                        st.push_back(Val{true, op == air::OP_NEG ? bb::neg(aa.mont) : bb::inv(aa.mont), ""});
                    } else {
                        Val v{false, 0, fresh()};
                        snprintf(buf, sizeof buf, " u32 %s = %s(%s);\n", v.name.c_str(), op == air::OP_NEG ? "neg" : "inv", aa.name.c_str());
                        src += buf;
                        st.push_back(v);
                    }
                }
            }
            const Val& c = st.back();
            char lit[16];
            snprintf(lit, sizeof lit, "0x%08xu", c.mont);
            snprintf(buf, sizeof buf, " acc = fold(acc, %s, __ldg(ap + %zu));\n", c.lit ? lit : c.name.c_str(), k);
            src += buf;
            ops += spans[k].len;
            k++;
        }
        src += " return acc;\n}\n";
        n_groups++;
    }
    src += R"(
extern "C" __global__ void __launch_bounds__(256) pbq(const u32* __restrict__ mat, u64 m, int log_n, const uint4* __restrict__ ap,
                                                       u32 zinv0, u32 zinv1, u32* __restrict__ out, int apply_zinv,
                                                       const u32* __restrict__ raw_in, u32* __restrict__ raw_out) {
    const u64 r = (u64)blockIdx.x * 256ull + threadIdx.x;
    if (r >= m) return;
    const u32* b = mat + r;
    uint4 acc = make_uint4(0u, 0u, 0u, 0u);
    if (raw_in) acc = make_uint4(raw_in[r], raw_in[m + r], raw_in[2 * m + r], raw_in[3 * m + r]);      // fold of the earlier chunks
)";
    for (size_t g = 0; g < n_groups; g++) {
        snprintf(buf, sizeof buf, "    acc = g%zu(b, m, ap, acc);\n", g);
        src += buf;
    }
    src += R"(
    if (raw_out) { raw_out[r] = acc.x; raw_out[m + r] = acc.y; raw_out[2 * m + r] = acc.z; raw_out[3 * m + r] = acc.w; return; }
    if (apply_zinv) {
        const u64 n = 1ull << log_n, chunk = r >> log_n, j = r & (n - 1);
        const u32 z = chunk ? zinv1 : zinv0;
        out[(chunk * 4 + 0) * n + j] = mul(acc.x, z); out[(chunk * 4 + 1) * n + j] = mul(acc.y, z);
        out[(chunk * 4 + 2) * n + j] = mul(acc.z, z); out[(chunk * 4 + 3) * n + j] = mul(acc.w, z);
    } else {
        out[r] = acc.x; out[m + r] = acc.y; out[2 * m + r] = acc.z; out[3 * m + r] = acc.w;
    }
}
)";
    return src;
}

// on-disk cubin cache (PB_JIT_CACHE=<dir>, default /tmp/powdr_b200_jit; PB_JIT_CACHE=off disables): key generation is seconds of NVRTC
// per AIR, and the ranks of a multi-GPU job (or repeated runs) compile identical modules
inline std::string cache_path(const std::string& src) {
    const char* dir = getenv("PB_JIT_CACHE");
    if (dir && std::string(dir) == "off") return "";
    std::string d = dir ? dir : "/tmp/powdr_b200_jit";
    mkdir(d.c_str(), 0777);
    uint64_t h1 = 1469598103934665603ull, h2 = 0x9e3779b97f4a7c15ull;
    for (unsigned char c : src) { h1 = (h1 ^ c) * 1099511628211ull; h2 = (h2 + c) * 0xff51afd7ed558ccdull; h2 ^= h2 >> 29; }
    char name[96];
    snprintf(name, sizeof name, "/sm90a_%016llx%016llx_%zu.cubin", (unsigned long long)h1, (unsigned long long)h2, src.size());
    return d + name;
}

// one chunk: source -> cubin (thread-safe: distinct NVRTC programs)
inline int compile_chunk(const std::string& src, std::vector<char>& cubin) {
    const std::string cpath = cache_path(src);
    if (!cpath.empty())
        if (FILE* f = fopen(cpath.c_str(), "rb")) {
            fseek(f, 0, SEEK_END);
            const long n = ftell(f);
            fseek(f, 0, SEEK_SET);
            cubin.resize(n > 0 ? (size_t)n : 0);
            const bool ok = n > 0 && fread(cubin.data(), 1, (size_t)n, f) == (size_t)n;
            fclose(f);
            if (ok) return 0;
        }
    Api& a = api();
    nvrtcProgram prog;
    if (a.CreateProgram(&prog, src.c_str(), "pb_air.cu", 0, nullptr, nullptr) != NVRTC_SUCCESS) return 4;
    const char* opts[] = {"--gpu-architecture=sm_90a", "-std=c++17", "-lineinfo"};
    nvrtcResult rc = a.CompileProgram(prog, 3, opts);
    if (rc != NVRTC_SUCCESS) {
        if (getenv("PB_AIR_JIT_VERBOSE")) {
            size_t ls = 0;
            a.GetProgramLogSize(prog, &ls);
            std::vector<char> log(ls + 1, 0);
            a.GetProgramLog(prog, log.data());
            fprintf(stderr, "[powdr_b200] NVRTC failed (%d):\n%s\n", (int)rc, log.data());
        }
        a.DestroyProgram(&prog);
        return 5;
    }
    size_t sz = 0;
    a.GetCUBINSize(prog, &sz);
    cubin.resize(sz);
    a.GetCUBIN(prog, cubin.data());
    a.DestroyProgram(&prog);
    if (!cpath.empty()) {                      // write-then-rename: a concurrent reader never sees a partial file
        const std::string tmp = cpath + "." + std::to_string((long)getpid()) + "." + std::to_string((unsigned long)(uintptr_t)&cubin);
        if (FILE* f = fopen(tmp.c_str(), "wb")) {
            const bool ok = fwrite(cubin.data(), 1, cubin.size(), f) == cubin.size();
            fclose(f);
            if (ok) rename(tmp.c_str(), cpath.c_str()); else remove(tmp.c_str());
        }
    }
    return 0;
}

// returns 0 and fills `out` on success; non-zero when the JIT path is unavailable (caller keeps the interpreter).
// Measured (8 shared cores): one module for a 41 k-word AIR (3771 constraints) took 537 s in ptxas; 4 k-word chunks compiled
// on all host threads bring key generation back to seconds (the running fold crosses chunks through a [4][rows] buffer,
// +1 % traffic for the keccak shape).
inline int build(const std::vector<uint32_t>& code, const std::vector<air::Span>& spans, const std::vector<uint32_t>& pool, Kernel* out,
                 size_t* cubin_bytes = nullptr) {
    if (getenv("PB_AIR_NO_JIT")) return 1;
    if (code.size() > 1000000) return 2;                       // keep compile time bounded; huge AIRs stay on the interpreter
    Api& a = api();
    if (!a.nvrtc_ok || (out && !a.ok)) return 3;
    const size_t chunk_words = 2000;      // keccak shape (7.2 k words): 4 modules, 2.7 s instead of 7.8 s; sha256 shape: 13 s; 141 k-word pre-opt machine: 30 s
    std::vector<size_t> bounds{0};
    for (size_t k = 0, w = 0; k < spans.size(); k++) {
        if (w > 0 && w + spans[k].len > chunk_words) { bounds.push_back(k); w = 0; }
        w += spans[k].len;
    }
    bounds.push_back(spans.size());
    const size_t n_chunks = bounds.size() - 1;
    std::vector<std::vector<char>> cubins(n_chunks);
    std::vector<int> rcs(n_chunks, 0);
    std::atomic<size_t> next{0};
    auto worker = [&]() {
        for (size_t c = next.fetch_add(1); c < n_chunks; c = next.fetch_add(1)) {
            const std::string src = generate(code, spans, pool, bounds[c], bounds[c + 1]);
            rcs[c] = compile_chunk(src, cubins[c]);
            if (const char* dump = getenv("PB_AIR_JIT_DUMP")) {       // debugging aid: <path>.<chunk>.cu / .cubin (cuobjdump -sass / -res-usage)
                const std::string base = std::string(dump) + "." + std::to_string(c);
                if (FILE* f = fopen((base + ".cu").c_str(), "w")) { fwrite(src.data(), 1, src.size(), f); fclose(f); }
                if (FILE* f = fopen((base + ".cubin").c_str(), "wb")) { fwrite(cubins[c].data(), 1, cubins[c].size(), f); fclose(f); }
            }
        }
    };
    const size_t n_threads = std::min<size_t>(n_chunks, std::max(1u, std::thread::hardware_concurrency()));
    std::vector<std::thread> pool_threads;
    for (size_t t = 1; t < n_threads; t++) pool_threads.emplace_back(worker);
    worker();
    for (auto& t : pool_threads) t.join();
    size_t total = 0;
    for (size_t c = 0; c < n_chunks; c++) {
        if (rcs[c]) return rcs[c];
        total += cubins[c].size();
    }
    if (cubin_bytes) *cubin_bytes = total;
    if (!out) return 0;
    for (size_t c = 0; c < n_chunks; c++) {
        CUmodule mod = nullptr;
        CUfunction fn = nullptr;
        if (a.ModuleLoadData(&mod, cubins[c].data()) != CUDA_SUCCESS || a.ModuleGetFunction(&fn, mod, "pbq") != CUDA_SUCCESS) {
            if (mod) a.ModuleUnload(mod);
            for (CUmodule m2 : out->mods) a.ModuleUnload(m2);
            out->mods.clear();
            out->fns.clear();
            return 6;
        }
        out->mods.push_back(mod);
        out->fns.push_back(fn);
    }
    return 0;
}

// raw: [4][m] scratch for the running fold between chunks (needed only when the kernel has more than one chunk)
inline int launch(const Kernel& k, cudaStream_t st, const uint32_t* mat, unsigned long long m, int log_n, const uint32_t* ap, uint32_t zinv0,
                  uint32_t zinv1, uint32_t* out, int apply_zinv, uint32_t* raw) {
    if (k.fns.size() > 1 && !raw) return 699;
    for (size_t c = 0; c < k.fns.size(); c++) {
        const uint32_t* raw_in = c > 0 ? raw : nullptr;
        uint32_t* raw_out = c + 1 < k.fns.size() ? raw : nullptr;
        void* args[] = {(void*)&mat, (void*)&m, (void*)&log_n, (void*)&ap, (void*)&zinv0, (void*)&zinv1, (void*)&out, (void*)&apply_zinv,
                        (void*)&raw_in, (void*)&raw_out};
        CUresult rc = api().LaunchKernel(k.fns[c], (unsigned)((m + 255) / 256), 1, 1, 256, 1, 1, 0, (CUstream)st, args, nullptr);
        if (rc != CUDA_SUCCESS) return 700 + (int)rc;
    }
    return 0;
}

inline void destroy(Kernel& k) {
    for (CUmodule m : k.mods) api().ModuleUnload(m);
    k.mods.clear();
    k.fns.clear();
}

}  // namespace airjit
