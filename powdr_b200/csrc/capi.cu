// C ABI + host orchestration of the powdr_b200 hot path (include/powdr_b200.h).  Single translation unit: the kernels
// live in the .cuh files included below.  Host code here plays the role of the reference's Rust host side
// (bytecode packing ~ emit_expr, /root/reference/openvm/src/powdr_extension/trace_generator/cuda/mod.rs:49-81;
// launch wrappers ~ /root/reference/openvm/src/cuda_abi.rs:97-135,174-223; stage order ~ engine.prove behind
// /root/reference/openvm-riscv/src/lib.rs:327-332).  No CPU fallback exists: every proving entry point needs a CUDA device.  The
// verifier (verify.inl) and the proof's byte form (proof_bytes.inl) are host code and need none.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <array>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <thread>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../include/pb_poseidon2_constants.h"
#include "../../include/powdr_b200.h"
#include "air.cuh"
#include "air_jit.cuh"
#include "bb31.cuh"
#include "deep.cuh"
#include "fri.cuh"
#include "logup_jit.cuh"
#include "bus_jit.cuh"
#include "ntt.cuh"
#include "ntt_fast.cuh"
#include "ntt_tma.cuh"
#include "poseidon2.cuh"
#include "tracegen.cuh"
#include "transcript_host.h"

#define CK(x)                                  \
    do {                                       \
        cudaError_t e__ = (x);                 \
        if (e__ != cudaSuccess) return (int)e__; \
    } while (0)
#define RC(x)                          \
    do {                               \
        const int r__ = (x);           \
        if (r__) return r__;           \
    } while (0)
#define LAUNCHED(ctx) ((ctx)->launches++)

namespace {

// ---------------- host-side field helpers (Montgomery, same bb:: code as the device) ----------------
inline uint32_t h_to_m(uint32_t c) { return bb::to_monty(c % bb::P); }
inline uint32_t h_from_m(uint32_t m) { return bb::from_monty(m); }
inline uint32_t h_root_of_unity_m(int log_n) { return bb::pow(h_to_m(bb::GEN), (uint64_t)(bb::P - 1) >> log_n); }
inline bb::E4 h_e4_from_canon(const uint32_t v[4]) { bb::E4 r; for (int i = 0; i < 4; i++) r.c[i] = h_to_m(v[i]); return r; }

// the transcript's permutation runs on the host (transcript_host.cpp: AVX-512 with a scalar fallback)
using pbhost::P2Host;
inline void host_permute(uint32_t s[16], const P2Host& k) { pbhost::permute(s, k); }
// the host permutation's constants from canonical ones (pb_ctx_set_poseidon2's arguments)
inline P2Host host_p2(const uint32_t rc_ext[8][16], const uint32_t rc_int[13], const uint32_t diag_m1[16]) {
    P2Host k;
    for (int r = 0; r < 8; r++) for (int i = 0; i < 16; i++) k.rc_ext[r][i] = h_to_m(rc_ext[r][i]);
    for (int r = 0; r < 13; r++) k.rc_int[r] = h_to_m(rc_int[r]);
    for (int i = 0; i < 16; i++) k.diag[i] = h_to_m(diag_m1[i]);
    return k;
}

// DuplexChallenger<BabyBear, Perm16, 16, 8> on Montgomery values (SURVEY.md App. C.6)
struct Challenger {
    const P2Host* k;
    uint32_t sponge[16] = {0};
    uint32_t in_buf[8];
    int n_in = 0;
    uint32_t out_buf[8];
    int n_out = 0;
    void duplexing() {
        for (int i = 0; i < n_in; i++) sponge[i] = in_buf[i];
        n_in = 0;
        host_permute(sponge, *k);
        memcpy(out_buf, sponge, 32);
        n_out = 8;
    }
    void observe(const uint32_t* v, int n) {
        for (int i = 0; i < n; i++) {
            n_out = 0;
            in_buf[n_in++] = v[i];
            if (n_in == 8) duplexing();
        }
    }
    uint32_t sample() {
        if (n_in > 0 || n_out == 0) duplexing();
        return out_buf[--n_out];
    }
    bb::E4 sample_ext() { bb::E4 r; for (int i = 0; i < 4; i++) r.c[i] = sample(); return r; }
};

struct TwiddleSet {
    int n, log_blowup;
    uint32_t shift;      // canonical
    uint2 ninv;          // Shoup pair of 1/N
    uint2* d_inv;        // [2^n]           tw_inv[2^u + k] = w_{2^(u+1)}^{-k}            (Shoup pairs: w, floor(w 2^32/p))
    uint2* d_fwd;        // [cosets][2^n]   tw_fwd[c][2^u + k] = S_c^(2^(n-1-u)) * w_{2^(u+1)}^{k},  S_c = shift * w_{N 2^b}^c
};

// device buffer that grows on demand and frees itself; move-only (noexcept, so that a std::vector of holders can resize)
template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    ~DevBuf() { if (p) cudaFree(p); }
    int ensure(size_t n) {
        if (n <= cap) return 0;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        cudaError_t e = cudaMalloc((void**)&p, n * sizeof(T));
        if (e != cudaSuccess) return (int)e;
        cap = n;
        return 0;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

__global__ void to_monty_kernel(uint32_t* a, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i] = bb::to_monty(a[i]);
}
__global__ void from_monty_kernel(uint32_t* a, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i] = bb::from_monty(a[i]);
}

}  // namespace

struct pb_air {
    uint32_t width = 0, n_constraints = 0;
    DevBuf<uint32_t> d_code;
    DevBuf<air::Span> d_spans;
    DevBuf<uint32_t> d_pool;
    DevBuf<uint32_t> d_alpha_pows;      // [C][4]
    size_t n_code = 0, n_pool = 0;
    airjit::Kernel jit;                 // NVRTC-compiled straight-line evaluator of this AIR
    bool jit_ok = false;
    // LogUp / bus interactions (pb_air_set_interactions): program, generated kernels, per-proof constant buffers
    bool has_lu = false;
    logup::Program lu;
    logup::Kernels lujit;
    DevBuf<uint4> d_kc;                 // [n_ints]   alpha_lu + beta^k (bus+1) + literal arguments
    DevBuf<uint4> d_bt;                 // [max_args + 1] beta powers
    DevBuf<uint4> d_apl;                // [n_chunks] alpha^(n_chunks + 2 - c)
};

struct pb_bus {
    busjit::Kernel k;
    std::vector<unsigned> grid_y;
};

// one chip of a proof (chips.inl): its matrices stay resident until the query phase.  pb_prove_segment uses slot 0.  The sharded provers
// (shard_api.inl) hold their row blocks here; their `perm` is [my trace rows x the padded permutation columns | row sums | my permutation
// columns, whole].  On one GPU a chip's LDEs are 2^lb row blocks (rowblock.inl), and `lde` and `perm_lde` hold one of them: a resident
// chip (lb = 0) has one block, its whole LDE; a row-blocked chip (lb > 0) keeps its main coefficients in `coef` and its permutation
// coefficients in `perm`, and each phase that reads a block recomputes it.
struct McChip {
    size_t log_n = 0, width = 0, wp = 0, n_chunks = 0, e_main = 0, e_perm = 0, e_q = 0, lb = 0;
    const pb_air* air = nullptr;
    const uint32_t* d_trace = nullptr;
    DevBuf<uint32_t> lde, perm, perm_lde, qnat, qlde, coef;
    bb::E4 cumsum = {{0u, 0u, 0u, 0u}};
};

// a committed matrix, column-major [width][2^log_h]; w: the chip whose main (perm = false) or permutation LDE it is, when each of its row
// blocks is to be recomputed into p before it is read (lde_block)
struct Mat { const uint32_t* p; size_t width; size_t log_h; McChip* w = nullptr; bool perm = false; };

namespace shard { struct Xfer; }        // one chip's slice of a batched exchange (shard_api.inl)

struct pb_ctx {
    int device = 0;
    int n_sms = 1;                    // multiprocessor count of `device` (sizes the LDE column batches)
    cudaStream_t stream = nullptr;
    uint64_t launches = 0;
    P2Host p2;
    std::vector<TwiddleSet> tws;
    uint32_t* d_fold_tab = nullptr;   // w_L^{-bitrev(j)}, j < L/2, Montgomery
    int fold_tab_log_len = 0;
    DevBuf<uint32_t> tmp, tmp2;       // LDE intermediates (L2-sized)
    DevBuf<const uint32_t*> coltab;
    // proof workspaces: the matrices of every prover live in the chip slots and the three trees
    std::vector<McChip> chips;
    DevBuf<uint32_t> tree_main, tree_perm, tree_q;   // main, permutation and quotient commitments (node-major layers)
    DevBuf<uint32_t> ro[32];                         // reduced-opening codeword of each LDE height below the tallest
    DevBuf<uint32_t> ws_trace, ws_q, ws_f0, ws_state, ws_ys;
    DevBuf<uint4> ws_w, ws_part;          // barycentric weights [N], per-CTA partial sums of the openings
    DevBuf<uint2> ws_gp;                  // gamma powers of the reduced opening, canonical (one uint4 per column)
    DevBuf<uint32_t> ws_fri_words, ws_fri_trees, ws_qidx, ws_qout;
    DevBuf<uint32_t> ws_shard_send, ws_shard_recv, ws_shard_coef, ws_gather, ws_gather2;   // multi-GPU segment (shard_api.inl)
    DevBuf<uint32_t> ws_qraw;             // running constraint fold between the chunks of a JIT-compiled AIR, [4][rows]
    DevBuf<uint32_t> ws_rowsum, ws_scan_tot, ws_lu_raw, ws_lu_s, ws_pow;   // LogUp phase + PoW
    DevBuf<uint32_t> ws_mc_dig;           // digests of the shorter height groups until the tree reaches their level
    uint32_t n_queries = 100, pow_bits = 16;
    size_t mem_budget = 0;                // pb_ctx_set_memory_budget (0: free device memory + what the proof workspaces hold)
    uint32_t last_lb = 0;                 // log2 of the row blocks of the last proof (0: resident); sharded: per rank block
    uint64_t proof_serial = 0;            // proofs begun on this context (invalidate_proofs): a group's query phase checks it is still its proof
    DevBuf<uint32_t> ws_fri_ch, ws_fri_log;  // device challenger state and the (root, beta) log of the FRI commit phase
    DevBuf<uint32_t> ws_sh_qall;             // every rank's share of the query openings
    DevBuf<shard::Xfer> ws_sh_tab;           // chip table of the batched exchanges
    DevBuf<uint32_t> ws_sh_q, ws_sh_sub;     // row-blocked sharded quotient: the rank's [chip][4][Ms], one sub-block's q | S | phi
    // The last proof, read by the query phase of the prover that made it (everything else stays resident on the device).
    enum class Prover { segment, chips, sharded, chips_sharded };
    struct {
        bool valid = false;
        Prover by = Prover::segment;
        size_t K = 0, hmax = 0, hperm = 0;   // chips; log2 of the tallest LDE, of the tallest one with a permutation trace
        uint32_t n_layers = 0;
        size_t word_off[33] = {0}, tree_off[33] = {0};
        Challenger ch;                       // transcript state after the proof of work
        std::vector<uint32_t> ys;            // opened values, Montgomery, [n_opened][4]
        // The context holds row block `rank` of G = 2^g of every committed matrix with the subtree over it, and of every row-sharded
        // FRI layer; a replicated layer is held whole by rank 0.  One GPU: G = 1.  top_*: the tree over each commitment's G subtree
        // roots, node-major like every tree (2G - 1 nodes, Montgomery)
        int G = 1, g = 0, rank = 0;
        bool layer_sharded[33] = {false};
        uint32_t top_main[31][8], top_perm[31][8], top_q[31][8], top_fri[32][31][8];
    } last;
    cudaStream_t copy_stream = nullptr;   // H2D chunks of the host-input pipeline
    cudaEvent_t ev_copy[2] = {nullptr}, ev_free[2] = {nullptr};
    cudaEvent_t ev[12] = {nullptr};         // stage boundaries of pb_last_stage_ms (stage_clocks)
    float stage_ms[PB_N_STAGES] = {0};     // h2d, lde, merkle, logup_gen, logup_commit, quotient, qlde, qmerkle, open(+deep), fri, pow, total
    // live timing of the dominant kernel (Poseidon2 leaf hashing over column-major matrices): event pairs on the stream
    static constexpr int KPROF = 16;
    cudaEvent_t kp_a[KPROF] = {nullptr}, kp_b[KPROF] = {nullptr};
    double kp_bytes[KPROF] = {0};
    int kp_n = 0;
};

namespace {

int upload_p2(pb_ctx* ctx, const uint32_t rc_ext[8][16], const uint32_t rc_int[13], const uint32_t diag[16]) {
    p2::Consts c;
    for (int r = 0; r < 8; r++)
        for (int i = 0; i < 16; i++) {
            uint32_t m = h_to_m(rc_ext[r][i]);
            ctx->p2.rc_ext[r][i] = m;
            c.rc_ext_mp[r][i] = m - bb::P;
        }
    for (int r = 0; r < 13; r++) {
        uint32_t m = h_to_m(rc_int[r]);
        ctx->p2.rc_int[r] = m;
        c.rc_int_mp[r] = m - bb::P;
    }
    bool p3 = true;
    for (int i = 0; i < 16; i++) {
        const uint32_t w = diag[i] % bb::P;
        ctx->p2.diag[i] = h_to_m(w);
        c.diag_w[i] = w;
        c.diag_wp[i] = (uint32_t)(((uint64_t)w << 32) / bb::P);
        p3 = p3 && w == PB_P2_DIAG_M1[i];
    }
    c.p3_diag = p3 ? 1u : 0u;
    CK(cudaMemcpyToSymbolAsync(p2::c_p2, &c, sizeof c, 0, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

int get_twiddles(pb_ctx* ctx, int n, int log_blowup, uint32_t shift, const TwiddleSet** out) {
    for (auto& t : ctx->tws)
        if (t.n == n && t.log_blowup == log_blowup && t.shift == shift) { *out = &t; return 0; }
    const size_t N = (size_t)1 << n;
    const int cosets = 1 << log_blowup;
    // entries are Shoup pairs (w canonical, floor(w 2^32 / p)); powers are walked in Montgomery form and converted on store
    std::vector<uint2> inv(N), fwd(N * cosets);
    inv[0] = make_uint2(0u, 0u);
    for (int u = 0; u < n; u++) {
        uint32_t w = bb::inv(h_root_of_unity_m(u + 1)), x = bb::R1;
        for (size_t k = 0; k < ((size_t)1 << u); k++) { inv[((size_t)1 << u) + k] = bb::shoup_pair(h_from_m(x)); x = bb::mul(x, w); }
    }
    const uint32_t shift_m = h_to_m(shift);
    const uint32_t w_ext = h_root_of_unity_m(n + log_blowup);
    for (int c = 0; c < cosets; c++) {
        uint32_t sc = bb::mul(shift_m, bb::pow(w_ext, (uint64_t)c));
        uint2* f = fwd.data() + (size_t)c * N;
        f[0] = make_uint2(0u, 0u);
        // factor for stage u is S_c^(2^(n-1-u)): walk u from n-1 down, squaring
        uint32_t fac = sc;
        for (int u = n - 1; u >= 0; u--) {
            uint32_t w = h_root_of_unity_m(u + 1), x = fac;
            for (size_t k = 0; k < ((size_t)1 << u); k++) { f[((size_t)1 << u) + k] = bb::shoup_pair(h_from_m(x)); x = bb::mul(x, w); }
            fac = bb::mul(fac, fac);
        }
    }
    TwiddleSet t;
    t.n = n; t.log_blowup = log_blowup; t.shift = shift;
    t.ninv = bb::shoup_pair(h_from_m(bb::inv(h_to_m((uint32_t)(N % bb::P)))));
    CK(cudaMalloc((void**)&t.d_inv, N * sizeof(uint2)));
    CK(cudaMalloc((void**)&t.d_fwd, N * cosets * sizeof(uint2)));
    CK(cudaMemcpyAsync(t.d_inv, inv.data(), N * sizeof(uint2), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(t.d_fwd, fwd.data(), N * cosets * sizeof(uint2), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    // bounded cache: a multi-chip segment cycles through (height, shift) pairs -- 3 shifts per height -- so keep them all
    // unless the tables get large (FIFO eviction above 64 sets or 4 GiB)
    auto bytes_of = [](const TwiddleSet& s) { return (((size_t)1 << s.n) * ((size_t)1 + ((size_t)1 << s.log_blowup))) * sizeof(uint2); };
    size_t total = bytes_of(t);
    for (auto& s : ctx->tws) total += bytes_of(s);
    while (!ctx->tws.empty() && (ctx->tws.size() >= 64 || total > ((size_t)4 << 30))) {
        total -= bytes_of(ctx->tws.front());
        cudaFree(ctx->tws.front().d_inv);
        cudaFree(ctx->tws.front().d_fwd);
        ctx->tws.erase(ctx->tws.begin());
    }
    ctx->tws.push_back(t);
    *out = &ctx->tws.back();
    return 0;
}

int get_fold_table(pb_ctx* ctx, int log_len) {
    if (ctx->d_fold_tab && ctx->fold_tab_log_len >= log_len) return 0;
    if (ctx->d_fold_tab) { cudaFree(ctx->d_fold_tab); ctx->d_fold_tab = nullptr; }
    const size_t half = (size_t)1 << (log_len - 1);
    std::vector<uint32_t> nat(half), tab(half);
    uint32_t w = bb::inv(h_root_of_unity_m(log_len)), x = bb::R1;
    for (size_t k = 0; k < half; k++) { nat[k] = x; x = bb::mul(x, w); }
    for (size_t j = 0; j < half; j++) {
        uint32_t r = 0;
        for (int b = 0; b < log_len - 1; b++) r |= ((j >> b) & 1u) << (log_len - 2 - b);
        tab[j] = nat[r];
    }
    CK(cudaMalloc((void**)&ctx->d_fold_tab, half * 4));
    CK(cudaMemcpyAsync(ctx->d_fold_tab, tab.data(), half * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->fold_tab_log_len = log_len;
    return 0;
}

// Merkle layers above the leaves: node-major, layer k+1 follows layer k.  Levels with more than MERKLE_COOP nodes are throughput
// work: compress_block_kernel, one thread per permutation, up to 10 levels per launch.  Below that every level is ONE permutation
// latency however few nodes it has, and 16 lanes per permutation shorten that latency, so they run on compress_coop_kernel:
// 128-node subtrees per CTA, then the last <= 128 nodes in one CTA.  On wider levels the one-thread-per-permutation form wins.
constexpr size_t MERKLE_COOP = 1024;     // nodes
constexpr size_t LEAF_COOP = 1024;       // rows: leaf sponges of shorter matrices run 16 lanes per row as well
int merkle_upper(pb_ctx* ctx, uint32_t* d_layers, size_t log_h) {
    size_t n = (size_t)1 << log_h;
    uint32_t* prev = d_layers;
    while (n > 1) {
        int kb = 0;
        if (n <= MERKLE_COOP) {
            while (kb < 7 && ((size_t)1 << (kb + 1)) <= n) kb++;
            const unsigned threads = 16u * (unsigned)std::max<size_t>(2, ((size_t)1 << kb) / 2);       // one group per first-level parent
            p2::compress_coop_kernel<<<(unsigned)(n >> kb), threads, 0, ctx->stream>>>(prev, n, kb);
        } else {
            while (kb < 10 && (n >> (kb + 1)) >= MERKLE_COOP) kb++;
            const unsigned threads = (unsigned)std::min<size_t>(256, std::max<size_t>(32, ((size_t)1 << kb) / 2));
            p2::compress_block_kernel<<<(unsigned)(n >> kb), threads, 0, ctx->stream>>>(reinterpret_cast<uint4*>(prev), n, kb);
        }
        LAUNCHED(ctx);
        for (int l = 0; l < kb; l++) { prev += 8 * n; n >>= 1; }
    }
    CK(cudaGetLastError());
    return 0;
}

int read_root(pb_ctx* ctx, const uint32_t* d_layers, size_t log_h, uint32_t root_m[8]) {
    const size_t root_off = 8 * (((size_t)2 << log_h) - 2);
    CK(cudaMemcpyAsync(root_m, d_layers + root_off, 32, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

// leaf digests of 2^log_h rows over the column-major columns `cols` into d_out (8 words per row), timed for pb_leaf_kernel_profile
int leaf_hash_cols(pb_ctx* ctx, const std::vector<const uint32_t*>& cols, size_t log_h, uint32_t* d_out) {
    const size_t h = (size_t)1 << log_h;
    RC(ctx->coltab.ensure(std::max<size_t>(1, cols.size())));
    // (pageable source: staged before the call returns; the table itself is reused in stream order)
    CK(cudaMemcpyAsync(ctx->coltab.p, cols.data(), cols.size() * sizeof(void*), cudaMemcpyHostToDevice, ctx->stream));
    const int slot = ctx->kp_n < pb_ctx::KPROF ? ctx->kp_n : -1;
    if (slot >= 0) CK(cudaEventRecord(ctx->kp_a[slot], ctx->stream));
    if (h <= LEAF_COOP)
        p2::leaf_hash_cols_coop_kernel<<<(unsigned)((16 * h + 255) / 256), 256, 0, ctx->stream>>>(ctx->coltab.p, (uint32_t)cols.size(), h, d_out);
    else
        p2::leaf_hash_cols_kernel<<<(unsigned)((h + p2::LEAF_THREADS - 1) / p2::LEAF_THREADS), p2::LEAF_THREADS, 0, ctx->stream>>>(ctx->coltab.p, (uint32_t)cols.size(), h, d_out);
    LAUNCHED(ctx);
    if (slot >= 0) {
        CK(cudaEventRecord(ctx->kp_b[slot], ctx->stream));
        ctx->kp_bytes[slot] = 4.0 * (double)h * (double)cols.size() + 32.0 * (double)h;   // algorithmic bytes: matrix in, digests out
        ctx->kp_n++;
    }
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// The two halves of the LDE (shared by pb_lde_batch and pb_lde_shard), with the pass plan of each log_n fixed at compile time

// Column batch: 16 tiles of 2^LDE_BATCH_LOG_TILE elements per SM (66 columns at 2^20 on 132 SMs).  On the H100 the passes run
// at 40-75 % of HBM bandwidth and 3-6 butterflies/clk/SM (scripts/lde_kernels.py); batches of 2-16 columns, alone or round-robin
// over 2-8 streams so that the K1->K2->K3 intermediates of the batches in flight fit the 50 MB L2, measured no faster at 2022 or
// 3348 columns (DESIGN.md §4).  PB_LDE_BATCH overrides the batch size.
constexpr int LDE_BATCH_LOG_TILE = 15;
size_t lde_column_batch(const pb_ctx* ctx, size_t N, size_t width) {
    const size_t tiles_per_col = std::max<size_t>(1, N >> LDE_BATCH_LOG_TILE);
    size_t batch = std::max<size_t>(1, (size_t)ctx->n_sms * 16 / tiles_per_col);
    if (const char* e = getenv("PB_LDE_BATCH")) batch = std::max<size_t>(1, (size_t)atol(e));
    batch = std::min<size_t>(std::min<size_t>(batch, width), 32768);
    return (width + (width + batch - 1) / batch - 1) / ((width + batch - 1) / batch);     // equal-sized batches (no runt batch)
}

// K1: inverse high bits, nb natural-order columns (stride N) of src into coef (stride N)
template <int LOG_N>
void k1_pass(pb_ctx* ctx, const TwiddleSet* tw, const uint32_t* src, unsigned nb, uint32_t* coef) {
    constexpr int LO = nttf::n_lo_of(LOG_N), HI = LOG_N - LO;
    constexpr size_t N = (size_t)1 << LOG_N;
    const dim3 g1(1u << (LO - nttf::log_lc_of(HI)), nb);
    nttf::strided_kernel<HI, LO, true><<<g1, nttf::THREADS, nttf::tile_bytes(HI), ctx->stream>>>(src, N, 0u, coef, N, 0, tw->d_inv);
    LAUNCHED(ctx);
}

// K2a: inverse low bits, src (stride N; may be coef) into coef (stride N), scaled by 1/N
template <int LOG_N>
void k2a_pass(pb_ctx* ctx, const TwiddleSet* tw, const uint32_t* src, unsigned nb, uint32_t* coef) {
    constexpr int LO = nttf::n_lo_of(LOG_N), HI = LOG_N - LO;
    constexpr size_t N = (size_t)1 << LOG_N;
    const size_t total_blocks = (size_t)nb << HI;
    // n_lo == 10: the TMA-staged kernel (ntt_tma.cuh) where its preconditions hold
    if (!ntttma::launch_inverse(LOG_N, LO, ctx->stream, src, coef, nb, tw->d_inv, tw->ninv)) {
        const dim3 g2((unsigned)((total_blocks + ((size_t)1 << nttf::log_lc_of(LO)) - 1) >> nttf::log_lc_of(LO)));
        nttf::transposed_kernel<LO, true><<<g2, nttf::THREADS, nttf::tile_bytes(LO), ctx->stream>>>(src, N, coef, LOG_N, 0, total_blocks,
                                                                                                    tw->d_inv, tw->ninv);
    }
    LAUNCHED(ctx);
}

// K2b: forward low bits, coefficients (stride N) -> scratch [nb][cosets][N]
template <int LOG_N>
void k2b_pass(pb_ctx* ctx, const TwiddleSet* tw, int log_blowup, const uint32_t* coef, unsigned nb, uint32_t* scratch) {
    constexpr int LO = nttf::n_lo_of(LOG_N), HI = LOG_N - LO;
    constexpr size_t N = (size_t)1 << LOG_N;
    const size_t total_blocks = (size_t)nb << HI;
    const dim3 g2((unsigned)((total_blocks + ((size_t)1 << nttf::log_lc_of(LO)) - 1) >> nttf::log_lc_of(LO)), 1, 1u << log_blowup);
    nttf::transposed_kernel<LO, false><<<g2, nttf::THREADS, nttf::tile_bytes(LO), ctx->stream>>>(coef, N, scratch, LOG_N, log_blowup,
                                                                                                 total_blocks, tw->d_fwd, make_uint2(0u, 0u));
    LAUNCHED(ctx);
}

// K3 (or, without high bits, the bit-reversed store): scratch [nb][cosets][N] -> out[col * out_stride + bitrev_b(c) * N + bitrev_n(k)];
// the scratch rows are grouped by 2^lg (nttf::strided_kernel), 0 = natural order
template <int LOG_N>
void k3_pass(pb_ctx* ctx, const TwiddleSet* tw, int log_blowup, unsigned nb, const uint32_t* scratch, uint32_t lg, uint32_t* out, size_t out_stride) {
    constexpr int LO = nttf::n_lo_of(LOG_N), HI = LOG_N - LO;
    const unsigned cosets = 1u << log_blowup;
    if constexpr (HI > 0) {
        const dim3 g3(1u << (LO - nttf::log_lc_of(HI)), nb, cosets);
        nttf::strided_kernel<HI, LO, false><<<g3, nttf::THREADS, nttf::tile_bytes(HI), ctx->stream>>>(scratch, 0, lg, out, out_stride, log_blowup,
                                                                                                      tw->d_fwd);
    } else {
        const size_t tot = ((size_t)nb * cosets) << LOG_N;
        ntt::bitrev_store_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, ctx->stream>>>(scratch, out, out_stride, LOG_N, log_blowup, nb);
    }
    LAUNCHED(ctx);
}

// K1 + K2a: nb natural-order columns (stride N) -> coefficients in bit-reversed slots, scaled by 1/N, in coef (stride N)
template <int LOG_N>
void inverse_passes(pb_ctx* ctx, const TwiddleSet* tw, const uint32_t* src, unsigned nb, uint32_t* coef) {
    if constexpr (LOG_N > nttf::n_lo_of(LOG_N)) {
        k1_pass<LOG_N>(ctx, tw, src, nb, coef);
        src = coef;
    }
    k2a_pass<LOG_N>(ctx, tw, src, nb, coef);
}

// K2b + K3: coefficients (bit-reversed slots, stride N) -> 2^log_blowup coset evaluations per column, bit-reversed rows,
// out[col * out_stride + bitrev_b(c) * N + bitrev_n(k)];  scratch holds [nb][cosets][N]
template <int LOG_N>
void forward_passes(pb_ctx* ctx, const TwiddleSet* tw, int log_blowup, const uint32_t* coef, unsigned nb, uint32_t* scratch, uint32_t* out,
                    size_t out_stride) {
    k2b_pass<LOG_N>(ctx, tw, log_blowup, coef, nb, scratch);
    k3_pass<LOG_N>(ctx, tw, log_blowup, nb, scratch, 0u, out, out_stride);
}

// the whole LDE of nb natural-order columns (stride N) into out: inverse_passes into tmp, then forward_passes through scratch, except
// that where the TMA kernels apply (n_lo = 10) K2a and K2b run as one pass and the coefficients never reach HBM
template <int LOG_N>
void lde_passes(pb_ctx* ctx, const TwiddleSet* tw, int log_blowup, const uint32_t* src, unsigned nb, uint32_t* tmp, uint32_t* scratch,
                uint32_t* out, size_t out_stride) {
    constexpr int LO = nttf::n_lo_of(LOG_N);
    if constexpr (LOG_N > LO) {
        k1_pass<LOG_N>(ctx, tw, src, nb, tmp);
        uint32_t lg = 0;
        if (ntttma::launch_low_bits(LOG_N, LO, ctx->stream, tmp, scratch, nb, log_blowup, tw->d_inv, tw->ninv, tw->d_fwd)) {
            LAUNCHED(ctx);
            lg = ntttma::LOG_ROW_GROUP;
        } else {
            k2a_pass<LOG_N>(ctx, tw, tmp, nb, tmp);
            k2b_pass<LOG_N>(ctx, tw, log_blowup, tmp, nb, scratch);
        }
        k3_pass<LOG_N>(ctx, tw, log_blowup, nb, scratch, lg, out, out_stride);
    } else {
        inverse_passes<LOG_N>(ctx, tw, src, nb, tmp);
        forward_passes<LOG_N>(ctx, tw, log_blowup, tmp, nb, scratch, out, out_stride);
    }
}

// dynamic shared memory opt-in of the passes' kernels on the current device
template <int LOG_N>
int opt_in_passes() {
    constexpr int LO = nttf::n_lo_of(LOG_N), HI = LOG_N - LO, SMEM = 4 << nttf::LOG_TILE;
    CK(cudaFuncSetAttribute(nttf::transposed_kernel<LO, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    CK(cudaFuncSetAttribute(nttf::transposed_kernel<LO, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    if constexpr (HI > 0) {
        CK(cudaFuncSetAttribute(nttf::strided_kernel<HI, LO, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
        CK(cudaFuncSetAttribute(nttf::strided_kernel<HI, LO, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    }
    return 0;
}

struct NttPlan {
    void (*inverse)(pb_ctx*, const TwiddleSet*, const uint32_t*, unsigned, uint32_t*);
    void (*forward)(pb_ctx*, const TwiddleSet*, int, const uint32_t*, unsigned, uint32_t*, uint32_t*, size_t);
    void (*lde)(pb_ctx*, const TwiddleSet*, int, const uint32_t*, unsigned, uint32_t*, uint32_t*, uint32_t*, size_t);
    int (*opt_in)();
};
template <size_t... I>
constexpr std::array<NttPlan, sizeof...(I)> make_ntt_plans(std::index_sequence<I...>) {
    return {{{inverse_passes<(int)I + 1>, forward_passes<(int)I + 1>, lde_passes<(int)I + 1>, opt_in_passes<(int)I + 1>}...}};
}
constexpr auto NTT_PLANS = make_ntt_plans(std::make_index_sequence<24>());     // NTT_PLANS[log_n - 1], 1 <= log_n <= 24

void ntt_inverse_cols(pb_ctx* ctx, int log_n, const TwiddleSet* tw, const uint32_t* src, unsigned nb, uint32_t* coef) {
    NTT_PLANS[log_n - 1].inverse(ctx, tw, src, nb, coef);
}
void ntt_forward_cols(pb_ctx* ctx, int log_n, const TwiddleSet* tw, int log_blowup, const uint32_t* coef, unsigned nb, uint32_t* scratch,
                      uint32_t* out, size_t out_stride) {
    NTT_PLANS[log_n - 1].forward(ctx, tw, log_blowup, coef, nb, scratch, out, out_stride);
}
void ntt_lde_cols(pb_ctx* ctx, int log_n, const TwiddleSet* tw, int log_blowup, const uint32_t* src, unsigned nb, uint32_t* tmp, uint32_t* scratch,
                  uint32_t* out, size_t out_stride) {
    NTT_PLANS[log_n - 1].lde(ctx, tw, log_blowup, src, nb, tmp, scratch, out, out_stride);
}

}  // namespace

// =====================================================================================================================
extern "C" {

int pb_ctx_create(pb_ctx_t** out, int device, void* cuda_stream) {
    if (!out) return PB_ERR_INVALID_ARG;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) return PB_ERR_NO_DEVICE;
    CK(cudaSetDevice(device));
    pb_ctx* ctx = new pb_ctx();
    ctx->device = device;
    ctx->stream = (cudaStream_t)cuda_stream;
    // any failure below releases what was created so far (pb_ctx_destroy tolerates a half-built context)
    auto init = [&]() -> int {
        CK(cudaDeviceGetAttribute(&ctx->n_sms, cudaDevAttrMultiProcessorCount, device));
        for (auto& e : ctx->ev) CK(cudaEventCreate(&e));
        CK(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
        for (int i = 0; i < 2; i++) {
            CK(cudaEventCreateWithFlags(&ctx->ev_copy[i], cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&ctx->ev_free[i], cudaEventDisableTiming));
        }
        for (int i = 0; i < pb_ctx::KPROF; i++) { CK(cudaEventCreate(&ctx->kp_a[i])); CK(cudaEventCreate(&ctx->kp_b[i])); }
        // the runtime applies a kernel's shared memory opt-in to the current device only: every context does its own
        for (const NttPlan& p : NTT_PLANS) RC(p.opt_in());
        CK(cudaFuncSetAttribute(ntttma::transposed_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ntttma::SMEM_BYTES));
        CK(cudaFuncSetAttribute(ntttma::lde_low_bits_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ntttma::LOW_BITS_SMEM_BYTES));
        return upload_p2(ctx, PB_P2_RC_EXT, PB_P2_RC_INT, PB_P2_DIAG_M1);
    };
    const int rc = init();
    if (rc) { pb_ctx_destroy(ctx); return rc; }
    *out = ctx;
    return 0;
}

int pb_ctx_destroy(pb_ctx_t* ctx) {
    if (!ctx) return 0;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (auto& t : ctx->tws) { cudaFree(t.d_inv); cudaFree(t.d_fwd); }
    if (ctx->d_fold_tab) cudaFree(ctx->d_fold_tab);
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    for (int i = 0; i < 2; i++) { if (ctx->ev_copy[i]) cudaEventDestroy(ctx->ev_copy[i]); if (ctx->ev_free[i]) cudaEventDestroy(ctx->ev_free[i]); }
    for (auto& e : ctx->ev) if (e) cudaEventDestroy(e);
    for (int i = 0; i < pb_ctx::KPROF; i++) { if (ctx->kp_a[i]) cudaEventDestroy(ctx->kp_a[i]); if (ctx->kp_b[i]) cudaEventDestroy(ctx->kp_b[i]); }
    delete ctx;                                  // the workspaces free themselves
    return 0;
}

// the transcript's host-side permutation with the default (Plonky3) instance, canonical words in and out; needs no device
int pb_host_poseidon2_permute(uint32_t state[16], int reps, int force_scalar, int* used_avx512) {
    if (!state || reps < 0) return PB_ERR_INVALID_ARG;
    const P2Host k = host_p2(PB_P2_RC_EXT, PB_P2_RC_INT, PB_P2_DIAG_M1);
    uint32_t s[16];
    for (int i = 0; i < 16; i++) s[i] = h_to_m(state[i]);
    for (int i = 0; i < reps; i++) { if (force_scalar) pbhost::permute_scalar(s, k); else pbhost::permute(s, k); }
    for (int i = 0; i < 16; i++) state[i] = h_from_m(s[i]);
    if (used_avx512) *used_avx512 = force_scalar ? 0 : pbhost::uses_avx512();
    return 0;
}

int pb_ctx_synchronize(pb_ctx_t* ctx) { CK(cudaStreamSynchronize(ctx->stream)); return 0; }

int pb_ctx_set_poseidon2(pb_ctx_t* ctx, const uint32_t rc_ext[8][16], const uint32_t rc_int[13], const uint32_t diag_m1[16]) {
    if (!ctx || !rc_ext || !rc_int || !diag_m1) return PB_ERR_INVALID_ARG;
    // NOTE: the device-side constants are one __constant__ symbol per process and GPU: every context on this GPU hashes with
    // the last instantiation set (documented in include/powdr_b200.h); the host-side transcript constants are per context.
    CK(cudaSetDevice(ctx->device));
    return upload_p2(ctx, rc_ext, rc_int, diag_m1);
}

int pb_host_alloc(void** out, size_t bytes) { CK(cudaHostAlloc(out, bytes, cudaHostAllocDefault)); return 0; }
int pb_host_free(void* p) { CK(cudaFreeHost(p)); return 0; }
int pb_device_alloc(void** out, size_t bytes) { CK(cudaMalloc(out, bytes)); return 0; }
int pb_device_free(void* p) { CK(cudaFree(p)); return 0; }

int pb_copy_h2d(pb_ctx_t* ctx, void* d, const void* h, size_t bytes) {
    CK(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return 0;
}
int pb_copy_d2h(pb_ctx_t* ctx, void* h, const void* d, size_t bytes) {
    CK(cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}
int pb_memset_zero(pb_ctx_t* ctx, void* d, size_t bytes) {
    CK(cudaMemsetAsync(d, 0, bytes, ctx->stream));
    return 0;
}

int pb_to_monty(pb_ctx_t* ctx, uint32_t* d, size_t n) {
    if (!n) return 0;
    to_monty_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d, n);
    LAUNCHED(ctx);
    CK(cudaGetLastError());
    return 0;
}
int pb_from_monty(pb_ctx_t* ctx, uint32_t* d, size_t n) {
    if (!n) return 0;
    from_monty_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d, n);
    LAUNCHED(ctx);
    CK(cudaGetLastError());
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
int pb_lde_batch(pb_ctx_t* ctx, const uint32_t* d_trace, size_t log_n, size_t width, uint32_t log_blowup, uint32_t shift,
                 uint32_t* d_lde) {
    if (!ctx || !d_trace || !d_lde) return PB_ERR_INVALID_ARG;
    if (log_n < 1 || log_n > 24 || log_blowup < 1 || log_blowup > 3 || shift == 0 || shift >= bb::P) return PB_ERR_UNSUPPORTED;
    if (width == 0) return 0;
    const int n = (int)log_n;
    const size_t N = (size_t)1 << n;
    const int cosets = 1 << log_blowup;
    const TwiddleSet* tw;
    int rc = get_twiddles(ctx, n, (int)log_blowup, shift, &tw);
    if (rc) return rc;
    const size_t batch = lde_column_batch(ctx, N, width);
    rc = ctx->tmp.ensure(batch * N); if (rc) return rc;
    rc = ctx->tmp2.ensure(batch * N * cosets); if (rc) return rc;
    for (size_t c0 = 0; c0 < width; c0 += batch) {
        const unsigned nb = (unsigned)std::min(batch, width - c0);
        ntt_lde_cols(ctx, n, tw, (int)log_blowup, d_trace + c0 * N, nb, ctx->tmp.p, ctx->tmp2.p, d_lde + c0 * N * cosets, N * cosets);
    }
    CK(cudaGetLastError());
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// reference-format bytecode -> validated, packed program (one word per instruction + Montgomery constant pool)
static int pack_program(const uint32_t* bc, size_t n_words, const pb_expr_span_t* cons, size_t n_constraints, uint32_t width,
                        std::vector<uint32_t>& code, std::vector<uint32_t>& pool, std::vector<air::Span>& spans) {
    std::unordered_map<uint32_t, uint32_t> pool_idx;
    for (size_t k = 0; k < n_constraints; k++) {
        const size_t off = cons[k].off, len = cons[k].len;
        if (off + len > n_words) return PB_ERR_BAD_BYTECODE;
        air::Span sp{(uint32_t)code.size(), 0};
        int depth = 0;
        for (size_t ip = off; ip < off + len;) {
            const uint32_t op = bc[ip++];
            if (op == air::OP_PUSH_APC || op == air::OP_PUSH_CONST) {
                if (ip >= off + len) return PB_ERR_BAD_BYTECODE;
                const uint32_t arg = bc[ip++];
                if (++depth > air::STACK_CAPACITY) return PB_ERR_STACK_DEPTH;
                if (op == air::OP_PUSH_APC) {
                    if (arg >= width) return PB_ERR_BAD_BYTECODE;
                    code.push_back((op << 28) | arg);
                } else {
                    auto it = pool_idx.find(arg % bb::P);
                    uint32_t idx;
                    if (it == pool_idx.end()) {
                        idx = (uint32_t)pool.size();
                        pool_idx[arg % bb::P] = idx;
                        pool.push_back(h_to_m(arg));
                    } else idx = it->second;
                    code.push_back((op << 28) | idx);
                }
            } else if (op == air::OP_ADD || op == air::OP_SUB || op == air::OP_MUL) {
                if (depth < 2) return PB_ERR_BAD_BYTECODE;
                depth--;
                code.push_back(op << 28);
            } else if (op == air::OP_NEG || op == air::OP_INV_OR_ZERO) {
                if (depth < 1) return PB_ERR_BAD_BYTECODE;
                code.push_back(op << 28);
            } else return PB_ERR_BAD_BYTECODE;
        }
        if (depth != 1) return PB_ERR_BAD_BYTECODE;
        sp.len = (uint32_t)code.size() - sp.off;
        spans.push_back(sp);
    }
    return 0;
}

int pb_air_jit_compile_only(const uint32_t* bc, size_t n_words, const pb_expr_span_t* cons, size_t n_constraints, uint32_t width,
                            size_t* cubin_bytes) {
    if ((!bc && n_words) || (!cons && n_constraints)) return PB_ERR_INVALID_ARG;
    std::vector<uint32_t> code, pool;
    std::vector<air::Span> spans;
    int rc = pack_program(bc, n_words, cons, n_constraints, width, code, pool, spans);
    if (rc) return rc;
    size_t total = 0;
    rc = airjit::build(code, spans, pool, nullptr, &total);
    if (cubin_bytes) *cubin_bytes = total;
    return rc ? PB_ERR_UNSUPPORTED : 0;
}

int pb_air_compile(pb_ctx_t* ctx, const uint32_t* bc, size_t n_words, const pb_expr_span_t* cons, size_t n_constraints,
                   uint32_t width, pb_air_t** out) {
    if (!ctx || !out || (!bc && n_words) || (!cons && n_constraints)) return PB_ERR_INVALID_ARG;
    std::vector<uint32_t> code, pool;
    std::vector<air::Span> spans;
    {
        int prc = pack_program(bc, n_words, cons, n_constraints, width, code, pool, spans);
        if (prc) return prc;
    }
    std::unique_ptr<pb_air> a(new pb_air());          // an early return below frees it and its buffers
    a->width = width;
    a->n_constraints = (uint32_t)n_constraints;
    a->n_code = code.size();
    a->n_pool = pool.size();
    RC(a->d_code.ensure(std::max<size_t>(1, code.size())));
    RC(a->d_spans.ensure(std::max<size_t>(1, spans.size())));
    RC(a->d_pool.ensure(std::max<size_t>(1, pool.size())));
    RC(a->d_alpha_pows.ensure(4 * std::max<size_t>(1, n_constraints)));
    CK(cudaMemcpyAsync(a->d_code.p, code.data(), code.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(a->d_spans.p, spans.data(), spans.size() * sizeof(air::Span), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(a->d_pool.p, pool.data(), pool.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    a->jit_ok = n_constraints > 0 && airjit::build(code, spans, pool, &a->jit) == 0;   // straight-line per-AIR kernel (air_jit.cuh)
    *out = a.release();
    return 0;
}

int pb_air_is_jit(const pb_air_t* a) { return a && a->jit_ok ? 1 : 0; }

int pb_air_free(pb_air_t* a) {
    if (!a) return 0;
    if (a->jit_ok) airjit::destroy(a->jit);
    if (a->has_lu) logup::destroy(a->lujit);
    delete a;
    return 0;
}

static int upload_alpha_pows(pb_ctx* ctx, const pb_air* a, bb::E4 alpha, size_t extra = 0) {
    // alpha_pows[k] = alpha^(C-1-k+extra): `extra` = number of constraints folded after the AIR's own (the LogUp ones)
    const size_t C = a->n_constraints;
    std::vector<uint32_t> ap(4 * std::max<size_t>(1, C));
    bb::E4 cur = {{bb::R1, 0, 0, 0}};
    for (size_t e = 0; e < extra; e++) cur = bb::e4_mul(cur, alpha);
    for (size_t k = C; k-- > 0;) {          // alpha_pows[k] = alpha^(C-1-k)
        memcpy(&ap[4 * k], cur.c, 16);
        cur = bb::e4_mul(cur, alpha);
    }
    CK(cudaMemcpyAsync(a->d_alpha_pows.p, ap.data(), 16 * C, cudaMemcpyHostToDevice, ctx->stream));
    return 0;
}

// Z_H(x) = x^N - 1 on the two cosets s*H and s*w_2N*H of the LDE domain (log_blowup 1) is s^N - 1 and -s^N - 1:
// sn = s^N, zinv0 / zinv1 = their inverses (Montgomery)
static void zh_inverses(size_t log_n, uint32_t shift_m, uint32_t* sn, uint32_t* zinv0, uint32_t* zinv1) {
    *sn = bb::pow(shift_m, (uint64_t)1 << log_n);
    *zinv0 = bb::inv(bb::sub(*sn, bb::R1));
    *zinv1 = bb::inv(bb::sub(bb::neg(*sn), bb::R1));
}

int pb_quotient(pb_ctx_t* ctx, const pb_air_t* a, const uint32_t* d_lde, size_t log_n, uint32_t log_blowup, uint32_t shift,
                const uint32_t alpha[4], uint32_t* d_q) {
    if (!ctx || !a || !d_lde || !alpha || !d_q) return PB_ERR_INVALID_ARG;
    if (log_blowup != 1 || log_n < 1 || log_n > 26) return PB_ERR_UNSUPPORTED;
    int rc = upload_alpha_pows(ctx, a, h_e4_from_canon(alpha));
    if (rc) return rc;
    uint32_t sn, zinv0, zinv1;
    zh_inverses(log_n, h_to_m(shift), &sn, &zinv0, &zinv1);
    const size_t m = (size_t)2 << log_n;
    if (a->jit_ok) {
        if (a->jit.fns.size() > 1) { rc = ctx->ws_qraw.ensure(4 * m); if (rc) return rc; }
        rc = airjit::launch(a->jit, ctx->stream, d_lde, m, (int)log_n, a->d_alpha_pows.p, zinv0, zinv1, d_q, 1, ctx->ws_qraw.p);
        LAUNCHED(ctx);
        return rc;
    }
    air::quotient_kernel<<<(unsigned)((m + air::THREADS - 1) / air::THREADS), air::THREADS, 0, ctx->stream>>>(
        a->d_code.p, a->d_spans.p, a->n_constraints, a->d_pool.p, d_lde, (int)log_n, a->d_alpha_pows.p, zinv0, zinv1, d_q, 1);
    LAUNCHED(ctx);
    CK(cudaGetLastError());
    return 0;
}

static int constraint_fold_m(pb_ctx* ctx, const pb_air* a, const uint32_t* d_mat, size_t height, bb::E4 alpha_m, size_t extra, uint32_t* d_out);
int pb_constraint_fold(pb_ctx_t* ctx, const pb_air_t* a, const uint32_t* d_mat, size_t height, const uint32_t alpha[4], uint32_t* d_out) {
    if (!ctx || !a || !d_mat || !alpha || !d_out) return PB_ERR_INVALID_ARG;
    if (!height) return 0;
    return constraint_fold_m(ctx, a, d_mat, height, h_e4_from_canon(alpha), 0, d_out);
}
static int constraint_fold_m(pb_ctx* ctx, const pb_air* a, const uint32_t* d_mat, size_t height, bb::E4 alpha_m, size_t extra, uint32_t* d_out) {
    int rc = upload_alpha_pows(ctx, a, alpha_m, extra);
    if (rc) return rc;
    if (a->n_constraints == 0) { CK(cudaMemsetAsync(d_out, 0, 16 * height, ctx->stream)); return 0; }
    if (a->jit_ok) {
        if (a->jit.fns.size() > 1) { rc = ctx->ws_qraw.ensure(4 * height); if (rc) return rc; }
        rc = airjit::launch(a->jit, ctx->stream, d_mat, height, 0, a->d_alpha_pows.p, 0u, 0u, d_out, 0, ctx->ws_qraw.p);
        LAUNCHED(ctx);
        return rc;
    }
    air::constraint_fold_kernel<<<(unsigned)((height + air::THREADS - 1) / air::THREADS), air::THREADS, 0, ctx->stream>>>(
        a->d_code.p, a->d_spans.p, a->n_constraints, a->d_pool.p, d_mat, height, a->d_alpha_pows.p, d_out);
    LAUNCHED(ctx);
    CK(cudaGetLastError());
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
int pb_merkle_commit(pb_ctx_t* ctx, const uint32_t* const* d_mats, const size_t* widths, size_t n_mats, size_t log_h,
                     uint32_t* d_layers, uint32_t root_out[8]) {
    if (!ctx || !d_mats || !widths || !n_mats || !d_layers) return PB_ERR_INVALID_ARG;
    if (log_h > 30) return PB_ERR_UNSUPPORTED;
    const size_t h = (size_t)1 << log_h;
    std::vector<const uint32_t*> cols;
    for (size_t i = 0; i < n_mats; i++)
        for (size_t c = 0; c < widths[i]; c++) cols.push_back(d_mats[i] + c * h);
    int rc = leaf_hash_cols(ctx, cols, log_h, d_layers);
    if (rc) return rc;
    rc = merkle_upper(ctx, d_layers, log_h);
    if (rc) return rc;
    if (root_out) {
        uint32_t r[8];
        rc = read_root(ctx, d_layers, log_h, r);
        if (rc) return rc;
        for (int i = 0; i < 8; i++) root_out[i] = h_from_m(r[i]);
    }
    return 0;
}

int pb_merkle_commit_rows8(pb_ctx_t* ctx, const uint32_t* d_rows, size_t log_h, uint32_t* d_layers, uint32_t root_out[8]) {
    if (!ctx || !d_rows || !d_layers) return PB_ERR_INVALID_ARG;
    const size_t h = (size_t)1 << log_h;
    if (h <= LEAF_COOP)
        p2::leaf_hash_rows8_coop_kernel<<<(unsigned)((16 * h + 255) / 256), 256, 0, ctx->stream>>>(d_rows, h, d_layers);
    else
        p2::leaf_hash_rows8_kernel<<<(unsigned)((h + 255) / 256), 256, 0, ctx->stream>>>(reinterpret_cast<const uint4*>(d_rows), h, d_layers);
    LAUNCHED(ctx);
    int rc = merkle_upper(ctx, d_layers, log_h);
    if (rc) return rc;
    if (root_out) {
        uint32_t r[8];
        rc = read_root(ctx, d_layers, log_h, r);
        if (rc) return rc;
        for (int i = 0; i < 8; i++) root_out[i] = h_from_m(r[i]);
    }
    return 0;
}

int pb_poseidon2_permute(pb_ctx_t* ctx, uint32_t* d_states, size_t n, int reps) {
    if (!ctx || !d_states) return PB_ERR_INVALID_ARG;
    if (!n) return 0;
    p2::permute_states_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d_states, n, reps);
    LAUNCHED(ctx);
    CK(cudaGetLastError());
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// outputs [j0, j0 + n_out) of the folded codeword only when n_out != 0 (d_in / d_out then point at that block: inputs 2*j0.., outputs j0..)
static int fri_fold_m(pb_ctx* ctx, const uint32_t* d_in, size_t log_len, uint32_t shift_m, bb::E4 beta_m, uint32_t* d_out, size_t j0 = 0,
                      size_t n_out = 0) {
    int rc = get_fold_table(ctx, (int)log_len);
    if (rc) return rc;
    const size_t half = n_out ? n_out : (size_t)1 << (log_len - 1);
    const uint32_t two_inv = bb::inv(h_to_m(2));
    const uint32_t c = bb::mul(two_inv, bb::inv(shift_m));          // (2*shift)^-1
    bb::E4 beta_c = bb::e4_scale(beta_m, c);
    // table prefix property: w_L^{-bitrev_{logL-1}(j)} for a shorter layer is the prefix of the longer layer's table
    fri::fold_kernel<<<(unsigned)((half + 255) / 256), 256, 0, ctx->stream>>>(reinterpret_cast<const uint4*>(d_in),
                                                                              reinterpret_cast<uint4*>(d_out), half, ctx->d_fold_tab + j0,
                                                                              beta_c, two_inv);
    LAUNCHED(ctx);
    CK(cudaGetLastError());
    return 0;
}

int pb_fri_fold(pb_ctx_t* ctx, const uint32_t* d_in, size_t log_len, uint32_t shift, const uint32_t beta[4], uint32_t* d_out) {
    if (!ctx || !d_in || !d_out || !beta) return PB_ERR_INVALID_ARG;
    if (log_len < 1 || log_len > 27 || shift == 0 || shift >= bb::P) return PB_ERR_UNSUPPORTED;
    return fri_fold_m(ctx, d_in, log_len, h_to_m(shift), h_e4_from_canon(beta), d_out);
}

// FRI commit phase, device-driven: from layer `layer0`, whose codeword of length 2^log_len0 is at ws_fri_words + word_off[layer0] and
// whose tree goes to ws_fri_trees + tree_off[layer0], the codeword is committed and folded down to length 2 without a host round trip
// per layer (p2::fri_challenge_kernel keeps the duplex state on the device and hands the challenge to the fold through memory).  Layer
// codewords / trees stay in ws_fri_words / ws_fri_trees, which the caller has sized, at word_off / tree_off for the query phase.
// inject (optional, [32]): inject[h] is added to the folded codeword when it reaches length 2^h (multi-chip segments).
// Afterwards ONE read-back of (roots, challenges, final values) and the host replays the transcript: `ch` advances exactly as if
// it had driven the phase, and any difference from what the device sampled is PB_ERR_INTERNAL.
static int fri_commit_phase(pb_ctx* ctx, Challenger& ch, uint32_t layer0, size_t log_len0, uint32_t* const* inject, size_t* word_off, size_t* tree_off,
                            uint32_t* n_layers, uint32_t fri_roots[32][8], uint32_t fri_betas[32][4], uint32_t fin_m[8], cudaEvent_t after_last_kernel) {
    cudaStream_t st = ctx->stream;
    int rc;
    if (ch.n_in != 0) return PB_ERR_INTERNAL;              // the phase starts right after a sampled challenge: no pending input
    if ((rc = ctx->ws_fri_ch.ensure(16))) return rc;
    if ((rc = ctx->ws_fri_log.ensure(32 * 12))) return rc;
    if ((rc = get_fold_table(ctx, (int)log_len0))) return rc;
    uint32_t* d_sponge = ctx->ws_fri_ch.p;
    CK(cudaMemcpyAsync(d_sponge, ch.sponge, 64, cudaMemcpyHostToDevice, st));    // pageable source: staged before the call returns
    size_t log_len = log_len0, woff = word_off[layer0], toff = tree_off[layer0];
    uint32_t* f = ctx->ws_fri_words.p + woff;
    uint32_t shift_m = h_to_m(bb::GEN), layer = layer0;
    for (uint32_t l = 0; l < layer0; l++) shift_m = bb::mul(shift_m, shift_m);
    const uint32_t two_inv = bb::inv(h_to_m(2));
    while (log_len > 1) {
        uint32_t* tree = ctx->ws_fri_trees.p + toff;
        word_off[layer] = woff;
        tree_off[layer] = toff;
        if ((rc = pb_merkle_commit_rows8(ctx, f, log_len - 1, tree, nullptr))) return rc;
        uint32_t* lg = ctx->ws_fri_log.p + 12 * layer;
        p2::fri_challenge_kernel<<<1, 32, 0, st>>>(d_sponge, tree + 8 * (((size_t)2 << (log_len - 1)) - 2), lg);
        uint32_t* g = f + ((size_t)4 << log_len);
        const size_t half = (size_t)1 << (log_len - 1);
        fri::fold_dev_beta_kernel<<<(unsigned)((half + 255) / 256), 256, 0, st>>>(reinterpret_cast<const uint4*>(f), reinterpret_cast<uint4*>(g), half, ctx->d_fold_tab,
                                                                                lg + 8, bb::mul(two_inv, bb::inv(shift_m)), two_inv);
        ctx->launches += 2;
        woff += (size_t)4 << log_len;
        toff += 8 * (((size_t)2 << (log_len - 1)) - 1);
        f = g;
        shift_m = bb::mul(shift_m, shift_m);
        log_len--;
        layer++;
        if (inject && log_len > 1 && inject[log_len]) {
            const size_t nw = (size_t)4 << log_len;
            fri::add_words_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, st>>>(f, inject[log_len], nw);
            LAUNCHED(ctx);
        }
    }
    CK(cudaGetLastError());
    uint32_t log_h[32 * 12];
    CK(cudaMemcpyAsync(fin_m, f, 32, cudaMemcpyDeviceToHost, st));
    if (layer > layer0) CK(cudaMemcpyAsync(log_h + 12 * layer0, ctx->ws_fri_log.p + 12 * layer0, 48 * (size_t)(layer - layer0), cudaMemcpyDeviceToHost, st));
    if (after_last_kernel) CK(cudaEventRecord(after_last_kernel, st));
    CK(cudaStreamSynchronize(st));
    for (uint32_t l = layer0; l < layer; l++) {
        ch.observe(log_h + 12 * l, 8);
        const bb::E4 beta = ch.sample_ext();
        if (memcmp(beta.c, log_h + 12 * l + 8, 16) != 0) return PB_ERR_INTERNAL;
        for (int i = 0; i < 8; i++) fri_roots[l][i] = h_from_m(log_h[12 * l + i]);
        for (int i = 0; i < 4; i++) fri_betas[l][i] = h_from_m(beta.c[i]);
    }
    *n_layers = layer;
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
static int eval_weighted_m(pb_ctx* ctx, const uint32_t* d_mat, size_t N, size_t width, bb::E4 pref, uint32_t* d_ys);
// openings: y_k = f_k(zeta) for columns given as evaluations over shift*H (natural order); d_ys: [width][4] Montgomery
static int eval_at_point_m(pb_ctx* ctx, const uint32_t* d_mat, size_t log_n, size_t width, uint32_t shift_m, bb::E4 zeta_m, uint32_t* d_ys) {
    const size_t N = (size_t)1 << log_n;
    if (width == 0) return 0;
    int rc = ctx->ws_w.ensure(N);
    if (rc) return rc;
    // f(zeta) = g(zeta/shift) with g's evaluations over H:  g(z) = (z^N - 1)/N * sum_i g_i * w^i / (z - w^i)
    const bb::E4 z = bb::e4_scale(zeta_m, bb::inv(shift_m));
    deep::bary_weights_kernel<<<(unsigned)((N + 255) / 256), 256, 0, ctx->stream>>>(ctx->ws_w.p, (int)log_n, h_root_of_unity_m((int)log_n), z);
    LAUNCHED(ctx);
    bb::E4 zn = z;
    for (size_t i = 0; i < log_n; i++) zn = bb::e4_mul(zn, zn);
    zn.c[0] = bb::sub(zn.c[0], bb::R1);
    const bb::E4 pref = bb::e4_scale(zn, bb::inv(h_to_m((uint32_t)(N % bb::P))));
    return eval_weighted_m(ctx, d_mat, N, width, pref, d_ys);
}

// y_k = pref * sum_i mat[k][i] * ws_w[i]
static int eval_weighted_m(pb_ctx* ctx, const uint32_t* d_mat, size_t N, size_t width, bb::E4 pref, uint32_t* d_ys) {
    const uint32_t rows_per_cta = (uint32_t)std::max<size_t>(deep::EV_THREADS, std::min<size_t>(N, (size_t)1 << 15));
    const uint32_t splits = (uint32_t)((N + rows_per_cta - 1) / rows_per_cta);
    RC(ctx->ws_part.ensure(width * splits));
    dim3 grid((unsigned)((width + deep::EV_COLS - 1) / deep::EV_COLS), splits);
    deep::eval_partial_kernel<<<grid, deep::EV_THREADS, 0, ctx->stream>>>(d_mat, N, (uint32_t)width, ctx->ws_w.p, ctx->ws_part.p, rows_per_cta);
    LAUNCHED(ctx);
    deep::eval_finalize_kernel<<<(unsigned)((width + 127) / 128), 128, 0, ctx->stream>>>(ctx->ws_part.p, (uint32_t)width, splits, pref,
                                                                                        reinterpret_cast<uint4*>(d_ys));
    LAUNCHED(ctx);
    CK(cudaGetLastError());
    return 0;
}

// reduced opening over shift*H' (bit-reversed rows).  `cols[j]` is opened at point zs[grp[j]]; e[j] is its position in the order in
// which the opened values are observed: its gamma exponent and the index of its value in ys_m (host, [..][4] Montgomery).  Rows
// [row0, row0 + n_rows) of the domain only when n_rows != 0 (cols[] then point at that row block).
// Columns of group 0 go in runs of equal stride; a run of group-1 columns that repeats a group-0 run (same base, stride, count: the
// permutation trace opened at zeta and at zeta*w) is attached to it, so those columns are read from HBM once.  One launch per
// DQ_MAX_SEGS runs: the first writes d_out, the later ones add to it.
static int deep_quotient_groups_m(pb_ctx* ctx, const std::vector<const uint32_t*>& cols, const std::vector<uint32_t>& grp, const std::vector<uint32_t>& e,
                                  const std::vector<bb::E4>& zs, size_t log_m, uint32_t shift_m, bb::E4 gamma_m, const uint32_t* ys_m, uint32_t* d_out,
                                  size_t row0 = 0, size_t n_rows = 0) {
    const size_t n_cols = cols.size(), M = n_rows ? n_rows : (size_t)1 << log_m;
    if (n_cols == 0 || grp.size() != n_cols || e.size() != n_cols || zs.empty()) return PB_ERR_INVALID_ARG;
    if (zs.size() > 2) return PB_ERR_UNSUPPORTED;
    std::vector<bb::E4> gp(n_cols);                   // gamma^e[j]: one product along a run of consecutive exponents
    std::vector<uint4> gs(n_cols);
    for (size_t j = 0; j < n_cols; j++) {
        if (grp[j] >= zs.size()) return PB_ERR_INVALID_ARG;
        if (j && e[j] == e[j - 1] + 1) {
            gp[j] = bb::e4_mul(gp[j - 1], gamma_m);
        } else {
            bb::E4 r = {{bb::R1, 0u, 0u, 0u}}, base = gamma_m;
            for (uint32_t x = e[j]; x; x >>= 1) { if (x & 1) r = bb::e4_mul(r, base); base = bb::e4_mul(base, base); }
            gp[j] = r;
        }
        gs[j] = make_uint4(h_from_m(gp[j].c[0]), h_from_m(gp[j].c[1]), h_from_m(gp[j].c[2]), h_from_m(gp[j].c[3]));
    }
    int rc = ctx->ws_gp.ensure(2 * n_cols);          // uint2 elements: one uint4 per column
    if (rc) return rc;
    CK(cudaMemcpyAsync(ctx->ws_gp.p, gs.data(), gs.size() * sizeof(uint4), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));           // gs is a host temporary
    struct Run { const uint32_t* base; size_t stride; uint32_t count, off, off2; };
    // A group-0 run must start where a group-1 run starts: two matrices that happen to be adjacent in memory (the main LDE of one chip
    // and the permutation LDE of the next) would otherwise merge into one run that no group-1 run mirrors.
    std::vector<const uint32_t*> second_starts;
    for (size_t j = 0; j < n_cols; j++)
        if (grp[j] == 1 && (j == 0 || grp[j - 1] != 1)) second_starts.push_back(cols[j]);
    auto starts_second = [&](const uint32_t* p) { return std::find(second_starts.begin(), second_starts.end(), p) != second_starts.end(); };
    std::vector<Run> runs;
    for (size_t j = 0; j < n_cols;) {
        if (grp[j] != 0) { j++; continue; }
        size_t k = j + 1;
        const ptrdiff_t st = (k < n_cols && grp[k] == 0) ? cols[k] - cols[j] : 0;
        while (k < n_cols && grp[k] == 0 && st > 0 && cols[k] - cols[k - 1] == st && !starts_second(cols[k])) k++;
        if (st <= 0) k = j + 1;
        runs.push_back(Run{cols[j], st > 0 ? (size_t)st : 0, (uint32_t)(k - j), (uint32_t)j, deep::DQ_NO_SECOND});
        j = k;
    }
    for (size_t j = 0; j < n_cols;) {           // group-1 runs must mirror a group-0 run
        if (grp[j] != 1) { j++; continue; }
        size_t k = j + 1;
        while (k < n_cols && grp[k] == 1) k++;
        bool placed = false;
        for (size_t sgi = 0; sgi < runs.size() && !placed; sgi++) {
            Run& r = runs[sgi];
            if (r.base == cols[j] && r.count == (uint32_t)(k - j) && r.off2 == deep::DQ_NO_SECOND && (k - j < 2 || (size_t)(cols[j + 1] - cols[j]) == r.stride)) {
                bool same = true;
                for (size_t t = j; t < k && same; t++) same = cols[t] == r.base + (t - j) * r.stride;
                if (same) { r.off2 = (uint32_t)j; placed = true; }
            }
        }
        if (!placed) return PB_ERR_UNSUPPORTED;
        j = k;
    }
    for (size_t r0 = 0; r0 < runs.size(); r0 += deep::DQ_MAX_SEGS) {
        deep::DeepSegs segs{};
        bb::E4 ysum[2] = {{{0u, 0u, 0u, 0u}}, {{0u, 0u, 0u, 0u}}};      // sum of gamma^e[j] y_j over this launch's columns, per point
        auto add_y = [&](int pt, size_t j) {
            bb::E4 y;
            memcpy(y.c, ys_m + 4 * (size_t)e[j], 16);
            ysum[pt] = bb::e4_add(ysum[pt], bb::e4_mul(gp[j], y));
        };
        bool two = false;
        for (size_t i = r0; i < std::min(runs.size(), r0 + deep::DQ_MAX_SEGS); i++) {
            const Run& r = runs[i];
            segs.base[segs.n] = r.base;
            segs.stride[segs.n] = r.stride;
            segs.count[segs.n] = r.count;
            segs.gp_off[segs.n] = r.off;
            segs.gp_off2[segs.n] = r.off2;
            segs.n++;
            for (uint32_t t = 0; t < r.count; t++) add_y(0, r.off + t);
            if (r.off2 != deep::DQ_NO_SECOND) {
                two = true;
                for (uint32_t t = 0; t < r.count; t++) add_y(1, r.off2 + t);
            }
        }
        deep::deep_quotient_kernel<<<(unsigned)((M + 255) / 256), 256, 0, ctx->stream>>>(segs, M, (int)log_m, row0, shift_m, h_root_of_unity_m((int)log_m),
                                                                                        reinterpret_cast<const uint4*>(ctx->ws_gp.p), ysum[0], zs[0],
                                                                                        two ? ysum[1] : ysum[0], two ? zs[1] : zs[0], two ? 1 : 0,
                                                                                        reinterpret_cast<uint4*>(d_out), r0 > 0 ? 1 : 0);
        LAUNCHED(ctx);
    }
    CK(cudaGetLastError());
    return 0;
}
// the same values for columns given as coefficients in bit-reversed slots, scaled as the inverse LDE passes leave them (the true
// coefficients): y_k = sum_j coef[k][j] * z^bitrev(j)
static int eval_coefs_at_point_m(pb_ctx* ctx, const uint32_t* d_coef, size_t log_n, size_t width, bb::E4 z, uint32_t* d_ys) {
    const size_t N = (size_t)1 << log_n;
    if (width == 0) return 0;
    RC(ctx->ws_w.ensure(N));
    deep::ZPow2 zp{};
    bb::E4 x = z;
    for (size_t k = 0; k < log_n; k++) { zp.p[k] = x; x = bb::e4_mul(x, x); }
    deep::monomial_weights_kernel<<<(unsigned)((N + 255) / 256), 256, 0, ctx->stream>>>(ctx->ws_w.p, (int)log_n, zp);
    LAUNCHED(ctx);
    return eval_weighted_m(ctx, d_coef, N, width, bb::E4{{bb::R1, 0u, 0u, 0u}}, d_ys);
}

int pb_eval_at_point(pb_ctx_t* ctx, const uint32_t* d_mat, size_t log_n, size_t width, uint32_t shift, const uint32_t zeta[4], uint32_t* d_ys) {
    if (!ctx || !d_mat || !zeta || !d_ys) return PB_ERR_INVALID_ARG;
    if (log_n < 1 || log_n > 27 || shift == 0 || shift >= bb::P) return PB_ERR_UNSUPPORTED;
    return eval_at_point_m(ctx, d_mat, log_n, width, h_to_m(shift), h_e4_from_canon(zeta), d_ys);
}

int pb_deep_quotient(pb_ctx_t* ctx, const uint32_t* const* d_mats, const size_t* widths, size_t n_mats, size_t log_m, uint32_t shift,
                     const uint32_t zeta[4], const uint32_t gamma[4], const uint32_t* d_ys, uint32_t* d_out) {
    if (!ctx || !d_mats || !widths || !n_mats || !zeta || !gamma || !d_ys || !d_out) return PB_ERR_INVALID_ARG;
    if (log_m < 1 || log_m > 27 || shift == 0 || shift >= bb::P) return PB_ERR_UNSUPPORTED;
    std::vector<const uint32_t*> cols;
    for (size_t i = 0; i < n_mats; i++)
        for (size_t c = 0; c < widths[i]; c++) cols.push_back(d_mats[i] + (c << log_m));
    std::vector<uint32_t> ys(4 * cols.size());
    CK(cudaMemcpyAsync(ys.data(), d_ys, 16 * cols.size(), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    std::vector<uint32_t> e(cols.size());
    for (size_t j = 0; j < e.size(); j++) e[j] = (uint32_t)j;
    return deep_quotient_groups_m(ctx, cols, std::vector<uint32_t>(cols.size(), 0u), e, {h_e4_from_canon(zeta)}, log_m, h_to_m(shift),
                                  h_e4_from_canon(gamma), ys.data(), d_out);
}

#include "segment.inl"
#include "chips.inl"
#include "verify.inl"
#include "proof_bytes.inl"

int pb_last_stage_ms(pb_ctx_t* ctx, float ms[PB_N_STAGES]) {
    if (!ctx || !ms) return PB_ERR_INVALID_ARG;
    memcpy(ms, ctx->stage_ms, sizeof ctx->stage_ms);
    return 0;
}

uint64_t pb_launch_count(pb_ctx_t* ctx) { return ctx ? ctx->launches : 0; }

int pb_leaf_kernel_profile(pb_ctx_t* ctx, int* n_launches, double* total_ms, double* total_bytes) {
    if (!ctx || !n_launches || !total_ms || !total_bytes) return PB_ERR_INVALID_ARG;
    CK(cudaStreamSynchronize(ctx->stream));
    *n_launches = ctx->kp_n; *total_ms = 0; *total_bytes = 0;
    for (int i = 0; i < ctx->kp_n; i++) {
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, ctx->kp_a[i], ctx->kp_b[i]));
        *total_ms += ms;
        *total_bytes += ctx->kp_bytes[i];
    }
    ctx->kp_n = 0;
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// stage 0: the reference's exact entry points (default stream, async, cudaGetLastError as the return value)
int _apc_tracegen(uint32_t* d_output, size_t H, const OriginalAir* d_airs, const Subst* d_subs, size_t n_subs, int num_apc_calls) {
    if (H == 0 || (H & (H - 1)) != 0) return PB_ERR_INVALID_ARG;     // the reference asserts a power-of-two height
    if (n_subs == 0) return 0;
    const unsigned per = tg::GATHER_THREADS * tg::GATHER_ROWS_PER_THREAD;
    const size_t max_y = 65535;
    for (size_t s0 = 0; s0 < n_subs; s0 += max_y) {
        dim3 grid((unsigned)((H + per - 1) / per), (unsigned)std::min(max_y, n_subs - s0));
        tg::apc_tracegen_kernel<<<grid, tg::GATHER_THREADS>>>(d_output, H, reinterpret_cast<const tg::OriginalAir*>(d_airs),
                                                              reinterpret_cast<const tg::Subst*>(d_subs) + s0, num_apc_calls);
    }
    return (int)cudaGetLastError();
}

int _apc_apply_derived_expr(uint32_t* d_output, size_t H, int num_apc_calls, const DerivedExprSpec* d_specs, size_t n_cols,
                            const uint32_t* d_bytecode) {
    if (n_cols == 0) return 0;
    tg::apc_apply_derived_expr_kernel<<<(unsigned)((H + 255) / 256), 256>>>(
        d_output, H, num_apc_calls, reinterpret_cast<const tg::DerivedExprSpec*>(d_specs), n_cols, d_bytecode);
    return (int)cudaGetLastError();
}

int _apc_apply_bus(const uint32_t* d_output, int num_apc_calls, const uint32_t* d_bytecode, size_t bytecode_len,
                   const DevInteraction* d_interactions, size_t n_interactions, const ExprSpan* d_arg_spans, size_t n_arg_spans,
                   uint32_t var_range_bus_id, uint32_t* d_var_hist, size_t var_num_bins, uint32_t tuple2_bus_id,
                   uint32_t* d_tuple2_hist, uint32_t sz0, uint32_t sz1, uint32_t bitwise_bus_id, uint32_t* d_bitwise_hist) {
    (void)bytecode_len; (void)n_arg_spans;
    if (num_apc_calls <= 0) return 0;
    tg::apc_apply_bus_kernel<<<(unsigned)((num_apc_calls + 127) / 128), 128>>>(
        d_output, num_apc_calls, d_bytecode, reinterpret_cast<const tg::DevInteraction*>(d_interactions), n_interactions,
        reinterpret_cast<const tg::ExprSpan*>(d_arg_spans), var_range_bus_id, d_var_hist, var_num_bins, tuple2_bus_id, d_tuple2_hist,
        sz0, sz1, bitwise_bus_id, d_bitwise_hist);
    return (int)cudaGetLastError();
}

// ---- stage 0, generated periphery kernel (bus_jit.cuh): same histograms as _apc_apply_bus, straight-line code per AIR ----
int pb_bus_compile(pb_ctx_t* ctx, const uint32_t* bc, size_t n_words, const ExprSpan* arg_spans, size_t n_arg_spans, const DevInteraction* ints, size_t n_ints,
                   uint32_t width, uint32_t var_range_bus_id, uint32_t tuple2_bus_id, uint32_t bitwise_bus_id, pb_bus_t** out) {
    // ctx == NULL && out == NULL: host-only check of the code generator (packs, generates, compiles for sm_90a; no device needed)
    const bool compile_only = !ctx && !out;
    if ((!compile_only && (!ctx || !out)) || (!bc && n_words) || (!arg_spans && n_arg_spans) || (!ints && n_ints)) return PB_ERR_INVALID_ARG;
    std::vector<uint32_t> code, pool;
    std::vector<air::Span> spans;
    std::vector<pb_expr_span_t> sp(n_arg_spans);
    for (size_t i = 0; i < n_arg_spans; i++) { sp[i].off = arg_spans[i].off; sp[i].len = arg_spans[i].len; }
    int rc = pack_program(bc, n_words, sp.data(), n_arg_spans, width, code, pool, spans);
    if (rc) return rc;
    std::vector<logup::Interaction> all;
    for (size_t i = 0; i < n_ints; i++) {
        if ((size_t)ints[i].args_index_off + ints[i].num_args + 1 > n_arg_spans) return PB_ERR_BAD_BYTECODE;
        all.push_back(logup::Interaction{ints[i].bus_id, ints[i].num_args, ints[i].args_index_off});
    }
    if (compile_only) return busjit::build(code, spans, pool, all, var_range_bus_id, tuple2_bus_id, bitwise_bus_id, nullptr, nullptr) ? PB_ERR_UNSUPPORTED : 0;
    pb_bus* b = new pb_bus();
    if (busjit::build(code, spans, pool, all, var_range_bus_id, tuple2_bus_id, bitwise_bus_id, &b->k, &b->grid_y)) { busjit::destroy(b->k); delete b; return PB_ERR_UNSUPPORTED; }
    *out = b;
    return 0;
}

int pb_bus_free(pb_bus_t* b) {
    if (!b) return 0;
    busjit::destroy(b->k);
    delete b;
    return 0;
}

int pb_bus_apply(pb_ctx_t* ctx, const pb_bus_t* b, const uint32_t* d_trace, size_t H, int num_apc_calls, uint32_t* d_var_hist, size_t var_num_bins,
                 uint32_t* d_tuple2_hist, uint32_t sz0, uint32_t sz1, uint32_t* d_bitwise_hist) {
    if (!ctx || !b || !d_trace) return PB_ERR_INVALID_ARG;
    if (num_apc_calls <= 0) return 0;
    unsigned long long h = H;
    uint32_t vb = (uint32_t)var_num_bins;
    for (size_t k = 0; k < b->k.fns.size(); k++) {
        void* args[] = {(void*)&d_trace, (void*)&h, (void*)&num_apc_calls, (void*)&d_var_hist, (void*)&vb, (void*)&d_tuple2_hist, (void*)&sz0, (void*)&sz1,
                        (void*)&d_bitwise_hist};
        CUresult rc = airjit::api().LaunchKernel(b->k.fns[k], (unsigned)((num_apc_calls + 127) / 128), b->grid_y[k], 1, 128, 1, 1, 0, (CUstream)ctx->stream, args, nullptr);
        if (rc != CUDA_SUCCESS) return 700 + (int)rc;
        LAUNCHED(ctx);
    }
    return 0;
}

#include "shard_api.inl"
#include "rowblock.inl"
#include "group.inl"

}  // extern "C"
