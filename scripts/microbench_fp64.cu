// Does the FP64 pipe of the H100 give the BabyBear kernels a second multiplier?  (sm_90a has full-rate FP64.)
// A modular product in doubles: h = a*b (rounded), l = fma(a,b,-h) (exact low part), q = rint(h/p), r = (h - q*p) + l: six
// DP instructions, result in the symmetric range |r| <= 0.51 p for any |a|,|b| < 2^31.5, so products chain with no correction.
// nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o microbench_fp64 scripts/microbench_fp64.cu ; ./microbench_fp64
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "../powdr_b200/csrc/bb31.cuh"

constexpr int ITERS = 2048;

__device__ __forceinline__ double fpmul(double a, double b) {
    const double P = 2013265921.0, PINV = 1.0 / 2013265921.0, MAGIC = 6755399441055744.0;
    const double h = a * b;
    const double l = fma(a, b, -h);
    const double q = fma(h, PINV, MAGIC) - MAGIC;
    const double t = fma(-q, P, h);
    return t + l;
}

// KIND 0: DFMA, 1: DMUL, 2: DADD, 3: fpmul chains, 4: mixed NI int (signed Montgomery) + NF fp chains
template <int KIND, int NI, int NF>
__global__ void __launch_bounds__(256) k(uint32_t* out, uint32_t seed) {
    double d[NF > 0 ? NF : 1];
    int32_t x[NI > 0 ? NI : 1];
    const double yd = (double)((seed * 2654435761u) % 1000003u) - 500000.0;
    const int32_t yi = (int32_t)((seed * 40503u) % bb::P);
#pragma unroll
    for (int i = 0; i < NF; i++) d[i] = (double)((threadIdx.x * 2654435761u + i * 40503u + seed) % bb::P) - 1006632960.0;
#pragma unroll
    for (int i = 0; i < NI; i++) x[i] = (int32_t)((threadIdx.x * 2246822519u + i * 40503u + seed) % bb::P);
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int i = 0; i < (NI > NF ? NI : NF); i++) {
            if (i < NF) {
                if (KIND == 0) d[i] = fma(d[i], 1.0000001, yd);
                if (KIND == 1) d[i] = d[i] * 1.0000001;
                if (KIND == 2) d[i] = d[i] + yd;
                if (KIND >= 3) d[i] = fpmul(d[i], yd);
            }
            if (i < NI) x[i] = bb::smul(x[i], yi);
        }
    }
    uint32_t acc = 0;
#pragma unroll
    for (int i = 0; i < NF; i++) acc ^= (uint32_t)__double2loint(d[i] + 6755399441055744.0);
#pragma unroll
    for (int i = 0; i < NI; i++) acc ^= (uint32_t)x[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

template <int KIND, int NI, int NF>
void run(const char* name) {
    int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    int blocks = sms * 8;
    uint32_t* d; cudaMalloc(&d, blocks * 256 * 4);
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    k<KIND, NI, NF><<<blocks, 256>>>(d, 3);
    cudaDeviceSynchronize();
    float best = 1e9;
    for (int r = 0; r < 5; r++) {
        cudaEventRecord(a); k<KIND, NI, NF><<<blocks, 256>>>(d, 3 + r); cudaEventRecord(b); cudaEventSynchronize(b);
        float ms; cudaEventElapsedTime(&ms, a, b); if (ms < best) best = ms;
    }
    double total = (double)blocks * 256 * ITERS * (NI + NF);
    int clk; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
    printf("%-44s %8.3f ms  %8.2f Gop/s  (%.2f op/clk/SM at %d MHz max)\n", name, best, total / best * 1e-6,
           total / (best * 1e-3) / sms / (clk * 1e3), clk / 1000);
    cudaFree(d);
}

// exactness check of fpmul against 64-bit integer arithmetic on random signed operands
__global__ void check(uint32_t seed, unsigned long long* bad) {
    uint64_t s = seed + 0x9E3779B97F4A7C15ull * (blockIdx.x * blockDim.x + threadIdx.x + 1);
    for (int it = 0; it < 4096; it++) {
        s ^= s << 13; s ^= s >> 7; s ^= s << 17;
        const int64_t a = (int64_t)(s % 4026531842ull) - 2013265921ll;            // (-p, p)
        s ^= s << 13; s ^= s >> 7; s ^= s << 17;
        const int64_t b = (int64_t)(s % 6039797763ull) - 2013265921ll;            // (-p, 2p)
        const double r = fpmul((double)a, (double)b);
        const int64_t ri = (int64_t)r;
        int64_t e = (a * b - ri) % 2013265921ll;
        if (e != 0 || ri > 1026765620ll || ri < -1026765620ll || (double)ri != r) atomicAdd(bad, 1ull);
    }
}

int main() {
    unsigned long long* bad; cudaMalloc(&bad, 8); cudaMemset(bad, 0, 8);
    check<<<1024, 256>>>(12345u, bad);
    unsigned long long hb = 0; cudaMemcpy(&hb, bad, 8, cudaMemcpyDeviceToHost);
    printf("fpmul exactness: %llu mismatches in %d products\n", hb, 1024 * 256 * 4096);
    run<0, 0, 8>("DFMA");
    run<1, 0, 8>("DMUL");
    run<2, 0, 8>("DADD");
    run<3, 0, 8>("fp64 modular product (6 DP instr)");
    run<4, 8, 0>("signed Montgomery product (int)");
    run<4, 4, 4>("mixed 4 int + 4 fp chains");
    run<4, 5, 3>("mixed 5 int + 3 fp chains");
    run<4, 6, 2>("mixed 6 int + 2 fp chains");
    run<4, 6, 4>("mixed 6 int + 4 fp chains");
    run<4, 8, 4>("mixed 8 int + 4 fp chains");
    return 0;
}
