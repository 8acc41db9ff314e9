// Integer-pipe micro-benchmarks that decide which roof binds the BabyBear kernels (SURVEY.md §7 step 0, App. D).
// nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o microbench scripts/microbench.cu ; ./microbench
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "../powdr_b200/csrc/bb31.cuh"

constexpr int ITERS = 4096;
constexpr int ILP = 8;

template <int KIND>
__global__ void __launch_bounds__(256) k(uint32_t* out, uint32_t seed) {
    uint32_t x[ILP], y = seed | 1;
#pragma unroll
    for (int i = 0; i < ILP; i++) x[i] = (threadIdx.x * 2654435761u + i * 40503u + seed) % bb::P;
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int i = 0; i < ILP; i++) {
            if (KIND == 0) x[i] = x[i] * y + 12345u;                                   // IMAD
            if (KIND == 1) x[i] = x[i] + y + 7u;                                       // IADD3
            if (KIND == 2) x[i] = bb::add(x[i], y);                                    // modular add
            if (KIND == 3) x[i] = bb::mul(x[i], y);                                    // canonical Montgomery mul
            if (KIND == 4) x[i] = (uint32_t)bb::smul((int32_t)x[i], (int32_t)y);       // signed Montgomery mul
            if (KIND == 5) { uint64_t t = (uint64_t)x[i] * y + (((uint64_t)x[i]) << 32 | y); x[i] = (uint32_t)(t >> 32) ^ (uint32_t)t; }   // IMAD.WIDE w/ 64-bit addend
            if (KIND == 6) x[i] = __umulhi(x[i], y) + 3u;                              // IMAD.HI
            if (KIND == 7) { uint32_t t = bb::mul(x[(i + 1) % ILP], y); uint32_t a = x[i]; x[i] = bb::add(a, t); x[(i + 1) % ILP] = bb::sub(a, t); }  // butterfly
            if (KIND == 8) x[i] = bb::mul_lazy(x[i], y);                               // lazy mul (no correction)
            if (KIND == 10) { uint32_t t = x[i] + 0x87ffffffu; x[i] = t < x[i] ? t : x[i]; x[i] += (uint32_t)it; }   // VIADDMNMX + IADD
            if (KIND == 11) { x[i] = x[i] + x[(i + 1) % ILP] + y; y ^= x[i]; }                                        // IADD3 (3 regs) + LOP3
            if (KIND == 12) { x[i] = bb::mul_shoup(x[i], make_uint2(y, 0x12345677u)); }                               // Shoup constant product
            if (KIND == 13) { uint32_t a = x[i], b = x[(i + 1) % ILP]; x[i] = bb::add(a, b); x[(i + 1) % ILP] = bb::mul_shoup(a - b + bb::P, make_uint2(y, 0x12345677u)); }  // DIF butterfly
            if (KIND == 14) { uint64_t t = (uint64_t)x[i] * y; x[i] = (uint32_t)t + (uint32_t)(t >> 32); }             // IMAD.WIDE + IADD
            if (KIND == 9) { x[i] = bb::mul(x[i], y); x[i] = bb::add(x[i], y); x[i] = bb::add(x[i], x[(i+1)%ILP]); x[i] = bb::add(x[i], 5u);}  // 1 mul : 3 add mix
        }
    }
    uint32_t acc = 0;
#pragma unroll
    for (int i = 0; i < ILP; i++) acc ^= x[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

template <int KIND>
void run(const char* name, double ops_per_iter) {
    int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    int blocks = sms * 8;
    uint32_t* d; cudaMalloc(&d, blocks * 256 * 4);
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    k<KIND><<<blocks, 256>>>(d, 3);
    cudaDeviceSynchronize();
    float best = 1e9;
    for (int r = 0; r < 5; r++) {
        cudaEventRecord(a); k<KIND><<<blocks, 256>>>(d, 3 + r); cudaEventRecord(b); cudaEventSynchronize(b);
        float ms; cudaEventElapsedTime(&ms, a, b); if (ms < best) best = ms;
    }
    double total = (double)blocks * 256 * ITERS * ILP * ops_per_iter;
    int clk; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
    printf("%-34s %8.3f ms  %8.2f Gop/s  (%.1f op/clk/SM at %d MHz max)\n", name, best, total / best * 1e-6,
           total / (best * 1e-3) / sms / (clk * 1e3), clk / 1000);
    cudaFree(d);
}

int main() {
    run<0>("IMAD (32-bit mad)", 1);
    run<1>("IADD3", 1);
    run<6>("IMAD.HI", 1);
    run<5>("IMAD.WIDE + 64-bit addend", 1);
    run<2>("modular add (IADD3+VIADDMNMX)", 1);
    run<8>("Montgomery mul, lazy [0,2p)", 1);
    run<3>("Montgomery mul, canonical", 1);
    run<4>("Montgomery mul, signed", 1);
    run<7>("radix-2 butterfly (mul+add+sub)", 1);
    run<9>("1 mul + 3 add mix", 4);
    run<10>("VIADDMNMX + IADD", 1);
    run<11>("IADD3 + LOP3", 1);
    run<14>("IMAD.WIDE + IADD", 1);
    run<12>("Shoup constant product", 1);
    run<13>("DIF butterfly (Shoup, lazy diff)", 1);
    return 0;
}
