// Issue-rate microbenchmark for the integer instruction mix of BabyBear arithmetic and Keccak on sm_90a.
// Each kernel runs ILP=8 independent dependency chains per thread, 1024 threads x 2 blocks per SM, 4096 iterations.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#define ITER 4096
#define ILP 8
template <int OP> __global__ void k(uint32_t* out, uint32_t seed, uint32_t c) {
    uint32_t a[ILP], b = seed ^ threadIdx.x;
#pragma unroll
    for (int i = 0; i < ILP; i++) a[i] = b * (i + 3) + 1;
    for (int it = 0; it < ITER; it++) {
#pragma unroll
        for (int i = 0; i < ILP; i++) {
            if (OP == 0) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(c), "r"(b));
            if (OP == 1) asm volatile("mad.hi.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(c), "r"(b));
            if (OP == 2) { uint64_t w; asm volatile("mul.wide.u32 %0, %1, %2;" : "=l"(w) : "r"(a[i]), "r"(c)); a[i] = (uint32_t)w ^ (uint32_t)(w >> 32); }
            if (OP == 3) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(c), "r"(b));
            if (OP == 4) asm volatile("shf.l.wrap.b32 %0, %0, %1, 7;" : "+r"(a[i]) : "r"(b));
            if (OP == 5) asm volatile("add.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(c));
            if (OP == 6) { uint32_t s = a[i] + c; a[i] = min(s, s - 0x78000001u); }
            if (OP == 7) {   // Montgomery product (WIDE + lo + HI + sub + min)
                uint64_t t = (uint64_t)a[i] * c; uint32_t m = (uint32_t)t * 0x88000001u;
                uint32_t u = (uint32_t)(t >> 32) - __umulhi(m, 0x78000001u); a[i] = min(u, u + 0x78000001u);
            }
            if (OP == 8) {   // Shoup product: q = hi(w' * y); r = w*y - q*p  (lo, lo, HI), then one conditional subtract
                uint32_t q = __umulhi(b, a[i]); uint32_t r = c * a[i] - q * 0x78000001u; a[i] = min(r, r - 0x78000001u);
            }
            if (OP == 9) asm volatile("mul.lo.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(c));
        }
    }
    uint32_t s = 0;
#pragma unroll
    for (int i = 0; i < ILP; i++) s ^= a[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
template <int OP> void run(const char* name, int per_iter_instr) {
    int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    const int blocks = 2 * sms;
    uint32_t* d; cudaMalloc(&d, blocks * 1024 * 4);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    k<OP><<<blocks, 1024>>>(d, 1, 0x12345671u);
    cudaEventRecord(e0);
    k<OP><<<blocks, 1024>>>(d, 2, 0x12345671u);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    double ops = (double)blocks * 1024 * ITER * ILP;
    int clk; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
    printf("%-28s %8.3f ms  %7.2f Gop/s  = %6.2f lane-ops/clk/SM at %d MHz (%d instr/op)\n", name, ms, ops / ms / 1e6, ops / (ms * 1e-3) / sms / (clk * 1e3), clk / 1000, per_iter_instr);
    cudaFree(d);
}
int main() {
    run<0>("IMAD.lo (mad.lo)", 1); run<9>("IMUL.lo", 1); run<1>("IMAD.HI (mad.hi)", 1); run<2>("IMAD.WIDE + xor", 2); run<3>("LOP3", 1); run<4>("SHF", 1);
    run<5>("IADD", 1); run<6>("add mod p (IADD+VIADDMNMX)", 2); run<7>("Montgomery mul", 5); run<8>("Shoup mul", 5);
    return 0;
}
