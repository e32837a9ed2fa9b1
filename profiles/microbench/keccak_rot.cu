// Keccak-f throughput vs the number of rotations moved from SHF (INT ALU pipe) to multiply-adds (FMA pipe).
// Build one binary per mask:  nvcc -DKK_FMA_ROT_MASK=<mask>ull ...
#include <cstdio>
#include <cstdint>
#include "../../valida_b200/csrc/keccak.cuh"
__global__ void __launch_bounds__(128) k(uint32_t* out, uint32_t seed) {
    uint2 A[25];
#pragma unroll
    for (int i = 0; i < 25; i++) A[i] = make_uint2(seed * (i + 1) + threadIdx.x, blockIdx.x ^ (i * 77));
    for (int it = 0; it < 16; it++) kk::keccak_f(A);
    uint32_t s = 0;
#pragma unroll
    for (int i = 0; i < 25; i++) s ^= A[i].x ^ A[i].y;
    out[blockIdx.x * 128 + threadIdx.x] = s;
}
int main() {
    int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    const int blocks = sms * 64;
    uint32_t* d; cudaMalloc(&d, blocks * 128 * 4);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    k<<<blocks, 128>>>(d, 1);
    cudaEventRecord(e0);
    for (int r = 0; r < 5; r++) k<<<blocks, 128>>>(d, 2 + r);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    double perms = 5.0 * blocks * 128 * 16;
    uint32_t h; cudaMemcpy(&h, d, 4, cudaMemcpyDeviceToHost);
    printf("mask %016llx : %.3f ms, %.3f G Keccak-f/s (check %08x)\n", (unsigned long long)(KK_FMA_ROT_MASK), ms, perms / ms / 1e6, h);
    return 0;
}
