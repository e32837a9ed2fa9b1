// Probe for the multi-GPU data path: (1) does CUDA IPC work between two PROCESSES on this box (one rank per GPU,
// torchrun style), (2) what do kernel-issued peer stores / loads over NVLink sustain.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o p2p_probe p2p_probe.cu ; run with >= 2 GPUs visible.
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <unistd.h>
#include <sys/wait.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("FAIL %s: %s (line %d)\n", #x, cudaGetErrorString(e), __LINE__); fflush(stdout); exit(2); } } while (0)

__global__ void copy_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) dst[i] = src[i];
}
__global__ void copy4_kernel(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) dst[i] = src[i];
}

static float time_copy(const void* src, void* dst, size_t bytes, bool wide, int blocks) {
    cudaEvent_t a, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
    for (int w = 0; w < 2; w++) {
        if (wide) copy_kernel<<<blocks, 512>>>((const uint4*)src, (uint4*)dst, bytes / 16);
        else copy4_kernel<<<blocks, 512>>>((const uint32_t*)src, (uint32_t*)dst, bytes / 4);
    }
    CK(cudaDeviceSynchronize());
    CK(cudaEventRecord(a));
    const int reps = 5;
    for (int r = 0; r < reps; r++) {
        if (wide) copy_kernel<<<blocks, 512>>>((const uint4*)src, (uint4*)dst, bytes / 16);
        else copy4_kernel<<<blocks, 512>>>((const uint32_t*)src, (uint32_t*)dst, bytes / 4);
    }
    CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b));
    float ms = 0; CK(cudaEventElapsedTime(&ms, a, b));
    return ms / reps;
}

int main() {
    const size_t bytes = 1ull << 30;   // no CUDA call before the fork
    int p2c[2], c2p[2];
    if (pipe(p2c) || pipe(c2p)) return 1;
    pid_t pid = fork();
    if (pid == 0) {   // child: rank 1 on device 1, opens rank 0's allocation
        CK(cudaSetDevice(1));
        cudaIpcMemHandle_t h;
        if (read(p2c[0], &h, sizeof h) != (ssize_t)sizeof h) return 3;
        void* peer = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&peer, h, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) { printf("IPC open FAILED: %s\n", cudaGetErrorString(e)); fflush(stdout); char c = 'x'; (void)!write(c2p[1], &c, 1); return 0; }
        printf("IPC open ok\n");
        void* local = nullptr; CK(cudaMalloc(&local, bytes)); CK(cudaMemset(local, 0x5a, bytes));
        int sms; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 1));
        for (int blocks : {sms, 4 * sms, 16 * sms}) {
            float w16 = time_copy(local, peer, bytes, true, blocks), r16 = time_copy(peer, local, bytes, true, blocks);
            float w4 = time_copy(local, peer, bytes, false, blocks), r4 = time_copy(peer, local, bytes, false, blocks);
            printf("IPC blocks=%d: peer store 16B %.0f GB/s, peer load 16B %.0f GB/s, store 4B %.0f GB/s, load 4B %.0f GB/s\n", blocks,
                   bytes / w16 / 1e6, bytes / r16 / 1e6, bytes / w4 / 1e6, bytes / r4 / 1e6);
        }
        float l = time_copy(local, (char*)local + bytes / 2, bytes / 2, true, 2368);
        printf("local copy (read+write) %.0f GB/s\n", 2 * (bytes / 2) / l / 1e6);
        // check what rank 0 sees
        CK(cudaMemset(local, 0x11, 4096)); copy_kernel<<<1, 256>>>((const uint4*)local, (uint4*)peer, 256); CK(cudaDeviceSynchronize());
        CK(cudaIpcCloseMemHandle(peer));
        fflush(stdout);
        char c = 'k'; (void)!write(c2p[1], &c, 1);
        return 0;
    }
    int n = 0; CK(cudaGetDeviceCount(&n));
    printf("devices: %d\n", n);
    CK(cudaSetDevice(0));
    void* buf = nullptr; CK(cudaMalloc(&buf, bytes)); CK(cudaMemset(buf, 0, bytes));
    cudaIpcMemHandle_t h; CK(cudaIpcGetMemHandle(&h, buf));
    if (write(p2c[1], &h, sizeof h) != (ssize_t)sizeof h) return 1;
    char c = 0; (void)!read(c2p[0], &c, 1);
    int st = 0; waitpid(pid, &st, 0);
    if (c == 'k') { uint32_t v = 0; CK(cudaMemcpy(&v, buf, 4, cudaMemcpyDeviceToHost)); printf("rank 0 sees 0x%08x (expect 0x11111111)\n", v); }
    // in-process peer access (thread-per-GPU mode)
    int can = 0; CK(cudaDeviceCanAccessPeer(&can, 0, 1));
    printf("in-process canAccessPeer(0,1) = %d\n", can);
    if (can) {
        CK(cudaDeviceEnablePeerAccess(1, 0));
        CK(cudaSetDevice(1)); void* b1 = nullptr; CK(cudaMalloc(&b1, bytes)); CK(cudaMemset(b1, 1, bytes)); CK(cudaDeviceSynchronize());
        CK(cudaSetDevice(0));
        float w16 = time_copy(buf, b1, bytes, true, 2368), r16 = time_copy(b1, buf, bytes, true, 2368);
        printf("in-process: peer store %.0f GB/s, peer load %.0f GB/s\n", bytes / w16 / 1e6, bytes / r16 / 1e6);
    }
    return 0;
}
