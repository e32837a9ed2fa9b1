// The pieces of the calls that list what they find: vgpu_check_failures, vgpu_diff_witness and vgpu_check_buses.
#pragma once
#include "ctx.h"

// The sum of x over a CTA of WARPS warps, on every thread.
template <int WARPS>
__device__ __forceinline__ uint32_t vg_cta_total(uint32_t x) {
    __shared__ uint32_t warp_total[WARPS];
    x = __reduce_add_sync(0xffffffffu, x);
    if ((threadIdx.x & 31) == 0) warp_total[threadIdx.x >> 5] = x;
    __syncthreads();
    x = 0;
#pragma unroll
    for (int w = 0; w < WARPS; w++) x += warp_total[w];
    return x;
}

// The sum of x over the lower threads of a CTA of WARPS warps.
template <int WARPS>
__device__ __forceinline__ uint32_t vg_cta_exclusive(uint32_t x) {
    __shared__ uint32_t warp_total[WARPS];
    const uint32_t lane = threadIdx.x & 31;
    uint32_t s = x;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, s, d);
        if (lane >= (uint32_t)d) s += y;
    }
    if (lane == 31) warp_total[threadIdx.x >> 5] = s;
    __syncthreads();
    s -= x;
    for (uint32_t w = 0; w < (threadIdx.x >> 5); w++) s += warp_total[w];
    return s;
}

// check.cu — one CTA: off[j] = the exclusive prefix sum of the m per-CTA counts, *total their sum, *end = 1 + the last CTA with a
// count that starts below cap (0: none)
int32_t vg_cta_scan(vgpu_ctx* ctx, const uint32_t* count, uint32_t m, uint64_t cap, unsigned long long* off, unsigned long long* total, uint32_t* end);

// Every rank's list, in rank order, copied to host[0, *listed), *listed <= room.  n[r]: what rank r found (one count per rank when
// `gather`, else one), of which it lists the first min(n[r], cap).  write(slot) enqueues this rank's list at its block of the longest
// such list; when `gather` one all-gather exchanges the blocks.  Nothing is enqueued when no rank lists anything.
template <class T, class Write>
int32_t vg_gather_lists(vgpu_ctx* ctx, bool gather, const std::vector<uint64_t>& n, uint64_t cap, Write&& write, T* host, uint64_t room,
                        uint64_t* listed) {
    static_assert(sizeof(T) % 4 == 0, "lists are exchanged as words");
    uint64_t block = 0;
    for (uint64_t x : n) block = std::max(block, std::min(x, cap));
    *listed = 0;
    if (!block) return 0;
    VgBuf ents(ctx);
    VG_TRY(ents.alloc(n.size() * block * sizeof(T)));
    VG_TRY(write(ents.as<T>() + (gather ? (uint64_t)ctx->comm_rank : 0) * block));
    if (gather) VG_TRY(vg_comm_allgather_inplace(ctx, ents.as<uint32_t>(), block * sizeof(T) / 4));
    for (size_t r = 0; r < n.size(); r++) {
        const uint64_t k = std::min({n[r], cap, room - *listed});
        if (k) VG_CUDA(ctx, cudaMemcpyAsync(host + *listed, ents.as<T>() + r * block, k * sizeof(T), cudaMemcpyDeviceToHost, ctx->stream));
        *listed += k;
    }
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}
