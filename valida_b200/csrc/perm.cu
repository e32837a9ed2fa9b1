// K5 — LogUp permutation trace on the device: generate_permutation_trace (machine/src/chip.rs:121-208)
// with generate_rlc_elements (291-331), reduce_row (335-352) and
// batch_multiplicative_inverse_allowing_zero (util/src/lib.rs:21-43; zeros stay zero).
// The reference walks rows serially with a Vec per row; here:
//   (a) one thread per row builds every interaction's denominator  alpha_bus + sum_j beta^j * field_j
//       from the column-major main/preprocessed traces (coalesced column reads);
//   (b) the ext5 inversion is batched per thread over 8 rows spaced one grid apart (Montgomery trick,
//       one Frobenius-norm inversion per 8 elements), so every access stays coalesced;
//   (c) the signed running sum phi is a 3-kernel block scan over the five limbs (addition mod p is
//       limb-wise in F_p[X]/(X^5-2)).
// Output layout = RowMajorMatrix<Challenge>::flatten_to_base, column-major on device: column 5m+l.
#include "ctx.h"
#include "devchip.h"
#include <memory>

namespace {

using bb::E5;

__device__ __forceinline__ uint32_t pair_col_eval(const DevPairCol& pc, const uint32_t* main, uint64_t mcs, const uint32_t* prep, uint64_t pcs, uint64_t row) {
    uint32_t v = pc.constant;
    for (uint32_t t = 0; t < pc.n_terms; t++) {
        uint32_t x = pc.is_prep[t] ? __ldg(prep + (uint64_t)pc.column[t] * pcs + row) : __ldg(main + (uint64_t)pc.column[t] * mcs + row);
        v = bb::add(v, bb::mul(x, pc.weight[t]));
    }
    return v;
}

// The chip descriptor travels in the kernel parameters (constant bank): descriptor reads are uniform constant loads.
__global__ void __launch_bounds__(256) perm_denominators_kernel(const __grid_constant__ DevChip chip_, const uint32_t* __restrict__ main, uint64_t mcs,
                                                               const uint32_t* __restrict__ prep, uint64_t pcs, uint64_t h, uint32_t* __restrict__ perm, uint64_t qcs) {
    const DevChip* chip = &chip_;
    uint64_t n = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= h) return;
    for (uint32_t m = 0; m < chip->n_interactions; m++) {
        const DevInteraction& it = chip->interactions[m];
        bb::Lazy5 ra; ra.init();        // sum_j beta^j * field_j as raw 64-bit products, reduced once
        for (uint32_t j = 0; j < it.n_fields; j++) ra.fma_base(chip->betas[j], pair_col_eval(it.fields[j], main, mcs, prep, pcs, n));
        const E5 rlc = bb::e5_add(it.alpha, ra.value());
#pragma unroll
        for (int l = 0; l < 5; l++) perm[(uint64_t)(5 * m + l) * qcs + n] = rlc.c[l];
    }
}

constexpr int INV_BATCH = 8;
constexpr int INV_MINB = 5;   // resident CTAs per SM: the register cap of 8 spills (88-byte stack frame)
// In-place inverse of `count` ext5 columns (column group g uses base columns 5g..5g+4); zero stays zero.
__global__ void __launch_bounds__(128, INV_MINB) ext_batch_inverse_kernel(uint32_t* __restrict__ data, uint64_t cs, uint64_t h, uint32_t groups) {
    uint64_t stride = (h + INV_BATCH - 1) / INV_BATCH;
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= stride) return;
    for (uint32_t g = 0; g < groups; g++) {
        uint32_t* base = data + (uint64_t)(5 * g) * cs;
        E5 pref[INV_BATCH];
        E5 acc = bb::e5_one();
#pragma unroll
        for (int i = 0; i < INV_BATCH; i++) {
            uint64_t n = t + (uint64_t)i * stride;
            pref[i] = acc;
            if (n < h) {
                E5 d;
#pragma unroll
                for (int l = 0; l < 5; l++) d.c[l] = base[(uint64_t)l * cs + n];
                if (!bb::e5_is_zero(d)) acc = bb::e5_mul(acc, d);
            }
        }
        E5 inv = bb::e5_inv(acc);
#pragma unroll
        for (int i = INV_BATCH - 1; i >= 0; i--) {
            uint64_t n = t + (uint64_t)i * stride;
            if (n < h) {
                E5 d;
#pragma unroll
                for (int l = 0; l < 5; l++) d.c[l] = base[(uint64_t)l * cs + n];
                if (!bb::e5_is_zero(d)) {
                    E5 r = bb::e5_mul(inv, pref[i]);
                    inv = bb::e5_mul(inv, d);
#pragma unroll
                    for (int l = 0; l < 5; l++) base[(uint64_t)l * cs + n] = r.c[l];
                }
            }
        }
    }
}

// term[n] = sum_m (+-) q[n][m] * count_m(n), written into the phi columns (5k..5k+4)
__global__ void __launch_bounds__(256) perm_terms_kernel(const __grid_constant__ DevChip chip_, const uint32_t* __restrict__ main, uint64_t mcs,
                                                        const uint32_t* __restrict__ prep, uint64_t pcs, uint64_t h, uint32_t* __restrict__ perm, uint64_t qcs) {
    const DevChip* chip = &chip_;
    uint64_t n = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= h) return;
    uint32_t k = chip->n_interactions;
    E5 term = bb::e5_zero();
    for (uint32_t m = 0; m < k; m++) {
        const DevInteraction& it = chip->interactions[m];
        uint32_t mult = pair_col_eval(it.count, main, mcs, prep, pcs, n);
        E5 q;
#pragma unroll
        for (int l = 0; l < 5; l++) q.c[l] = perm[(uint64_t)(5 * m + l) * qcs + n];
        E5 t = bb::e5_mul_base(q, mult);
        term = it.is_send ? bb::e5_add(term, t) : bb::e5_sub(term, t);
    }
#pragma unroll
    for (int l = 0; l < 5; l++) perm[(uint64_t)(5 * k + l) * qcs + n] = term.c[l];
}

// Inclusive prefix sums mod p.  Each block scans SCAN_CHUNK consecutive elements of column blockIdx.y.
constexpr int SCAN_THREADS = 256, SCAN_PER_THREAD = 8, SCAN_CHUNK = SCAN_THREADS * SCAN_PER_THREAD;
__global__ void __launch_bounds__(SCAN_THREADS) scan_chunks_kernel(uint32_t* __restrict__ data, uint64_t cs, uint64_t n, uint32_t* __restrict__ chunk_sums, uint64_t sums_cs) {
    __shared__ uint32_t buf[SCAN_CHUNK];
    __shared__ uint32_t wsum[SCAN_THREADS / 32];
    uint32_t* col = data + (uint64_t)blockIdx.y * cs;
    uint64_t base = (uint64_t)blockIdx.x * SCAN_CHUNK;
    for (int i = threadIdx.x; i < SCAN_CHUNK; i += SCAN_THREADS) buf[i] = base + i < n ? col[base + i] : 0;
    __syncthreads();
    uint32_t loc[SCAN_PER_THREAD];
    uint32_t run = 0;
#pragma unroll
    for (int i = 0; i < SCAN_PER_THREAD; i++) { run = bb::add(run, buf[threadIdx.x * SCAN_PER_THREAD + i]); loc[i] = run; }
    // exclusive scan of per-thread totals across the block
    uint32_t v = run;
    int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint32_t u = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v = bb::add(v, u); }
    if (lane == 31) wsum[wid] = v;
    __syncthreads();
    if (wid == 0) {
        uint32_t w = lane < SCAN_THREADS / 32 ? wsum[lane] : 0;
#pragma unroll
        for (int o = 1; o < SCAN_THREADS / 32; o <<= 1) { uint32_t u = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w = bb::add(w, u); }
        if (lane < SCAN_THREADS / 32) wsum[lane] = w;
    }
    __syncthreads();
    uint32_t offset = bb::sub(v, run);                    // exclusive within warp
    if (wid > 0) offset = bb::add(offset, wsum[wid - 1]);
    __syncthreads();
#pragma unroll
    for (int i = 0; i < SCAN_PER_THREAD; i++) buf[threadIdx.x * SCAN_PER_THREAD + i] = bb::add(loc[i], offset);
    __syncthreads();
    for (int i = threadIdx.x; i < SCAN_CHUNK; i += SCAN_THREADS) if (base + i < n) col[base + i] = buf[i];
    if (threadIdx.x == SCAN_THREADS - 1 && chunk_sums) chunk_sums[(uint64_t)blockIdx.y * sums_cs + blockIdx.x] = bb::add(loc[SCAN_PER_THREAD - 1], offset);
}
// Serial-over-chunks inclusive scan of a short array by ONE block per column (used on the chunk sums).
__global__ void __launch_bounds__(1024) scan_small_kernel(uint32_t* __restrict__ data, uint64_t cs, uint64_t n) {
    __shared__ uint32_t wsum[32];
    __shared__ uint32_t carry_s;
    uint32_t* col = data + (uint64_t)blockIdx.y * cs;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (uint64_t base = 0; base < n; base += 1024) {
        uint64_t i = base + threadIdx.x;
        uint32_t x = i < n ? col[i] : 0, v = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { uint32_t u = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v = bb::add(v, u); }
        if (lane == 31) wsum[wid] = v;
        __syncthreads();
        if (wid == 0) {
            uint32_t w = wsum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { uint32_t u = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w = bb::add(w, u); }
            wsum[lane] = w;
        }
        __syncthreads();
        uint32_t r = bb::add(v, carry_s);
        if (wid > 0) r = bb::add(r, wsum[wid - 1]);
        if (i < n) col[i] = r;
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = r;
        __syncthreads();
    }
}
__global__ void __launch_bounds__(256) scan_add_offsets_kernel(uint32_t* __restrict__ data, uint64_t cs, uint64_t n, const uint32_t* __restrict__ chunk_sums, uint64_t sums_cs) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t chunk = i / SCAN_CHUNK;
    if (chunk == 0) return;
    uint32_t* col = data + (uint64_t)blockIdx.y * cs;
    col[i] = bb::add(col[i], chunk_sums[(uint64_t)blockIdx.y * sums_cs + chunk - 1]);
}

// totals[l] = last element of column l (the sum of this rank's rows after the local scan)
__global__ void perm_totals_kernel(const uint32_t* __restrict__ phi, uint64_t cs, uint64_t n, uint32_t* __restrict__ totals) {
    if (threadIdx.x < 5) totals[threadIdx.x] = phi[(uint64_t)threadIdx.x * cs + n - 1];
}
// split proof: phi of this rank's rows += the totals of the ranks before it (totals: [rank][limb])
__global__ void __launch_bounds__(256) scan_add_rank_offset_kernel(uint32_t* __restrict__ phi, uint64_t cs, uint64_t n, const uint32_t* __restrict__ totals, uint32_t rank) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t off = 0;
    for (uint32_t p = 0; p < rank; p++) off = bb::add(off, totals[p * 5 + blockIdx.y]);
    uint32_t* col = phi + (uint64_t)blockIdx.y * cs;
    col[i] = bb::add(col[i], off);
}

}  // namespace

// Inclusive prefix sum (mod p) of `ncols` columns of length n, in place.
int32_t vg_prefix_sum_columns(vgpu_ctx* ctx, uint32_t* data, uint64_t cs, uint64_t n, uint32_t ncols) {
    uint64_t chunks = (n + SCAN_CHUNK - 1) / SCAN_CHUNK;
    VgBuf sums(ctx);
    if (chunks > 1) VG_TRY(sums.alloc(chunks * ncols * 4));
    scan_chunks_kernel<<<dim3((unsigned)chunks, ncols), SCAN_THREADS, 0, ctx->stream>>>(data, cs, n, sums.as<uint32_t>(), chunks);
    VG_LAUNCH_CHECK(ctx);
    if (chunks > 1) {
        scan_small_kernel<<<dim3(1, ncols), 1024, 0, ctx->stream>>>(sums.as<uint32_t>(), chunks, chunks);
        VG_LAUNCH_CHECK(ctx);
        scan_add_offsets_kernel<<<dim3((unsigned)((n + 255) / 256), ncols), 256, 0, ctx->stream>>>(data, cs, n, sums.as<uint32_t>(), chunks);
        VG_LAUNCH_CHECK(ctx);
    }
    return 0;
}

int32_t vg_ext_batch_inverse(vgpu_ctx* ctx, uint32_t* data, uint64_t cs, uint64_t h, uint32_t groups) {
    if (!groups || !h) return 0;
    uint64_t stride = (h + INV_BATCH - 1) / INV_BATCH;
    ext_batch_inverse_kernel<<<(unsigned)((stride + 127) / 128), 128, 0, ctx->stream>>>(data, cs, h, groups);
    VG_LAUNCH_CHECK(ctx);
    return 0;
}

// generate_permutation_trace without a host synchronisation.  d_totals (device, 5 * vg_perm_totals_ranks() words, [rank][limb])
// receives the per-rank sums of the signed terms; the cumulative sum is their sum over the ranks (one rank unless the chip's
// rows are split).  Split proof, tall chip: `main` / `prep` are this rank's row shard (VG_ROWS) or the whole trace (VG_FULL, of which
// this rank's rows are used); the result is the row shard of the permutation trace.
int32_t vg_perm_trace_enqueue(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep_or_null,
                              const uint32_t challenges[15], vgpu_dmat** out_perm, uint32_t* d_totals, uint32_t* n_totals) {
    if (!chip || !main || !out_perm) VG_FAIL(ctx, "perm_trace: null argument");
    if (main->bitrev_rows) VG_FAIL(ctx, "perm_trace: main trace rows are stored bit-reversed");
    if (main->gw != chip->width) VG_FAIL(ctx, "perm_trace: main width %llu != chip width %u", (unsigned long long)main->gw, chip->width);
    if (chip->preprocessed_width && (!prep_or_null || prep_or_null->gw != chip->preprocessed_width || prep_or_null->gh != main->gh)) {
        // interactions of BasicMachine never read preprocessed columns, but the shape must still be coherent when given
        if (prep_or_null) VG_FAIL(ctx, "perm_trace: preprocessed trace shape mismatch");
    }
    VG_TRY(vg_dmat_materialize(ctx, main));
    VG_TRY(vg_dmat_materialize(ctx, prep_or_null));
    auto dchip_h = std::make_unique<DevChip>();
    VG_TRY(vg_build_devchip(ctx, chip, challenges, dchip_h.get()));
    const DevChip& dchip = *dchip_h;
    const VgRun run = vg_trace_run(ctx, main->gh);
    const bool split = run.split;
    if (!split && main->dist != VG_FULL) VG_FAIL(ctx, "perm_trace: the trace is a shard but too short to be split");
    const uint64_t h = run.count;                            // rows swept here
    uint32_t k = chip->n_interactions;
    VgMat perm;
    VG_TRY(vg_dmat_alloc_run(ctx, main->gh, 5 * (k + 1), split, false, &perm));
    const uint32_t* md = vg_run_rows(main, run);
    const uint32_t* pd = vg_run_rows(prep_or_null, run);
    uint64_t pcs = prep_or_null ? prep_or_null->col_stride : 0;
    unsigned blocks = (unsigned)((h + 255) / 256);
    uint32_t* phi = perm->d + (uint64_t)(5 * k) * perm->col_stride;
    {
        KScope ks(ctx, KC_PERM, 4.0 * (double)h * (chip->width + 5.0 * (k + 1)));
        if (k) {
            perm_denominators_kernel<<<blocks, 256, 0, ctx->stream>>>(dchip, md, main->col_stride, pd, pcs, h, perm->d, perm->col_stride);
            VG_LAUNCH_CHECK(ctx);
            VG_TRY(vg_ext_batch_inverse(ctx, perm->d, perm->col_stride, h, k));
        }
        perm_terms_kernel<<<blocks, 256, 0, ctx->stream>>>(dchip, md, main->col_stride, pd, pcs, h, perm->d, perm->col_stride);
        VG_LAUNCH_CHECK(ctx);
        VG_TRY(vg_prefix_sum_columns(ctx, phi, perm->col_stride, h, 5));
        perm_totals_kernel<<<1, 32, 0, ctx->stream>>>(phi, perm->col_stride, h, d_totals + (split ? 5 * ctx->comm_rank : 0));
        VG_LAUNCH_CHECK(ctx);
    }
    if (split) {
        VG_TRY(vg_comm_allgather_inplace(ctx, d_totals, 5));
        KScope ks2(ctx, KC_PERM, 0.0);
        scan_add_rank_offset_kernel<<<dim3(blocks, 5), 256, 0, ctx->stream>>>(phi, perm->col_stride, h, d_totals, (uint32_t)ctx->comm_rank);
        VG_LAUNCH_CHECK(ctx);
    }
    *n_totals = split ? (uint32_t)ctx->comm_size : 1;
    *out_perm = perm.release();
    return 0;
}
uint32_t vg_perm_totals_ranks(const vgpu_ctx* ctx) { return vg_sharded(ctx) ? (uint32_t)ctx->comm_size : 1; }

void vg_perm_totals_fold(const uint32_t* totals, uint32_t n, uint32_t out[5]) {
    for (int l = 0; l < 5; l++) {
        uint32_t a = 0;
        for (uint32_t r = 0; r < n; r++) a = bb::add(a, totals[r * 5 + l]);
        out[l] = a;
    }
}

extern "C" int32_t vgpu_perm_trace(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep_or_null,
                                   const uint32_t challenges[15], vgpu_dmat** out_perm, uint32_t cumulative_sum_out[5]) {
    VG_TRY(vg_enter(ctx));
    VgBuf d_tot(ctx);
    const uint32_t slots = vg_perm_totals_ranks(ctx);
    VG_TRY(d_tot.alloc(slots * 5 * 4));
    uint32_t nt = 0;
    VG_TRY(vg_perm_trace_enqueue(ctx, chip, main, prep_or_null, challenges, out_perm, d_tot.as<uint32_t>(), &nt));
    if (cumulative_sum_out) {
        uint32_t tot[16 * 5];
        cudaError_t e = cudaMemcpyAsync(tot, d_tot.p, nt * 5 * 4, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) VG_FAIL(ctx, "perm_trace: reading the cumulative sum failed: %s", cudaGetErrorString(e));
        vg_perm_totals_fold(tot, nt, cumulative_sum_out);
        for (int l = 0; l < 5; l++) cumulative_sum_out[l] = bb::from_monty(cumulative_sum_out[l]);
    }
    return 0;
}
