// vgpu_diff_witness: every cell of a caller's witness that differs from what Chip::generate_trace writes for the run the logs record.
// The expected witness comes from the device builder of vgpu_witness_device (witness.h), one chip at a time: a chip is built (this
// rank's run of it when split), compared, and freed before the next is built.  Each comparison (one per main trace, and one per
// preprocessed trace of chips 1 and 12) is the pattern of vgpu_check_failures:
//   1. count: one thread per row walks the row's columns in both matrices (column-major, so each load is coalesced over the warp);
//      a CTA keeps per-column counts and its lowest differing row in shared memory and stores its count; only a CTA that found a
//      difference touches the per-column counts and the chip's lowest row in global memory (a clean witness makes no global atomic);
//   2. when the trace differs somewhere and the list still has room: one scan of the CTA counts (vg_cta_scan), then a write pass in
//      which the CTAs whose differences start below the cap count each thread's differences again, scan them over the CTA and write
//      each thread's cells in column order at the CTA's prefix: the list is in (row, column) order whatever the schedule.
// Words are compared as stored (Montgomery); only the reported words are made canonical.
#include "ctx.h"
#include "devchip.h"
#include "lists.cuh"
#include "witness.h"
#include "host/vmlog.h"
#include <algorithm>
#include <tuple>

struct vgpu_vmlog;
extern "C" const VgVmLogs* vg_vmlog_view(const vgpu_vmlog* l);

namespace {

constexpr int DIFF_THREADS = 256, DIFF_WARPS = DIFF_THREADS / 32, DIFF_MAX_COLS = 128, DIFF_BATCH = 8;
static_assert(sizeof(vgpu_cell_diff) == 32, "vgpu_cell_diff is 8 words");

struct DParams {
    const uint32_t* have; uint64_t hcs;             // the caller's matrix, at local row 0 of the rows compared
    const uint32_t* want; uint64_t wcs;             // generate_trace's, at the same row
    uint64_t g0, n;                                 // global row of local row 0; rows compared
    uint32_t width, chip, trace;
    uint32_t* cta_count;                            // differing cells of each CTA
    unsigned long long* cols;                       // count pass: differing cells per column of this trace
    unsigned long long* first;                      // count pass: the chip's lowest differing global row (~0: none)
    const unsigned long long* cta_off;              // write pass: exclusive prefix sum of cta_count
    vgpu_cell_diff* out; uint64_t cap;              // write pass: entries [0, cap) of this comparison's list
};

// Calls f(column, have, want) for every differing cell of local row i, in column order; DIFF_BATCH columns of both matrices are loaded
// before any is compared.
template <class F>
__device__ __forceinline__ void row_diffs(const DParams& p, uint64_t i, F&& f) {
    const uint32_t* a = p.have + i;
    const uint32_t* b = p.want + i;
    for (uint32_t c0 = 0; c0 < p.width; c0 += DIFF_BATCH) {
        uint32_t x[DIFF_BATCH], y[DIFF_BATCH];
#pragma unroll
        for (int k = 0; k < DIFF_BATCH; k++) {
            const uint32_t c = c0 + k;
            x[k] = c < p.width ? __ldg(a + (uint64_t)c * p.hcs) : 0u;
            y[k] = c < p.width ? __ldg(b + (uint64_t)c * p.wcs) : 0u;
        }
#pragma unroll
        for (int k = 0; k < DIFF_BATCH; k++)
            if (x[k] != y[k]) f(c0 + k, x[k], y[k]);
    }
}

__global__ void __launch_bounds__(DIFF_THREADS) diff_count_kernel(const __grid_constant__ DParams p) {
    __shared__ uint32_t hist[DIFF_MAX_COLS];
    __shared__ uint32_t low;                                 // the CTA's lowest thread with a difference
    for (uint32_t t = threadIdx.x; t < p.width; t += blockDim.x) hist[t] = 0;
    if (threadIdx.x == 0) low = 0xffffffffu;
    __syncthreads();
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t mine = 0;
    if (i < p.n) row_diffs(p, i, [&](uint32_t c, uint32_t, uint32_t) { atomicAdd(&hist[c], 1u); mine++; });
    if (mine) atomicMin(&low, threadIdx.x);
    const uint32_t total = vg_cta_total<DIFF_WARPS>(mine);
    if (threadIdx.x == 0) p.cta_count[blockIdx.x] = total;
    if (!total) return;
    if (threadIdx.x == 0) atomicMin(p.first, (unsigned long long)(p.g0 + (uint64_t)blockIdx.x * blockDim.x + low));
    for (uint32_t t = threadIdx.x; t < p.width; t += blockDim.x)
        if (hist[t]) atomicAdd(p.cols + t, (unsigned long long)hist[t]);
}

__global__ void __launch_bounds__(DIFF_THREADS) diff_write_kernel(const __grid_constant__ DParams p) {
    const uint32_t total = p.cta_count[blockIdx.x];
    const unsigned long long base = p.cta_off[blockIdx.x];
    if (!total || base >= p.cap) return;                     // alike for the whole CTA
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t mine = 0;
    if (i < p.n) row_diffs(p, i, [&](uint32_t, uint32_t, uint32_t) { mine++; });
    // the thread's first entry: the differences of the CTA's lower threads
    uint32_t pos = vg_cta_exclusive<DIFF_WARPS>(mine);
    const uint32_t end = (uint32_t)min((unsigned long long)total, p.cap - base);
    if (!mine || pos >= end) return;
    vgpu_cell_diff* out = p.out + base;
    const int64_t row = (int64_t)(p.g0 + i);
    row_diffs(p, i, [&](uint32_t c, uint32_t h, uint32_t w) {
        if (pos < end) out[pos] = vgpu_cell_diff{p.chip, p.trace, c, row, bb::from_monty(h), bb::from_monty(w)};
        pos++;
    });
}

unsigned blocks_of(uint64_t n) { return (unsigned)((n + DIFF_THREADS - 1) / DIFF_THREADS); }

// the first per-column count of chip c's main trace (c < 14), of the program (c = 14) and of the range (c = 15) preprocessed trace
uint64_t column_base(int c) {
    uint64_t b = 0;
    for (int i = 0; i < std::min(c, VGPU_NUM_CHIPS); i++) b += vgpu_basic_machine_chip(i)->width;
    return b + (c > VGPU_NUM_CHIPS ? vgpu_basic_machine_chip(1)->preprocessed_width : 0);
}

}  // namespace

extern "C" uint64_t vgpu_witness_column_count(void) {
    return column_base(VGPU_NUM_CHIPS + 1) + vgpu_basic_machine_chip(12)->preprocessed_width;
}

// Per rank, u64 words [lowest differing row of each chip (14) | differing cells of each column]: all-gathered on a split context; the
// ranks' cell counts then size one block of entries per rank, which one more all-gather exchanges, and every rank merges the blocks.
extern "C" int32_t vgpu_diff_witness(vgpu_ctx* ctx, const vgpu_vmlog* log, const vgpu_dmat* const main[VGPU_NUM_CHIPS], const vgpu_dmat* const prep[2],
                                     uint64_t cap, vgpu_cell_diff* out, uint64_t* n_out, uint64_t* total,
                                     vgpu_diff_summary summary[VGPU_NUM_CHIPS], uint64_t* per_column_or_null) {
    if (!ctx) return -1;
    if (!log || !main || !prep) VG_FAIL(ctx, "diff_witness: null argument");
    if (!n_out || !total || !summary || (cap && !out)) VG_FAIL(ctx, "diff_witness: null output");
    VG_TRY(vg_check_machine(ctx, "diff_witness", main, prep));
    const VgVmLogs& L = *vg_vmlog_view(log);
    if (!L.n_cpu) VG_FAIL(ctx, "diff_witness: the run has no cycles");
    VG_TRY(vg_enter(ctx));
    const bool gather = vg_sharded(ctx);
    const uint32_t N = gather ? (uint32_t)ctx->comm_size : 1, me = gather ? (uint32_t)ctx->comm_rank : 0;
    const uint64_t ncol = vgpu_witness_column_count(), words = VGPU_NUM_CHIPS + ncol;
    VgWitnessBuilder wb(ctx, L);
    VG_TRY(wb.start());
    VgBuf counts(ctx), scal(ctx);
    VG_TRY(counts.alloc((size_t)N * words * 8));
    VG_TRY(scal.alloc(16));                                  // the scan's total (u64) and end (u32)
    unsigned long long* mine = counts.as<unsigned long long>() + (uint64_t)me * words;
    VG_CUDA(ctx, cudaMemsetAsync(mine, 0xff, VGPU_NUM_CHIPS * 8, ctx->stream));
    VG_CUDA(ctx, cudaMemsetAsync(mine + VGPU_NUM_CHIPS, 0, ncol * 8, ctx->stream));
    // this rank's first min(its cells, cap) entries: straight into out on a lone context, else gathered below
    std::vector<vgpu_cell_diff> local;
    uint64_t listed = 0;
    // Compares this rank's run of one trace of chip c with generate_trace's (cb: its first per-column count), then lists its
    // differences while the list has room.
    auto compare = [&](int c, uint32_t trace, const vgpu_dmat* have, const vgpu_dmat* want, const VgRun& run, uint64_t cb) -> int32_t {
        VG_TRY(vg_dmat_materialize(ctx, have));
        if (!run.count) return 0;
        const unsigned grid = blocks_of(run.count);
        VgBuf cta(ctx);
        VG_TRY(cta.alloc((size_t)grid * 4));
        DParams p{};
        p.have = vg_run_rows(have, run); p.hcs = have->col_stride;
        p.want = vg_run_rows(want, run); p.wcs = want->col_stride;
        p.g0 = run.begin; p.n = run.count;
        p.width = (uint32_t)have->gw; p.chip = (uint32_t)c; p.trace = trace;
        p.cta_count = cta.as<uint32_t>(); p.cols = mine + VGPU_NUM_CHIPS + cb; p.first = mine + c;
        {
            KScope ks(ctx, KC_CHECK, 8.0 * (double)run.count * p.width);
            diff_count_kernel<<<grid, DIFF_THREADS, 0, ctx->stream>>>(p);
            VG_LAUNCH_CHECK(ctx);
        }
        std::vector<unsigned long long> cc(p.width);
        VG_CUDA(ctx, cudaMemcpyAsync(cc.data(), p.cols, cc.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
        VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        uint64_t found = 0;
        for (unsigned long long x : cc) found += x;
        if (!found || listed >= cap) return 0;
        const uint64_t room = cap - listed, k = std::min(found, room);
        VgBuf off(ctx), ents(ctx);
        VG_TRY(off.alloc((size_t)grid * 8));
        VG_TRY(ents.alloc(k * sizeof(vgpu_cell_diff)));
        VG_TRY(vg_cta_scan(ctx, p.cta_count, grid, room, off.as<unsigned long long>(), scal.as<unsigned long long>(), (uint32_t*)(scal.as<unsigned long long>() + 1)));
        p.cta_off = off.as<unsigned long long>(); p.out = ents.as<vgpu_cell_diff>(); p.cap = room;
        {
            KScope ks(ctx, KC_CHECK, 0.0);
            diff_write_kernel<<<grid, DIFF_THREADS, 0, ctx->stream>>>(p);
            VG_LAUNCH_CHECK(ctx);
        }
        if (gather) local.resize(listed + k);
        VG_CUDA(ctx, cudaMemcpyAsync((gather ? local.data() : out) + listed, ents.p, k * sizeof(vgpu_cell_diff), cudaMemcpyDeviceToHost, ctx->stream));
        VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        listed += k;
        return 0;
    };
    for (int c = 0; c < VGPU_NUM_CHIPS; c++) {
        const uint64_t h = wb.height(c);
        if (h != main[c]->gh) continue;                      // reported in the summary, not compared
        VgRun run;
        if (!vg_reports_trace(ctx, h, &run)) continue;
        VgMat want;                                          // back to the cache once its comparison is done
        VG_TRY(wb.main(c, &want));
        VG_TRY(compare(c, VGPU_TRACE_MAIN, main[c], want.get(), run, column_base(c)));
        if (const vgpu_dmat* pr = vg_machine_prep(prep, c)) {
            const int w = c == 12;
            VG_TRY(wb.prep(w, &want));
            VG_TRY(compare(c, VGPU_TRACE_PREPROCESSED, pr, want.get(), run, column_base(VGPU_NUM_CHIPS + w)));
        }
    }
    if (gather) VG_TRY(vg_comm_allgather_inplace(ctx, counts.as<uint32_t>(), words * 2));
    std::vector<unsigned long long> hc((size_t)N * words);
    VG_CUDA(ctx, cudaMemcpyAsync(hc.data(), counts.p, hc.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    // the ranks' rows are disjoint (a chip every rank holds whole is compared by rank 0 alone): counts add, lowest rows take the min
    std::vector<uint64_t> per_rank(N, 0), cols(ncol, 0);
    unsigned long long first[VGPU_NUM_CHIPS];
    std::fill(first, first + VGPU_NUM_CHIPS, ~0ull);
    uint64_t all = 0;
    for (uint32_t r = 0; r < N; r++) {
        const unsigned long long* b = hc.data() + (size_t)r * words;
        for (int c = 0; c < VGPU_NUM_CHIPS; c++) first[c] = std::min(first[c], b[c]);
        for (uint64_t j = 0; j < ncol; j++) { cols[j] += b[VGPU_NUM_CHIPS + j]; per_rank[r] += b[VGPU_NUM_CHIPS + j]; }
        all += per_rank[r];
    }
    if (gather) {
        // each rank's list is ascending; the first cap of the union are among the ranks' first cap
        std::vector<vgpu_cell_diff> merged;
        for (uint64_t x : per_rank) merged.resize(merged.size() + std::min(x, cap));
        uint64_t gathered = 0;
        VG_TRY(vg_gather_lists(ctx, true, per_rank, cap, [&](vgpu_cell_diff* slot) -> int32_t {
            if (listed) VG_CUDA(ctx, cudaMemcpyAsync(slot, local.data(), listed * sizeof(vgpu_cell_diff), cudaMemcpyHostToDevice, ctx->stream));
            return 0;
        }, merged.data(), merged.size(), &gathered));
        std::sort(merged.begin(), merged.end(), [](const vgpu_cell_diff& a, const vgpu_cell_diff& b) {
            return std::tie(a.chip, a.trace, a.row, a.column) < std::tie(b.chip, b.trace, b.row, b.column);
        });
        std::copy(merged.begin(), merged.begin() + std::min<uint64_t>(merged.size(), cap), out);
    }
    *n_out = std::min(all, cap);
    *total = all;
    for (int c = 0; c < VGPU_NUM_CHIPS; c++) {
        vgpu_diff_summary& s = summary[c];
        s.height_have = main[c]->gh;
        s.height_want = wb.height(c);
        s.cells = 0;
        const uint64_t b = column_base(c), w = vgpu_basic_machine_chip(c)->width;
        for (uint64_t j = b; j < b + w; j++) s.cells += cols[j];
        if (c == 1 || c == 12) {
            const uint64_t pb = column_base(VGPU_NUM_CHIPS + (c == 12)), pw = vgpu_basic_machine_chip(c)->preprocessed_width;
            for (uint64_t j = pb; j < pb + pw; j++) s.cells += cols[j];
        }
        s.first_row = first[c] == ~0ull ? -1 : (int64_t)first[c];
    }
    if (per_column_or_null) std::copy(cols.begin(), cols.end(), per_column_or_null);
    return 0;
}
