// vgpu_free_cells: every main-trace cell of a chip's witness that no check pins.  Cell (r, c) is free when
//   1. no Air::eval assertion depends on it: every assertion keeps its value when the cell changes, on row r (the cell as L(c)) and
//      on row (r - 1) mod h with that row's own selectors (the cell as N(c)); on a one-row chip the cell is both L(c) and N(c) of the
//      one evaluation.  Every constraint has degree <= 3 (log_quotient_degree = 1), so its value is a polynomial of degree <= 3 in the
//      cell, constant exactly when it is equal at cell + 0, + 1, + 2 and + 3: one evaluation of the AIR text with 4-lane values (F4)
//      decides it exactly;
//   2. no bus event depends on it: no interaction's count gives the column a non-zero summed weight, and on a row where an
//      interaction's count is not 0 none of its fields does.  (Two events of one row could only cancel on one bus with opposite
//      signs; Shift32, the one chip that sends and receives on one bus, uses different opcodes unless its count is 0.)
// The LogUp constraints are left to 2: they see the main trace only through the events.  Preprocessed and permutation cells are not
// judged (the verifier fixes the first, the main trace and the challenges the second).
// Only the columns the AIR text reads on the local / next row (explain.cu's catalogue) are evaluated, and a column the buses or the
// local evaluation already pin is not evaluated again.
// Two kernels, one thread per row of the run, in the pattern of vgpu_check_failures: a mask pass counts each CTA's free cells and
// keeps per-column counts in shared memory (a CTA with nothing free touches no global memory); after vg_cta_scan, a write pass in the
// CTAs whose cells start below the cap recomputes the masks and writes each thread's cells in column order at its prefix, so the list
// is in (row, column) order.  A split chip's run needs the row before its first row and the row after its last: each rank packs its
// first and last main rows into a small block (check_copy_kernel) and one all-gather exchanges them (no peer pointers: a borrowed
// shard is caller memory).
#include "cells.cuh"
#include "lists.cuh"

namespace {

constexpr int FREE_THREADS = 128, FREE_WARPS = FREE_THREADS / 32, FREE_MAX_COLS = CELLS_MAX_COLS;
static_assert(sizeof(vgpu_free_cell) == 16, "vgpu_free_cell is 4 words");

struct LaneBuilder : VgLanes {
    bool dep;                                       // some assertion's value changed with the cell
    __device__ __forceinline__ void z(const V& x) { dep |= (x.v[1] != x.v[0]) | (x.v[2] != x.v[0]) | (x.v[3] != x.v[0]); }
};

struct MParams {
    const uint32_t* main; uint64_t mcs;             // local row 0 of the rows swept
    const uint32_t* prep; uint64_t pcs;             // null without a preprocessed trace
    const uint32_t* before; uint64_t bcs;           // the row before local row 0 ((g0 - 1) mod h)
    const uint32_t* after; uint64_t acs;            // the row after local row n - 1
    uint64_t g0, n, h;                              // global row of local row 0; rows swept; global height
    uint64_t air_l[2], air_n[2];                    // columns the AIR text reads on the local / next row (bit c % 64 of word c / 64)
    uint64_t cols[2];                               // the chip's columns
    VgBusMasks bus;
    uint32_t k, width;
    uint32_t* cta_count;                            // free cells of each CTA
    unsigned long long* per_col;                    // mask pass: free cells per column
    const unsigned long long* cta_off;              // write pass: exclusive prefix sum of cta_count
    vgpu_free_cell* out; uint64_t cap;              // write pass: entries [0, cap) of this rank's list
};

// The free columns of local row i: f0 (columns 0..63), f1 (64..127).
template <int CHIP>
__device__ __forceinline__ void free_mask(const MParams& p, uint64_t i, uint64_t& f0, uint64_t& f1) {
    const uint32_t* row = p.main + i;
    uint64_t pin0 = p.bus.count_cols[0], pin1 = p.bus.count_cols[1];
    for (uint32_t m = 0; m < p.k; m++)
        if (logup::pair_col(p.bus.count[m], row, p.mcs, p.prep ? p.prep + i : nullptr, p.pcs) != 0) {
            pin0 |= p.bus.fields[m][0];
            pin1 |= p.bus.fields[m][1];
        }
    const uint64_t g = p.g0 + i, one_row = p.h == 1;
    LaneBuilder b;
    // jobs 0, 1: the row's own evaluation, the cell as L(c) (and as N(c) on a one-row chip); jobs 2, 3: the previous row's, the cell
    // as N(c).  A column already pinned is skipped.
#pragma unroll 1
    for (int w = 0; w < 4; w++) {
        const bool prev = w >= 2;
        if (prev && one_row) break;
        const uint64_t reads = prev ? p.air_n[w & 1] : (one_row ? p.air_l[w] | p.air_n[w] : p.air_l[w]);
        uint64_t todo = reads & ~((w & 1) ? pin1 : pin0);
        const uint64_t ge = prev ? (g ? g : p.h) - 1 : g;          // the evaluated row
        const bool is_last = ge + 1 == p.h;
        b.first = air::Lift<F4>::from_monty_word(ge == 0 ? bb::R1 : 0u);
        b.last = air::Lift<F4>::from_monty_word(is_last ? bb::R1 : 0u);
        b.trans = air::Lift<F4>::from_monty_word(is_last ? 0u : bb::R1);
        if (prev) {
            b.lrow = i ? row - 1 : p.before; b.lcs = i ? p.mcs : p.bcs;
            b.nrow = row; b.ncs = p.mcs;
        } else {
            b.lrow = row; b.lcs = p.mcs;
            b.nrow = i + 1 < p.n ? row + 1 : p.after; b.ncs = i + 1 < p.n ? p.mcs : p.acs;
        }
        while (todo) {
            const int bit = __ffsll((long long)todo) - 1;
            todo &= todo - 1;
            const int c = 64 * (w & 1) + bit;
            b.tl = prev ? -1 : c;
            b.tn = prev || one_row ? c : -1;
            b.dep = false;
            air::eval_chip<CHIP>(b);
            if (b.dep) {
                if (w & 1) pin1 |= 1ull << bit;
                else pin0 |= 1ull << bit;
            }
        }
    }
    f0 = p.cols[0] & ~pin0;
    f1 = p.cols[1] & ~pin1;
}

template <int CHIP>
__global__ void __launch_bounds__(FREE_THREADS, 1) free_mask_kernel(const __grid_constant__ MParams p) {
    __shared__ uint32_t hist[FREE_MAX_COLS];
    for (uint32_t t = threadIdx.x; t < p.width; t += blockDim.x) hist[t] = 0;
    __syncthreads();
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t f0 = 0, f1 = 0;
    if (i < p.n) free_mask<CHIP>(p, i, f0, f1);
    // one shared atomic per warp and column with a free cell
    const uint64_t any = __reduce_or_sync(0xffffffffu, (uint32_t)(f0 | (f0 >> 32))) | __reduce_or_sync(0xffffffffu, (uint32_t)(f1 | (f1 >> 32)));
    if (any)
        for (uint32_t c = 0; c < p.width; c++) {
            const unsigned v = __ballot_sync(0xffffffffu, ((c < 64 ? f0 : f1) >> (c & 63)) & 1);
            if (v && (threadIdx.x & 31) == 0) atomicAdd(&hist[c], (unsigned)__popc(v));
        }
    const uint32_t total = vg_cta_total<FREE_WARPS>((uint32_t)(__popcll(f0) + __popcll(f1)));
    if (!total) return;
    if (threadIdx.x == 0) p.cta_count[blockIdx.x] = total;
    for (uint32_t t = threadIdx.x; t < p.width; t += blockDim.x)
        if (hist[t]) atomicAdd(p.per_col + t, (unsigned long long)hist[t]);
}

template <int CHIP>
__global__ void __launch_bounds__(FREE_THREADS, 1) free_write_kernel(const __grid_constant__ MParams p) {
    const uint32_t total = p.cta_count[blockIdx.x];
    const unsigned long long base = p.cta_off[blockIdx.x];
    if (!total || base >= p.cap) return;                     // alike for the whole CTA
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t f0 = 0, f1 = 0;
    if (i < p.n) free_mask<CHIP>(p, i, f0, f1);
    const uint32_t mine = (uint32_t)(__popcll(f0) + __popcll(f1));
    // the thread's first entry: the free cells of the CTA's lower threads
    uint32_t pos = vg_cta_exclusive<FREE_WARPS>(mine);
    const uint32_t end = (uint32_t)min((unsigned long long)total, p.cap - base);
    if (!mine || pos >= end) return;
    vgpu_free_cell* out = p.out + base;
    const int64_t row = (int64_t)(p.g0 + i);
    for (int w = 0; w < 2; w++)
        for (uint64_t m = w ? f1 : f0; m && pos < end; m &= m - 1, pos++) {
            out[pos].row = row;
            out[pos].column = 64 * w + (__ffsll((long long)m) - 1);
        }
}

}  // namespace

extern "C" int32_t vgpu_free_cells(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep_or_null,
                                   uint64_t cap, vgpu_free_cell* out, uint64_t* n_out, uint64_t* total, uint64_t* rows_per_column) {
    if (!ctx) return -1;
    if (!n_out || !total || (cap && !out)) VG_FAIL(ctx, "free_cells: null output");
    if (!chip || !main) VG_FAIL(ctx, "free_cells: null argument");
    if (chip->n_interactions > VGPU_MAX_INTERACTIONS) VG_FAIL(ctx, "free_cells: %u interactions exceed %d", chip->n_interactions, VGPU_MAX_INTERACTIONS);
    if (chip->width > FREE_MAX_COLS) VG_FAIL(ctx, "free_cells: %u columns exceed %d", chip->width, FREE_MAX_COLS);
    VG_TRY(vg_check_shapes(ctx, chip, main, prep_or_null, nullptr, true));
    VG_TRY(vg_enter(ctx));
    VG_TRY(vg_dmat_materialize(ctx, main));
    VG_TRY(vg_dmat_materialize(ctx, prep_or_null));
    const uint64_t h = main->gh;
    const uint32_t w = chip->width;
    const VgRun run = vg_trace_run(ctx, h);
    const uint32_t N = run.split ? (uint32_t)ctx->comm_size : 1, me = run.split ? (uint32_t)ctx->comm_rank : 0;
    const uint32_t ctas = (uint32_t)((run.count + FREE_THREADS - 1) / FREE_THREADS);
    const uint64_t words = 1 + (uint64_t)w;                  // per rank: [free cells | free cells per column], u64
    auto p = std::make_unique<MParams>();
    p->main = vg_run_rows(main, run); p->mcs = main->col_stride;
    p->prep = vg_run_rows(prep_or_null, run); p->pcs = prep_or_null ? prep_or_null->col_stride : 0;
    p->g0 = run.begin; p->n = run.count; p->h = h; p->width = w; p->k = chip->n_interactions;
    vg_air_reads(chip->chip_id, p->air_l, p->air_n);
    for (uint32_t c = 0; c < w; c++) p->cols[c >> 6] |= 1ull << (c & 63);
    VG_TRY(vg_bus_masks(ctx, chip, &p->bus));
    VgBuf counts(ctx), cta(ctx), off(ctx), endb(ctx), edges(ctx);
    VG_TRY(counts.alloc(N * words * 8));
    VG_TRY(cta.alloc(ctas * 4ull));
    VG_TRY(off.alloc(ctas * 8ull));
    VG_TRY(endb.alloc(4));
    unsigned long long* mine = counts.as<unsigned long long>() + (uint64_t)me * words;
    VG_CUDA(ctx, cudaMemsetAsync(mine, 0, words * 8, ctx->stream));
    VG_CUDA(ctx, cudaMemsetAsync(cta.p, 0, ctas * 4ull, ctx->stream));
    VG_TRY(vg_edge_rows(ctx, run, p->main, p->mcs, h, w, edges, &p->before, &p->bcs, &p->after, &p->acs));
    p->cta_count = cta.as<uint32_t>(); p->per_col = mine + 1;
    {
        KScope ks(ctx, KC_CHECK, 4.0 * (double)run.count * w);
        air::with_chip(chip->chip_id, [&](auto c) { free_mask_kernel<decltype(c)::value><<<ctas, FREE_THREADS, 0, ctx->stream>>>(*p); });
        VG_LAUNCH_CHECK(ctx);
    }
    VG_TRY(vg_cta_scan(ctx, cta.as<uint32_t>(), ctas, cap, off.as<unsigned long long>(), mine, endb.as<uint32_t>()));
    if (run.split) VG_TRY(vg_comm_allgather_inplace(ctx, counts.as<uint32_t>(), 2 * words));
    std::vector<unsigned long long> hc((size_t)N * words);
    uint32_t end = 0;
    VG_CUDA(ctx, cudaMemcpyAsync(hc.data(), counts.p, hc.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaMemcpyAsync(&end, endb.p, 4, cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    std::vector<uint64_t> found(N);
    uint64_t all = 0;
    for (uint32_t r = 0; r < N; r++) all += found[r] = hc[(size_t)r * words];
    // rank r's cells are rows of its run, below rank r + 1's: the list is the ranks' lists in rank order
    p->cta_off = off.as<unsigned long long>(); p->cap = cap;
    VG_TRY(vg_gather_lists(ctx, run.split, found, cap, [&](vgpu_free_cell* slot) -> int32_t {
        if (!end) return 0;
        p->out = slot;
        KScope ks(ctx, KC_CHECK, 4.0 * (double)std::min<uint64_t>(run.count, (uint64_t)end * FREE_THREADS) * w);
        air::with_chip(chip->chip_id, [&](auto c) { free_write_kernel<decltype(c)::value><<<end, FREE_THREADS, 0, ctx->stream>>>(*p); });
        VG_LAUNCH_CHECK(ctx);
        return 0;
    }, out, cap, n_out));
    *total = all;
    if (rows_per_column)
        for (uint32_t c = 0; c < w; c++) {
            uint64_t s = 0;
            for (uint32_t r = 0; r < N; r++) s += hc[(size_t)r * words + 1 + c];
            rows_per_column[c] = s;
        }
    return 0;
}
