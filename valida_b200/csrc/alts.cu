// vgpu_cell_alternatives: the other values the AIR accepts in a main-trace cell of a chip's witness.  For cell (r, c) holding x0, S is
// the set of Air::eval assertions whose value depends on the cell: those of row r's evaluation (the cell as L(c)) and of row
// (r - 1) mod h's, with that row's own selectors (the cell as N(c)); on a one-row chip the one evaluation, the cell as both.  Each is a
// polynomial of degree <= 3 in t = X - x0 (log_quotient_degree = 1), so its values at t = 0..3 (one 4-lane evaluation, F4) determine it.
// The cell is listed when S is not empty and its polynomials share a root t != 0 in F_p; the values are x0 + those roots.  A cell with S
// empty is vgpu_free_cells' (free.cu); a listed cell is flagged when a bus event reads it (free.cu's rule), not skipped.
// Two kernels, one thread per row of the run, in the pattern of vgpu_free_cells: a count pass folds, for each column the AIR reads, the
// row's evaluation and then the previous row's into the cell's gcd (polyroots.cuh), finds its roots, and keeps per-column counts
// (listed, bus-free) in shared memory; a CTA with nothing listed touches no global memory.  After vg_cta_scan, a write pass in the
// CTAs whose entries start below the cap finds each thread's listed columns, scans them over the CTA, and recomputes and writes each
// entry at its prefix, so the list is in (row, column) order.  A split run's edge rows come from vg_edge_rows (cells.cuh).
#include "cells.cuh"
#include "lists.cuh"
#include "polyroots.cuh"

namespace {

constexpr int ALT_THREADS = 128, ALT_WARPS = ALT_THREADS / 32;
static_assert(sizeof(vgpu_cell_alternative) == 40, "vgpu_cell_alternative is 10 words");

// z() folds every assertion that is not constant in the cell into g, the gcd of S so far (zero: S empty so far).  A non-zero constant
// gcd has no roots, and stays.
struct AltBuilder : VgLanes {
    poly::P3 g;
    __device__ __forceinline__ void z(const V& x) {
        if (((x.v[1] != x.v[0]) | (x.v[2] != x.v[0]) | (x.v[3] != x.v[0])) && poly::deg(g) != 0) g = poly::gcd(g, poly::interp(x.v));
    }
};

struct AParams {
    const uint32_t* main; uint64_t mcs;             // local row 0 of the rows swept
    const uint32_t* prep; uint64_t pcs;             // null without a preprocessed trace
    const uint32_t* before; uint64_t bcs;           // the row before local row 0 ((g0 - 1) mod h)
    const uint32_t* after; uint64_t acs;            // the row after local row n - 1
    uint64_t g0, n, h;                              // global row of local row 0; rows swept; global height
    uint64_t air_l[2], air_n[2];                    // columns the AIR text reads on the local / next row (bit c % 64 of word c / 64)
    VgBusMasks bus;
    uint32_t k, width;
    uint32_t* cta_count;                            // listed cells of each CTA
    unsigned long long* per_col;                    // count pass: listed cells per column, then bus-free ones per column
    unsigned long long* failed;                     // count pass: ~(row * 256 + column) of the first cell whose roots were not split
    const unsigned long long* cta_off;              // write pass: exclusive prefix sum of cta_count
    vgpu_cell_alternative* out; uint64_t cap;       // write pass: entries [0, cap) of this rank's list
};

// The other values of local row i's cell in column c (canonical, ascending): their number, or -1 (roots not split).
template <int CHIP>
__device__ __forceinline__ int cell_values(const AParams& p, uint64_t i, int c, uint32_t v[3]) {
    const uint32_t* row = p.main + i;
    const uint64_t g = p.g0 + i;
    const bool one_row = p.h == 1;
    const uint64_t bit = 1ull << (c & 63);
    AltBuilder b;
    b.g = poly::P3{{0, 0, 0, 0}};
    // job 0: the row's own evaluation, the cell as L(c) (and as N(c) on a one-row chip); job 1: the previous row's, the cell as N(c)
#pragma unroll 1
    for (int job = 0; job < 2; job++) {
        const bool prev = job == 1;
        if (prev ? one_row || !(p.air_n[c >> 6] & bit) : !((p.air_l[c >> 6] | (one_row ? p.air_n[c >> 6] : 0)) & bit)) continue;
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
        b.tl = prev ? -1 : c;
        b.tn = prev || one_row ? c : -1;
        air::eval_chip<CHIP>(b);
    }
    if (poly::deg(b.g) < 1) return 0;                               // S empty, or no common root at all
    return poly::other_roots(b.g, __ldg(row + (uint64_t)c * p.mcs), v);
}

// The columns a bus event of local row i reads (bit c % 64 of word c / 64).
__device__ __forceinline__ void bus_read(const AParams& p, uint64_t i, uint64_t& pin0, uint64_t& pin1) {
    pin0 = p.bus.count_cols[0]; pin1 = p.bus.count_cols[1];
    for (uint32_t m = 0; m < p.k; m++)
        if (logup::pair_col(p.bus.count[m], p.main + i, p.mcs, p.prep ? p.prep + i : nullptr, p.pcs) != 0) {
            pin0 |= p.bus.fields[m][0];
            pin1 |= p.bus.fields[m][1];
        }
}

template <int CHIP>
__global__ void __launch_bounds__(ALT_THREADS, 1) alt_count_kernel(const __grid_constant__ AParams p) {
    __shared__ uint32_t hist[2 * CELLS_MAX_COLS];                  // listed, then bus-free, per column
    for (uint32_t t = threadIdx.x; t < p.width; t += blockDim.x) hist[t] = hist[CELLS_MAX_COLS + t] = 0;
    __syncthreads();
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t listed = 0;
    if (i < p.n) {
        uint64_t pin0, pin1;
        bus_read(p, i, pin0, pin1);
        uint64_t t0 = p.air_l[0] | p.air_n[0], t1 = p.air_l[1] | p.air_n[1];
        while (t0 | t1) {
            int c;
            if (t0) { c = __ffsll((long long)t0) - 1; t0 &= t0 - 1; }
            else { c = 64 + __ffsll((long long)t1) - 1; t1 &= t1 - 1; }
            uint32_t v[3];
            const int nv = cell_values<CHIP>(p, i, c, v);
            if (nv < 0) atomicMax(p.failed, ~((unsigned long long)(p.g0 + i) * 256 + c));
            if (nv <= 0) continue;
            listed++;
            atomicAdd(&hist[c], 1u);
            if (!(((c < 64 ? pin0 : pin1) >> (c & 63)) & 1)) atomicAdd(&hist[CELLS_MAX_COLS + c], 1u);
        }
    }
    const uint32_t total = vg_cta_total<ALT_WARPS>(listed);
    if (!total) return;
    if (threadIdx.x == 0) p.cta_count[blockIdx.x] = total;
    for (uint32_t t = threadIdx.x; t < p.width; t += blockDim.x) {
        if (hist[t]) atomicAdd(p.per_col + t, (unsigned long long)hist[t]);
        if (hist[CELLS_MAX_COLS + t]) atomicAdd(p.per_col + p.width + t, (unsigned long long)hist[CELLS_MAX_COLS + t]);
    }
}

template <int CHIP>
__global__ void __launch_bounds__(ALT_THREADS, 1) alt_write_kernel(const __grid_constant__ AParams p) {
    const uint32_t total = p.cta_count[blockIdx.x];
    const unsigned long long base = p.cta_off[blockIdx.x];
    if (!total || base >= p.cap) return;                     // alike for the whole CTA
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < p.n;
    uint64_t pin0 = 0, pin1 = 0;
    if (live) bus_read(p, i, pin0, pin1);
    // pass 0 finds the thread's listed columns (l0, l1), pass 1 recomputes and writes them at the thread's place in the CTA's list
    uint64_t l0 = 0, l1 = 0, t0 = live ? p.air_l[0] | p.air_n[0] : 0, t1 = live ? p.air_l[1] | p.air_n[1] : 0;
    uint32_t pos = 0, end = 0;
    vgpu_cell_alternative* out = p.out + base;
#pragma unroll 1
    for (int pass = 0; pass < 2; pass++) {
        if (pass == 1) {
            pos = vg_cta_exclusive<ALT_WARPS>((uint32_t)(__popcll(l0) + __popcll(l1)));
            end = (uint32_t)min((unsigned long long)total, p.cap - base);
            t0 = pos < end ? l0 : 0; t1 = pos < end ? l1 : 0;
        }
        while (t0 | t1) {
            int c;
            if (t0) { c = __ffsll((long long)t0) - 1; t0 &= t0 - 1; }
            else { c = 64 + __ffsll((long long)t1) - 1; t1 &= t1 - 1; }
            uint32_t v[3];
            const int nv = cell_values<CHIP>(p, i, c, v);
            if (nv <= 0) continue;
            if (pass == 0) {
                if (c < 64) l0 |= 1ull << c;
                else l1 |= 1ull << (c - 64);
                continue;
            }
            vgpu_cell_alternative e;
            e.row = (int64_t)(p.g0 + i);
            e.column = (uint32_t)c;
            e.value = bb::from_monty(__ldg(p.main + i + (uint64_t)c * p.mcs));
            e.n_values = (uint32_t)nv;
            e.values[0] = v[0]; e.values[1] = nv > 1 ? v[1] : 0; e.values[2] = nv > 2 ? v[2] : 0;
            e.bus = (uint32_t)((((c < 64 ? pin0 : pin1) >> (c & 63)) & 1));
            e.reserved = 0;
            out[pos] = e;
            if (++pos >= end) break;
        }
    }
}

}  // namespace

extern "C" int32_t vgpu_cell_alternatives(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep_or_null,
                                          uint64_t cap, vgpu_cell_alternative* out, uint64_t* n_out, uint64_t* total,
                                          uint64_t* total_bus_free, uint64_t* per_column_or_null) {
    if (!ctx) return -1;
    if (!n_out || !total || !total_bus_free || (cap && !out)) VG_FAIL(ctx, "cell_alternatives: null output");
    if (!chip || !main) VG_FAIL(ctx, "cell_alternatives: null argument");
    if (chip->n_interactions > VGPU_MAX_INTERACTIONS) VG_FAIL(ctx, "cell_alternatives: %u interactions exceed %d", chip->n_interactions, VGPU_MAX_INTERACTIONS);
    if (chip->width > CELLS_MAX_COLS) VG_FAIL(ctx, "cell_alternatives: %u columns exceed %d", chip->width, CELLS_MAX_COLS);
    VG_TRY(vg_check_shapes(ctx, chip, main, prep_or_null, nullptr, true));
    VG_TRY(vg_enter(ctx));
    VG_TRY(vg_dmat_materialize(ctx, main));
    VG_TRY(vg_dmat_materialize(ctx, prep_or_null));
    const uint64_t h = main->gh;
    const uint32_t w = chip->width;
    const VgRun run = vg_trace_run(ctx, h);
    const uint32_t N = run.split ? (uint32_t)ctx->comm_size : 1, me = run.split ? (uint32_t)ctx->comm_rank : 0;
    const uint32_t ctas = (uint32_t)((run.count + ALT_THREADS - 1) / ALT_THREADS);
    const uint64_t words = 2 + 2 * (uint64_t)w;              // per rank: [listed | ~first unsplit cell | listed per column | bus-free per column]
    auto p = std::make_unique<AParams>();
    p->main = vg_run_rows(main, run); p->mcs = main->col_stride;
    p->prep = vg_run_rows(prep_or_null, run); p->pcs = prep_or_null ? prep_or_null->col_stride : 0;
    p->g0 = run.begin; p->n = run.count; p->h = h; p->width = w; p->k = chip->n_interactions;
    vg_air_reads(chip->chip_id, p->air_l, p->air_n);
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
    p->cta_count = cta.as<uint32_t>(); p->failed = mine + 1; p->per_col = mine + 2;
    {
        KScope ks(ctx, KC_CHECK, 4.0 * (double)run.count * w);
        air::with_chip(chip->chip_id, [&](auto c) { alt_count_kernel<decltype(c)::value><<<ctas, ALT_THREADS, 0, ctx->stream>>>(*p); });
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
    uint64_t all = 0, failed = 0;
    for (uint32_t r = 0; r < N; r++) {
        all += found[r] = hc[(size_t)r * words];
        failed = std::max<uint64_t>(failed, hc[(size_t)r * words + 1]);
    }
    if (failed)
        VG_FAIL(ctx, "cell_alternatives: the common roots of the cell at row %llu, column %llu were not split in %d tries",
                (unsigned long long)(~failed >> 8), (unsigned long long)(~failed & 255), poly::SPLIT_TRIES);
    // rank r's cells are rows of its run, below rank r + 1's: the list is the ranks' lists in rank order
    p->cta_off = off.as<unsigned long long>(); p->cap = cap;
    VG_TRY(vg_gather_lists(ctx, run.split, found, cap, [&](vgpu_cell_alternative* slot) -> int32_t {
        if (!end) return 0;
        p->out = slot;
        KScope ks(ctx, KC_CHECK, 4.0 * (double)std::min<uint64_t>(run.count, (uint64_t)end * ALT_THREADS) * w);
        air::with_chip(chip->chip_id, [&](auto c) { alt_write_kernel<decltype(c)::value><<<end, ALT_THREADS, 0, ctx->stream>>>(*p); });
        VG_LAUNCH_CHECK(ctx);
        return 0;
    }, out, cap, n_out));
    *total = all;
    uint64_t bus_free = 0;
    for (uint32_t c = 0; c < w; c++) {
        uint64_t s = 0, f = 0;
        for (uint32_t r = 0; r < N; r++) {
            s += hc[(size_t)r * words + 2 + c];
            f += hc[(size_t)r * words + 2 + w + c];
        }
        bus_free += f;
        if (per_column_or_null) { per_column_or_null[c] = s; per_column_or_null[w + c] = f; }
    }
    *total_bus_free = bus_free;
    return 0;
}
