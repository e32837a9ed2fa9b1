// check_constraints (machine/src/check_constraints.rs:14-84; debug builds of the reference's prove, derive/src/lib.rs:246-253) on the
// device: every constraint of a chip's Air::eval and of eval_permutation_constraints on every row g of the TRACE, with row (g+1) mod h
// as "next" and the debug selectors is_first_row = [g == 0], is_last_row = [g == h-1], is_transition = 1 - is_last_row.
// One thread per natural trace row reads the column-major traces (coalesced) through the same AIR text as the quotient sweep
// (airs.cuh, logup.cuh), so constraint i here is constraint i there: the chip's assertions in eval order, one per interaction,
// then the LogUp transition, first-row and last-row constraints.  The cumulative sum is read on the device from the permutation
// trace's last row and last column (check_constraints.rs:33).
// One launch sweeps a RUN of rows: local rows [0, n) of matrices entered at global row g0, the next row of local row n-1 being local
// row `wrap`.  A whole trace is one run (g0 = 0, n = h, wrap = 0).  A split proof's rank r holds the run vg_trace_run(ctx, h): it
// sweeps all its rows but the last, whose next row is rank (r+1) mod N's first row; every rank packs its first row (and its last
// row's running sum) into a small block, one all-gather exchanges the blocks, and the last row is swept from a 2-row window (own
// last row, next rank's first row; column-major, stride 2) as a run of one row whose next row is window row 1.  No peer pointers:
// a borrowed shard is caller memory, outside the symmetric heap.
// Every call plans its runs in one CheckSet: vgpu_check_constraints takes each chip's whole trace as its run on any context; the
// other calls take this rank's run.  vgpu_check_witness and prove's debug mode drive one VgMachineCheck (devchip.h), which builds the
// permutation traces and sweeps them through a CheckSet.  check_kernel and vgpu_check_failures' two passes set up and evaluate a row
// with the same eval_row.
// Result per chip: the first failing (row, constraint) as ONE 64-bit key (global row << 8 | constraint, atomicMin) and the number of
// rows with at least one failure; both are aggregated per warp, so a clean trace costs no atomic at all.
#include "ctx.h"
#include "devchip.h"
#include "airs.cuh"
#include "logup.cuh"
#include "lists.cuh"
#include "open.h"
#include <functional>
#include <memory>

namespace {

using bb::E5;
using air::F;

constexpr uint32_t CHECK_NONE = 0xffffffffu;
constexpr uint32_t CHECK_MAX_CONSTRAINTS = 256;   // the constraint index takes the low 8 bits of the key

struct CParams {
    const uint32_t* main; uint64_t mcs;             // every matrix pointer is at local row 0 of the run
    const uint32_t* prep; uint64_t pcs;             // null without a preprocessed trace
    const uint32_t* perm; uint64_t qcs;             // flattened permutation trace, 5(k+1) columns
    const uint32_t* cumsum; uint64_t ccs;           // the cumulative sum's 5 words, ccs apart (read only by the row g = h-1)
    uint64_t g0, n, h, wrap;                        // global row of local row 0; rows swept; global height; next row of local row n-1
    unsigned long long* first;                      // min over failing rows of (row << 8 | first failing constraint); ~0: none
    unsigned long long* count;                      // rows with at least one failing constraint
    DevChip chip;
};

// What every check kernel's builder holds: the thread's row and its next row (main trace, pointers already offset to the rows),
// the selectors, and the index of the next constraint.  Each builder adds what it does with a constraint that does not vanish.
struct RowBuilder {
    using V = air::F;
    const uint32_t* lrow; const uint32_t* nrow; uint64_t cs;
    F first, last, trans;
    uint32_t idx;
    __device__ __forceinline__ F L(int c) const { return F{__ldg(lrow + (uint64_t)c * cs)}; }
    __device__ __forceinline__ F N(int c) const { return F{__ldg(nrow + (uint64_t)c * cs)}; }
    __device__ __forceinline__ void section(const char*) {}
};

// Sets up local row i of the run and evaluates every constraint on it, in eval order, into b.
template <int CHIP, class B>
__device__ __forceinline__ void eval_row(const CParams& p, uint64_t i, B& b) {
    // the global row is p.g0 + i, recomputed where it is used: a register kept for it makes two chips spill
    const bool is_last = p.g0 + i + 1 == p.h;
    const uint64_t n = i + 1 < p.n ? i + 1 : p.wrap;       // a one-row chip is its own next row
    b.lrow = p.main + i; b.nrow = p.main + n; b.cs = p.mcs;
    b.first = F{p.g0 + i == 0 ? bb::R1 : 0u};
    b.last = F{is_last ? bb::R1 : 0u};
    b.trans = F{is_last ? 0u : bb::R1};
    b.idx = 0;
    air::eval_chip<CHIP>(b);
    E5 cumsum;
#pragma unroll
    for (int l = 0; l < 5; l++) cumsum.c[l] = __ldg(p.cumsum + (uint64_t)l * p.ccs);
    logup::eval_constraints(b, p.chip, b.lrow, b.nrow, p.mcs, p.prep ? p.prep + i : nullptr, p.prep ? p.prep + n : nullptr, p.pcs,
                            p.perm + i, p.perm + n, p.qcs, cumsum);
}

struct CheckBuilder : RowBuilder {
    uint32_t bad;                                              // the first constraint that did not vanish
    __device__ __forceinline__ void z(F x) { if (x.v != 0 && bad == CHECK_NONE) bad = idx; idx++; }
    __device__ __forceinline__ void z_ext(const E5& x) { if (!bb::e5_is_zero(x) && bad == CHECK_NONE) bad = idx; idx++; }
};

template <int CHIP>
__global__ void __launch_bounds__(128) check_kernel(const __grid_constant__ CParams p) {
    const uint64_t i_raw = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = i_raw < p.n;
    const uint64_t i = active ? i_raw : p.n - 1;          // idle lanes shadow the last row (the warp vote needs every lane)
    CheckBuilder b;
    b.bad = CHECK_NONE;
    eval_row<CHIP>(p, i, b);
    const bool fail = active && b.bad != CHECK_NONE;
    const unsigned vote = __ballot_sync(0xffffffffu, fail);
    // the lowest failing lane holds the warp's lowest row, hence its smallest key
    if (vote && (threadIdx.x & 31) == (unsigned)(__ffs(vote) - 1)) {
        atomicMin(p.first, ((unsigned long long)(p.g0 + i) << 8) | b.bad);
        atomicAdd(p.count, (unsigned long long)__popc(vote));
    }
}

// n words of a strided source into a strided destination, per segment (one CTA each): the boundary rows of a split chip in and
// out of the exchanged block and the windows.
struct CopySeg { const uint32_t* src; uint64_t scs; uint32_t* dst; uint64_t dcs; uint32_t n; };
constexpr int COPY_SEGS = 7;
struct CopyList { CopySeg s[COPY_SEGS]; };
__global__ void __launch_bounds__(64) check_copy_kernel(const __grid_constant__ CopyList l) {
    const CopySeg& s = l.s[blockIdx.x];
    for (uint32_t c = threadIdx.x; c < s.n; c += blockDim.x) s.dst[(uint64_t)c * s.dcs] = __ldg(s.src + (uint64_t)c * s.scs);
}

int32_t copy_segments(vgpu_ctx* ctx, const CopyList& l, int nseg) {
    KScope ks(ctx, KC_CHECK, 0.0);
    check_copy_kernel<<<nseg, 64, 0, ctx->stream>>>(l);
    VG_LAUNCH_CHECK(ctx);
    return 0;
}

// Enqueues one run's sweep; p holds everything but the chip, which is built here from the challenges.
int32_t enqueue_sweep(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const uint32_t challenges[15], CParams& p) {
    if (!p.n) return 0;
    VG_TRY(vg_build_devchip(ctx, chip, challenges, &p.chip));
    KScope ks(ctx, KC_CHECK, 4.0 * (double)p.n * (double)(chip->width + chip->preprocessed_width + 5.0 * (chip->n_interactions + 1)));
    air::with_chip(chip->chip_id, [&](auto c) { check_kernel<decltype(c)::value><<<(unsigned)((p.n + 127) / 128), 128, 0, ctx->stream>>>(p); });
    VG_LAUNCH_CHECK(ctx);
    return 0;
}

// ---- every failure (vgpu_check_failures) ------------------------------------------------------------------------------------------
// The same rows and text as check_kernel, in kernels of their own so that check_kernel stays as it is.  Pass 1 counts: a CTA keeps a
// shared histogram of its failures per constraint and, only when it found one, stores its count and adds the histogram to the
// call's (a clean witness makes no global atomic).  A scan of the per-CTA counts gives each CTA its first entry; pass 2 runs only in
// the CTAs with failures that start below the cap, counts each thread's failures again, scans them over the CTA and writes each
// thread's entries in constraint order: the list is ordered by row, then constraint, whatever the schedule.
struct FParams {
    CParams c;                               // the run (c.first / c.count unused)
    uint32_t* cta_count;                     // failures of each CTA of every sweep of the call; this sweep's CTAs from cta0
    const unsigned long long* cta_off;       // pass 2: exclusive prefix sum of cta_count
    unsigned long long* hist;                // pass 1: failures per constraint (= failing rows, a constraint fails once per row)
    vgpu_check_failure* out; uint64_t cap;   // pass 2: entries [0, cap) of the list
    uint32_t cta0;
};

__shared__ uint32_t fail_hist[CHECK_MAX_CONSTRAINTS];

struct FailCountBuilder : RowBuilder {
    bool active;
    // every lane reaches every constraint (the text has no branch on values): one shared atomic per warp and failing constraint
    __device__ __forceinline__ void tally(bool bad) {
        const unsigned v = __ballot_sync(0xffffffffu, active && bad);
        if (v && (threadIdx.x & 31) == 0) atomicAdd(&fail_hist[idx], (unsigned)__popc(v));
        idx++;
    }
    __device__ __forceinline__ void z(F x) { tally(x.v != 0); }
    __device__ __forceinline__ void z_ext(const E5& x) { tally(!bb::e5_is_zero(x)); }
};

// Counts the thread's failures while pos < end is false; then writes those at entries [pos, end) of the CTA's part of the list.
struct FailWriteBuilder : RowBuilder {
    uint32_t pos, end;
    vgpu_check_failure* out;                 // the CTA's first entry
    uint64_t row;
    __device__ __forceinline__ void put(const uint32_t* v, int limbs) {
        vgpu_check_failure* e = out + pos;
        e->row = (int64_t)row;
        e->constraint = idx;
        for (int l = 0; l < 5; l++) e->value[l] = l < limbs ? bb::from_monty(v[l]) : 0u;
    }
    __device__ __forceinline__ void z(F x) {
        if (x.v != 0) { if (pos < end) put(&x.v, 1); pos++; }
        idx++;
    }
    __device__ __forceinline__ void z_ext(const E5& x) {
        if (!bb::e5_is_zero(x)) { if (pos < end) put(x.c, 5); pos++; }
        idx++;
    }
};

template <int CHIP>
__global__ void __maxnreg__(128) fail_count_kernel(const __grid_constant__ FParams f) {
    const CParams& p = f.c;
    for (uint32_t t = threadIdx.x; t < CHECK_MAX_CONSTRAINTS; t += blockDim.x) fail_hist[t] = 0;
    __syncthreads();
    const uint64_t i_raw = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    FailCountBuilder b;
    b.active = i_raw < p.n;
    const uint64_t i = b.active ? i_raw : p.n - 1;        // idle lanes shadow the last row (the warp vote needs every lane)
    eval_row<CHIP>(p, i, b);
    __syncthreads();
    uint32_t s = 0;
    for (uint32_t t = threadIdx.x; t < CHECK_MAX_CONSTRAINTS; t += blockDim.x) s += fail_hist[t];
    const uint32_t total = vg_cta_total<4>(s);
    if (!total) return;
    if (threadIdx.x == 0) f.cta_count[f.cta0 + blockIdx.x] = total;
    for (uint32_t t = threadIdx.x; t < CHECK_MAX_CONSTRAINTS; t += blockDim.x)
        if (fail_hist[t]) atomicAdd(f.hist + t, (unsigned long long)fail_hist[t]);
}

template <int CHIP>
__global__ void __maxnreg__(128) fail_write_kernel(const __grid_constant__ FParams f) {
    const CParams& p = f.c;
    const uint32_t cta = f.cta0 + blockIdx.x, total = f.cta_count[cta];
    const unsigned long long base = f.cta_off[cta];
    if (!total || base >= f.cap) return;                  // alike for the whole CTA
    const uint64_t i_raw = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = i_raw < p.n;
    const uint64_t i = active ? i_raw : p.n - 1;
    FailWriteBuilder b;
    b.out = f.out + base; b.row = p.g0 + i;
    b.pos = 0; b.end = 0;
    eval_row<CHIP>(p, i, b);
    // the thread's first entry: the failures of the CTA's lower threads
    const uint32_t mine = active ? b.pos : 0, first = vg_cta_exclusive<4>(mine);
    const uint32_t end = (uint32_t)min((unsigned long long)total, f.cap - base);
    if (!mine || first >= end) return;
    b.pos = first; b.end = end;
    eval_row<CHIP>(p, i, b);
}

// One CTA: the exclusive prefix sum of the m per-CTA counts, their total, and *end = 1 + the last CTA with failures that starts below
// cap (0: none), which bounds pass 2's grids.
__global__ void __launch_bounds__(1024) fail_scan_kernel(const uint32_t* count, uint32_t m, uint64_t cap, unsigned long long* off,
                                                         unsigned long long* total, uint32_t* end) {
    __shared__ unsigned long long warp_sum[32];
    __shared__ uint32_t warp_end[32];
    const uint32_t per = (m + 1023) / 1024, a = min(m, threadIdx.x * per), e = min(m, a + per), lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long s = 0;
    for (uint32_t j = a; j < e; j++) s += count[j];
    unsigned long long x = s;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= (uint32_t)d) x += y;
    }
    if (lane == 31) warp_sum[warp] = x;
    __syncthreads();
    if (warp == 0) {
        unsigned long long w = warp_sum[lane];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, w, d);
            if (lane >= (uint32_t)d) w += y;
        }
        warp_sum[lane] = w;
    }
    __syncthreads();
    unsigned long long at = x - s + (warp ? warp_sum[warp - 1] : 0);
    uint32_t last = 0;
    for (uint32_t j = a; j < e; j++) {
        off[j] = at;
        if (count[j] && at < cap) last = j + 1;
        at += count[j];
    }
    if (threadIdx.x == 1023) *total = at;               // its range ends at m
    last = __reduce_max_sync(0xffffffffu, last);
    if (lane == 0) warp_end[warp] = last;
    __syncthreads();
    if (warp == 0) {
        last = __reduce_max_sync(0xffffffffu, warp_end[lane]);
        if (lane == 0) *end = last;
    }
}

}  // namespace

// The check of n chips on this rank of a split context (or of a lone one, where every chip is whole and nothing crosses ranks).
// Per chip, sweep() enqueues the run's rows (all but the last when the chip is split) and packs the split chip's boundary words;
// finish() then makes ONE all-gather of every split chip's block, sweeps the windows, and makes ONE all-gather of the verdicts.
// Every rank plans from global heights alone, so all ranks make the same collectives.  `whole`: every chip is one run of its whole
// traces, on any context (vgpu_check_constraints); no collective, one verdict slot.
class CheckSet {
  public:
    CheckSet(vgpu_ctx* ctx, uint32_t n, bool whole = false) : ctx_(ctx), n_(n), whole_(whole), chips_(n), block_(ctx), win_(ctx), store_(ctx) {}

    // the layout, from the chips and their global heights (before any sweep)
    void plan(uint32_t i, const vgpu_chip_desc* chip, uint64_t h) {
        Chip& c = chips_[i];
        c.desc = chip; c.run = whole_ ? VgRun{0, h, false} : vg_trace_run(ctx_, h); c.h = h;
        c.wm = chip->width; c.wp = chip->preprocessed_width; c.wq = 5 * (chip->n_interactions + 1);
        if (c.run.split) {
            c.at = words_; words_ += c.wm + c.wp + c.wq + 5;
            c.win_at = win_words_; win_words_ += 2 * (c.wm + c.wp + c.wq);
            any_split_ = true;
        }
    }
    // verdicts: verdict_bytes() of device memory for the verdicts (VgMachineCheck's copy-back buffer); null: allocated here
    int32_t alloc(unsigned long long* verdicts = nullptr) {
        const uint32_t N = any_split_ ? (uint32_t)ctx_->comm_size : 1;
        if (words_) VG_TRY(block_.alloc((size_t)N * words_ * 4));
        if (win_words_) VG_TRY(win_.alloc(win_words_ * 4));
        if (!verdicts) {
            VG_TRY(store_.alloc(verdict_bytes()));
            verdicts = store_.as<unsigned long long>();
        }
        verdicts_ = verdicts;
        unsigned long long* mine = own_verdicts();
        VG_CUDA(ctx_, cudaMemsetAsync(mine, 0xff, n_ * sizeof(unsigned long long), ctx_->stream));
        VG_CUDA(ctx_, cudaMemsetAsync(mine + n_, 0, n_ * sizeof(unsigned long long), ctx_->stream));
        return 0;
    }
    // Launches one run's sweep (p complete but for the chip): vgpu_check_failures' passes; by default enqueue_sweep's check_kernel.
    using Sweep = std::function<int32_t(const vgpu_chip_desc*, CParams&)>;
    // Enqueues chip i's sweep of this rank's run (arguments validated); what it reads of perm is read before later work on the stream.
    int32_t sweep(uint32_t i, const vgpu_dmat* main, const vgpu_dmat* prep, const vgpu_dmat* perm, const uint32_t challenges[15],
                  const Sweep& run = nullptr) {
        Chip& c = chips_[i];
        VG_TRY(vg_dmat_materialize(ctx_, main));
        VG_TRY(vg_dmat_materialize(ctx_, prep));
        VG_TRY(vg_dmat_materialize(ctx_, perm));
        const uint64_t row0 = c.run.begin, cnt = c.run.count, k = c.desc->n_interactions;
        const uint32_t *md = vg_run_rows(main, c.run), *pd = vg_run_rows(prep, c.run), *qd = vg_run_rows(perm, c.run);
        const uint64_t mcs = main->col_stride, pcs = prep ? prep->col_stride : 0, qcs = perm->col_stride;
        auto pp = std::make_unique<CParams>();
        CParams& p = *pp;
        p.main = md; p.mcs = mcs; p.prep = pd; p.pcs = pcs; p.perm = qd; p.qcs = qcs;
        // the running sum of the run's last row: the cumulative sum when the run ends the trace; otherwise read by no swept row
        p.cumsum = qd + 5 * k * qcs + cnt - 1; p.ccs = qcs;
        p.g0 = row0; p.h = c.h;
        p.n = c.run.split ? cnt - 1 : cnt;
        p.wrap = c.run.split ? p.n : 0;
        p.first = own_verdicts() + i; p.count = own_verdicts() + n_ + i;
        VG_TRY(run ? run(c.desc, p) : enqueue_sweep(ctx_, c.desc, challenges, p));
        if (!c.run.split) return 0;
        // the block this rank sends (first rows, last running sum) and the window's row 0 (this rank's last row)
        uint32_t* blk = block_.as<uint32_t>() + (uint64_t)ctx_->comm_rank * words_ + c.at;
        uint32_t* win = win_.as<uint32_t>() + c.win_at;
        CopyList l{};
        l.s[0] = {md, mcs, blk, 1, c.wm};
        l.s[1] = {pd, pcs, blk + c.wm, 1, pd ? c.wp : 0};
        l.s[2] = {qd, qcs, blk + c.wm + c.wp, 1, c.wq};
        l.s[3] = {qd + 5 * k * qcs + cnt - 1, qcs, blk + c.wm + c.wp + c.wq, 1, 5};
        l.s[4] = {md + cnt - 1, mcs, win, 2, c.wm};
        l.s[5] = {pd ? pd + cnt - 1 : nullptr, pcs, win + 2 * c.wm, 2, pd ? c.wp : 0};
        l.s[6] = {qd + cnt - 1, qcs, win + 2 * (c.wm + c.wp), 2, c.wq};
        return copy_segments(ctx_, l, 7);
    }
    // The exchange of the boundary blocks, the window sweeps and the exchange of the verdicts.
    int32_t finish(const uint32_t challenges[15]) {
        if (!any_split_) return 0;
        VG_TRY(windows(challenges));
        return vg_comm_allgather_inplace(ctx_, (uint32_t*)verdicts_, 4 * (uint64_t)n_);
    }
    // The exchange of the boundary blocks and the window sweeps (each the last row of a split chip's run, after its other rows).
    int32_t windows(const uint32_t challenges[15], const Sweep& run = nullptr) {
        if (!any_split_) return 0;
        const uint32_t N = (uint32_t)ctx_->comm_size, next = ((uint32_t)ctx_->comm_rank + 1) % N;
        VG_TRY(vg_comm_allgather_inplace(ctx_, block_.as<uint32_t>(), words_));
        for (uint32_t i = 0; i < n_; i++) {
            Chip& c = chips_[i];
            if (!c.run.split) continue;
            const uint32_t* nb = block_.as<uint32_t>() + (uint64_t)next * words_ + c.at;
            uint32_t* win = win_.as<uint32_t>() + c.win_at;
            CopyList l{};
            l.s[0] = {nb, 1, win + 1, 2, c.wm};
            l.s[1] = {nb + c.wm, 1, win + 2 * c.wm + 1, 2, c.wp};
            l.s[2] = {nb + c.wm + c.wp, 1, win + 2 * (c.wm + c.wp) + 1, 2, c.wq};
            VG_TRY(copy_segments(ctx_, l, 3));
            auto pp = std::make_unique<CParams>();
            CParams& p = *pp;
            p.main = win; p.mcs = 2;
            p.prep = c.wp ? win + 2 * c.wm : nullptr; p.pcs = 2;
            p.perm = win + 2 * (c.wm + c.wp); p.qcs = 2;
            p.cumsum = block_.as<uint32_t>() + (uint64_t)(N - 1) * words_ + c.at + c.wm + c.wp + c.wq; p.ccs = 1;   // the last rank's
            p.g0 = c.run.begin + c.run.count - 1; p.n = 1; p.h = c.h; p.wrap = 1;
            p.first = own_verdicts() + i; p.count = own_verdicts() + n_ + i;
            VG_TRY(run ? run(c.desc, p) : enqueue_sweep(ctx_, c.desc, challenges, p));
        }
        return 0;
    }
    // every rank's verdicts, as finish() left them on the device
    const void* verdicts() const { return verdicts_; }
    size_t verdict_bytes() const { return (any_split_ ? (size_t)ctx_->comm_size : 1) * 2 * n_ * sizeof(unsigned long long); }
    // all: verdict_bytes() copied to the host -> out: [first keys n | failing-row counts n].  A split chip's rows are spread over the
    // ranks (min of the keys, sum of the counts); any other chip was swept whole by every rank and counts once, as rank 0 reports it.
    void reduce(const unsigned long long* all, unsigned long long* out) const {
        const uint32_t N = any_split_ ? (uint32_t)ctx_->comm_size : 1;
        for (uint32_t i = 0; i < n_; i++) {
            unsigned long long key = all[i], cnt = all[n_ + i];
            for (uint32_t r = 1; chips_[i].run.split && r < N; r++) {
                key = std::min(key, all[(size_t)r * 2 * n_ + i]);
                cnt += all[(size_t)r * 2 * n_ + n_ + i];
            }
            out[i] = key; out[n_ + i] = cnt;
        }
    }

  private:
    struct Chip { const vgpu_chip_desc* desc = nullptr; VgRun run{}; uint64_t h = 0, at = 0, win_at = 0; uint32_t wm = 0, wp = 0, wq = 0; };
    unsigned long long* own_verdicts() const {
        return verdicts_ + (any_split_ ? (size_t)ctx_->comm_rank : 0) * 2 * n_;
    }

    vgpu_ctx* ctx_;
    uint32_t n_;
    bool whole_;
    std::vector<Chip> chips_;
    uint64_t words_ = 0, win_words_ = 0;     // per-rank block words; window words of this rank
    bool any_split_ = false;
    VgBuf block_, win_, store_;
    unsigned long long* verdicts_ = nullptr;
};

namespace {

void decode(unsigned long long first, unsigned long long count, int64_t* row, uint32_t* constraint, uint64_t* failing_rows) {
    *row = first == ~0ull ? -1 : (int64_t)(first >> 8);
    *constraint = first == ~0ull ? 0 : (uint32_t)(first & 0xff);
    *failing_rows = count;
}

// One chip's check, its arguments validated: whole traces, or this rank's run (on a lone context, the whole trace).
int32_t check_chip(vgpu_ctx* ctx, bool whole, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep, const vgpu_dmat* perm,
                   const uint32_t challenges[15], int64_t* first_row, uint32_t* first_constraint, uint64_t* failing_rows) {
    VG_TRY(vg_enter(ctx));
    CheckSet set(ctx, 1, whole);
    set.plan(0, chip, main->gh);
    VG_TRY(set.alloc());
    VG_TRY(set.sweep(0, main, prep, perm, challenges));
    VG_TRY(set.finish(challenges));
    std::vector<unsigned long long> all(set.verdict_bytes() / sizeof(unsigned long long));
    VG_CUDA(ctx, cudaMemcpyAsync(all.data(), set.verdicts(), set.verdict_bytes(), cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    unsigned long long fc[2];
    set.reduce(all.data(), fc);
    decode(fc[0], fc[1], first_row, first_constraint, failing_rows);
    return 0;
}

}  // namespace

VgMachineCheck::VgMachineCheck(vgpu_ctx* ctx, const vgpu_dmat* const main[VGPU_NUM_CHIPS], const vgpu_dmat* const prep[2],
                               const uint32_t challenges[15], bool check)
    : ctx_(ctx), main_(main), prep_(prep), challenges_(challenges), set_(check ? new CheckSet(ctx, VGPU_NUM_CHIPS) : nullptr), res_(ctx) {}

VgMachineCheck::~VgMachineCheck() = default;

int32_t VgMachineCheck::alloc() {
    slots_ = vg_perm_totals_ranks(ctx_);
    if (set_)
        for (int i = 0; i < VGPU_NUM_CHIPS; i++) set_->plan(i, vgpu_basic_machine_chip(i), main_[i]->gh);
    tot_at_ = set_ ? set_->verdict_bytes() / 4 : 0;
    VG_TRY(res_.alloc((tot_at_ + (size_t)VGPU_NUM_CHIPS * slots_ * 5) * 4));
    return set_ ? set_->alloc(res_.as<unsigned long long>()) : 0;
}

int32_t VgMachineCheck::perm(int i, VgMat* out) {
    vgpu_dmat* pm = nullptr;
    VG_TRY(vg_perm_trace_enqueue(ctx_, vgpu_basic_machine_chip(i), main_[i], prep_for(i), challenges_, &pm,
                                 res_.as<uint32_t>() + tot_at_ + (size_t)i * slots_ * 5, &nt_[i]));
    out->reset(pm);
    return 0;
}

int32_t VgMachineCheck::sweep(int i, const vgpu_dmat* perm) {
    // prove's debug mode refuses here what check_constraints refuses; vgpu_check_witness has refused it before enqueueing anything
    VG_TRY(vg_check_shapes(ctx_, vgpu_basic_machine_chip(i), main_[i], prep_for(i), perm, vg_sharded(ctx_)));
    return set_->sweep(i, main_[i], prep_for(i), perm, challenges_);
}

int32_t VgMachineCheck::finish(uint32_t sums[VGPU_NUM_CHIPS][5], vgpu_check_report report[VGPU_NUM_CHIPS]) {
    if (set_) VG_TRY(set_->finish(challenges_));
    std::vector<uint32_t> host(tot_at_ + (size_t)VGPU_NUM_CHIPS * slots_ * 5);
    VG_CUDA(ctx_, cudaMemcpyAsync(host.data(), res_.p, host.size() * 4, cudaMemcpyDeviceToHost, ctx_->stream));
    VG_CUDA(ctx_, cudaStreamSynchronize(ctx_->stream));
    unsigned long long chk[2 * VGPU_NUM_CHIPS];
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) { chk[i] = ~0ull; chk[VGPU_NUM_CHIPS + i] = 0; }
    if (set_) set_->reduce((const unsigned long long*)host.data(), chk);
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) {
        vg_perm_totals_fold(host.data() + tot_at_ + (size_t)i * slots_ * 5, nt_[i], sums[i]);
        decode(chk[i], chk[VGPU_NUM_CHIPS + i], &report[i].first_row, &report[i].first_constraint, &report[i].failing_rows);
        for (int l = 0; l < 5; l++) report[i].cumulative_sum[l] = bb::from_monty(sums[i][l]);
    }
    return 0;
}

// Refuses, before anything is enqueued and alike on every rank (global shapes and this context's run rule only), what the sweep
// cannot check.  perm may be null (vgpu_check_witness builds it).  shards: row shards of this rank's run are accepted.
int32_t vg_check_shapes(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep, const vgpu_dmat* perm, bool shards) {
    if (chip->chip_id >= VGPU_NUM_CHIPS) VG_FAIL(ctx, "check_constraints: unknown chip id %u", chip->chip_id);
    for (const vgpu_dmat* m : {main, prep, perm}) {
        if (!m) continue;
        if (!shards && (m->dist != VG_FULL || m->bitrev_rows)) VG_FAIL(ctx, "check_constraints: whole matrices in natural row order only (not row shards)");
        if (m->bitrev_rows) VG_FAIL(ctx, "check_constraints: a matrix stores its rows bit-reversed (quotient chunks); the check reads traces in natural row order");
    }
    if (main->gw != chip->width) VG_FAIL(ctx, "check_constraints: main width %llu != chip width %u", (unsigned long long)main->gw, chip->width);
    const uint64_t pw = 5ull * (chip->n_interactions + 1);
    if (perm && perm->gw != pw) VG_FAIL(ctx, "check_constraints: permutation trace width %llu != 5 (k + 1) = %llu", (unsigned long long)perm->gw, (unsigned long long)pw);
    if (chip->preprocessed_width && !prep) VG_FAIL(ctx, "check_constraints: chip %u needs its preprocessed trace (%u columns)", chip->chip_id, chip->preprocessed_width);
    if (!chip->preprocessed_width && prep) VG_FAIL(ctx, "check_constraints: chip %u has no preprocessed trace", chip->chip_id);
    if (prep && prep->gw != chip->preprocessed_width) VG_FAIL(ctx, "check_constraints: preprocessed width %llu != %u", (unsigned long long)prep->gw, chip->preprocessed_width);
    const uint64_t h = main->gh;
    if (h == 0 || (h & (h - 1))) VG_FAIL(ctx, "check_constraints: trace height %llu is not a power of two", (unsigned long long)h);
    if ((perm && perm->gh != h) || (prep && prep->gh != h)) VG_FAIL(ctx, "check_constraints: the main, preprocessed and permutation traces differ in height");
    const VgRun run = vg_trace_run(ctx, h);
    for (const vgpu_dmat* m : {main, prep, perm})
        if (m && m->dist == VG_ROWS && !(run.split && m->row0 == run.begin && m->h == run.count))
            VG_FAIL(ctx, "check_constraints: a row shard holding rows [%llu, %llu) of a trace of height %llu is not this context's run of that "
                    "height, rows [%llu, %llu)%s", (unsigned long long)m->row0, (unsigned long long)(m->row0 + m->h), (unsigned long long)h,
                    (unsigned long long)run.begin, (unsigned long long)(run.begin + run.count), run.split ? "" : " (the trace is not split here)");
    const uint32_t N = vg_chip_constraints(chip);
    if (N > CHECK_MAX_CONSTRAINTS) VG_FAIL(ctx, "check_constraints: %u constraints exceed the 8-bit index (%u)", N, CHECK_MAX_CONSTRAINTS);
    return 0;
}

int32_t vg_check_machine(vgpu_ctx* ctx, const char* what, const vgpu_dmat* const main[VGPU_NUM_CHIPS], const vgpu_dmat* const prep[2]) {
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) {
        if (!main[i]) VG_FAIL(ctx, "%s: chip %d has no trace", what, i);
        VG_TRY(vg_check_shapes(ctx, vgpu_basic_machine_chip(i), main[i], vg_machine_prep(prep, i), nullptr, true));
    }
    return 0;
}

int32_t vg_cta_scan(vgpu_ctx* ctx, const uint32_t* count, uint32_t m, uint64_t cap, unsigned long long* off, unsigned long long* total, uint32_t* end) {
    KScope ks(ctx, KC_CHECK, 16.0 * m);
    fail_scan_kernel<<<1, 1024, 0, ctx->stream>>>(count, m, cap, off, total, end);
    VG_LAUNCH_CHECK(ctx);
    return 0;
}

int32_t vg_copy_segments(vgpu_ctx* ctx, const VgCopySeg* segs, int n) {
    if (n > COPY_SEGS) VG_FAIL(ctx, "copy_segments: %d segments exceed %d", n, COPY_SEGS);
    CopyList l{};
    for (int i = 0; i < n; i++) l.s[i] = {segs[i].src, segs[i].scs, segs[i].dst, segs[i].dcs, segs[i].n};
    return copy_segments(ctx, l, n);
}

bool vg_sums_cancel(const vgpu_check_report report[VGPU_NUM_CHIPS]) {
    for (int l = 0; l < 5; l++) {
        uint64_t s = 0;
        for (int i = 0; i < VGPU_NUM_CHIPS; i++) s += report[i].cumulative_sum[l];
        if (s % bb::P) return false;
    }
    return true;
}

extern "C" int32_t vgpu_check_constraints(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep_or_null,
                                          const vgpu_dmat* perm, const uint32_t challenges[15],
                                          int64_t* first_row, uint32_t* first_constraint, uint64_t* failing_rows) {
    if (!first_row || !first_constraint || !failing_rows) VG_FAIL(ctx, "check_constraints: null output");
    if (!chip || !main || !perm || !challenges) VG_FAIL(ctx, "check_constraints: null argument");
    VG_TRY(vg_check_shapes(ctx, chip, main, prep_or_null, perm, false));
    return check_chip(ctx, true, chip, main, prep_or_null, perm, challenges, first_row, first_constraint, failing_rows);
}

extern "C" int32_t vgpu_check_constraints_local(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep_or_null,
                                                const vgpu_dmat* perm, const uint32_t challenges[15],
                                                int64_t* first_row, uint32_t* first_constraint, uint64_t* failing_rows) {
    if (!first_row || !first_constraint || !failing_rows) VG_FAIL(ctx, "check_constraints_local: null output");
    if (!chip || !main || !perm || !challenges) VG_FAIL(ctx, "check_constraints_local: null argument");
    VG_TRY(vg_check_shapes(ctx, chip, main, prep_or_null, perm, true));
    return check_chip(ctx, false, chip, main, prep_or_null, perm, challenges, first_row, first_constraint, failing_rows);
}

extern "C" int32_t vgpu_check_witness(vgpu_ctx* ctx, const vgpu_dmat* const main[VGPU_NUM_CHIPS], const vgpu_dmat* const prep[2],
                                      const uint32_t challenges[15], vgpu_check_report report[VGPU_NUM_CHIPS], int32_t* sums_cancel) {
    if (!main || !prep || !challenges || !report || !sums_cancel) VG_FAIL(ctx, "check_witness: null argument");
    VG_TRY(vg_check_machine(ctx, "check_witness", main, prep));
    VgMachineCheck mc(ctx, main, prep, challenges, true);
    VG_TRY(vg_enter(ctx));
    VG_TRY(mc.alloc());
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) {
        VgMat perm;                                   // back to the cache once the sweep that reads it is enqueued
        VG_TRY(mc.perm(i, &perm));
        VG_TRY(mc.sweep(i, perm.get()));
    }
    uint32_t sums[VGPU_NUM_CHIPS][5];
    VG_TRY(mc.finish(sums, report));
    *sums_cancel = vg_sums_cancel(report) ? 1 : 0;
    return 0;
}

extern "C" int32_t vgpu_chip_constraint_count(const vgpu_chip_desc* chip, uint32_t* air_constraints, uint32_t* total) {
    if (!vg_chip_ok(chip) || !air_constraints || !total) return -1;
    *air_constraints = vg_chip_base_constraints(chip->chip_id);
    *total = vg_chip_constraints(chip);
    return 0;
}

// Per rank, [total, failures per constraint] (u64 words), all-gathered when the chip is split; then the ranks' lists, gathered.  Rank
// r's entries are rows of its run, below rank r + 1's: the list is the ranks' lists in rank order.
extern "C" int32_t vgpu_check_failures(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep_or_null,
                                       const vgpu_dmat* perm, const uint32_t challenges[15], uint64_t cap, vgpu_check_failure* out,
                                       uint64_t* n_out, uint64_t* total_failures, uint64_t* rows_per_constraint) {
    if (!n_out || !total_failures || (cap && !out)) VG_FAIL(ctx, "check_failures: null output");
    if (!chip || !main || !perm || !challenges) VG_FAIL(ctx, "check_failures: null argument");
    VG_TRY(vg_check_shapes(ctx, chip, main, prep_or_null, perm, true));
    VG_TRY(vg_enter(ctx));
    const uint32_t nc = vg_chip_constraints(chip);
    const VgRun run = vg_trace_run(ctx, main->gh);
    const uint32_t N = run.split ? (uint32_t)ctx->comm_size : 1, me = run.split ? (uint32_t)ctx->comm_rank : 0;
    // the run's sweep of its rows but the last, then the window of the last row, when split; else one sweep of the whole trace
    const uint32_t ctas = (uint32_t)((run.count - run.split + 127) / 128) + run.split;
    const uint64_t words = 2 * (1 + (uint64_t)nc);
    CheckSet set(ctx, 1);
    set.plan(0, chip, main->gh);
    VG_TRY(set.alloc());
    VgBuf counts(ctx), cta(ctx), off(ctx), endb(ctx);
    VG_TRY(counts.alloc(N * words * 4));
    VG_TRY(cta.alloc(ctas * 4ull));
    VG_TRY(off.alloc(ctas * 8ull));
    VG_TRY(endb.alloc(4));
    unsigned long long* mine = counts.as<unsigned long long>() + (uint64_t)me * (1 + nc);
    VG_CUDA(ctx, cudaMemsetAsync(mine, 0, words * 4, ctx->stream));
    VG_CUDA(ctx, cudaMemsetAsync(cta.p, 0, ctas * 4ull, ctx->stream));
    std::vector<std::unique_ptr<FParams>> sweeps;
    uint32_t used = 0;
    auto pass1 = [&](const vgpu_chip_desc* d, CParams& p) -> int32_t {
        if (!p.n) return 0;
        auto f = std::make_unique<FParams>();
        f->c = p;
        VG_TRY(vg_build_devchip(ctx, d, challenges, &f->c.chip));
        f->cta_count = cta.as<uint32_t>(); f->cta_off = off.as<unsigned long long>(); f->hist = mine + 1; f->cta0 = used;
        const uint32_t blocks = (uint32_t)((p.n + 127) / 128);
        used += blocks;
        KScope ks(ctx, KC_CHECK, 4.0 * (double)p.n * (double)(d->width + d->preprocessed_width + 5.0 * (d->n_interactions + 1)));
        air::with_chip(d->chip_id, [&](auto c) { fail_count_kernel<decltype(c)::value><<<blocks, 128, 0, ctx->stream>>>(*f); });
        VG_LAUNCH_CHECK(ctx);
        sweeps.push_back(std::move(f));
        return 0;
    };
    VG_TRY(set.sweep(0, main, prep_or_null, perm, challenges, pass1));
    VG_TRY(set.windows(challenges, pass1));
    VG_TRY(vg_cta_scan(ctx, cta.as<uint32_t>(), used, cap, off.as<unsigned long long>(), mine, endb.as<uint32_t>()));
    if (run.split) VG_TRY(vg_comm_allgather_inplace(ctx, counts.as<uint32_t>(), words));
    std::vector<unsigned long long> hc((size_t)N * (1 + nc));
    uint32_t end = 0;
    VG_CUDA(ctx, cudaMemcpyAsync(hc.data(), counts.p, hc.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaMemcpyAsync(&end, endb.p, 4, cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    std::vector<uint64_t> found(N);
    uint64_t total = 0;
    for (uint32_t r = 0; r < N; r++) total += found[r] = hc[(size_t)r * (1 + nc)];
    VG_TRY(vg_gather_lists(ctx, run.split, found, cap, [&](vgpu_check_failure* slot) -> int32_t {
        for (auto& f : sweeps) {
            if (end <= f->cta0) break;
            f->out = slot; f->cap = cap;
            const FParams& fp = *f;
            const uint32_t grid = std::min<uint32_t>(end - f->cta0, (uint32_t)((f->c.n + 127) / 128));
            KScope ks(ctx, KC_CHECK, 0.0);
            air::with_chip(chip->chip_id, [&](auto c) { fail_write_kernel<decltype(c)::value><<<grid, 128, 0, ctx->stream>>>(fp); });
            VG_LAUNCH_CHECK(ctx);
        }
        return 0;
    }, out, cap, n_out));
    *total_failures = total;
    if (rows_per_constraint)
        for (uint32_t c = 0; c < nc; c++) {
            uint64_t s = 0;
            for (uint32_t r = 0; r < N; r++) s += hc[(size_t)r * (1 + nc) + 1 + c];
            rows_per_constraint[c] = s;
        }
    return 0;
}
