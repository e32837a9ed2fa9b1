// check_constraints (machine/src/check_constraints.rs:14-84; debug builds of the reference's prove, derive/src/lib.rs:246-253) on the
// device: every constraint of a chip's Air::eval and of eval_permutation_constraints on every row i of the TRACE, with row (i+1) mod h
// as "next" and the debug selectors is_first_row = [i == 0], is_last_row = [i == h-1], is_transition = 1 - is_last_row.
// One thread per natural trace row reads the column-major traces (coalesced) through the same AIR text as the quotient sweep
// (airs.cuh, logup.cuh), so constraint i here is constraint i there: the chip's assertions in eval order, one per interaction,
// then the LogUp transition, first-row and last-row constraints.  The cumulative sum is read on the device from the permutation
// trace's last row and last column (check_constraints.rs:33).
// Result per chip: the first failing (row, constraint) as ONE 64-bit key (row << 8 | constraint, atomicMin) and the number of rows
// with at least one failure; both are aggregated per warp, so a clean trace costs no atomic at all.
#include "ctx.h"
#include "devchip.h"
#include "airs.cuh"
#include "logup.cuh"
#include "open.h"
#include <memory>

namespace {

using bb::E5;
using air::F;

constexpr uint32_t CHECK_NONE = 0xffffffffu;
constexpr uint32_t CHECK_MAX_CONSTRAINTS = 256;   // the constraint index takes the low 8 bits of the key

struct CParams {
    const uint32_t* main; uint64_t mcs;
    const uint32_t* prep; uint64_t pcs;             // null without a preprocessed trace
    const uint32_t* perm; uint64_t qcs;             // flattened permutation trace, h x 5(k+1)
    uint64_t h;
    unsigned long long* first;                      // min over failing rows of (row << 8 | first failing constraint); ~0: none
    unsigned long long* count;                      // rows with at least one failing constraint
    DevChip chip;
};

struct CheckBuilder {
    using V = air::F;
    const uint32_t* lrow; const uint32_t* nrow; uint64_t cs;   // pointers already offset to the row
    F first, last, trans;
    uint32_t idx, bad;                                         // next constraint index; first one that did not vanish
    __device__ __forceinline__ F L(int c) const { return F{__ldg(lrow + (uint64_t)c * cs)}; }
    __device__ __forceinline__ F N(int c) const { return F{__ldg(nrow + (uint64_t)c * cs)}; }
    __device__ __forceinline__ void z(F x) { if (x.v != 0 && bad == CHECK_NONE) bad = idx; idx++; }
    __device__ __forceinline__ void z_ext(const E5& x) { if (!bb::e5_is_zero(x) && bad == CHECK_NONE) bad = idx; idx++; }
};

template <int CHIP>
__global__ void __launch_bounds__(128) check_kernel(const __grid_constant__ CParams p) {
    const uint64_t i_raw = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = i_raw < p.h;
    const uint64_t i = active ? i_raw : p.h - 1;          // idle lanes shadow the last row (the warp vote needs every lane)
    const bool is_last = i + 1 == p.h;
    const uint64_t n = is_last ? 0 : i + 1;                // a one-row chip is its own next row
    CheckBuilder b;
    b.lrow = p.main + i; b.nrow = p.main + n; b.cs = p.mcs;
    b.first = F{i == 0 ? bb::R1 : 0u};
    b.last = F{is_last ? bb::R1 : 0u};
    b.trans = F{is_last ? 0u : bb::R1};
    b.idx = 0; b.bad = CHECK_NONE;
    air::eval_chip<CHIP>(b);
    const uint32_t k = p.chip.n_interactions;
    E5 cumsum;
#pragma unroll
    for (int l = 0; l < 5; l++) cumsum.c[l] = __ldg(p.perm + (uint64_t)(5 * k + l) * p.qcs + p.h - 1);
    logup::eval_constraints(b, p.chip, b.lrow, b.nrow, p.mcs, p.prep ? p.prep + i : nullptr, p.prep ? p.prep + n : nullptr, p.pcs,
                            p.perm + i, p.perm + n, p.qcs, cumsum);
    const bool fail = active && b.bad != CHECK_NONE;
    const unsigned vote = __ballot_sync(0xffffffffu, fail);
    // the lowest failing lane holds the warp's lowest row, hence its smallest key
    if (vote && (threadIdx.x & 31) == (unsigned)(__ffs(vote) - 1)) {
        atomicMin(p.first, ((unsigned long long)i << 8) | b.bad);
        atomicAdd(p.count, (unsigned long long)__popc(vote));
    }
}

}  // namespace

// Validates the arguments (before anything is enqueued) and enqueues the sweep of one chip.  d_first / d_count must hold ~0 / 0.
int32_t vg_check_enqueue(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep, const vgpu_dmat* perm,
                         const uint32_t challenges[15], unsigned long long* d_first, unsigned long long* d_count) {
    if (!chip || !main || !perm || !challenges) VG_FAIL(ctx, "check_constraints: null argument");
    if (chip->chip_id >= VGPU_NUM_CHIPS) VG_FAIL(ctx, "check_constraints: unknown chip id %u", chip->chip_id);
    for (const vgpu_dmat* m : {main, prep, perm})
        if (m && (m->dist != VG_FULL || m->bitrev_rows)) VG_FAIL(ctx, "check_constraints: whole matrices in natural row order only (not row shards)");
    if (main->gw != chip->width) VG_FAIL(ctx, "check_constraints: main width %llu != chip width %u", (unsigned long long)main->gw, chip->width);
    const uint64_t pw = 5ull * (chip->n_interactions + 1);
    if (perm->gw != pw) VG_FAIL(ctx, "check_constraints: permutation trace width %llu != 5 (k + 1) = %llu", (unsigned long long)perm->gw, (unsigned long long)pw);
    if (chip->preprocessed_width && !prep) VG_FAIL(ctx, "check_constraints: chip %u needs its preprocessed trace (%u columns)", chip->chip_id, chip->preprocessed_width);
    if (!chip->preprocessed_width && prep) VG_FAIL(ctx, "check_constraints: chip %u has no preprocessed trace", chip->chip_id);
    if (prep && prep->gw != chip->preprocessed_width) VG_FAIL(ctx, "check_constraints: preprocessed width %llu != %u", (unsigned long long)prep->gw, chip->preprocessed_width);
    const uint64_t h = main->gh;
    if (h == 0 || (h & (h - 1))) VG_FAIL(ctx, "check_constraints: trace height %llu is not a power of two", (unsigned long long)h);
    if (perm->gh != h || (prep && prep->gh != h)) VG_FAIL(ctx, "check_constraints: the main, preprocessed and permutation traces differ in height");
    const uint32_t N = vg_chip_base_constraints(chip->chip_id) + chip->n_interactions + 3;
    if (N > CHECK_MAX_CONSTRAINTS) VG_FAIL(ctx, "check_constraints: %u constraints exceed the 8-bit index (%u)", N, CHECK_MAX_CONSTRAINTS);
    VG_TRY(vg_dmat_materialize(ctx, main));
    VG_TRY(vg_dmat_materialize(ctx, prep));
    VG_TRY(vg_dmat_materialize(ctx, perm));
    auto pp = std::make_unique<CParams>();
    CParams& p = *pp;
    VG_TRY(vg_build_devchip(ctx, chip, challenges, &p.chip));
    p.main = main->d; p.mcs = main->col_stride;
    p.prep = prep ? prep->d : nullptr; p.pcs = prep ? prep->col_stride : 0;
    p.perm = perm->d; p.qcs = perm->col_stride;
    p.h = h; p.first = d_first; p.count = d_count;
    KScope ks(ctx, KC_CHECK, 4.0 * (double)h * (double)(main->gw + perm->gw + (prep ? prep->gw : 0)));
    air::with_chip(chip->chip_id, [&](auto c) { check_kernel<decltype(c)::value><<<(unsigned)((h + 127) / 128), 128, 0, ctx->stream>>>(p); });
    VG_LAUNCH_CHECK(ctx);
    return 0;
}

void vg_check_decode(const unsigned long long first_count[2], int64_t* row, uint32_t* constraint, uint64_t* failing_rows) {
    const unsigned long long key = first_count[0];
    *row = key == ~0ull ? -1 : (int64_t)(key >> 8);
    *constraint = key == ~0ull ? 0 : (uint32_t)(key & 0xff);
    *failing_rows = first_count[1];
}

extern "C" int32_t vgpu_check_constraints(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep_or_null,
                                          const vgpu_dmat* perm, const uint32_t challenges[15],
                                          int64_t* first_row, uint32_t* first_constraint, uint64_t* failing_rows) {
    if (!first_row || !first_constraint || !failing_rows) VG_FAIL(ctx, "check_constraints: null output");
    VG_TRY(vg_enter(ctx));
    VgBuf buf(ctx);
    VG_TRY(buf.alloc(2 * sizeof(unsigned long long)));
    unsigned long long* d = buf.as<unsigned long long>();
    VG_CUDA(ctx, cudaMemsetAsync(d, 0xff, sizeof(unsigned long long), ctx->stream));
    VG_CUDA(ctx, cudaMemsetAsync(d + 1, 0, sizeof(unsigned long long), ctx->stream));
    VG_TRY(vg_check_enqueue(ctx, chip, main, prep_or_null, perm, challenges, d, d + 1));
    unsigned long long h[2];
    VG_CUDA(ctx, cudaMemcpyAsync(h, d, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    vg_check_decode(h, first_row, first_constraint, failing_rows);
    return 0;
}
