// The pieces the single-cell witness reports share: vgpu_free_cells (free.cu) and vgpu_cell_alternatives (alts.cu).
//   - F4 and VgLanes: a row's Air::eval with 4-lane values, the cell under test at +0, +1, +2 and +3 and every other cell broadcast;
//   - VgBusMasks: what the bus events of a row read: every count's columns and, on a row whose count m is not 0, m's fields' columns
//     (a kernel ORs in the fields' masks of the counts that are not 0 on its row);
//   - vg_edge_rows: a split run's row before its first row and row after its last, from one all-gather of every rank's first and last
//     main rows (packed by check_copy_kernel; no peer pointers: a borrowed shard is caller memory).
#pragma once
#include "ctx.h"
#include "devchip.h"
#include "airs.cuh"
#include "logup.cuh"

namespace {

constexpr int CELLS_MAX_COLS = 128;

// one expression's value with the cell under test at +0, +1, +2 and +3 (Montgomery)
struct F4 {
    uint32_t v[4];
};
BB_HD F4 operator+(const F4& a, const F4& b) { return F4{{bb::add(a.v[0], b.v[0]), bb::add(a.v[1], b.v[1]), bb::add(a.v[2], b.v[2]), bb::add(a.v[3], b.v[3])}}; }
BB_HD F4 operator-(const F4& a, const F4& b) { return F4{{bb::sub(a.v[0], b.v[0]), bb::sub(a.v[1], b.v[1]), bb::sub(a.v[2], b.v[2]), bb::sub(a.v[3], b.v[3])}}; }
BB_HD F4 operator*(const F4& a, const F4& b) { return F4{{bb::mul(a.v[0], b.v[0]), bb::mul(a.v[1], b.v[1]), bb::mul(a.v[2], b.v[2]), bb::mul(a.v[3], b.v[3])}}; }

}  // namespace

namespace air {
template <> struct Lift<F4> { static BB_HD F4 from_monty_word(uint32_t m) { return F4{{m, m, m, m}}; } };
}  // namespace air

namespace {

// The reads of a builder over F4; a builder adds z() and its state.
struct VgLanes {
    using V = F4;
    const uint32_t* lrow; uint64_t lcs;             // the evaluated row and its next row, each with its column stride
    const uint32_t* nrow; uint64_t ncs;
    V first, last, trans;
    int tl, tn;                                     // the column under test as L(c) / as N(c) (-1: none)
    __device__ __forceinline__ static V at(uint32_t x, bool test) {
        if (!test) return V{{x, x, x, x}};
        const uint32_t x1 = bb::add(x, bb::R1), x2 = bb::add(x1, bb::R1);
        return V{{x, x1, x2, bb::add(x2, bb::R1)}};
    }
    __device__ __forceinline__ V L(int c) const { return at(__ldg(lrow + (uint64_t)c * lcs), c == tl); }
    __device__ __forceinline__ V N(int c) const { return at(__ldg(nrow + (uint64_t)c * ncs), c == tn); }
    __device__ __forceinline__ void section(const char*) {}
};

struct VgBusMasks {
    uint64_t count_cols[2];                         // columns some interaction's count gives a non-zero weight (bit c % 64 of word c / 64)
    uint64_t fields[VGPU_MAX_INTERACTIONS][2];      // columns interaction m's fields give a non-zero weight
    DevPairCol count[VGPU_MAX_INTERACTIONS];
};
static_assert(sizeof(VgBusMasks) % 8 == 0, "no tail padding: a kernel's parameters keep their offsets");

// the main columns a VirtualPairCol gives a non-zero summed weight (preprocessed terms are the verifier's)
inline void vg_weighted_columns(const vgpu_pair_col& pc, uint64_t mask[2]) {
    uint64_t sum[CELLS_MAX_COLS] = {};
    for (uint32_t t = 0; t < pc.n_terms && t < VGPU_MAX_TERMS; t++)
        if (!pc.terms[t].is_preprocessed && pc.terms[t].column < CELLS_MAX_COLS)
            sum[pc.terms[t].column] = (sum[pc.terms[t].column] + pc.terms[t].weight % bb::P) % bb::P;
    for (uint32_t c = 0; c < CELLS_MAX_COLS; c++)
        if (sum[c]) mask[c >> 6] |= 1ull << (c & 63);
}

inline int32_t vg_bus_masks(vgpu_ctx* ctx, const vgpu_chip_desc* chip, VgBusMasks* m) {
    auto dev = std::make_unique<DevChip>();
    const uint32_t no_challenges[15] = {};
    VG_TRY(vg_build_devchip(ctx, chip, no_challenges, dev.get()));
    for (uint32_t i = 0; i < chip->n_interactions; i++) {
        const vgpu_interaction& it = chip->interactions[i];
        vg_weighted_columns(it.count, m->count_cols);
        for (uint32_t f = 0; f < it.n_fields; f++) vg_weighted_columns(it.fields[f], m->fields[i]);
        m->count[i] = dev->interactions[i].count;
    }
    return 0;
}

// The rows around this rank's run (local row 0 at `rows`, column stride mcs, `count` rows, w columns): the row before local row 0
// (before, bcs) and the row after the last (after, acs).  Split: one all-gather of [first row | last row] per rank into `edges`; else
// the trace's wrap-around rows.
inline int32_t vg_edge_rows(vgpu_ctx* ctx, const VgRun& run, const uint32_t* rows, uint64_t mcs, uint64_t h, uint32_t w, VgBuf& edges,
                            const uint32_t** before, uint64_t* bcs, const uint32_t** after, uint64_t* acs) {
    if (!run.split) {
        *before = rows + h - 1; *bcs = mcs;
        *after = rows; *acs = mcs;
        return 0;
    }
    const uint32_t N = (uint32_t)ctx->comm_size, me = (uint32_t)ctx->comm_rank;
    VG_TRY(edges.alloc((size_t)N * 2 * w * 4));
    uint32_t* blk = edges.as<uint32_t>() + (uint64_t)me * 2 * w;
    const VgCopySeg segs[2] = {{rows, mcs, blk, 1, w}, {rows + run.count - 1, mcs, blk + w, 1, w}};
    VG_TRY(vg_copy_segments(ctx, segs, 2));
    VG_TRY(vg_comm_allgather_inplace(ctx, edges.as<uint32_t>(), 2 * (uint64_t)w));
    // the row before ours is the previous rank's last, the row after the next's first
    *before = edges.as<uint32_t>() + (uint64_t)((me + N - 1) % N) * 2 * w + w; *bcs = 1;
    *after = edges.as<uint32_t>() + (uint64_t)((me + 1) % N) * 2 * w; *acs = 1;
    return 0;
}

}  // namespace
