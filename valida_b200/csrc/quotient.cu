// K6 + K7 — fused constraint / quotient sweep with the chunk split, one kernel per chip.
// Replaces quotient() / quotient_values() (machine/src/quotient.rs:18-238), ProverConstraintFolder
// (machine/src/folding_builder.rs:32-125), eval_permutation_constraints (machine/src/chip.rs:210-289)
// and p3-uni-stark's decompose_and_flatten / ZerofierOnCoset for log_quotient_degree = 1.
//
// The reference gathers LDE rows through a bit-reversed view element by element; here one thread owns
// one STORAGE row of the committed (bit-reversed) LDEs; lanes (2r, 2r+1) hold the natural rows
// (j, j+h) with j = bitrev(r): x and -x.  That pair is exactly what the even/odd chunk split needs,
// so the quotient values never touch HBM: each lane folds all constraints of its row, divides by Z_H,
// the pair exchanges its ext5 value with one shuffle, and the even / odd lane writes the even / odd
// chunk limbs.  Every trace load and every chunk store is a fully coalesced 4-byte-per-lane access
// (the chunk matrix is left in bit-reversed row order; the quotient commit's iNTT reads it that way).
// (A pair per thread with a natural-order scatter, the first version, moved several times the algorithmic bytes.)
// alpha-folding: acc = sum_i c_i * alpha^(N-1-i) with precomputed powers — the same value as the
// reference's Horner recurrence acc = acc*alpha + c_i, at 5 instead of 25 multiplications for the
// base-field constraints.  The sum is accumulated LAZILY (bb::Lazy5: raw 64-bit products, one IMAD.WIDE
// per limb and constraint, a fold every fourth) and reduced once per row; the powers sit in the kernel
// parameters (constant bank), so a base-field constraint costs ~7 instructions instead of 50.
// The selectors need 1/((x-1)(x-g^-1)) on both rows of a pair: the product over the pair is symmetric,
// vg_selector_inverses() inverts it for every pair of a height with the Montgomery batch trick (one
// Fermat inversion per 8 pairs) instead of one Fermat inversion (~46 multiplications) per row.
#include "ctx.h"
#include "devchip.h"
#include "airs.cuh"
#include "logup.cuh"
#include <cstring>
#include <memory>

namespace {

using bb::E5;
using air::F;

constexpr uint32_t Q_MAX_CONSTRAINTS = 128;   // bitwise: 88 base + interactions + 3

struct QParams {
    // Base pointers are VIRTUAL: base + (global storage row) is the element, whether the matrix is whole or this rank's row
    // shard (then base = shard - first row).  The *_n bases serve the "next" rows: natural row i + 2 of every row of the launch's
    // range lies in ONE rank's shard (vgpu_quotient's next-row table), read through its peer pointer over NVLink.
    const uint32_t* main; const uint32_t* main_n; uint64_t mcs;
    const uint32_t* prep; const uint32_t* prep_n; uint64_t pcs;
    const uint32_t* perm; const uint32_t* perm_n; uint64_t qcs;
    uint32_t* out; uint64_t ocs;            // h x 10 chunk matrix (virtual base: + chunk row)
    const uint32_t* selinv;                 // selinv[r] = 1 / ((x-1)(x-glast)(-x-1)(-x-glast)), x = s * w^bitrev(r)  (virtual base: + pair)
    uint32_t log_h;
    uint64_t row_begin, row_end;            // storage rows of the LDE swept by this launch (a rank's range when the sweep is split)
    uint32_t s;                             // coset shift (Montgomery)
    uint32_t glast;                         // g_subgroup^-1
    uint32_t zh[2], zinv[2];                // Z_H on even / odd natural rows, and inverses
    uint32_t odd_scale;                     // 1 / (2 s)
    uint32_t half;                          // 1 / 2
    E5 cumsum;
    const uint32_t* root_lo; const uint32_t* root_hi;
    uint32_t apow[Q_MAX_CONSTRAINTS][5];    // apow[i] = alpha^(N-1-i)
    DevChip chip;                           // interaction descriptors + LogUp randomness: read through the constant bank (uniform loads),
                                            // not through dependent global loads (ncu r1b: 27-54 % of the stall samples sat on those);
                                            // staging them in shared memory instead measured 6 % slower (9.08 vs 8.57 ms per proof)
};

struct DevBuilder {
    using V = air::F;
    const uint32_t* lrow; const uint32_t* nrow; uint64_t cs;   // pointers already offset to the row
    F first, last, trans;
    const uint32_t (*apow)[5]; uint32_t idx; bb::Lazy5 acc;
    __device__ __forceinline__ F L(int c) const { return F{__ldg(lrow + (uint64_t)c * cs)}; }
    __device__ __forceinline__ F N(int c) const { return F{__ldg(nrow + (uint64_t)c * cs)}; }
    __device__ __forceinline__ E5 pw() const { E5 a; for (int l = 0; l < 5; l++) a.c[l] = apow[idx][l]; return a; }
    __device__ __forceinline__ void z(F x) { acc.fma_base(pw(), x.v); idx++; }
    __device__ __forceinline__ void z_ext(const E5& x) { acc.fma_ext(pw(), x, bb::e5_dbl(x)); idx++; }
    __device__ __forceinline__ void section(const char*) {}
};

__device__ __forceinline__ uint32_t qroot_pow(const QParams& p, uint64_t e) {
    return vg_pow_lookup(p.root_lo, p.root_hi, e & ((1ull << VG_LOG_NMAX) - 1));
}
// Resident-CTA target (register cap) of the sweep.  It is latency bound (ncu r1b: issue slots 43-57 % busy at 5 CTAs per
// SM), so more resident warps beat fewer spills: measured 11.4 / 8.9 / 8.6 ms per proof at 2-4 / 6 / 8 CTAs per SM.
constexpr int QUOTIENT_MINB = 8;
template <int CHIP>
__global__ void __launch_bounds__(128, QUOTIENT_MINB) quotient_kernel(const __grid_constant__ QParams p) {
    const uint64_t h = 1ull << p.log_h, H = 2 * h;
    const uint64_t rho_raw = p.row_begin + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;     // storage row of the committed LDEs
    const bool active = rho_raw < p.row_end;
    const uint64_t rho = active ? rho_raw : p.row_begin + (rho_raw & 1);           // idle lanes shadow the first pair of the range (shuffles need every lane)
    const uint32_t e = (uint32_t)(rho & 1);                                        // 0: x = +x0 (natural row j), 1: x = -x0 (natural row j + h)
    const uint64_t r = rho >> 1;
    const uint32_t j = bb::reverse_bits((uint32_t)r, (int)p.log_h);
    // next row: natural (i + 2) mod 2h  ->  pair bitrev((j + 2) mod h), element e ^ carry
    const uint64_t t = (uint64_t)j + 2;
    const uint32_t a = (uint32_t)(t & (h - 1));
    const uint32_t swap = (uint32_t)((t >> p.log_h) & 1);
    const uint64_t nrow = 2 * (uint64_t)bb::reverse_bits(a, (int)p.log_h) + (e ^ swap);
    const uint32_t x0 = bb::mul(p.s, qroot_pow(p, (uint64_t)j << (VG_LOG_NMAX - p.log_h - 1)));
    const uint32_t x = e ? bb::neg(x0) : x0;
    // selectors 1/(x-1), 1/(x-glast): both lanes of a pair invert the same symmetric product
    uint32_t inv_first, inv_last;
    {
        const uint32_t nx0 = bb::neg(x0);
        const uint32_t d0 = bb::sub(x0, bb::R1), d1 = bb::sub(x0, p.glast), d2 = bb::sub(nx0, bb::R1), d3 = bb::sub(nx0, p.glast);
        const uint32_t p01 = bb::mul(d0, d1), p23 = bb::mul(d2, d3);
        const uint32_t all = __ldg(p.selinv + r);
        const uint32_t i01 = bb::mul(all, p23), i23 = bb::mul(all, p01);
        inv_first = e ? bb::mul(i23, d3) : bb::mul(i01, d1);
        inv_last = e ? bb::mul(i23, d2) : bb::mul(i01, d0);
    }
    const DevChip& chip = p.chip;
    const uint32_t parity = (uint32_t)(((uint64_t)j + (e ? h : 0)) & 1);
    const uint32_t zh = p.zh[parity];
    DevBuilder b;
    b.lrow = p.main + rho; b.nrow = p.main_n + nrow; b.cs = p.mcs;
    b.first = F{bb::mul(zh, inv_first)};
    b.last = F{bb::mul(zh, inv_last)};
    b.trans = F{bb::sub(x, p.glast)};
    b.apow = p.apow; b.idx = 0; b.acc.init();
    air::eval_chip<CHIP>(b);
    logup::eval_constraints(b, chip, b.lrow, b.nrow, p.mcs, p.prep ? p.prep + rho : nullptr, p.prep ? p.prep_n + nrow : nullptr, p.pcs,
                            p.perm + rho, p.perm_n + nrow, p.qcs, p.cumsum);
    const E5 q = bb::e5_mul_base(b.acc.value(), p.zinv[parity]);
    // decompose_and_flatten across the lane pair: even = (q(x) + q(-x))/2, odd = (q(x) - q(-x)) / (2 s g^j)
    E5 other;
#pragma unroll
    for (int l = 0; l < 5; l++) other.c[l] = __shfl_xor_sync(0xffffffffu, q.c[l], 1);
    E5 outv;
    if (e == 0) {
        outv = bb::e5_mul_base(bb::e5_add(q, other), p.half);
    } else {
        const uint32_t ginv_j = qroot_pow(p, (1ull << VG_LOG_NMAX) - ((uint64_t)j << (VG_LOG_NMAX - p.log_h - 1)));
        outv = bb::e5_mul_base(bb::e5_sub(other, q), bb::mul(p.odd_scale, ginv_j));
    }
    if (active) {
        // chunk row j is written at row r = bitrev(j): the chunk matrix leaves this kernel in bit-reversed row order
        // (coalesced), which the commit's inverse transform consumes directly
#pragma unroll
        for (int l = 0; l < 5; l++) p.out[(uint64_t)(5 * e + l) * p.ocs + r] = outv.c[l];
    }
}

// selinv[r] = 1 / ((x0-1)(x0-glast)(-x0-1)(-x0-glast)), x0 = s * w_2h^bitrev(r), for the pairs [begin, begin + count).
// Montgomery batch trick over SEL_BATCH pairs per thread, pairs of one thread a grid apart (coalesced).
constexpr int SEL_BATCH = 8;
__global__ void __launch_bounds__(256) selector_inverse_kernel(uint32_t* __restrict__ out, uint64_t begin, uint64_t count, uint32_t log_h, uint32_t s, uint32_t glast,
                                                               const uint32_t* __restrict__ root_lo, const uint32_t* __restrict__ root_hi) {
    const uint64_t stride = (count + SEL_BATCH - 1) / SEL_BATCH;
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= stride) return;
    uint32_t v[SEL_BATCH], pref[SEL_BATCH];
    uint32_t acc = bb::R1;
#pragma unroll
    for (int i = 0; i < SEL_BATCH; i++) {
        const uint64_t r = begin + t + (uint64_t)i * stride;
        v[i] = bb::R1;
        if (t + (uint64_t)i * stride < count) {
            const uint32_t j = bb::reverse_bits((uint32_t)r, (int)log_h);
            const uint64_t e = ((uint64_t)j << (VG_LOG_NMAX - log_h - 1)) & ((1ull << VG_LOG_NMAX) - 1);
            const uint32_t x0 = bb::mul(s, vg_pow_lookup(root_lo, root_hi, e));
            const uint32_t nx0 = bb::neg(x0);
            v[i] = bb::mul(bb::mul(bb::sub(x0, bb::R1), bb::sub(x0, glast)), bb::mul(bb::sub(nx0, bb::R1), bb::sub(nx0, glast)));
        }
        pref[i] = acc;
        acc = bb::mul(acc, v[i]);
    }
    uint32_t inv = bb::inv(acc);
#pragma unroll
    for (int i = SEL_BATCH - 1; i >= 0; i--) {
        if (t + (uint64_t)i * stride < count) out[begin + t + (uint64_t)i * stride] = bb::mul(inv, pref[i]);
        inv = bb::mul(inv, v[i]);
    }
}

struct CountBuilder {
    using V = air::F;
    F first{0}, last{0}, trans{0};
    uint32_t n = 0;
    BB_HD F L(int) const { return F{0}; }
    BB_HD F N(int) const { return F{0}; }
    BB_HD void z(F) { n++; }
    BB_HD void section(const char*) {}
};

}  // namespace

uint32_t vg_chip_base_constraints(uint32_t chip_id) {
    CountBuilder c;
    air::with_chip(chip_id, [&](auto chip) { air::eval_chip<decltype(chip)::value>(c); });
    return c.n;
}

extern "C" int32_t vgpu_quotient(vgpu_ctx* ctx, const vgpu_chip_desc* chip, uint32_t log_degree, const vgpu_dmat* prep_lde,
                                 const vgpu_dmat* main_lde, const vgpu_dmat* perm_lde, const uint32_t cumulative_sum[5],
                                 const uint32_t perm_challenges[15], const uint32_t alpha[5], vgpu_dmat** out_chunks) {
    if (!chip || !main_lde || !perm_lde || !out_chunks) VG_FAIL(ctx, "quotient: null argument");
    VG_TRY(vg_enter(ctx));
    const uint64_t h = 1ull << log_degree;
    if (main_lde->gh != 2 * h || perm_lde->gh != 2 * h) VG_FAIL(ctx, "quotient: LDE height must be 2 * 2^log_degree");
    if (main_lde->gw != chip->width || perm_lde->gw != 5 * (chip->n_interactions + 1)) VG_FAIL(ctx, "quotient: LDE width does not match the chip");
    if (chip->chip_id >= VGPU_NUM_CHIPS) VG_FAIL(ctx, "quotient: unknown chip id %u", chip->chip_id);
    // split proof: the committed LDEs of a tall chip are row shards (all three the same run of rows), of a short chip whole
    const bool split = main_lde->dist == VG_ROWS;
    if ((perm_lde->dist == VG_ROWS) != split || (prep_lde && (prep_lde->dist == VG_ROWS) != split)) VG_FAIL(ctx, "quotient: the LDEs are not distributed alike");
    // alpha powers for N = base + k + 3 constraints
    const uint32_t N = vg_chip_constraints(chip);
    if (N > Q_MAX_CONSTRAINTS) { VG_FAIL(ctx, "quotient: %u constraints exceed the parameter table (%u)", N, Q_MAX_CONSTRAINTS); }
    auto pp = std::make_unique<QParams>();
    QParams& p = *pp;
    std::memset(&p, 0, sizeof p);
    VG_TRY(vg_build_devchip(ctx, chip, perm_challenges, &p.chip));
    E5 al; for (int i = 0; i < 5; i++) al.c[i] = bb::to_monty(alpha[i] % bb::P);
    { E5 a = bb::e5_one(); for (uint32_t i = 0; i < N; i++) { for (int l = 0; l < 5; l++) p.apow[N - 1 - i][l] = a.c[l]; a = bb::e5_mul(a, al); } }
    p.row_begin = split ? main_lde->row0 : 0;
    p.row_end = split ? main_lde->row0 + main_lde->h : 2 * h;
    if ((p.row_begin & 1) || (p.row_end & 1)) VG_FAIL(ctx, "quotient: a row shard must hold whole (x, -x) pairs");
    // The next-row table: the 2h storage rows are V units (ctx.h); unit u holds the rows of natural index i = bitrev(u) mod V, so the
    // next rows (i + 2) of all its rows lie in unit bitrev((bitrev(u) + 2) mod V), which one rank holds.  Consecutive units of this
    // rank's run whose next rows one rank holds form one launch: a single launch at a power-of-two comm_size (every unit of a run
    // then names the same rank), at most one per unit otherwise.  next_rank[k]: the rank holding the next rows of local range k.
    std::vector<uint64_t> range_end;             // storage rows: range k is [range_end[k - 1] (or row_begin), range_end[k])
    std::vector<int> next_rank;
    if (!split) { range_end.push_back(p.row_end); next_rank.push_back(ctx->comm_rank); }
    else {
        const int G = ctx->comm_size;
        const uint64_t V = vg_units(G), urows = 2 * h / V;
        int lgv = 0; while ((1ull << lgv) < V) lgv++;
        if (p.row_begin % urows || p.row_end % urows) VG_FAIL(ctx, "quotient: a row shard must hold whole units");
        for (uint64_t u = p.row_begin / urows; u < p.row_end / urows; u++) {
            const uint32_t un = bb::reverse_bits((bb::reverse_bits((uint32_t)u, lgv) + 2) & (uint32_t)(V - 1), lgv);
            int d = 0;
            while (vg_unit_begin(G, d + 1) <= un) d++;
            if (!next_rank.empty() && next_rank.back() == d) range_end.back() = (u + 1) * urows;
            else { range_end.push_back((u + 1) * urows); next_rank.push_back(d); }
        }
    }
    // virtual bases of a matrix: local rows, and the rows of rank d
    auto base_of = [&](const vgpu_dmat* m) { return m->d - (split ? m->row0 : 0); };
    auto next_of = [&](const vgpu_dmat* m, int d) -> const uint32_t* {
        if (!split || d == ctx->comm_rank) return base_of(m);
        if (!m->symm) return nullptr;
        return vg_peer_ptr(ctx, m->d, d) - vg_run_bound(m->gh, ctx->comm_size, d);
    };
    for (int d : next_rank)
        if (!next_of(main_lde, d) || !next_of(perm_lde, d) || (prep_lde && !next_of(prep_lde, d)))
            VG_FAIL(ctx, "quotient: a row shard read by a peer must live in the symmetric heap");
    VgMat out;
    VG_TRY(vg_dmat_alloc_run(ctx, h, 10, split, false, &out));
    out->bitrev_rows = true;
    p.main = base_of(main_lde); p.mcs = main_lde->col_stride;
    p.prep = prep_lde ? base_of(prep_lde) : nullptr; p.pcs = prep_lde ? prep_lde->col_stride : 0;
    p.perm = base_of(perm_lde); p.qcs = perm_lde->col_stride;
    p.out = out->d - p.row_begin / 2; p.ocs = out->col_stride;
    p.log_h = log_degree;
    p.s = bb::to_monty(bb::GEN_CANON);
    uint32_t g_sub = bb::two_adic_generator_monty((int)log_degree);
    p.glast = bb::inv(g_sub);
    uint32_t s_pow_n = p.s;
    for (uint32_t i = 0; i < log_degree; i++) s_pow_n = bb::sqr(s_pow_n);
    p.zh[0] = bb::sub(s_pow_n, bb::R1);
    p.zh[1] = bb::sub(bb::neg(s_pow_n), bb::R1);
    p.zinv[0] = bb::inv(p.zh[0]); p.zinv[1] = bb::inv(p.zh[1]);
    p.half = bb::inv(bb::to_monty(2));
    p.odd_scale = bb::mul(p.half, bb::inv(p.s));
    for (int i = 0; i < 5; i++) p.cumsum.c[i] = bb::to_monty(cumulative_sum[i] % bb::P);
    p.root_lo = ctx->root_table.lo; p.root_hi = ctx->root_table.hi;
    const uint64_t pb = p.row_begin / 2, pc = (p.row_end - p.row_begin) / 2;     // pairs swept here
    VgBuf selinv(ctx);
    VG_TRY(selinv.alloc(pc * 4));
    p.selinv = selinv.as<uint32_t>() - pb;
    {
        KScope ks(ctx, KC_QUOTIENT, 4.0 * (double)(p.row_end - p.row_begin) * (main_lde->gw + perm_lde->gw + (prep_lde ? prep_lde->gw : 0)) + 20.0 * (double)(p.row_end - p.row_begin));
        const uint64_t stride = (pc + SEL_BATCH - 1) / SEL_BATCH;
        selector_inverse_kernel<<<(unsigned)((stride + 255) / 256), 256, 0, ctx->stream>>>(selinv.as<uint32_t>() - pb, pb, pc, log_degree, p.s, p.glast, p.root_lo, p.root_hi);
        ctx->launches++;
        const uint64_t row_begin = p.row_begin, row_end = p.row_end;
        for (size_t k = 0; k < next_rank.size(); k++) {
            p.row_begin = k ? range_end[k - 1] : row_begin; p.row_end = range_end[k];
            p.main_n = next_of(main_lde, next_rank[k]); p.prep_n = prep_lde ? next_of(prep_lde, next_rank[k]) : nullptr; p.perm_n = next_of(perm_lde, next_rank[k]);
            air::with_chip(chip->chip_id, [&](auto c) {
                quotient_kernel<decltype(c)::value><<<(unsigned)((p.row_end - p.row_begin + 127) / 128), 128, 0, ctx->stream>>>(p);
            });
        }
        p.row_begin = row_begin; p.row_end = row_end;
    }
    selinv.reset();
    VG_LAUNCH_CHECK(ctx);
    *out_chunks = out.release();
    return 0;
}
