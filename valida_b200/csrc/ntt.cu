// K1/K2 — batched BabyBear NTT / iNTT / coset-LDE over column-major device matrices (sm_90a).
// Replaces p3-dft's TwoAdicSubgroupDft::{dft_batch, idft_batch, coset_lde_batch} as reached from
// TwoAdicFriPcs::commit_shifted_batches (reference call sites derive/src/lib.rs:309,330,355,372;
// DFT selected at basic/src/bin/valida.rs:379).
//
// Design (GPU-first, not the reference's row-major butterfly network):
//  * a length-n column transform is split n = n1*n2 ("four-step"); each pass stages a tile of T
//    sub-transforms of length L in shared memory and runs ALL log2(L) DIF stages there, four stages
//    at a time in registers (radix-16 units: 16 loads, 32 butterflies, 16 stores per thread-unit, one
//    __syncthreads per four stages), so a column crosses HBM twice per transform for n <= 2^24;
//  * element(r, g) = base + r*rs + g*gs; the thread->element map makes the unit-stride index the
//    fastest one in both the load and the store.  Strided ("column") passes keep L <= 2^10 so that
//    T >= 16 adjacent groups give >= 64-byte segments; contiguous ("row") passes take up to 2^14;
//  * bit reversal is never a separate pass: loads/stores may permute within the tile (free in smem),
//    and a column pass may store its tile transposed (T contiguous runs of L);
//  * coset LDE = iNTT natural->bit-reversed coefficients (column pass + row pass, in place) with
//    shift^k/n folded into the store, then two forward coset transforms bit-reversed coefficients ->
//    bit-reversed evaluations (row pass + column pass with transposed store) written straight into
//    the two halves of the committed (bit-reversed) LDE;
//  * twiddles: a two-level power table of w_(2^27) in global memory (L2-resident) feeds a per-CTA
//    shared table of w_L^j.
#include "ctx.h"

namespace {

using bb::mul; using bb::add; using bb::sub;

struct PassParams {
    const uint32_t* src; uint32_t* dst;
    uint64_t src_cs, dst_cs;          // column strides
    uint64_t src_rs, src_gs;          // element(r, g) = col + r*src_rs + g*src_gs
    uint64_t dst_rs, dst_gs;          // output slot pos of group g -> col + pos*dst_rs + g*dst_gs
    uint32_t log_len;                 // L = 2^log_len
    uint32_t tile;                    // T groups per CTA
    uint64_t groups;                  // groups per column (n / L)
    uint32_t inverse;                 // twiddle direction
    uint32_t src_bitrev;              // 1: memory element r holds natural index bitrev(r) (load into slot bitrev(r))
    uint32_t dst_natural;             // 1: natural output k stored at pos = k ; 0: raw DIF order pos = bitrev(k)
    uint32_t g_bits;                  // if nonzero, multipliers see gval = bitrev(g, g_bits) instead of g
    // pre-multiplier: x *= w_NMAX^((rnat*pre_r + gval*pre_g) << pre_shift), rnat = natural index of the element in its group
    uint32_t pre_mode; uint32_t pre_r, pre_g, pre_shift;   // exponent = (rnat*pre_r + gval*pre_g) << pre_shift  (< 2^27)
    // post-multiplier on natural output k: mode 1: w_NMAX^(+-(gval*k) * post_unit) ; mode 2: table[gval*post_g + k*post_k] ; mode 3: constant
    uint32_t post_mode; uint32_t post_shift, post_g, post_k; uint32_t post_scale;   // mode 1 exponent = (gval*k) << post_shift
    const uint32_t* root_hi;                            // w_NMAX two-level table, hi part: w^(4096 j)
    const uint32_t* root3;                              // w_NMAX three-level table (3 x 512 entries, stays in L1)
    const uint32_t* tab_lo; const uint32_t* tab_hi;     // shift tables (mode 2)
    uint32_t tab_base;                                  // the table's base (shift) in Montgomery form
    uint32_t tab_step;                                  // base^(k_stride * post_k): running-product step of the store phase (host-computed)
};

__device__ __forceinline__ uint32_t root_pow(const PassParams& p, uint32_t e) {
    // the shared-memory tiles leave ~24 KB of L1: the 144 KB two-level table misses to L2 on every element,
    // the 6 KB three-level one hits (one more multiply, ~10x less latency)
    const uint32_t a = __ldg(p.root3 + (e & 511)), b = __ldg(p.root3 + 512 + ((e >> 9) & 511)), c = __ldg(p.root3 + 1024 + ((e >> 18) & 511));
    return mul(mul(a, b), c);
}

// one spare word per 16 (conflict-free stride-16 access of the last radix-16 step) plus one per 512
// (spreads bit-reversed accesses, whose lanes differ only in the top five index bits, over all banks)
__device__ __forceinline__ uint32_t pad(uint32_t i) { return i + (i >> 4) + (i >> 9); }

// Padded-tile offset of register-unit element m relative to element 0 of the unit.  With i = blk*2^(LQ+RHO) + m*2^LQ + j
// (j < 2^LQ) both floor terms of pad(i) split into a unit-constant part and a part that depends on m alone, so the
// sixteen shared-memory accesses of a unit are one computed address plus compile-time immediates:
//   i >> 4 : LQ >= 4 -> m*2^(LQ-4) ;  LQ < 4 (and LQ+RHO >= 4) -> m >> (4-LQ)
//   i >> 9 : LQ >= 9 -> m*2^(LQ-9) ;  LQ < 9 <= LQ+RHO -> m >> (9-LQ) ;  LQ+RHO < 9 -> 0
template <int LQ, int RHO>
__device__ __forceinline__ constexpr uint32_t unit_off(uint32_t m) {
    uint32_t o = m << LQ;
    o += (LQ >= 4) ? (m << (LQ >= 4 ? LQ - 4 : 0)) : (m >> (LQ < 4 ? 4 - LQ : 0));
    if (LQ >= 9) o += m << (LQ >= 9 ? LQ - 9 : 0);
    else if (LQ + RHO >= 9) o += m >> (LQ < 9 ? 9 - LQ : 0);
    return o;
}

// RHO DIF stages (S .. S+RHO-1) of one register unit: the 2^RHO elements base + m*q, q = L >> (S+RHO).
// LOG_LEN and S are compile-time so that every shift, pad() term and twiddle offset folds to an immediate.
template <int RHO, int LOG_LEN, int S>
__device__ __forceinline__ void radix_unit(uint32_t* __restrict__ grp, const uint32_t* __restrict__ tw, uint32_t u) {
    constexpr int R = 1 << RHO;
    constexpr int LQ = LOG_LEN - S - RHO;
    constexpr bool IMM = (LQ + RHO >= 4);           // unit_off() is exact
    const uint32_t j = u & ((1u << LQ) - 1), blk = u >> LQ;
    const uint32_t base = (blk << (LQ + RHO)) + j;
    uint32_t* const g0 = grp + pad(base);
    uint32_t x[R];
#pragma unroll
    for (int m = 0; m < R; m++) x[m] = IMM ? g0[unit_off<LQ, RHO>(m)] : grp[pad(base + ((uint32_t)m << LQ))];
#pragma unroll
    for (int a = 0; a < RHO; a++) {
        const int half = R >> (a + 1);
        constexpr int E0 = LQ + S;                  // twiddle index of butterfly mm at stage a: (j << (S+a)) + (mm << (E0+a))
        const uint32_t tj = j << (S + a);
        const uint32_t* const tw0 = tw + tj + (tj >> 5);
#pragma unroll
        for (int m0 = 0; m0 < R; m0++) {
            if ((m0 & half) == 0) {
                const int m1 = m0 + half, mm = m0 & (half - 1);
                const uint32_t A = x[m0], B = x[m1];
                x[m0] = add(A, B);
                if (a == RHO - 1 && LQ == 0) x[m1] = sub(A, B);              // last stage of the transform: twiddle 1
                else {
                    // the Montgomery product reduces any 32-bit left factor: the difference goes in unreduced (A - B + p < 2^32)
                    const uint32_t d = A - B + bb::P;
                    uint32_t wv;
                    if (E0 + a >= 5) wv = tw0[((uint32_t)mm << (E0 + a)) + ((uint32_t)mm << (E0 + a >= 5 ? E0 + a - 5 : 0))];   // padded index splits likewise
                    else { const uint32_t ti = tj + ((uint32_t)mm << (E0 + a)); wv = tw[ti + (ti >> 5)]; }
                    x[m1] = mul(d, wv);
                }
            }
        }
    }
#pragma unroll
    for (int m = 0; m < R; m++) { if (IMM) g0[unit_off<LQ, RHO>(m)] = x[m]; else grp[pad(base + ((uint32_t)m << LQ))] = x[m]; }
}

template <int RHO, int LOG_LEN, int S>
__device__ __forceinline__ void radix_step(uint32_t* data, const uint32_t* tw, uint32_t T, uint32_t LS, uint32_t tid, uint32_t nt) {
    constexpr int LU = LOG_LEN - RHO;                  // log2(units per group)
    const uint32_t total_units = T << LU;
    for (uint32_t w = tid; w < total_units; w += nt) {
        const uint32_t t = w >> LU, u = w & ((1u << LU) - 1);
        radix_unit<RHO, LOG_LEN, S>(data + t * LS, tw, u);
    }
    __syncthreads();
}

// all stages of a length-2^LOG_LEN DIF, four at a time
template <int LOG_LEN, int S>
__device__ __forceinline__ void all_stages(uint32_t* data, const uint32_t* tw, uint32_t T, uint32_t LS, uint32_t tid, uint32_t nt) {
    if constexpr (LOG_LEN - S >= 4) {
        // prefer (4, 3, 3) over (4, 4, 2) style endings only when it saves a step: greedy 4s otherwise
        radix_step<4, LOG_LEN, S>(data, tw, T, LS, tid, nt);
        all_stages<LOG_LEN, S + 4>(data, tw, T, LS, tid, nt);
    } else if constexpr (LOG_LEN - S == 3) {
        radix_step<3, LOG_LEN, S>(data, tw, T, LS, tid, nt);
    } else if constexpr (LOG_LEN - S == 2) {
        radix_step<2, LOG_LEN, S>(data, tw, T, LS, tid, nt);
    } else if constexpr (LOG_LEN - S == 1) {
        radix_step<1, LOG_LEN, S>(data, tw, T, LS, tid, nt);
    }
}

// ---- standard-shape tile movement ---------------------------------------------------------------------------
// Every pass over a column longer than one tile runs 512 threads on a tile of exactly 2^14 elements
// (T = 2^(14 - LOG_LEN) sub-transforms of length L).  For that shape the per-thread sequence of 32 elements is a
// compile-time pattern: one base address / base slot per thread, everything else immediates (bit reversals of the
// step counter, padded-slot corrections, group pitches).  The generic index arithmetic below these helpers remains
// for short columns and unusual shapes; it executes more instructions per element than the butterflies do.
__host__ __device__ constexpr uint32_t cbrev(uint32_t x, int bits) {
    uint32_t r = 0;
    for (int i = 0; i < bits; i++) r |= ((x >> i) & 1u) << (bits - 1 - i);
    return r;
}
template <int LOG_LEN> struct Std {
    static constexpr int LOG_T = 14 - LOG_LEN;
    static constexpr uint32_t T = 1u << (LOG_T > 0 ? LOG_T : 0), L = 1u << LOG_LEN;
    static constexpr uint32_t LS = (L + (L >> 4) + (L >> 9)) | 1;
    static constexpr int LR0 = LOG_LEN - 5;      // strided ("column") view: 2^LR0 rows per step, 32 steps
    static constexpr int LB = LOG_LEN - 9;       // contiguous ("row") view: 2^LB steps of 512 per sub-transform
};
// padded slot of (B << 5) + c, c < 32, relative to the B part
__device__ __forceinline__ constexpr uint32_t off_b5(uint32_t c) { return c + (c >> 4); }
// strided view, natural slots r0 + (k << LR0), r0 < 2^LR0 <= 2^7: offset of step k
template <int LR0> __device__ __forceinline__ constexpr uint32_t off_strided(uint32_t k) {
    return (k << LR0) + (LR0 >= 4 ? (k << (LR0 >= 4 ? LR0 - 4 : 0)) : (k >> (LR0 < 4 ? 4 - LR0 : 0))) + (k >> (9 - LR0));
}
template <int LR0> __device__ __forceinline__ uint32_t base_strided(uint32_t r0) { return r0 + (LR0 >= 4 ? (r0 >> 4) : 0u); }
// contiguous view, bit-reversed slots (B << LB) + c with B = bitrev9(tid), c < 2^LB
template <int LB> __device__ __forceinline__ uint32_t base_rowrev(uint32_t B) { return (B << LB) + ((B << LB) >> 4) + (B >> (9 - LB)); }
template <int LB> __device__ __forceinline__ constexpr uint32_t off_rowrev(uint32_t c) { return c + (LB >= 4 ? (c >> 4) : 0u); }

// strided load (src_gs == 1): element r of sub-transform g0 + tt at src[r * src_rs + g0 + tt]
template <int LOG_LEN, bool BITREV>
__device__ __forceinline__ void load_strided_std(const PassParams& p, const uint32_t* __restrict__ src, uint32_t* __restrict__ data, uint64_t g0, uint32_t tid) {
    using S = Std<LOG_LEN>;
    const uint32_t tt = tid & (S::T - 1), r0 = tid >> S::LOG_T;
    const uint32_t* g = src + g0 + tt + (uint64_t)r0 * p.src_rs;
    const uint64_t ks = p.src_rs << S::LR0;
    uint32_t* sl;
    if (BITREV) { const uint32_t B = bb::reverse_bits(r0, S::LR0); sl = data + tt * S::LS + (B << 5) + (B << 1) + (B >> 4); }
    else sl = data + tt * S::LS + base_strided<S::LR0>(r0);
#pragma unroll
    for (int kb = 0; kb < 32; kb += 8) {
        uint32_t v[8];
#pragma unroll
        for (int u = 0; u < 8; u++) v[u] = __ldg(g + (uint64_t)(kb + u) * ks);
#pragma unroll
        for (int u = 0; u < 8; u++) sl[BITREV ? off_b5(cbrev(kb + u, 5)) : off_strided<S::LR0>(kb + u)] = v[u];
    }
}
// contiguous load (src_rs == 1): sub-transform g at src[g * src_gs + r]
template <int LOG_LEN, bool BITREV>
__device__ __forceinline__ void load_rows_std(const PassParams& p, const uint32_t* __restrict__ src, uint32_t* __restrict__ data, uint64_t g0, uint32_t tid) {
    using S = Std<LOG_LEN>;
    constexpr uint32_t I = 1u << S::LB;
    const uint32_t sb = BITREV ? base_rowrev<S::LB>(bb::reverse_bits(tid, 9)) : tid + (tid >> 4);
#pragma unroll
    for (uint32_t t = 0; t < S::T; t++) {
        const uint32_t* g = src + (g0 + t) * p.src_gs + tid;
        uint32_t* sl = data + t * S::LS + sb;
#pragma unroll
        for (uint32_t kb = 0; kb < I; kb += 8) {
            uint32_t v[8];
#pragma unroll
            for (uint32_t u = 0; u < 8 && kb + u < I; u++) v[u] = __ldg(g + 512 * (kb + u));
#pragma unroll
            for (uint32_t u = 0; u < 8 && kb + u < I; u++) sl[BITREV ? off_rowrev<S::LB>(cbrev(kb + u, S::LB)) : (kb + u) * 545u] = v[u];
        }
    }
}

// contiguous load of bit-reversed-ordered coefficients with the odd-coset pre-multiplier w^((rnat*pre_r + gval*pre_g) << pre_shift):
// memory position tid + 512 * bitrev(i) holds natural index rnat = (bitrev9(tid) << LB) + i, so walking i upwards turns the
// multiplier into a running product (one multiply per element, no table lookups)
template <int LOG_LEN>
__device__ __forceinline__ void load_rows_odd_std(const PassParams& p, const uint32_t* __restrict__ src, uint32_t* __restrict__ data, uint64_t g0, uint32_t tid) {
    using S = Std<LOG_LEN>;
    constexpr uint32_t I = 1u << S::LB;
    const uint32_t B = bb::reverse_bits(tid, 9);
    const uint32_t sb = base_rowrev<S::LB>(B);
    const uint32_t step = root_pow(p, p.pre_r << p.pre_shift);
#pragma unroll 8   // fully unrolled, the 16-group tile of L = 2^10 spills a register pair on sm_90a
    for (uint32_t t = 0; t < S::T; t++) {
        const uint32_t g = (uint32_t)g0 + t;
        const uint32_t gval = p.g_bits ? bb::reverse_bits(g, (int)p.g_bits) : g;
        uint32_t m = root_pow(p, (((B << S::LB) * p.pre_r) + gval * p.pre_g) << p.pre_shift);
        const uint32_t* gp = src + (uint64_t)g * p.src_gs + tid;
        uint32_t* sl = data + t * S::LS + sb;
#pragma unroll
        for (uint32_t ib = 0; ib < I; ib += 8) {
            uint32_t v[8];
#pragma unroll
            for (uint32_t u = 0; u < 8 && ib + u < I; u++) v[u] = __ldg(gp + 512 * cbrev(ib + u, S::LB));
#pragma unroll
            for (uint32_t u = 0; u < 8 && ib + u < I; u++) { sl[off_rowrev<S::LB>(ib + u)] = mul(v[u], m); m = mul(m, step); }
        }
    }
}

// multiplier state of one thread-local output sequence (natural output index k = k_start + i * k_stride)
__device__ __forceinline__ void post_begin(const PassParams& p, uint32_t gval, uint32_t k_start, uint32_t k_stride, uint32_t* m, uint32_t* step) {
    if (p.post_mode == 1) {
        uint32_t e0 = (gval * k_start) << p.post_shift, es = (gval * k_stride) << p.post_shift;
        if (p.inverse) { e0 = 0u - e0; es = 0u - es; }
        *m = root_pow(p, e0); *step = root_pow(p, es);
    } else if (p.post_mode == 2) {
        *m = vg_pow_lookup(p.tab_lo, p.tab_hi, gval * p.post_g + k_start * p.post_k);
        *step = p.tab_step;
    } else { *m = p.post_mode == 3 ? p.post_scale : bb::R1; *step = bb::R1; }
}
// contiguous store (dst_rs == 1), L >= 512: thread positions tid + 512 j of every sub-transform of the tile
template <int LOG_LEN, bool NAT>
__device__ __forceinline__ void store_rows_std(const PassParams& p, uint32_t* __restrict__ dst, const uint32_t* __restrict__ data, uint64_t g0, uint32_t tid) {
    using S = Std<LOG_LEN>;
    constexpr uint32_t I = 1u << S::LB;
    const uint32_t B = bb::reverse_bits(tid, 9);
    const uint32_t sb = NAT ? base_rowrev<S::LB>(B) : tid + (tid >> 4);
    const bool running = p.post_mode == 1 || p.post_mode == 2;
#pragma unroll
    for (uint32_t t = 0; t < S::T; t++) {
        const uint32_t g = (uint32_t)g0 + t;
        const uint32_t gval = p.g_bits ? bb::reverse_bits(g, (int)p.g_bits) : g;
        uint32_t m, step;
        post_begin(p, gval, NAT ? tid : (B << S::LB), NAT ? 512u : 1u, &m, &step);
        uint32_t* d = dst + (uint64_t)g * p.dst_gs + tid;
        const uint32_t* sl = data + t * S::LS + sb;
#pragma unroll
        for (uint32_t i = 0; i < I; i++) {
            // raw order: the i-th natural output of this thread sits at position tid + 512 * bitrev(i)
            const uint32_t j = NAT ? i : cbrev(i, S::LB);
            const uint32_t v = sl[NAT ? off_rowrev<S::LB>(cbrev(i, S::LB)) : j * 545u];
            d[512 * j] = p.post_mode ? mul(v, m) : v;
            if (running) m = mul(m, step);
        }
    }
}
// contiguous store (dst_rs == 1) of short sub-transforms (L < 512), no running multiplier: position tid & (L-1) of
// sub-transforms (tid >> LOG_LEN) + k * (512 / L)
template <int LOG_LEN, bool NAT>
__device__ __forceinline__ void store_short_rows_std(const PassParams& p, uint32_t* __restrict__ dst, const uint32_t* __restrict__ data, uint64_t g0, uint32_t tid) {
    using S = Std<LOG_LEN>;
    constexpr uint32_t GPS = 512u >> LOG_LEN;           // sub-transforms per step
    const uint32_t pos = tid & (S::L - 1), t0 = tid >> LOG_LEN;
    const uint32_t q = NAT ? bb::reverse_bits(pos, LOG_LEN) : pos;
    uint32_t* d = dst + (g0 + t0) * p.dst_gs + pos;
    const uint64_t ks = p.dst_gs * GPS;
    const uint32_t* sl = data + t0 * S::LS + pad(q);
#pragma unroll
    for (uint32_t kb = 0; kb < 32; kb += 8) {
        uint32_t v[8];
#pragma unroll
        for (uint32_t u = 0; u < 8; u++) v[u] = sl[(kb + u) * GPS * S::LS];
#pragma unroll
        for (uint32_t u = 0; u < 8; u++) d[(uint64_t)(kb + u) * ks] = p.post_mode == 3 ? mul(v[u], p.post_scale) : v[u];
    }
}
// strided store (dst_gs == 1): output position pos of sub-transform g at dst[pos * dst_rs + g]
template <int LOG_LEN, bool NAT>
__device__ __forceinline__ void store_strided_std(const PassParams& p, uint32_t* __restrict__ dst, const uint32_t* __restrict__ data, uint64_t g0, uint32_t tid) {
    using S = Std<LOG_LEN>;
    const uint32_t tt = tid & (S::T - 1), r0 = tid >> S::LOG_T;
    const uint32_t g = (uint32_t)g0 + tt;
    const uint32_t gval = p.g_bits ? bb::reverse_bits(g, (int)p.g_bits) : g;
    const uint32_t Bq = bb::reverse_bits(r0, S::LR0);
    uint32_t m, step;
    post_begin(p, gval, NAT ? r0 : (Bq << 5), NAT ? (1u << S::LR0) : 1u, &m, &step);
    const bool running = p.post_mode == 1 || p.post_mode == 2;
    uint32_t* d = dst + g + (uint64_t)r0 * p.dst_rs;
    const uint64_t ks = p.dst_rs << S::LR0;
    const uint32_t* sl = data + tt * S::LS + (NAT ? (Bq << 5) + (Bq << 1) + (Bq >> 4) : base_strided<S::LR0>(r0));
#pragma unroll
    for (uint32_t i = 0; i < 32; i++) {
        const uint32_t j = NAT ? i : cbrev(i, 5);       // position r0 + (j << LR0); its natural index advances by k_stride with i
        const uint32_t v = sl[NAT ? off_b5(cbrev(i, 5)) : off_strided<S::LR0>(j)];
        d[(uint64_t)j * ks] = p.post_mode ? mul(v, m) : v;
        if (running) m = mul(m, step);
    }
}

// One CTA = one tile of `tile` sub-transforms of one column.  grid.x = tiles_per_col, grid.y = column.
template <int LOG_LEN>
__global__ void __launch_bounds__(512) ntt_pass_kernel(PassParams p) {
    extern __shared__ uint32_t smem[];
    constexpr uint32_t L = 1u << LOG_LEN;
    const uint32_t T = p.tile;
    const uint32_t LS = (L + (L >> 4) + (L >> 9)) | 1;   // padded, odd group pitch
    uint32_t* tw = smem;                             // L/2 twiddles w_L^(+-j)
    uint32_t* data = smem + (L >= 2 ? L / 2 + L / 64 + 1 : 1);
    const uint32_t tid = threadIdx.x, nt = blockDim.x;
    const uint64_t col = blockIdx.y;
    const uint64_t g0 = (uint64_t)blockIdx.x * T;
    const uint32_t* src = p.src + col * p.src_cs;
    uint32_t* dst = p.dst + col * p.dst_cs;

    {   // w_L^j = w_NMAX^(j * NMAX/L); NMAX/L >= 2^13 so only the hi table is touched
        const uint64_t unit = (1ull << VG_LOG_NMAX) >> LOG_LEN;
        for (uint32_t j = tid; j < L / 2; j += nt) {
            uint64_t e = (uint64_t)j * unit;
            if (p.inverse && e) e = (1ull << VG_LOG_NMAX) - e;
            tw[j + (j >> 5)] = __ldg(p.root_hi + (e >> VG_POW_LO_BITS));
        }
    }
    // ---- load ----
    const uint32_t total = L * T;
    const uint32_t log_t = 31 - __clz(T);
    bool std_shape = false, loaded = false;
    if constexpr (LOG_LEN >= 8 && LOG_LEN <= 14) {
        std_shape = (T == Std<LOG_LEN>::T) && nt == 512;
        if constexpr (LOG_LEN >= 9) {
            if (std_shape && p.pre_mode && p.src_bitrev && p.src_rs == 1 && p.src_gs != 1) { load_rows_odd_std<LOG_LEN>(p, src, data, g0, tid); loaded = true; }
        }
        if (std_shape && !p.pre_mode) {
            if constexpr (LOG_LEN <= 12) {
                if (p.src_gs == 1) {
                    if (p.src_bitrev) load_strided_std<LOG_LEN, true>(p, src, data, g0, tid); else load_strided_std<LOG_LEN, false>(p, src, data, g0, tid);
                    loaded = true;
                }
            }
            if constexpr (LOG_LEN >= 9) {
                if (!loaded && p.src_rs == 1 && p.src_gs != 1) {
                    if (p.src_bitrev) load_rows_std<LOG_LEN, true>(p, src, data, g0, tid); else load_rows_std<LOG_LEN, false>(p, src, data, g0, tid);
                    loaded = true;
                }
            }
        }
    }
    if (!loaded) {   // generic shapes: 4 independent global loads in flight per thread
        const bool tfast = (p.src_gs == 1);
        const uint32_t log_nt = 31 - __clz(nt);
        if (p.pre_mode && p.src_bitrev && !tfast && L >= 4 * nt) {
            // odd-coset row pass: memory position r = tid + (j << log_nt) holds natural index
            // rnat = (bitrev(tid) << ibits) + bitrev(j); walking i = bitrev(j) upwards makes the pre-multiplier
            // w^((rnat*pre_r + gval*pre_g) << pre_shift) a running product
            const uint32_t ibits = LOG_LEN - log_nt, I = 1u << ibits;
            const uint32_t r_start = bb::reverse_bits(tid, (int)log_nt) << ibits;
            const uint32_t step = root_pow(p, p.pre_r << p.pre_shift);
            const uint32_t step2 = mul(step, step), step3 = mul(step2, step), step4 = mul(step2, step2);
            for (uint32_t t = 0; t < T; t++) {
                const uint32_t g = (uint32_t)g0 + t;
                const uint32_t gval = p.g_bits ? bb::reverse_bits(g, (int)p.g_bits) : g;
                uint32_t m = root_pow(p, (r_start * p.pre_r + gval * p.pre_g) << p.pre_shift);
                const uint32_t* srow = src + (uint64_t)g * p.src_gs;
                uint32_t* drow = data + t * LS;
                for (uint32_t i = 0; i < I; i += 4) {
                    uint32_t v[4];
#pragma unroll
                    for (int u = 0; u < 4; u++) v[u] = srow[tid + (bb::reverse_bits(i + u, (int)ibits) << log_nt)];
                    drow[pad(r_start + i)] = mul(v[0], m);
                    drow[pad(r_start + i + 1)] = mul(v[1], mul(m, step));
                    drow[pad(r_start + i + 2)] = mul(v[2], mul(m, step2));
                    drow[pad(r_start + i + 3)] = mul(v[3], mul(m, step3));
                    m = mul(m, step4);
                }
            }
        } else
        for (uint32_t idx0 = tid; idx0 < total; idx0 += 4 * nt) {
            uint32_t v[4], tt[4], rr[4];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const uint32_t idx = idx0 + u * nt;
                if (idx < total) {
                    if (tfast) { tt[u] = idx & (T - 1); rr[u] = idx >> log_t; } else { rr[u] = idx & (L - 1); tt[u] = idx >> LOG_LEN; }
                    v[u] = src[(uint64_t)rr[u] * p.src_rs + (g0 + tt[u]) * p.src_gs];
                }
            }
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const uint32_t idx = idx0 + u * nt;
                if (idx < total) {
                    const uint32_t rnat = p.src_bitrev ? bb::reverse_bits(rr[u], (int)LOG_LEN) : rr[u];
                    uint32_t x = v[u];
                    if (p.pre_mode) {
                        const uint32_t g = (uint32_t)g0 + tt[u];
                        const uint32_t gval = p.g_bits ? bb::reverse_bits(g, (int)p.g_bits) : g;
                        x = mul(x, root_pow(p, (rnat * p.pre_r + gval * p.pre_g) << p.pre_shift));
                    }
                    data[tt[u] * LS + pad(rnat)] = x;
                }
            }
        }
    }
    __syncthreads();
    // ---- all DIF stages, 4 at a time in registers ----
    all_stages<LOG_LEN, 0>(data, tw, T, LS, tid, nt);
    // ---- store (with optional post multiplier) ----
    // Thread-local view of the tile: fixed group t, positions pos = p0 + (j << lowbits), j < I.  The natural
    // output index k is then K0 + kk (raw order, kk = bitrev(j)) or p0 + (j << lowbits) (natural order): an
    // arithmetic progression, so the twiddle / coset multiplier is a running product (one multiply per
    // element, no table lookups, no per-element exponent arithmetic).
    bool stored = false;
    if constexpr (LOG_LEN >= 8 && LOG_LEN <= 14) {
        if (std_shape) {
            if constexpr (LOG_LEN <= 12) {
                if (p.dst_gs == 1) {
                    if (p.dst_natural) store_strided_std<LOG_LEN, true>(p, dst, data, g0, tid); else store_strided_std<LOG_LEN, false>(p, dst, data, g0, tid);
                    stored = true;
                }
            }
            if (!stored && p.dst_rs == 1 && p.dst_gs != 1) {
                if constexpr (LOG_LEN >= 9) {
                    if (p.dst_natural) store_rows_std<LOG_LEN, true>(p, dst, data, g0, tid); else store_rows_std<LOG_LEN, false>(p, dst, data, g0, tid);
                    stored = true;
                } else {
                    if (p.post_mode == 0 || p.post_mode == 3) {
                        if (p.dst_natural) store_short_rows_std<LOG_LEN, true>(p, dst, data, g0, tid); else store_short_rows_std<LOG_LEN, false>(p, dst, data, g0, tid);
                        stored = true;
                    }
                }
            }
        }
    }
    if (!stored) {
        const bool tfast = (p.dst_gs == 1);
        const uint32_t log_nt = 31 - __clz(nt);
        const bool fast = tfast ? (nt >= T && log_nt - log_t <= (uint32_t)LOG_LEN) : (L >= nt);
        if (fast && (p.post_mode == 1 || p.post_mode == 2)) {
            const uint32_t lowbits = tfast ? (log_nt - log_t) : log_nt;
            const uint32_t ibits = LOG_LEN - lowbits, I = 1u << ibits;
            const uint32_t p0 = tfast ? (tid >> log_t) : tid;
            const uint32_t ngroups_here = tfast ? 1u : T;                 // row-type: the same thread walks every group of the tile
            for (uint32_t tg = 0; tg < ngroups_here; tg++) {
                const uint32_t t = tfast ? (tid & (T - 1)) : tg;
                const uint32_t g = (uint32_t)g0 + t;
                const uint32_t gval = p.g_bits ? bb::reverse_bits(g, (int)p.g_bits) : g;
                // k runs over k_start + i * k_stride, i < I
                const uint32_t k_start = p.dst_natural ? p0 : (bb::reverse_bits(p0, (int)lowbits) << ibits);
                const uint32_t k_stride = p.dst_natural ? (1u << lowbits) : 1u;
                uint32_t m, step;
                post_begin(p, gval, k_start, k_stride, &m, &step);
                uint32_t* dcol = dst + (uint64_t)g * p.dst_gs;
                const uint32_t* drow = data + t * LS;
                for (uint32_t i = 0; i < I; i++) {
                    const uint32_t j = p.dst_natural ? i : bb::reverse_bits(i, (int)ibits);
                    const uint32_t pos = p0 + (j << lowbits);
                    const uint32_t q = p.dst_natural ? bb::reverse_bits(pos, (int)LOG_LEN) : pos;
                    dcol[(uint64_t)pos * p.dst_rs] = mul(drow[pad(q)], m);
                    m = mul(m, step);
                }
            }
        } else {
            for (uint32_t idx = tid; idx < total; idx += nt) {
                uint32_t t, pos;
                if (tfast) { t = idx & (T - 1); pos = idx >> log_t; } else { pos = idx & (L - 1); t = idx >> LOG_LEN; }
                const uint32_t brp = bb::reverse_bits(pos, (int)LOG_LEN);
                const uint32_t q = p.dst_natural ? brp : pos;      // smem slot holding the value stored at `pos`
                const uint32_t k = p.dst_natural ? pos : brp;      // its natural output index
                uint32_t v = data[t * LS + pad(q)];
                if (p.post_mode) {
                    const uint32_t g = (uint32_t)g0 + t;
                    const uint32_t gval = p.g_bits ? bb::reverse_bits(g, (int)p.g_bits) : g;
                    if (p.post_mode == 1) {
                        uint32_t e = (gval * k) << p.post_shift;          // < 2^27: gval*k < n and shift = 27 - log2(n)
                        if (p.inverse) e = (0u - e);                      // root_pow masks to 27 bits: w^(-e) = w^(2^27 - e)
                        v = mul(v, root_pow(p, e));
                    } else if (p.post_mode == 2) {
                        v = mul(v, vg_pow_lookup(p.tab_lo, p.tab_hi, gval * p.post_g + k * p.post_k));
                    } else {
                        v = mul(v, p.post_scale);
                    }
                }
                dst[(uint64_t)pos * p.dst_rs + (g0 + t) * p.dst_gs] = v;
            }
        }
    }
}

constexpr int LOG_ROW_MAX = 14;   // longest contiguous sub-transform staged in shared memory (64 KB)
constexpr int LOG_COL_MAX = 12;   // longest strided sub-transform (balanced nat->nat split)
constexpr int LOG_TILE_ELEMS = 14;

uint32_t choose_tile(int log_len, uint64_t groups) {
    int lt = LOG_TILE_ELEMS - log_len;
    if (lt < 0) lt = 0;
    if (lt > 6) lt = 6;
    uint32_t t = 1u << lt;
    while (t > groups) t >>= 1;
    return t ? t : 1;
}

int32_t launch_pass(vgpu_ctx* ctx, PassParams p, uint64_t w) {
    p.root_hi = ctx->root_table.hi; p.root3 = ctx->root3;
    const uint32_t L = 1u << p.log_len;
    p.tile = choose_tile((int)p.log_len, p.groups);
    const uint64_t tiles = p.groups / p.tile;
    const uint32_t LS = (L + (L >> 4) + (L >> 9)) | 1;
    const size_t smem = ((L >= 2 ? L / 2 + L / 64 + 1 : 1) + (size_t)p.tile * LS) * sizeof(uint32_t);
    const uint32_t total = L * p.tile;
    uint32_t threads = total / 16 >= 512 ? 512 : (total / 16 >= 32 ? total / 16 : 32);
    if (total >= (1u << 14) && threads > 256) threads = 256 * 2;
    using KernelFn = void (*)(PassParams);
    static const KernelFn kernels[15] = {ntt_pass_kernel<0>, ntt_pass_kernel<1>, ntt_pass_kernel<2>, ntt_pass_kernel<3>, ntt_pass_kernel<4>, ntt_pass_kernel<5>,
                                         ntt_pass_kernel<6>, ntt_pass_kernel<7>, ntt_pass_kernel<8>, ntt_pass_kernel<9>, ntt_pass_kernel<10>, ntt_pass_kernel<11>,
                                         ntt_pass_kernel<12>, ntt_pass_kernel<13>, ntt_pass_kernel<14>};
    if (p.log_len > 14) VG_FAIL(ctx, "ntt: sub-transform 2^%u exceeds the shared-memory tile", p.log_len);
    if (!ctx->ntt_attrs_set) { for (auto k : kernels) VG_CUDA(ctx, cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); ctx->ntt_attrs_set = true; }
    if (p.post_mode == 2) {   // step of the store phase's running product (see the kernel): base^(k_stride * post_k)
        uint32_t log_nt = 0; while ((1u << log_nt) < threads) log_nt++;
        uint32_t log_t = 0; while ((1u << log_t) < p.tile) log_t++;
        const bool tfast = (p.dst_gs == 1);
        const uint32_t lowbits = tfast ? (log_nt >= log_t ? log_nt - log_t : 0) : log_nt;
        const uint64_t k_stride = p.dst_natural ? (1ull << lowbits) : 1ull;
        p.tab_step = bb::pow(p.tab_base, k_stride * p.post_k);
    }
    for (uint64_t c0 = 0; c0 < w; c0 += 65535) {     // grid.y limit
        const uint64_t wc = w - c0 < 65535 ? w - c0 : 65535;
        PassParams q = p;
        q.src = p.src + c0 * p.src_cs; q.dst = p.dst + c0 * p.dst_cs;
        dim3 grid((unsigned)tiles, (unsigned)wc);
        KScope ks(ctx, KC_NTT, 8.0 * (double)(p.groups << p.log_len) * (double)wc);
        kernels[p.log_len]<<<grid, threads, smem, ctx->stream>>>(q);
        VG_LAUNCH_CHECK(ctx);
    }
    return 0;
}

// a one-row trace is a constant polynomial: its extension repeats the row (eight of BasicMachine's fourteen chips in a Fibonacci proof)
__global__ void repeat_row_kernel(const uint32_t* src, uint64_t src_cs, uint32_t* dst, uint64_t dst_cs, uint64_t H, uint64_t w) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H * w) return;
    dst[(i / H) * dst_cs + (i % H)] = src[(i / H) * src_cs];
}

__global__ void zero_pad_kernel(const uint32_t* src, uint64_t src_cs, uint32_t* dst, uint64_t dst_cs, uint64_t h, uint64_t H, uint64_t w) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H * w) return;
    uint64_t c = i / H, r = i % H;
    dst[c * dst_cs + r] = r < h ? src[c * src_cs + r] : 0;
}

// split for the passes that have one strided and one contiguous sub-transform
void split_col_row(int log_n, int* l_col, int* l_row) {
    if (log_n <= LOG_ROW_MAX) { *l_col = 0; *l_row = log_n; return; }
    int lc = log_n - LOG_ROW_MAX;
    if (lc > LOG_COL_MAX) lc = LOG_COL_MAX;          // then the contiguous part takes the rest (<= LOG_ROW_MAX for log_n <= 26)
    if (lc < 4) lc = 4;
    *l_col = lc; *l_row = log_n - lc;
}

}  // namespace

// natural -> natural transform of every column (forward: out[k] = sum_j in[j] w^(jk); inverse scales by 1/n).
int32_t vg_ntt_nat2nat(vgpu_ctx* ctx, const uint32_t* src, uint64_t src_cs, uint32_t* dst, uint64_t dst_cs, int log_n, uint64_t w,
                       bool inverse, const PowTable* coset, uint32_t* tmp, uint64_t tmp_cs) {
    const uint64_t n = 1ull << log_n;
    uint32_t ninv = inverse ? bb::inv(bb::to_monty((uint32_t)(n % bb::P))) : bb::R1;
    PassParams p{};
    p.inverse = inverse;
    if (log_n <= LOG_ROW_MAX) {
        p.src = src; p.src_cs = src_cs; p.dst = dst; p.dst_cs = dst_cs;
        p.src_rs = 1; p.src_gs = n; p.dst_rs = 1; p.dst_gs = n;
        p.log_len = log_n; p.groups = 1; p.dst_natural = 1;
        if (coset) { p.post_mode = 2; p.post_g = 0; p.post_k = 1; p.tab_lo = coset->lo; p.tab_hi = coset->hi; p.tab_base = coset->base; }
        else if (inverse) { p.post_mode = 3; p.post_scale = ninv; }
        return launch_pass(ctx, p, w);
    }
    // up to 2^24 both halves of the split are <= 2^12 (the fast strided tiles); above that the halves grow to 2^13 / 2^14 and fall back
    // on the generic tile movement: every size up to the field's two-adicity works, the sizes the prover uses are the fast ones
    if (log_n > VG_LOG_NMAX) VG_FAIL(ctx, "ntt: 2^%d exceeds BabyBear's two-adicity (2^%d)", log_n, VG_LOG_NMAX);
    const int l1 = (log_n + 1) / 2, l2 = log_n - l1;
    const uint64_t n1 = 1ull << l1, n2 = 1ull << l2;
    // pass 1: over i1 (stride n2) for each i2; times w_n^(+-i2*k1); transposed store tmp[i2][k1]
    p.src = src; p.src_cs = src_cs; p.dst = tmp; p.dst_cs = tmp_cs;
    p.src_rs = n2; p.src_gs = 1; p.dst_rs = 1; p.dst_gs = n1;
    p.log_len = l1; p.groups = n2; p.dst_natural = 1;
    p.post_mode = 1; p.post_shift = VG_LOG_NMAX - log_n;
    VG_TRY(launch_pass(ctx, p, w));
    // pass 2: tmp is [i2][k1]; over i2 (stride n1) for each k1; X[k1 + n1*k2] stored at that index
    PassParams q{};
    q.inverse = inverse;
    q.src = tmp; q.src_cs = tmp_cs; q.dst = dst; q.dst_cs = dst_cs;
    q.src_rs = n1; q.src_gs = 1; q.dst_rs = n1; q.dst_gs = 1;
    q.log_len = l2; q.groups = n1; q.dst_natural = 1;
    if (coset) { q.post_mode = 2; q.post_g = 1; q.post_k = (uint32_t)n1; q.tab_lo = coset->lo; q.tab_hi = coset->hi; q.tab_base = coset->base; }
    else if (inverse) { q.post_mode = 3; q.post_scale = ninv; }
    return launch_pass(ctx, q, w);
}

// iNTT natural evaluations -> coefficients in BIT-REVERSED order, coefficient K scaled by table[K]
// (= shift^K / n).  buf (column stride bcs) receives c[K] at position bitrev_n(K).
static int32_t intt_nat2bitrev_scaled(vgpu_ctx* ctx, const uint32_t* src, uint64_t src_cs, uint32_t* buf, uint64_t bcs, int log_n, uint64_t w, const PowTable* tab) {
    const uint64_t n = 1ull << log_n;
    int lc, lr;
    split_col_row(log_n, &lc, &lr);
    PassParams p{};
    p.inverse = 1;
    if (lc == 0) {
        p.src = src; p.src_cs = src_cs; p.dst = buf; p.dst_cs = bcs;
        p.src_rs = 1; p.src_gs = n; p.dst_rs = 1; p.dst_gs = n;
        p.log_len = log_n; p.groups = 1; p.dst_natural = 0;
        p.post_mode = 2; p.post_g = 0; p.post_k = 1; p.tab_lo = tab->lo; p.tab_hi = tab->hi; p.tab_base = tab->base;
        return launch_pass(ctx, p, w);
    }
    const uint64_t n1 = 1ull << lc, n2 = 1ull << lr;
    // column pass over i1 (stride n2): A[k1][i2] * w_n^(-i2*k1) stored raw at row bitrev(k1)
    p.src = src; p.src_cs = src_cs; p.dst = buf; p.dst_cs = bcs;
    p.src_rs = n2; p.src_gs = 1; p.dst_rs = n2; p.dst_gs = 1;
    p.log_len = lc; p.groups = n2; p.dst_natural = 0;
    p.post_mode = 1; p.post_shift = VG_LOG_NMAX - log_n;
    VG_TRY(launch_pass(ctx, p, w));
    // row pass on row q1 = bitrev(k1): over i2 -> k2 stored raw; K = k1 + n1*k2 = bitrev(q1) + n1*k
    PassParams q{};
    q.inverse = 1;
    q.src = buf; q.src_cs = bcs; q.dst = buf; q.dst_cs = bcs;
    q.src_rs = 1; q.src_gs = n2; q.dst_rs = 1; q.dst_gs = n2;
    q.log_len = lr; q.groups = n1; q.dst_natural = 0;
    q.g_bits = lc;
    q.post_mode = 2; q.post_g = 1; q.post_k = (uint32_t)n1; q.tab_lo = tab->lo; q.tab_hi = tab->hi; q.tab_base = tab->base;
    return launch_pass(ctx, q, w);
}

// forward coset transform: coefficients in bit-reversed order (c[K] at bitrev_n(K)) -> evaluations in
// bit-reversed order (E[m] at bitrev_n(m)), out of place.  odd != 0 multiplies c[K] by w_2n^K first.
// With inverse != 0 and tab != null the same two passes compute the INVERSE transform of bit-reversed-ordered
// evaluations (the quotient kernel's output order) into bit-reversed-ordered coefficients, coefficient K
// scaled by tab[K] (= shift^K / n).
static int32_t ntt_bitrev2bitrev(vgpu_ctx* ctx, const uint32_t* coef, uint64_t ccs, uint32_t* dst, uint64_t dst_cs, uint32_t* tmp, uint64_t tcs,
                                 int log_n, uint64_t w, bool odd, bool inverse = false, const PowTable* tab = nullptr) {
    const uint64_t n = 1ull << log_n;
    int lc, lr;
    split_col_row(log_n, &lc, &lr);
    PassParams p{};
    p.inverse = inverse ? 1 : 0;
    if (lc == 0) {
        p.src = coef; p.src_cs = ccs; p.dst = dst; p.dst_cs = dst_cs;
        p.src_rs = 1; p.src_gs = n; p.dst_rs = 1; p.dst_gs = n;
        p.log_len = log_n; p.groups = 1; p.src_bitrev = 1; p.dst_natural = 0;
        if (odd) { p.pre_mode = 1; p.pre_r = 1; p.pre_g = 0; p.pre_shift = VG_LOG_NMAX - (log_n + 1); }
        if (tab) { p.post_mode = 2; p.post_g = 0; p.post_k = 1; p.tab_lo = tab->lo; p.tab_hi = tab->hi; p.tab_base = tab->base; }
        return launch_pass(ctx, p, w);
    }
    const uint64_t n1 = 1ull << lc, n2 = 1ull << lr;
    // position (j1, j2) holds K = bitrev(j1) + n1*bitrev(j2) =: k1' + n1*k2'
    // row pass on row j1: transform over k2' (slot = bitrev(j2)) -> m2 ; times w_n^(k1'*m2) ; stored raw (position q <-> m2 = bitrev(q))
    p.src = coef; p.src_cs = ccs; p.dst = tmp; p.dst_cs = tcs;
    p.src_rs = 1; p.src_gs = n2; p.dst_rs = 1; p.dst_gs = n2;
    p.log_len = lr; p.groups = n1; p.src_bitrev = 1; p.dst_natural = 0;
    p.g_bits = lc;
    if (odd) { p.pre_mode = 1; p.pre_r = (uint32_t)n1; p.pre_g = 1; p.pre_shift = VG_LOG_NMAX - (log_n + 1); }
    p.post_mode = 1; p.post_shift = VG_LOG_NMAX - log_n;
    VG_TRY(launch_pass(ctx, p, w));
    // column pass over rows j1 (k1' = bitrev(j1)) for each column q: -> m1 ; E[m1*n2 + m2] goes to
    // bitrev_n = bitrev(m2)*n1 + bitrev(m1) = q*n1 + raw slot: transposed store, raw order
    PassParams q{};
    q.inverse = inverse ? 1 : 0;
    q.src = tmp; q.src_cs = tcs; q.dst = dst; q.dst_cs = dst_cs;
    q.src_rs = n2; q.src_gs = 1; q.dst_rs = 1; q.dst_gs = n1;
    q.log_len = lc; q.groups = n2; q.src_bitrev = 1; q.dst_natural = 0;
    if (tab) {   // natural output index K = m1*n2 + m2 with m1 = k and m2 = bitrev(column position g)
        q.g_bits = lr; q.post_mode = 2; q.post_g = 1; q.post_k = (uint32_t)n2;
        q.tab_lo = tab->lo; q.tab_hi = tab->hi; q.tab_base = tab->base;
    }
    return launch_pass(ctx, q, w);
}

// coset_lde_batch(mat, added_bits = 1, shift): dst (2h rows per column).
int32_t vg_coset_lde(vgpu_ctx* ctx, const uint32_t* src, uint64_t src_cs, uint64_t h, uint64_t w, uint32_t shift_canonical,
                     uint32_t* dst, uint64_t dst_cs, bool bit_reversed, bool src_bitrev, uint32_t log_blowup) {
    if (src_bitrev && !bit_reversed) VG_FAIL(ctx, "coset_lde: a bit-reversed-row input is only supported with bit-reversed output");
    if (bit_reversed && log_blowup != 1) VG_FAIL(ctx, "coset_lde: committed (bit-reversed) extensions are built for log_blowup = 1 only (FriConfig of basic/src/bin/valida.rs:385-390)");
    int log_n = 0;
    while ((1ull << log_n) < h) log_n++;
    if ((1ull << log_n) != h) VG_FAIL(ctx, "coset_lde: height %llu is not a power of two", (unsigned long long)h);
    // the height limit first: with log_blowup >= 1 the two-adicity check below would otherwise shadow it
    if (log_n > LOG_ROW_MAX + LOG_COL_MAX) VG_FAIL(ctx, "coset_lde: heights above 2^%d are not built", LOG_ROW_MAX + LOG_COL_MAX);
    if (log_n + (int)log_blowup > VG_LOG_NMAX) VG_FAIL(ctx, "coset_lde: LDE height 2^%d exceeds BabyBear two-adicity", log_n + (int)log_blowup);
    if (h == 1) {
        const uint64_t H = 1ull << log_blowup;
        repeat_row_kernel<<<(unsigned)((H * w + 127) / 128), 128, 0, ctx->stream>>>(src, src_cs, dst, dst_cs, H, w);
        VG_LAUNCH_CHECK(ctx);
        return 0;
    }
    const PowTable* tab = nullptr;
    uint32_t ninv_canon = bb::from_monty(bb::inv(bb::to_monty((uint32_t)(h % bb::P))));
    VG_TRY(vg_get_shift_table(ctx, shift_canonical, ninv_canon, h, &tab));
    // column batches bound the scratch; launches cover as many columns as possible (grid.y) so CTAs of
    // different phases overlap on each SM
    uint64_t batch = (2ull << 30) / (8 * h);   // coefficient + intermediate scratch <= 2 GB; whole matrices per launch
    if (batch < 1) batch = 1;
    if (batch > w) batch = w;
    VgBuf coef_buf(ctx), tmp_buf(ctx);
    VG_TRY(coef_buf.alloc(batch * h * 4));
    VG_TRY(tmp_buf.alloc(batch * h * 4));
    uint32_t *coef = coef_buf.as<uint32_t>(), *tmp = tmp_buf.as<uint32_t>();
    for (uint64_t c0 = 0; c0 < w; c0 += batch) {
        uint64_t wc = w - c0 < batch ? w - c0 : batch;
        if (bit_reversed) {
            VG_TRY(src_bitrev ? ntt_bitrev2bitrev(ctx, src + c0 * src_cs, src_cs, coef, h, tmp, h, log_n, wc, false, true, tab)
                              : intt_nat2bitrev_scaled(ctx, src + c0 * src_cs, src_cs, coef, h, log_n, wc, tab));
            VG_TRY(ntt_bitrev2bitrev(ctx, coef, h, dst + c0 * dst_cs, dst_cs, tmp, h, log_n, wc, false));
            VG_TRY(ntt_bitrev2bitrev(ctx, coef, h, dst + c0 * dst_cs + h, dst_cs, tmp, h, log_n, wc, true));
        } else {
            // natural-order output (API completeness, not on the proving path): zero-pad and transform at size h << log_blowup
            VG_TRY(vg_ntt_nat2nat(ctx, src + c0 * src_cs, src_cs, coef, h, log_n, wc, true, tab, tmp, h));
            const uint64_t H = h << log_blowup;
            VgBuf padb(ctx), tmp2(ctx);
            VG_TRY(padb.alloc(wc * H * 4));
            VG_TRY(tmp2.alloc(wc * H * 4));
            uint64_t tot = H * wc;
            zero_pad_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, ctx->stream>>>(coef, h, padb.as<uint32_t>(), H, h, H, wc);
            ctx->launches++;
            VG_TRY(vg_ntt_nat2nat(ctx, padb.as<uint32_t>(), H, dst + c0 * dst_cs, dst_cs, log_n + (int)log_blowup, wc, false, nullptr, tmp2.as<uint32_t>(), H));
        }
    }
    return 0;
}
