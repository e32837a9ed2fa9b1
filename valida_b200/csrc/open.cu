// K8/K9/K10 — kernels of TwoAdicFriPcs::open_multi_batches (derive/src/lib.rs:391-392) and of the
// p3-fri commit phase:
//   inverse denominators 1/(x - z) over a whole bit-reversed coset (one ext5 batch inversion per
//     height and point; the barycentric weights of K8 reuse them on the first-half rows),
//   K8  out-of-domain evaluation p(z) of every column from the first h storage rows (= g*H),
//   K9  reduced openings  ro[i] += alpha^off * (sum_c alpha^c p_c(x_i) - sum_c alpha^c p_c(z)) / (x_i - z),
//   K10 fold_even_odd with the next height's reduced openings added in.
// Ext5 vectors are limb-major (limb l of element i at v[l*cs + i]) so that every access is coalesced.
#include "ctx.h"
#include "devchip.h"
#include "open.h"
#include <algorithm>
#include <memory>

namespace {

using bb::E5;

__device__ __forceinline__ uint32_t oroot_pow(const uint32_t* lo, const uint32_t* hi, uint64_t e) {
    return vg_pow_lookup(lo, hi, e & ((1ull << VG_LOG_NMAX) - 1));
}
__device__ __forceinline__ E5 ld5(const uint32_t* v, uint64_t cs, uint64_t i) {
    E5 r;
#pragma unroll
    for (int l = 0; l < 5; l++) r.c[l] = v[(uint64_t)l * cs + i];
    return r;
}
__device__ __forceinline__ void st5(uint32_t* v, uint64_t cs, uint64_t i, const E5& x) {
#pragma unroll
    for (int l = 0; l < 5; l++) v[(uint64_t)l * cs + i] = x.c[l];
}

// out[i] = x_i - z,  x_i = s * w_H^bitrev(i)   (storage order of a committed LDE of height H = 2^log_h)
__global__ void __launch_bounds__(256) coset_minus_point_kernel(uint32_t* out /* virtual base: + global row */, uint64_t H /* limb stride */, uint64_t begin, uint64_t count, uint32_t log_h, uint32_t s, E5 z, const uint32_t* lo, const uint32_t* hi) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    i += begin;
    uint32_t nat = bb::reverse_bits((uint32_t)i, (int)log_h);
    uint32_t x = bb::mul(s, oroot_pow(lo, hi, (uint64_t)nat << (VG_LOG_NMAX - log_h)));
    E5 d = bb::e5_neg(z);
    d.c[0] = bb::add(d.c[0], x);
    st5(out, H, i, d);
}

// K8: out-of-domain evaluation.  With x/(x - z) = 1 + z/(x - z) the barycentric sum splits into
//     S_c(z) = sum_i p_c(x_i) + z * sum_i p_c(x_i) / (x_i - z)
// so the kernel needs no domain points at all: per column a base-field sum and, per point, an ext5 dot product with
// the inverse denominators — a (w x h) by (h x 5*NP) product over F_p.  Dot products are accumulated LAZILY
// (bb::madw / bb::lazy_fold: one IMAD.WIDE per term, one more per four terms), which makes the sweep bound by the
// half-rate IMAD.WIDE issue: 5 * NP * 1.25 of them per element.
// A CTA (16 warps) double-buffers tiles of 1024 rows of the inverse denominators in shared memory (cp.async) and its
// warps form a (column pair) x (row slice) grid over the tile: narrow matrices (the 2^24-row memory chip has 14 / 10
// columns) put several warps on the same column pair, so all 16 warps work whatever the width.  A lane owns four
// consecutive rows of a 128-row chunk: one 16-byte global load per column and one 16-byte shared load per limb.
constexpr int BARY_COLS = 2, BARY_WARPS = 16, BARY_THREADS = 32 * BARY_WARPS, BARY_TILE = 1024, BARY_CHUNKS = BARY_TILE / 128;
constexpr int BARY_OUT = 11;                       // per column: 2 points x 5 limbs, then the plain column sum
struct BaryParams {
    const uint32_t* mat; uint64_t mcs; uint64_t h; uint32_t w;   // h rows starting at row_begin
    uint64_t row_begin;
    const uint32_t* invden[2]; uint64_t ics; uint32_t npoints;
    uint32_t cpg, rs;        // columns per CTA (even, <= 32) and row slices per column pair: (cpg / 2) * rs <= 16 warps
    uint32_t* partial;       // [gridDim.x * rs][w][BARY_OUT]
};
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }

template <int NP>
__global__ void __launch_bounds__(BARY_THREADS, 1) bary_kernel(BaryParams p) {
    extern __shared__ __align__(16) uint32_t dsm[];          // [2][NP * 5][BARY_TILE]
    constexpr uint32_t BUF = NP * 5 * BARY_TILE;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t ncg = p.cpg / BARY_COLS;
    const uint32_t cw = wid % ncg, rsl = wid / ncg;
    const uint32_t c0 = blockIdx.y * p.cpg + cw * BARY_COLS;
    const bool worker = rsl < p.rs && c0 < p.w;
    const uint32_t* col[BARY_COLS];
#pragma unroll
    for (int c = 0; c < BARY_COLS; c++) col[c] = p.mat + (uint64_t)min(c0 + c, p.w - 1) * p.mcs + p.row_begin + 4 * lane;   // a surplus column shadows the last one (never written)
    uint64_t acc[BARY_COLS][NP][5];
    uint64_t sum[BARY_COLS];
#pragma unroll
    for (int c = 0; c < BARY_COLS; c++) { sum[c] = 0; for (int q = 0; q < NP; q++) for (int l = 0; l < 5; l++) acc[c][q][l] = 0; }
    const uint64_t ntiles = p.h / BARY_TILE;
    auto stage = [&](uint32_t buf, uint64_t t) {
        const uint64_t row0 = p.row_begin + t * BARY_TILE;
        for (uint32_t i = threadIdx.x; i < NP * 5 * (BARY_TILE / 4); i += BARY_THREADS) {
            const uint32_t ql = i / (BARY_TILE / 4), v = i % (BARY_TILE / 4);
            cp_async16(dsm + buf * BUF + ql * BARY_TILE + 4 * v, (ql < 5 ? p.invden[0] : p.invden[1]) + (uint64_t)(ql % 5) * p.ics + row0 + 4 * v);
        }
        cp_async_commit();
    };
    uint32_t buf = 0;
    if (blockIdx.x < ntiles) stage(0, blockIdx.x);
    for (uint64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const bool more = t + gridDim.x < ntiles;
        if (more) stage(buf ^ 1, t + gridDim.x);
        uint4 e[BARY_COLS];
        if (worker) {
#pragma unroll
            for (int c = 0; c < BARY_COLS; c++) e[c] = __ldg(reinterpret_cast<const uint4*>(col[c] + t * BARY_TILE + rsl * 128));
        }
        if (more) cp_async_wait<1>(); else cp_async_wait<0>();
        __syncthreads();
        if (worker) {
            const uint32_t* d = dsm + buf * BUF + 4 * lane;
            for (uint32_t ck = rsl; ck < BARY_CHUNKS; ck += p.rs) {
                uint4 nx[BARY_COLS];
                const bool pre = ck + p.rs < BARY_CHUNKS;
                if (pre) {
#pragma unroll
                    for (int c = 0; c < BARY_COLS; c++) nx[c] = __ldg(reinterpret_cast<const uint4*>(col[c] + t * BARY_TILE + (ck + p.rs) * 128));
                }
#pragma unroll
                for (int q = 0; q < NP; q++) {
#pragma unroll
                    for (int l = 0; l < 5; l++) {
                        const uint4 dv = *reinterpret_cast<const uint4*>(d + (q * 5 + l) * BARY_TILE + ck * 128);
#pragma unroll
                        for (int c = 0; c < BARY_COLS; c++) {
                            uint64_t a = acc[c][q][l];
                            a = bb::madw(e[c].x, dv.x, a); a = bb::madw(e[c].y, dv.y, a); a = bb::madw(e[c].z, dv.z, a); a = bb::madw(e[c].w, dv.w, a);
                            acc[c][q][l] = bb::lazy_fold(a);
                        }
                    }
                }
#pragma unroll
                for (int c = 0; c < BARY_COLS; c++) sum[c] += (uint64_t)e[c].x + e[c].y + e[c].z + e[c].w;
                if (pre) {
#pragma unroll
                    for (int c = 0; c < BARY_COLS; c++) e[c] = nx[c];
                }
            }
        }
        __syncthreads();
        buf ^= 1;
    }
    if (!worker) return;
    // reduce to field elements, then across the warp
#pragma unroll
    for (int c = 0; c < BARY_COLS; c++) {
        uint32_t v[BARY_OUT];
#pragma unroll
        for (int k = 0; k < BARY_OUT; k++) v[k] = 0;
#pragma unroll
        for (int q = 0; q < NP; q++)
#pragma unroll
            for (int l = 0; l < 5; l++) v[q * 5 + l] = bb::monty_reduce64(acc[c][q][l]);
        v[10] = (uint32_t)(sum[c] % bb::P);
#pragma unroll
        for (int k = 0; k < BARY_OUT; k++) {
            uint32_t x = v[k];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) x = bb::add(x, __shfl_xor_sync(0xffffffffu, x, o));
            if (lane == 0 && c0 + c < p.w) p.partial[(((uint64_t)blockIdx.x * p.rs + rsl) * p.w + c0 + c) * BARY_OUT + k] = x;
        }
    }
}
// heights below one tile (never on the critical path): a CTA per column, plain modular arithmetic
__global__ void __launch_bounds__(128) bary_small_kernel(BaryParams p) {
    __shared__ uint32_t red[4][BARY_OUT];
    const uint32_t c = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t* col = p.mat + (uint64_t)c * p.mcs + p.row_begin;
    E5 acc[2] = {bb::e5_zero(), bb::e5_zero()};
    uint32_t s = 0;
    for (uint64_t r = threadIdx.x; r < p.h; r += blockDim.x) {
        const uint32_t x = col[r];
        s = bb::add(s, x);
        for (uint32_t q = 0; q < p.npoints; q++) acc[q] = bb::e5_add(acc[q], bb::e5_mul_base(ld5(p.invden[q], p.ics, p.row_begin + r), x));
    }
    uint32_t v[BARY_OUT];
    for (int q = 0; q < 2; q++) for (int l = 0; l < 5; l++) v[q * 5 + l] = acc[q].c[l];
    v[10] = s;
    for (int k = 0; k < BARY_OUT; k++) {
        uint32_t x = v[k];
        for (int o = 16; o > 0; o >>= 1) x = bb::add(x, __shfl_xor_sync(0xffffffffu, x, o));
        if (lane == 0) red[wid][k] = x;
    }
    __syncthreads();
    if (threadIdx.x < BARY_OUT) {
        const uint32_t k = threadIdx.x;
        p.partial[(uint64_t)c * BARY_OUT + k] = bb::add(bb::add(red[0][k], red[1][k]), bb::add(red[2][k], red[3][k]));
    }
}

// K9: reduced openings.  One thread per LDE row i:
//     U(i)   = sum_c alpha^(off + c) p_c(x_i)                       (lazy dot product, powers in the kernel parameters)
//     ro[i] += (U - B_0) / (x_i - z_0)  +  (U * alpha^w - B_1) / (x_i - z_1),      B_q = alpha^(off_q) sum_c alpha^c p_c(z_q)
// which is the reference's  alpha^off_q * (sum_c alpha^c p_c(x_i) - sum_c alpha^c p_c(z_q)) / (x_i - z_q)  summed over the
// points (off_1 = off_0 + w): shifting the power table by off_0 removes one ext5 product per point from every row.
constexpr uint32_t RO_MAXW = 96;
struct RoParams {
    const uint32_t* mat; uint64_t mcs; uint64_t H; uint32_t w;
    const uint32_t* invden[2]; uint64_t ics; uint32_t npoints;
    E5 b[2]; E5 aw, aw2;              // B_q; alpha^w and 2 * alpha^w
    uint32_t* ro; uint64_t rcs;       // accumulator, limb-major, height H
    uint64_t row_begin, row_end;      // rows swept by this launch
    uint32_t first;                   // 1: this launch also subtracts B_q (0 on the later column blocks of a matrix wider than RO_MAXW)
    uint32_t apow[RO_MAXW][5];        // alpha^(off_0 + c)
};
// (Measured alternatives that did not help, 6.5-6.8 ms per proof each: loads two column groups ahead of the arithmetic;
// the power table in shared memory instead of indexed constant loads.  ncu r1b: issue slots 50 % busy, FMA pipe 34 %.)
template <int NP>
__global__ void __launch_bounds__(256) reduced_opening_kernel(const __grid_constant__ RoParams p) {
    const uint64_t i = p.row_begin + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.row_end) return;
    uint64_t a[5] = {0, 0, 0, 0, 0};
    const uint32_t* m = p.mat + i;
    uint32_t c = 0;
    for (; c + 8 <= p.w; c += 8) {   // eight loads in flight, two folds per limb
        uint32_t e[8];
#pragma unroll
        for (int u = 0; u < 8; u++) e[u] = __ldg(m + (uint64_t)(c + u) * p.mcs);
#pragma unroll
        for (int g = 0; g < 8; g += 4)
#pragma unroll
            for (int l = 0; l < 5; l++) {
                uint64_t t = a[l];
#pragma unroll
                for (int u = 0; u < 4; u++) t = bb::madw(e[g + u], p.apow[c + g + u][l], t);
                a[l] = bb::lazy_fold(t);
            }
    }
    for (; c < p.w; c++) {
        const uint32_t e0 = __ldg(m + (uint64_t)c * p.mcs);
#pragma unroll
        for (int l = 0; l < 5; l++) a[l] = bb::lazy_fold(bb::madw(e0, p.apow[c][l], a[l]));
    }
    E5 U;
#pragma unroll
    for (int l = 0; l < 5; l++) U.c[l] = bb::monty_reduce64(a[l]);
    bb::Lazy5 s; s.init();
    {
        const E5 w0 = p.first ? bb::e5_sub(U, p.b[0]) : U;
        s.fma_ext(ld5(p.invden[0], p.ics, i), w0, bb::e5_dbl(w0));
    }
    if (NP > 1) {
        bb::Lazy5 t; t.init();
        t.fma_ext(U, p.aw, p.aw2);
        E5 w1 = t.value();
        if (p.first) w1 = bb::e5_sub(w1, p.b[1]);
        s.fma_ext(ld5(p.invden[1], p.ics, i), w1, bb::e5_dbl(w1));
    }
    st5(p.ro, p.rcs, i, bb::e5_add(ld5(p.ro, p.rcs, i), s.value()));
}

// K10: out[i] = (lo + hi)/2 + (beta/2) * g_inv^bitrev(i) * (lo - hi)  (+ add[i]) for the `count` outputs starting at i0; `cur` holds
// the pairs of exactly those outputs (a rank's run, or everything with i0 = 0); out / add are virtual bases (+ global i)
__global__ void __launch_bounds__(256) fri_fold_kernel(const uint32_t* cur, uint64_t ccs, uint64_t i0, uint64_t count, uint32_t log_half, E5 half_beta, uint32_t one_half,
                                                      const uint32_t* add, uint64_t acs, uint32_t* out, uint64_t ocs, const uint32_t* lo, const uint32_t* hi) {
    const uint64_t il = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (il >= count) return;
    const uint64_t i = i0 + il;
    E5 a, b;
#pragma unroll
    for (int l = 0; l < 5; l++) { uint2 t = *reinterpret_cast<const uint2*>(cur + (uint64_t)l * ccs + 2 * il); a.c[l] = t.x; b.c[l] = t.y; }
    uint32_t nat = bb::reverse_bits((uint32_t)i, (int)log_half);
    // g_inv^nat, g = two_adic_generator(log_half + 1)
    uint64_t e = (uint64_t)nat << (VG_LOG_NMAX - log_half - 1);
    uint32_t gp = e ? oroot_pow(lo, hi, (1ull << VG_LOG_NMAX) - e) : bb::R1;
    E5 pw = bb::e5_mul_base(half_beta, gp);
    E5 r = bb::e5_add(bb::e5_mul_base(bb::e5_add(a, b), one_half), bb::e5_mul(pw, bb::e5_sub(a, b)));
    if (add) r = bb::e5_add(r, ld5(add, acs, i));
    st5(out, ocs, i, r);
}

// out[i] = sum over blocks of partial[b][i]
__global__ void __launch_bounds__(256) bary_reduce_kernel(const uint32_t* __restrict__ partial, uint32_t nblocks, uint32_t n, uint32_t* __restrict__ out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t acc = 0;
    for (uint32_t b = 0; b < nblocks; b++) acc = bb::add(acc, partial[(uint64_t)b * n + i]);
    out[i] = acc;
}

// a null pointer is a word another rank reports (split proof): it contributes 0 to the sum over the ranks
__global__ void __launch_bounds__(256) gather_words_kernel(const uint32_t* const* ptrs, uint64_t n, uint32_t* out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { const uint32_t* q = ptrs[i]; out[i] = q ? *q : 0u; }
}
__global__ void __launch_bounds__(256) sum_ranks_kernel(const uint32_t* __restrict__ all, uint32_t nranks, uint64_t n, uint32_t* __restrict__ out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t a = 0;
    for (uint32_t r = 0; r < nranks; r++) a += all[(uint64_t)r * n + i];     // exactly one rank reports a non-zero word
    out[i] = a;
}

}  // namespace

// 1/(x - z) without an extension-field inversion.  x is a base-field point, so the conjugates of x - z are x - frob^k(z):
//     1/(x - z) = Q(x) / M(x),   M(x) = prod_{k=0..4} (x - frob^k z)  (minimal polynomial of z: base-field coefficients),
//                                Q(x) = prod_{k=1..4} (x - frob^k z)  (degree 4, ext5 coefficients).
// Per element: the powers of x, two lazy dot products (M: 6 terms, Q: 5 x 5 terms) and a share of ONE base-field Fermat
// inversion per INVDEN_BATCH elements (Montgomery batch trick) — about 2.3x fewer instructions than forming x - z in
// ext5 and batch-inverting there (3 ext5 products per element plus a Frobenius-norm inversion per 8).  Measured per
// proof: 4.0 ms (ext5 batch inversion) -> 2.27 ms (batch 16, 96 registers) -> 2.07 ms (batch 8, 62 registers, 8 CTAs/SM).
struct InvdenParams {
    uint32_t* out; uint64_t H /* limb stride of out */, begin, count; uint32_t log_h, s;      // out: virtual base (+ global row)
    uint32_t mc[5];          // M(x) = x^5 + sum_j mc[j] x^j
    uint32_t qc[4][5];       // Q(x) = x^4 + sum_j qc[j] x^j   (qc[j] ext5, limb l at qc[j][l])
    const uint32_t* lo; const uint32_t* hi;
};
constexpr int INVDEN_BATCH = 8, INVDEN_MINB = 8;
__global__ void __launch_bounds__(128, INVDEN_MINB) invden_norm_kernel(const __grid_constant__ InvdenParams p) {
    const uint64_t stride = (p.count + INVDEN_BATCH - 1) / INVDEN_BATCH;
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= stride) return;
    auto point = [&](uint64_t i) {
        const uint32_t nat = bb::reverse_bits((uint32_t)i, (int)p.log_h);
        return bb::mul(p.s, oroot_pow(p.lo, p.hi, (uint64_t)nat << (VG_LOG_NMAX - p.log_h)));
    };
    uint32_t v[INVDEN_BATCH], pref[INVDEN_BATCH];
    uint32_t acc = bb::R1;
#pragma unroll
    for (int k = 0; k < INVDEN_BATCH; k++) {
        const uint64_t j = t + (uint64_t)k * stride;
        v[k] = bb::R1;
        if (j < p.count) {
            const uint32_t x = point(p.begin + j);
            const uint32_t x2 = bb::sqr(x), x3 = bb::mul(x2, x), x4 = bb::sqr(x2), x5 = bb::mul(x4, x);
            uint64_t m = bb::madw(p.mc[4], x4, bb::madw(p.mc[3], x3, bb::madw(p.mc[2], x2, bb::madw(p.mc[1], x, 0))));
            m = bb::madw(x5, bb::R1, bb::madw(p.mc[0], bb::R1, bb::lazy_fold(m)));
            v[k] = bb::monty_reduce64(m);
        }
        pref[k] = acc;
        acc = bb::mul(acc, v[k]);
    }
    uint32_t inv = bb::inv(acc);
#pragma unroll
    for (int k = INVDEN_BATCH - 1; k >= 0; k--) {
        const uint64_t j = t + (uint64_t)k * stride;
        const uint32_t minv = bb::mul(inv, pref[k]);
        inv = bb::mul(inv, v[k]);
        if (j < p.count) {
            const uint64_t i = p.begin + j;
            const uint32_t x = point(i);
            const uint32_t x2 = bb::sqr(x), x3 = bb::mul(x2, x), x4 = bb::sqr(x2);
#pragma unroll
            for (int l = 0; l < 5; l++) {
                uint64_t q = bb::madw(p.qc[3][l], x3, bb::madw(p.qc[2][l], x2, bb::madw(p.qc[1][l], x, bb::madw(p.qc[0][l], bb::R1, 0))));
                if (l == 0) q = bb::madw(x4, bb::R1, bb::lazy_fold(q));
                p.out[(uint64_t)l * p.H + i] = bb::mul(bb::monty_reduce64(q), minv);
            }
        }
    }
}

// 1/(x_i - z) for the rows [begin, begin + count) of the coset of height 2^log_H (committed order): out[l * count + (i - begin)]
int32_t vg_inverse_denominators(vgpu_ctx* ctx, uint32_t log_H, const E5& z, uint64_t begin, uint64_t count, uint32_t* out) {
    KScope ks(ctx, KC_INVDEN, 20.0 * (double)count);
    uint32_t* out_v = out - begin;
    if ((z.c[1] | z.c[2] | z.c[3] | z.c[4]) == 0) {
        // z in the base field may hit a coset point: the generic path keeps a zero denominator as zero
        coset_minus_point_kernel<<<(unsigned)((count + 255) / 256), 256, 0, ctx->stream>>>(out_v, count, begin, count, log_H, bb::to_monty(bb::GEN_CANON), z, ctx->root_table.lo, ctx->root_table.hi);
        VG_LAUNCH_CHECK(ctx);
        return vg_ext_batch_inverse(ctx, out, count, count, 1);
    }
    InvdenParams p{};
    p.out = out_v; p.H = count; p.begin = begin; p.count = count; p.log_h = log_H; p.s = bb::to_monty(bb::GEN_CANON);
    p.lo = ctx->root_table.lo; p.hi = ctx->root_table.hi;
    {   // poly(x) = prod (x - frob^k z): coefficients low to high, ext5 arithmetic on the host
        uint32_t zp[5];
        bb::e5_frob_consts(zp);
        E5 conj[5];
        conj[0] = z;
        for (int k = 1; k < 5; k++) conj[k] = bb::e5_frobenius(conj[k - 1], zp);
        auto times_x_minus = [](std::vector<E5>& poly, const E5& r) {
            std::vector<E5> n(poly.size() + 1, bb::e5_zero());
            for (size_t d = 0; d < poly.size(); d++) { n[d + 1] = bb::e5_add(n[d + 1], poly[d]); n[d] = bb::e5_sub(n[d], bb::e5_mul(poly[d], r)); }
            poly.swap(n);
        };
        std::vector<E5> q{bb::e5_one()};
        for (int k = 1; k < 5; k++) times_x_minus(q, conj[k]);
        std::vector<E5> m = q;
        times_x_minus(m, conj[0]);
        for (int j = 0; j < 5; j++) {
            if (m[j].c[1] | m[j].c[2] | m[j].c[3] | m[j].c[4]) VG_FAIL(ctx, "inverse denominators: the minimal polynomial left the base field");
            p.mc[j] = m[j].c[0];
        }
        for (int j = 0; j < 4; j++) for (int l = 0; l < 5; l++) p.qc[j][l] = q[j].c[l];
    }
    const uint64_t stride = (count + INVDEN_BATCH - 1) / INVDEN_BATCH;
    invden_norm_kernel<<<(unsigned)((stride + 127) / 128), 128, 0, ctx->stream>>>(p);
    VG_LAUNCH_CHECK(ctx);
    return 0;
}

// Enqueue the sums behind p_c(z_q) for every column c and point q (q < npoints <= 2) of a committed LDE (height H = 2h):
// d_out receives w * BARY_OUT words ([c][q*5 + l] = sum_i p_c(x_i) / (x_i - z_q), [c][10] = sum_i p_c(x_i)), stream-ordered, no
// host synchronisation — open_multi_batches reads the sums of every matrix back with ONE copy.
int32_t vg_eval_columns_enqueue(vgpu_ctx* ctx, const vgpu_dmat* lde, uint32_t npoints, const uint32_t* const* invden, uint64_t ics, uint32_t* d_out) {
    const uint64_t H = lde->gh, h = H / 2;
    const uint32_t gw = (uint32_t)lde->gw, nout_all = gw * BARY_OUT;
    // split proof: the first h committed rows are the coset g*H, the other h rows the coset g*w_2h*H — and EITHER coset determines
    // p(z).  So the first ceil(w/2) columns are summed over the rows of the first coset, the remaining columns over the rows of the
    // second: a rank sums its rows of each coset for that coset's columns (one part, or two when its run straddles row h), the
    // per-rank sums meet in one small all-gather and vg_eval_columns_finish normalises a column by the coset it was summed over.
    // invden: the caller's vector over the same rows as the matrix part held here.
    // sum_part: columns [c_begin, c_begin + w) over local rows [r0, r0 + rows) -> out (w * BARY_OUT words)
    auto sum_part = [&](uint64_t r0, uint64_t rows, uint32_t c_begin, uint32_t w, uint32_t* out) -> int32_t {
        BaryParams p{};
        p.mat = lde->d + (uint64_t)c_begin * lde->col_stride; p.mcs = lde->col_stride; p.h = rows; p.row_begin = r0; p.w = w;
        p.invden[0] = invden[0]; p.invden[1] = npoints > 1 ? invden[1] : invden[0]; p.ics = ics; p.npoints = npoints;
        uint32_t nblocks = 1;
        VgBuf partial(ctx);
        const uint32_t nout = w * BARY_OUT;
        if (rows >= BARY_TILE && rows % BARY_TILE == 0) {
            const unsigned by = (w + 31) / 32;
            p.cpg = 2 * (((w + by - 1) / by + 1) / 2);               // columns per CTA, even
            p.rs = std::min<uint32_t>(BARY_CHUNKS, BARY_WARPS / (p.cpg / BARY_COLS));
            const uint64_t ntiles = rows / BARY_TILE;
            const unsigned bx = (unsigned)std::min<uint64_t>(ntiles, std::max<uint64_t>(1, (uint64_t)ctx->sm_count / by));
            nblocks = bx * p.rs;
            VG_TRY(partial.alloc((size_t)nblocks * w * BARY_OUT * 4));
            p.partial = partial.as<uint32_t>();
            if (!ctx->bary_attrs_set) {
                VG_CUDA(ctx, cudaFuncSetAttribute(bary_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 1 * 5 * BARY_TILE * 4));
                VG_CUDA(ctx, cudaFuncSetAttribute(bary_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 2 * 5 * BARY_TILE * 4));
                ctx->bary_attrs_set = true;
            }
            KScope ks(ctx, KC_BARY, 4.0 * (double)rows * w);
            if (npoints > 1) bary_kernel<2><<<dim3(bx, by), BARY_THREADS, 2 * 2 * 5 * BARY_TILE * 4, ctx->stream>>>(p);
            else bary_kernel<1><<<dim3(bx, by), BARY_THREADS, 2 * 1 * 5 * BARY_TILE * 4, ctx->stream>>>(p);
            VG_LAUNCH_CHECK(ctx);
        } else {
            VG_TRY(partial.alloc((size_t)w * BARY_OUT * 4));
            p.partial = partial.as<uint32_t>();
            KScope ks(ctx, KC_BARY, 4.0 * (double)rows * w);
            bary_small_kernel<<<w, 128, 0, ctx->stream>>>(p);
            VG_LAUNCH_CHECK(ctx);
        }
        bary_reduce_kernel<<<(nout + 255) / 256, 256, 0, ctx->stream>>>(partial.as<uint32_t>(), nblocks, nout, out);
        VG_LAUNCH_CHECK(ctx);
        return 0;
    };
    if (lde->dist != VG_ROWS) return sum_part(0, h, 0, gw, d_out);
    const uint32_t w_first = vg_eval_columns_first_coset(gw);
    VgBuf gathered(ctx);                                                               // [rank 0 | rank 1 | ...], all columns each
    VG_TRY(gathered.alloc((size_t)nout_all * 4 * ctx->comm_size));
    uint32_t* mine = gathered.as<uint32_t>() + (size_t)nout_all * ctx->comm_rank;
    VG_CUDA(ctx, cudaMemsetAsync(mine, 0, (size_t)nout_all * 4, ctx->stream));         // the columns the other coset's rows sum
    const uint64_t g0 = lde->row0, g1 = lde->row0 + lde->h, mid = std::min(std::max(h, g0), g1);   // global rows; [g0, mid) in the first coset
    if (mid > g0 && w_first) VG_TRY(sum_part(0, mid - g0, 0, w_first, mine));
    if (g1 > mid && gw > w_first) VG_TRY(sum_part(mid - g0, g1 - mid, w_first, gw - w_first, mine + (size_t)w_first * BARY_OUT));
    VG_TRY(vg_comm_allgather_inplace(ctx, gathered.as<uint32_t>(), nout_all));
    bary_reduce_kernel<<<(nout_all + 255) / 256, 256, 0, ctx->stream>>>(gathered.as<uint32_t>(), (uint32_t)ctx->comm_size, nout_all, d_out);
    VG_LAUNCH_CHECK(ctx);
    return 0;
}

uint32_t vg_eval_columns_first_coset(uint32_t w) { return (w + 1) / 2; }

// host arithmetic on the sums of vg_eval_columns_enqueue:  p(z) = -(z^h - t^h) / (h t^h) * (sum_i p(x_i) + z sum_i p(x_i)/(x_i - z))
// over the coset t*H the sums ran over: t = s for columns < w_first, t = s * w_2h (t^h = -s^h) for the others (split proof).
void vg_eval_columns_finish(const uint32_t* sums, uint64_t H, uint32_t w, uint32_t npoints, const E5* z, std::vector<E5>* ys /* [q][c] */, uint32_t w_first) {
    const uint64_t h = H / 2;
    uint32_t log_h = 0; while ((1ull << log_h) < h) log_h++;
    uint32_t s = bb::to_monty(bb::GEN_CANON), sh = s;
    for (uint32_t i = 0; i < log_h; i++) sh = bb::sqr(sh);
    uint32_t denom_inv = bb::inv(bb::mul(bb::to_monty((uint32_t)(h % bb::P)), sh));
    ys->assign((size_t)npoints * w, bb::e5_zero());
    for (uint32_t q = 0; q < npoints; q++) {
        E5 zh = bb::e5_exp_pow2(z[q], (int)log_h);
        const E5 norm_a = bb::e5_neg(bb::e5_mul_base(bb::e5_sub_base(zh, sh), denom_inv));       // -(z^h - s^h) / (h s^h)
        const E5 norm_b = bb::e5_mul_base(bb::e5_add_base(zh, sh), denom_inv);                     // -(z^h + s^h) / (h (-s^h))
        for (uint32_t c = 0; c < w; c++) {
            E5 D;   // sum_i p_c(x_i) / (x_i - z_q)
            for (int l = 0; l < 5; l++) D.c[l] = sums[(size_t)c * BARY_OUT + q * 5 + l];
            const E5 S = bb::e5_add_base(bb::e5_mul(z[q], D), sums[(size_t)c * BARY_OUT + 10]);
            (*ys)[(size_t)q * w + c] = bb::e5_mul(S, c < w_first ? norm_a : norm_b);
        }
    }
}
uint32_t vg_eval_columns_words(uint32_t w) { return w * BARY_OUT; }

// ro[i] += sum_q alpha^(off_q) * (sum_c alpha^c p_c(x_i) - sum_y[q]) / (x_i - z_q),  off_1 = off_0 + w, over the rows of the
// matrix part held here (all rows, or this rank's run).  invden / ro: vectors over those same rows, limb stride vcs.
// apow_off[c] = alpha^(off_0 + c) (host, Montgomery), alpha_w = alpha^w, sum_y[q] = sum_c alpha^c p_c(z_q).
int32_t vg_reduced_opening_accumulate(vgpu_ctx* ctx, const vgpu_dmat* lde, const E5* apow_off, const E5& alpha_w, uint32_t npoints, const uint32_t* const* invden,
                                      uint64_t vcs, const E5* sum_y, uint32_t* ro) {
    auto p = std::make_unique<RoParams>();
    p->mcs = lde->col_stride; p->H = lde->h;
    p->npoints = npoints; p->ics = vcs;
    p->invden[0] = invden[0]; p->invden[1] = npoints > 1 ? invden[1] : invden[0];
    p->b[0] = bb::e5_mul(apow_off[0], sum_y[0]);                                        // alpha^off_0 * sum_y_0
    p->b[1] = npoints > 1 ? bb::e5_mul(bb::e5_mul(apow_off[0], alpha_w), sum_y[1]) : bb::e5_zero();
    p->aw = alpha_w;
    for (int l = 0; l < 5; l++) p->aw2.c[l] = bb::dbl(alpha_w.c[l]);
    p->ro = ro; p->rcs = vcs;
    const uint64_t rows = lde->h;
    p->row_begin = 0; p->row_end = rows;
    for (uint64_t c0 = 0; c0 < lde->w; c0 += RO_MAXW) {         // one launch unless the matrix is wider than the parameter table
        const uint32_t wc = (uint32_t)std::min<uint64_t>(RO_MAXW, lde->w - c0);
        p->mat = lde->d + c0 * lde->col_stride; p->w = wc; p->first = c0 == 0;
        for (uint32_t c = 0; c < wc; c++) for (int l = 0; l < 5; l++) p->apow[c][l] = apow_off[c0 + c].c[l];
        KScope ks(ctx, KC_REDUCED_OPENING, (double)rows * (4.0 * wc + 40.0));
        if (npoints > 1) reduced_opening_kernel<2><<<(unsigned)((rows + 255) / 256), 256, 0, ctx->stream>>>(*p);
        else reduced_opening_kernel<1><<<(unsigned)((rows + 255) / 256), 256, 0, ctx->stream>>>(*p);
        VG_LAUNCH_CHECK(ctx);
    }
    return 0;
}

// One FRI fold: `cur` holds the 2 * count values behind outputs [i0, i0 + count) of the n / 2 (limb stride ccs); out_v / add_v are
// virtual bases (+ global output index) with limb strides ocs / acs.
int32_t vg_fri_fold(vgpu_ctx* ctx, const uint32_t* cur, uint64_t ccs, uint64_t n, uint64_t i0, uint64_t count, const E5& beta,
                    const uint32_t* add_v, uint64_t acs, uint32_t* out_v, uint64_t ocs) {
    uint64_t half = n / 2;
    uint32_t log_half = 0; while ((1ull << log_half) < half) log_half++;
    uint32_t one_half = bb::inv(bb::to_monty(2));
    E5 half_beta = bb::e5_mul_base(beta, one_half);
    KScope ks(ctx, KC_FRI_FOLD, 60.0 * (double)count);
    fri_fold_kernel<<<(unsigned)((count + 255) / 256), 256, 0, ctx->stream>>>(cur, ccs, i0, count, log_half, half_beta, one_half, add_v, acs, out_v, ocs, ctx->root_table.lo, ctx->root_table.hi);
    VG_LAUNCH_CHECK(ctx);
    return 0;
}

// The words behind `ptrs` (null = reported by another rank of a split proof), summed over the ranks.
int32_t vg_gather_words(vgpu_ctx* ctx, const std::vector<const uint32_t*>& ptrs, std::vector<uint32_t>* out) {
    size_t n = ptrs.size();
    out->resize(n);
    if (!n) return 0;
    const bool all = vg_sharded(ctx);
    const size_t G = all ? (size_t)ctx->comm_size : 1;
    VgBuf dptr(ctx), dout_buf(ctx), dsum(ctx);
    VG_TRY(dptr.upload(ptrs.data(), n));
    VG_TRY(dout_buf.alloc(n * 4 * G));
    uint32_t* dout = dout_buf.as<uint32_t>();
    gather_words_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(dptr.as<const uint32_t*>(), n, dout + (all ? n * (size_t)ctx->comm_rank : 0));
    VG_LAUNCH_CHECK(ctx);
    const uint32_t* res = dout;
    if (all) {
        VG_TRY(vg_comm_allgather_inplace(ctx, dout, n));
        VG_TRY(dsum.alloc(n * 4));
        sum_ranks_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(dout, (uint32_t)G, n, dsum.as<uint32_t>());
        VG_LAUNCH_CHECK(ctx);
        res = dsum.as<uint32_t>();
    }
    VG_CUDA(ctx, cudaMemcpyAsync(out->data(), res, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}
