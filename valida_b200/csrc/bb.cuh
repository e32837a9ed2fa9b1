// BabyBear (p = 2^31 - 2^27 + 1) and its degree-5 binomial extension (X^5 = 2) for sm_90a.
// Replaces p3-baby-bear / p3-field arithmetic used throughout the reference's proving path
// (e.g. machine/src/chip.rs:174,194-197; machine/src/quotient.rs:199-226).
// Device words are in MONTGOMERY form (R = 2^32), the same storage p3_baby_bear::BabyBear uses,
// so a Rust caller's RowMajorMatrix<BabyBear>.values can be uploaded without conversion.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace bb {

constexpr uint32_t P = 0x78000001u;
constexpr uint32_t PINV = 0x88000001u;   // p^-1 mod 2^32
constexpr uint32_t R1 = 0x0ffffffeu;     // 2^32 mod p  (Montgomery form of 1)
constexpr uint32_t R2 = 1172168163u;     // 2^64 mod p  (to_monty multiplier)
constexpr uint32_t GEN_CANON = 31;

#ifdef __CUDACC__
#define BB_HD __host__ __device__ __forceinline__
#else
#define BB_HD inline
#endif

BB_HD uint32_t umin32(uint32_t a, uint32_t b) { return a < b ? a : b; }
BB_HD uint32_t add(uint32_t a, uint32_t b) { uint32_t s = a + b; return umin32(s, s - P); }
BB_HD uint32_t sub(uint32_t a, uint32_t b) { uint32_t d = a - b; return umin32(d, d + P); }
BB_HD uint32_t neg(uint32_t a) { return a ? P - a : 0; }
BB_HD uint32_t dbl(uint32_t a) { return add(a, a); }
// Montgomery product a*b/2^32 mod p, inputs < p (one of them may be any u32), output in [0,p).
BB_HD uint32_t mul(uint32_t a, uint32_t b) {
    uint64_t t = (uint64_t)a * b;
    uint32_t m = (uint32_t)t * PINV;
#ifdef __CUDA_ARCH__
    uint32_t u = (uint32_t)(t >> 32) - __umulhi(m, P);
#else
    uint32_t u = (uint32_t)(t >> 32) - (uint32_t)(((uint64_t)m * P) >> 32);
#endif
    return umin32(u, u + P);
}
BB_HD uint32_t sqr(uint32_t a) { return mul(a, a); }
BB_HD uint32_t to_monty(uint32_t canonical) { return mul(canonical, R2); }
BB_HD uint32_t from_monty(uint32_t m) { return mul(m, 1u); }
BB_HD uint32_t pow(uint32_t a_monty, uint64_t e) {
    uint32_t r = R1;
    while (e) { if (e & 1) r = mul(r, a_monty); a_monty = mul(a_monty, a_monty); e >>= 1; }
    return r;
}
BB_HD uint32_t inv(uint32_t a_monty) { return pow(a_monty, P - 2); }

// ---- degree-5 extension, coefficients in Montgomery form ---------------------------------------
struct E5 { uint32_t c[5]; };
BB_HD E5 e5_zero() { E5 r; for (int i = 0; i < 5; i++) r.c[i] = 0; return r; }
BB_HD E5 e5_one() { E5 r = e5_zero(); r.c[0] = R1; return r; }
BB_HD E5 e5_from_base(uint32_t b) { E5 r = e5_zero(); r.c[0] = b; return r; }
BB_HD bool e5_is_zero(const E5& a) { return (a.c[0] | a.c[1] | a.c[2] | a.c[3] | a.c[4]) == 0; }
BB_HD E5 e5_add(const E5& a, const E5& b) { E5 r; for (int i = 0; i < 5; i++) r.c[i] = add(a.c[i], b.c[i]); return r; }
BB_HD E5 e5_sub(const E5& a, const E5& b) { E5 r; for (int i = 0; i < 5; i++) r.c[i] = sub(a.c[i], b.c[i]); return r; }
BB_HD E5 e5_neg(const E5& a) { E5 r; for (int i = 0; i < 5; i++) r.c[i] = neg(a.c[i]); return r; }
BB_HD E5 e5_add_base(const E5& a, uint32_t b) { E5 r = a; r.c[0] = add(r.c[0], b); return r; }
BB_HD E5 e5_sub_base(const E5& a, uint32_t b) { E5 r = a; r.c[0] = sub(r.c[0], b); return r; }
BB_HD E5 e5_mul_base(const E5& a, uint32_t b) { E5 r; for (int i = 0; i < 5; i++) r.c[i] = mul(a.c[i], b); return r; }

// Reduce a 64-bit sum of <= 4 Montgomery partial products... general: x < 2^64 -> x * 2^-32 mod p in [0,p)
BB_HD uint32_t monty_reduce64(uint64_t t) {
    // t = hi*2^32 + lo ; standard reduction needs hi < p.  Fold hi first: hi*2^32 == hi*R1 (mod p) is not cheaper,
    // so split: reduce (lo part with hi' = hi mod p).
    uint32_t hi = (uint32_t)(t >> 32), lo = (uint32_t)t;
    // hi may be up to 2^32-1 >= p : bring into [0,p) with up to two subtractions (hi < 2^32 < 3p)
    hi = umin32(hi, hi - P); hi = umin32(hi, hi - P);
    uint32_t m = lo * PINV;
#ifdef __CUDA_ARCH__
    uint32_t u = hi - __umulhi(m, P);
#else
    uint32_t u = hi - (uint32_t)(((uint64_t)m * P) >> 32);
#endif
    return umin32(u, u + P);
}

#ifdef __CUDACC__
// ---- lazy ext5 accumulation on the device ----------------------------------------------------------------------
// a*b + c as ONE IMAD.WIDE (the C++ form `c + (uint64_t)a * b` is not reliably fused: ptxas was seen emitting a
// 64 x 32 multiply — IMAD.WIDE + IMAD + IADD3 — when the 32-bit factor came out of a predicated load).
__device__ __forceinline__ uint64_t madw(uint32_t a, uint32_t b, uint64_t c) {
    uint64_t r;
    asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(r) : "r"(a), "r"(b), "l"(c));
    return r;
}
// x = hi*2^32 + lo == hi*R1 + lo (mod p): value kept, size back under 2^60 + 2^32
__device__ __forceinline__ uint64_t lazy_fold(uint64_t a) { return madw((uint32_t)(a >> 32), R1, (uint64_t)(uint32_t)a); }

// Five 64-bit accumulators (one per ext5 limb) that absorb raw products of Montgomery words in lockstep.  Invariant:
// a folded limb is < 2^60 + 2^32 and every product is < p^2, so FOUR products may be pending before the next fold
// (4 p^2 + 2^60 + 2^32 = 1.737e19 < 2^64 = 1.845e19).  `np` is the pending count; in straight-line (unrolled) code it
// folds to a compile-time constant.  value() is the Montgomery reduction of the sum: sum(aR * bR) / R = sum(ab) R.
struct Lazy5 {
    uint64_t a[5]; int np;
    __device__ __forceinline__ void init() { for (int l = 0; l < 5; l++) a[l] = 0; np = 0; }
    __device__ __forceinline__ void fold() { for (int l = 0; l < 5; l++) a[l] = lazy_fold(a[l]); np = 0; }
    __device__ __forceinline__ void step() { if (np == 4) fold(); np++; }
    // += x * y, y in the base field (any 32-bit word times words < p keeps the bound only for y < p: callers pass reduced words)
    __device__ __forceinline__ void fma_base(const E5& x, uint32_t y) {
        step();
#pragma unroll
        for (int l = 0; l < 5; l++) a[l] = madw(x.c[l], y, a[l]);
    }
    // += x * y in F_p[X]/(X^5 - 2); y2 = 2*y (limb-wise, reduced) feeds the wrapped terms.  Round r adds x_r * y_(k-r) to limb k.
    __device__ __forceinline__ void fma_ext(const E5& x, const E5& y, const E5& y2) {
#pragma unroll
        for (int r = 0; r < 5; r++) {
            step();
#pragma unroll
            for (int k = 0; k < 5; k++) a[k] = madw(x.c[r], k >= r ? y.c[k - r] : y2.c[k - r + 5], a[k]);
        }
    }
    __device__ __forceinline__ E5 value() const { E5 r; for (int l = 0; l < 5; l++) r.c[l] = monty_reduce64(a[l]); return r; }
};
__device__ __forceinline__ E5 e5_dbl(const E5& a) { E5 r; for (int i = 0; i < 5; i++) r.c[i] = dbl(a.c[i]); return r; }
#endif

// Schoolbook product with X^5 = 2.  Products a_i*b_j < p^2 < 2^62, so up to 4 of them fit in 64 bits
// before one Montgomery reduction.
BB_HD E5 e5_mul(const E5& a, const E5& b) {
#ifdef __CUDA_ARCH__
    // device: 25 + 5 IMAD.WIDE and five reductions (the wrapped terms use 2*b) instead of nine reductions
    Lazy5 t; t.init(); t.fma_ext(a, b, e5_dbl(b));
    return t.value();
#else
    E5 r;
#define PR(i, j) ((uint64_t)a.c[i] * b.c[j])
    // low parts t_k = sum_{i+j=k}, high parts u_k = sum_{i+j=k+5} (to be doubled)
    uint32_t l0 = monty_reduce64(PR(0, 0));
    uint32_t l1 = monty_reduce64(PR(0, 1) + PR(1, 0));
    uint32_t l2 = monty_reduce64(PR(0, 2) + PR(1, 1) + PR(2, 0));
    uint32_t l3 = monty_reduce64(PR(0, 3) + PR(1, 2) + PR(2, 1) + PR(3, 0));
    uint32_t l4 = add(monty_reduce64(PR(0, 4) + PR(1, 3) + PR(2, 2) + PR(3, 1)), monty_reduce64(PR(4, 0)));
    uint32_t h0 = monty_reduce64(PR(1, 4) + PR(2, 3) + PR(3, 2) + PR(4, 1));
    uint32_t h1 = monty_reduce64(PR(2, 4) + PR(3, 3) + PR(4, 2));
    uint32_t h2 = monty_reduce64(PR(3, 4) + PR(4, 3));
    uint32_t h3 = monty_reduce64(PR(4, 4));
#undef PR
    r.c[0] = add(l0, dbl(h0));
    r.c[1] = add(l1, dbl(h1));
    r.c[2] = add(l2, dbl(h2));
    r.c[3] = add(l3, dbl(h3));
    r.c[4] = l4;
    return r;
#endif
}
BB_HD E5 e5_sqr(const E5& a) { return e5_mul(a, a); }
BB_HD E5 e5_pow(E5 a, uint64_t e) {
    E5 r = e5_one();
    while (e) { if (e & 1) r = e5_mul(r, a); a = e5_sqr(a); e >>= 1; }
    return r;
}
BB_HD E5 e5_exp_pow2(E5 a, int k) { while (k-- > 0) a = e5_sqr(a); return a; }
// Frobenius: coefficient i scaled by z^i, z = 2^((p-1)/5) (Montgomery constants below, set by frob_consts()).
BB_HD E5 e5_frobenius(const E5& a, const uint32_t zpow[5]) {
    E5 r; r.c[0] = a.c[0];
    for (int i = 1; i < 5; i++) r.c[i] = mul(a.c[i], zpow[i]);
    return r;
}
BB_HD void e5_frob_consts(uint32_t zpow[5]) {
    uint32_t z = pow(to_monty(2), (P - 1) / 5);
    zpow[0] = R1;
    for (int i = 1; i < 5; i++) zpow[i] = mul(zpow[i - 1], z);
}
BB_HD E5 e5_inv(const E5& a) {
    uint32_t zp[5];
    e5_frob_consts(zp);
    E5 f1 = e5_frobenius(a, zp), f2 = e5_frobenius(f1, zp), f3 = e5_frobenius(f2, zp), f4 = e5_frobenius(f3, zp);
    E5 prod = e5_mul(e5_mul(f1, f2), e5_mul(f3, f4));
    E5 n = e5_mul(a, prod);
    return e5_mul_base(prod, inv(n.c[0]));
}

BB_HD uint32_t reverse_bits(uint32_t x, int bits) {
#ifdef __CUDA_ARCH__
    return bits ? (__brev(x) >> (32 - bits)) : 0;
#else
    uint32_t r = 0;
    for (int i = 0; i < bits; i++) r = (r << 1) | ((x >> i) & 1);
    return r;
#endif
}

// canonical two_adic_generator(bits) = 0x1a427a41^(2^(27-bits))  (p3-baby-bear TwoAdicField)
BB_HD uint32_t two_adic_generator_monty(int bits) {
    uint32_t g = to_monty(0x1a427a41u);
    for (int i = 0; i < 27 - bits; i++) g = sqr(g);
    return g;
}

}  // namespace bb
