// Polynomials of degree <= 3 over BabyBear and their roots in F_p, on the device and the host (vgpu_cell_alternatives, alts.cu).
// A polynomial is in t = X - x0 for the cell's current value x0, its coefficients Montgomery words: c[0] + c[1] t + c[2] t^2 + c[3] t^3.
//   - interp: the polynomial through its values at t = 0, 1, 2, 3 (forward differences, Newton's form);
//   - gcd: a greatest common divisor up to a unit, by pseudo-remainders (no inversion: only the roots matter), fully unrolled;
//   - nonzero_roots: the distinct roots t != 0 in F_p: the part prime to t is made monic, its gcd with t^p - t (30 squarings modulo a
//     cubic) keeps its linear factors, which are split without random state (Tonelli-Shanks with the generator 31 as the non-residue for
//     a quadratic; gcd with (t + a)^((p-1)/2) - 1 for a = 1, 2, ..., SPLIT_TRIES for a cubic).
// No arrays are indexed by run-time values, so a kernel keeps all of it in registers.
#pragma once
#include "bb.cuh"

namespace poly {

constexpr uint32_t INV2 = 0x07ffffffu;      // 1/2 (Montgomery)
constexpr uint32_t INV6 = 0x52aaaaabu;      // 1/6
constexpr uint32_t NONRES = 0x0fffffbeu;    // 31, the field's generator: a quadratic non-residue
constexpr int SPLIT_TRIES = 32;             // shifts a tried to split a cubic with three roots

struct P3 {
    uint32_t c[4];
};

BB_HD int deg(const P3& a) { return a.c[3] ? 3 : a.c[2] ? 2 : a.c[1] ? 1 : a.c[0] ? 0 : -1; }
BB_HD uint32_t lead(const P3& a, int d) { return d == 3 ? a.c[3] : d == 2 ? a.c[2] : d == 1 ? a.c[1] : a.c[0]; }
// coefficient j of t^k * a (k in 0..3)
BB_HD uint32_t shifted(const P3& a, int k, int j) {
    uint32_t r = 0;
#pragma unroll
    for (int s = 0; s < 4; s++)
        if (s <= j && k == s) r = a.c[j - s];
    return r;
}

// The polynomial whose values at t = 0, 1, 2, 3 are v[0..3]: v0 + d1 t + d2 t(t-1)/2 + d3 t(t-1)(t-2)/6.
BB_HD P3 interp(const uint32_t v[4]) {
    const uint32_t d1 = bb::sub(v[1], v[0]);
    const uint32_t d2 = bb::add(bb::sub(v[2], bb::dbl(v[1])), v[0]);
    const uint32_t d3 = bb::sub(bb::add(bb::sub(v[3], v[0]), bb::add(bb::dbl(v[1]), v[1])), bb::add(bb::dbl(v[2]), v[2]));
    const uint32_t c3 = bb::mul(d3, INV6);
    return P3{{v[0], bb::add(bb::sub(d1, bb::mul(d2, INV2)), bb::dbl(c3)), bb::mul(bb::sub(d2, d3), INV2), c3}};
}

// gcd(a, b) up to a unit; gcd(0, b) = b.  Each step makes the higher of the two lower: a <- lc(b) a - lc(a) t^(da - db) b.  The sum of
// the degrees (at most 6) falls with every step, so seven steps end it.
BB_HD P3 gcd(P3 a, P3 b) {
    int da = deg(a), db = deg(b);
#pragma unroll
    for (int s = 0; s < 7; s++) {
        if (da < db) { const P3 x = a; a = b; b = x; const int y = da; da = db; db = y; }
        if (db < 0) break;
        const uint32_t la = lead(a, da), lb = lead(b, db);
        const int k = da - db;
#pragma unroll
        for (int j = 0; j < 4; j++) a.c[j] = bb::sub(bb::mul(lb, a.c[j]), bb::mul(la, shifted(b, k, j)));
        da = deg(a);
    }
    return da < db ? b : a;
}

// a / t^k for the largest k with t^k dividing a (a != 0)
BB_HD P3 strip_t(P3 a) {
#pragma unroll
    for (int s = 0; s < 3; s++)
        if (!a.c[0]) a = P3{{a.c[1], a.c[2], a.c[3], 0}};
    return a;
}

BB_HD P3 scale(const P3& a, uint32_t s) { return P3{{bb::mul(a.c[0], s), bb::mul(a.c[1], s), bb::mul(a.c[2], s), bb::mul(a.c[3], s)}}; }

// Residues modulo the monic cubic t^3 + e[2] t^2 + e[1] t + e[0] (e = m.c, m.c[3] ignored): degree <= 2.
BB_HD P3 mulmod(const P3& a, const P3& b, const P3& m) {
    uint32_t p0 = bb::mul(a.c[0], b.c[0]);
    uint32_t p1 = bb::add(bb::mul(a.c[0], b.c[1]), bb::mul(a.c[1], b.c[0]));
    uint32_t p2 = bb::add(bb::add(bb::mul(a.c[0], b.c[2]), bb::mul(a.c[1], b.c[1])), bb::mul(a.c[2], b.c[0]));
    uint32_t p3 = bb::add(bb::mul(a.c[1], b.c[2]), bb::mul(a.c[2], b.c[1]));
    const uint32_t p4 = bb::mul(a.c[2], b.c[2]);
    p3 = bb::sub(p3, bb::mul(p4, m.c[2])); p2 = bb::sub(p2, bb::mul(p4, m.c[1])); p1 = bb::sub(p1, bb::mul(p4, m.c[0]));
    p2 = bb::sub(p2, bb::mul(p3, m.c[2])); p1 = bb::sub(p1, bb::mul(p3, m.c[1])); p0 = bb::sub(p0, bb::mul(p3, m.c[0]));
    return P3{{p0, p1, p2, 0}};
}
// (t + s) a modulo m
BB_HD P3 mul_linear(const P3& a, uint32_t s, const P3& m) {
    const uint32_t h = a.c[2];
    return P3{{bb::sub(bb::mul(a.c[0], s), bb::mul(h, m.c[0])), bb::sub(bb::add(a.c[0], bb::mul(a.c[1], s)), bb::mul(h, m.c[1])),
               bb::sub(bb::add(a.c[1], bb::mul(a.c[2], s)), bb::mul(h, m.c[2])), 0}};
}
// (t + s)^e modulo m, e > 0
BB_HD P3 powmod_linear(uint32_t s, uint32_t e, const P3& m) {
    P3 r{{s, bb::R1, 0, 0}};
    int top = 31;
    while (!((e >> top) & 1)) top--;
    for (int i = top - 1; i >= 0; i--) {
        r = mulmod(r, r, m);
        if ((e >> i) & 1) r = mul_linear(r, s, m);
    }
    return r;
}

// A square root of the square n != 0 (Tonelli-Shanks; p - 1 = 15 * 2^27).
BB_HD uint32_t field_sqrt(uint32_t n) {
    uint32_t c = bb::pow(NONRES, 15), x = bb::pow(n, 8), t = bb::pow(n, 15);
    int m = 27;
    while (t != bb::R1) {
        int i = 0;
        for (uint32_t u = t; u != bb::R1 && i < m; u = bb::sqr(u)) i++;
        if (i >= m) return 0;                                   // not a square (not reached for n a square)
        uint32_t b = c;
        for (int j = 0; j < m - i - 1; j++) b = bb::sqr(b);
        x = bb::mul(x, b); c = bb::sqr(b); t = bb::mul(t, c); m = i;
    }
    return x;
}

// The two roots of the monic t^2 + b t + c with distinct roots in F_p.
BB_HD void quadratic_roots(uint32_t b, uint32_t c, uint32_t& r0, uint32_t& r1) {
    const uint32_t s = field_sqrt(bb::sub(bb::sqr(b), bb::dbl(bb::dbl(c))));
    r0 = bb::mul(bb::sub(s, b), INV2);
    r1 = bb::mul(bb::sub(bb::neg(s), b), INV2);
}

// The distinct roots t != 0 in F_p of a != 0 (Montgomery words, in no particular order): their number, or -1 when a cubic with three
// such roots was not split in SPLIT_TRIES shifts.
BB_HD int nonzero_roots(const P3& a, uint32_t r[3]) {
    P3 h = strip_t(a);
    const int d = deg(h);
    if (d <= 0) return 0;
    h = scale(h, bb::inv(lead(h, d)));
    if (d == 1) { r[0] = bb::neg(h.c[0]); return 1; }
    // the monic cubic m: h, or t h for a quadratic h (whose extra root 0 is stripped below)
    const P3 m = d == 3 ? h : P3{{0, h.c[0], h.c[1], bb::R1}};
    // t^p mod m, then the product of m's distinct linear factors: gcd(m, t^p - t)
    P3 x = powmod_linear(0, bb::P, m);
    x.c[1] = bb::sub(x.c[1], bb::R1);
    P3 g = strip_t(gcd(m, x));
    const int k = deg(g);
    if (k <= 0) return 0;
    g = scale(g, bb::inv(lead(g, k)));
    if (k == 1) { r[0] = bb::neg(g.c[0]); return 1; }
    if (k == 2) { quadratic_roots(g.c[1], g.c[0], r[0], r[1]); return 2; }
    // three roots: gcd(g, (t + a)^((p-1)/2) - 1) holds those with t + a a non-zero square
    for (uint32_t a = 1; a <= (uint32_t)SPLIT_TRIES; a++) {
        P3 q = powmod_linear(bb::to_monty(a), (bb::P - 1) / 2, g);
        q.c[0] = bb::sub(q.c[0], bb::R1);
        P3 s = gcd(g, q);
        const int ks = deg(s);
        if (ks != 1 && ks != 2) continue;
        s = scale(s, bb::inv(lead(s, ks)));
        if (ks == 1) {
            // g = (t - r0)(t^2 + (g2 + r0) t + (g1 + r0 (g2 + r0)))
            r[0] = bb::neg(s.c[0]);
            const uint32_t q1 = bb::add(g.c[2], r[0]);
            quadratic_roots(q1, bb::add(g.c[1], bb::mul(r[0], q1)), r[1], r[2]);
        } else {
            // the third root: the roots of g sum to -g2
            quadratic_roots(s.c[1], s.c[0], r[0], r[1]);
            r[2] = bb::sub(bb::neg(g.c[2]), bb::add(r[0], r[1]));
        }
        return 3;
    }
    return -1;
}

// The roots v != x0 of a polynomial g != 0 in t = X - x0 (x0 Montgomery): canonical words, ascending, in v[0, n); n, or -1 as above.
BB_HD int other_roots(const P3& g, uint32_t x0, uint32_t v[3]) {
    uint32_t r[3] = {0, 0, 0};
    const int n = nonzero_roots(g, r);
#pragma unroll
    for (int j = 0; j < 3; j++) v[j] = j < n ? bb::from_monty(bb::add(x0, r[j])) : 0xffffffffu;
    const auto order = [](uint32_t& a, uint32_t& b) { const uint32_t lo = a < b ? a : b; b = a < b ? b : a; a = lo; };
    order(v[0], v[1]); order(v[1], v[2]); order(v[0], v[1]);
    return n;
}

}  // namespace poly
