// Host instantiation of the product's cubic polynomial arithmetic (valida_b200/csrc/polyroots.cuh — the text alts.cu's kernels
// compile) driven from stdin: one operation per line, field elements as canonical decimal words, results on stdout.  Built with g++ by
// tests/test_poly_roots_host.py, which checks every answer in Python.  No GPU, no CUDA runtime call.
//   interp v0 v1 v2 v3     -> c0 c1 c2 c3            the polynomial in t with those values at t = 0, 1, 2, 3
//   gcd a0..a3 b0..b3      -> g0 g1 g2 g3            gcd(a, b) up to a unit
//   roots a0..a3 x0        -> n v0 v1 v2             other_roots: the roots v != x0 of a(X - x0), ascending (n = -1: not split)
#include <cstdio>
#include <cstring>
#include "polyroots.cuh"

static bool read_poly(poly::P3& a) {
    for (int i = 0; i < 4; i++) {
        unsigned x;
        if (scanf("%u", &x) != 1) return false;
        a.c[i] = bb::to_monty(x);
    }
    return true;
}

static void print_poly(const poly::P3& a) {
    printf("%u %u %u %u\n", bb::from_monty(a.c[0]), bb::from_monty(a.c[1]), bb::from_monty(a.c[2]), bb::from_monty(a.c[3]));
}

int main() {
    char op[32];
    while (scanf("%31s", op) == 1) {
        if (!strcmp(op, "interp")) {
            poly::P3 v;
            if (!read_poly(v)) return 1;
            print_poly(poly::interp(v.c));
        } else if (!strcmp(op, "gcd")) {
            poly::P3 a, b;
            if (!read_poly(a) || !read_poly(b)) return 1;
            print_poly(poly::gcd(a, b));
        } else if (!strcmp(op, "roots")) {
            poly::P3 a;
            unsigned x0;
            if (!read_poly(a) || scanf("%u", &x0) != 1) return 1;
            uint32_t v[3];
            const int n = poly::other_roots(a, bb::to_monty(x0), v);
            printf("%d %u %u %u\n", n, n > 0 ? v[0] : 0, n > 1 ? v[1] : 0, n > 2 ? v[2] : 0);
        } else return 2;
    }
    return 0;
}
