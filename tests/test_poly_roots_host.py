"""The product's cubic polynomial arithmetic over BabyBear (valida_b200/csrc/polyroots.cuh — what vgpu_cell_alternatives' kernels fold
and solve) instantiated on the host and checked against plain Python: interpolation against the defining sums, gcd against a monic
Euclid with inverses, and the roots other than the cell's value against polynomials built from planted roots — repeated roots,
irreducible quadratic factors, roots at 0 and p - 1, constants and the zero polynomial.  CPU only."""
import os
import random
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 2013265921


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("poly") / "poly_roots_check")
    subprocess.run(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "valida_b200", "csrc"), "-I", "/usr/local/cuda/include",
                    os.path.join(ROOT, "tests", "c", "poly_roots_check.cc"), "-o", out], check=True)
    return out


def run(exe, lines):
    r = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True)
    return [[int(x) for x in ln.split()] for ln in r.stdout.splitlines()]


def pmul(a, b):
    out = [0] * (len(a) + len(b) - 1)
    for i, x in enumerate(a):
        for j, y in enumerate(b):
            out[i + j] = (out[i + j] + x * y) % P
    return out


def trim(a):
    a = [x % P for x in a]
    while a and a[-1] == 0:
        a.pop()
    return a


def monic(a):
    a = trim(a)
    if not a:
        return a
    s = pow(a[-1], P - 2, P)
    return [x * s % P for x in a]


def pmod(a, b):
    a, b = trim(a), monic(b)
    while len(a) >= len(b):
        q, k = a[-1], len(a) - len(b)
        for i, y in enumerate(b):
            a[i + k] = (a[i + k] - q * y) % P
        a = trim(a)
    return a


def pgcd(a, b):
    a, b = trim(a), trim(b)
    while b:
        a, b = b, pmod(a, b)
    return monic(a)


def ev(a, x):
    return sum(c * pow(x, i, P) for i, c in enumerate(a)) % P


def nonresidue(rng):
    while True:
        n = rng.randrange(1, P)
        if pow(n, (P - 1) // 2, P) == P - 1:
            return n


def planted(rng):
    """A polynomial of degree <= 3 in t and its distinct roots in F_p."""
    kind = rng.randrange(8)
    special = [0, 1, P - 1, P - 2, rng.randrange(P)]
    root = lambda: rng.choice(special) if rng.random() < 0.3 else rng.randrange(P)  # noqa: E731
    unit = rng.randrange(1, P)
    if kind == 0:
        return [0, 0, 0, 0], None                     # the zero polynomial: every value is a root
    if kind == 1:
        return [unit, 0, 0, 0], set()                  # a non-zero constant
    if kind == 2:                                       # an irreducible quadratic, times a unit or a linear factor
        n = nonresidue(rng)
        q = [(-n) % P, 0, 1]
        if rng.random() < 0.5:
            return [x * unit % P for x in q] + [0], set()
        r = root()
        return pmul(q, [(-r) % P, 1]), {r}
    deg = rng.randrange(1, 4)
    rs = [root() for _ in range(deg)]
    if kind == 3 and deg >= 2:
        rs[1] = rs[0]                                   # a repeated root
    if kind == 4 and deg == 3:
        rs = [rs[0]] * 3
    a = [unit]
    for r in rs:
        a = pmul(a, [(-r) % P, 1])
    return a + [0] * (4 - len(a)), set(rs)


def test_interpolation_matches_the_defining_sums(exe):
    rng = random.Random(11)
    polys = [[0, 0, 0, 0], [1, 0, 0, 0], [0, 0, 0, 1], [P - 1] * 4] + [[rng.randrange(P) for _ in range(4)] for _ in range(300)]
    got = run(exe, ["interp %d %d %d %d" % tuple(ev(a, k) for k in range(4)) for a in polys])
    assert got == polys


def test_gcd_matches_euclid_with_inverses(exe):
    rng = random.Random(12)
    pairs = []
    for _ in range(400):
        a, _ = planted(rng)
        b, _ = planted(rng)
        if rng.random() < 0.4:                          # a common factor
            c = [rng.randrange(P), 1]
            a = (pmul(a[:3], c) + [0])[:4]
            b = (pmul(b[:3], c) + [0])[:4]
        pairs.append((a, b))
    got = run(exe, ["gcd %s %s" % (" ".join(map(str, a)), " ".join(map(str, b))) for a, b in pairs])
    for (a, b), g in zip(pairs, got):
        assert monic(g) == pgcd(a, b), (a, b, g)


def test_roots_other_than_the_value(exe):
    rng = random.Random(13)
    cases = []
    for _ in range(600):
        a, roots = planted(rng)
        if roots is None:
            continue
        x0 = rng.choice([0, 1, P - 1, rng.randrange(P)])
        cases.append((a, roots, x0))
    got = run(exe, ["roots %s %d" % (" ".join(map(str, a)), x0) for a, _, x0 in cases])
    for (a, roots, x0), (n, *v) in zip(cases, got):
        want = sorted((x0 + r) % P for r in roots if r)
        assert n == len(want) and v[:n] == want, (a, roots, x0, n, v)
        assert all(ev(a, (x - x0) % P) == 0 for x in v[:n])
