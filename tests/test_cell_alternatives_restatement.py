"""The definition of a cell's alternative values (vgpu_cell_alternatives, valida_b200/csrc/alts.cu) written independently in plain
Python, on the independent texts of the AIRs (AIRS, test_quotient_restatement.py) and the interactions (CHIPS,
test_perm_trace_restatement.py).

Main-trace cell (r, c) holding x0 has S: the Air::eval assertions whose value depends on it, on row r and on row (r - 1) mod h with that
row's own selectors (on a one-row chip the one evaluation).  Each is a polynomial of degree <= 3 in the cell; here it is interpolated
(Lagrange) through four RANDOM points, not x0 + 0..3.  The cell is listed when S is not empty and the polynomials share a root v != x0
in F_p: here their monic gcd (Euclid with inverses) is split by Cantor-Zassenhaus with Python's RNG.  bus: free_cells' rule.

Every value listed, substituted into AIRS, makes each assertion of S vanish, and the number of values is the number of distinct F_p
roots other than x0.  On the reference programs' witnesses the gaps are as found on the CPU before the device call existed: flags that
a bus-free value can flip.  CPU only."""
import random

import numpy as np
import pytest

from test_free_cells_restatement import air_values, bus_pinned, width
from test_perm_trace_restatement import P
from test_quotient_restatement import AIRS


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


def pmul(a, b):
    if not a or not b:
        return []
    out = [0] * (len(a) + len(b) - 1)
    for i, x in enumerate(a):
        for j, y in enumerate(b):
            out[i + j] = (out[i + j] + x * y) % P
    return out


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


def ppow(base, e, m):
    r, base = [1], pmod(base, m)
    while e:
        if e & 1:
            r = pmod(pmul(r, base), m)
        base = pmod(pmul(base, base), m)
        e >>= 1
    return r


def ev(a, x):
    return sum(c * pow(x, i, P) for i, c in enumerate(a)) % P


def lagrange(xs, ys):
    """The polynomial of degree < len(xs) through (xs, ys)."""
    out = []
    for i, (xi, yi) in enumerate(zip(xs, ys)):
        num, den = [1], 1
        for j, xj in enumerate(xs):
            if j != i:
                num = pmul(num, [(-xj) % P, 1])
                den = den * (xi - xj) % P
        s = yi * pow(den, P - 2, P) % P
        out = [(a + s * b) % P for a, b in zip(out + [0] * (len(num) - len(out)), num)]
    return trim(out)


def distinct_roots_part(g):
    """gcd(g, X^p - X): the product of g's distinct linear factors."""
    d = ppow([0, 1], P, g)
    d = d + [0] * (2 - len(d))
    d[1] = (d[1] - 1) % P
    return pgcd(g, d)


def cantor_zassenhaus(g, rng):
    """The roots of g, a product of distinct linear factors: split by gcd(g, (X + a)^((p-1)/2) - 1) for random a."""
    g = monic(g)
    if len(g) <= 1:
        return []
    if len(g) == 2:
        return [(-g[0]) % P]
    while True:
        h = ppow([rng.randrange(P), 1], (P - 1) // 2, g)
        h = [(h[0] - 1) % P] + h[1:] if h else [P - 1]
        d = pgcd(g, h)
        if 1 < len(d) < len(g):
            return cantor_zassenhaus(d, rng) + cantor_zassenhaus(pdiv(g, d), rng)


def pdiv(a, b):
    """a / b, exact."""
    a, b = trim(a), monic(b)
    q = [0] * (len(a) - len(b) + 1)
    while len(a) >= len(b):
        c, k = a[-1], len(a) - len(b)
        q[k] = c
        for i, y in enumerate(b):
            a[i + k] = (a[i + k] - c * y) % P
        a = trim(a)
    return q


def assertions(chip, main, r):
    """The values of the assertions of the evaluations that read row r: row r's, then row (r - 1) mod h's (one on a one-row chip)."""
    h = main.shape[0]
    return [v for q in sorted({r, (r - 1) % h}) for v in air_values(chip, main, q)]


def cell_polys(chip, main, r, c, rng):
    """S: (index in assertions(), polynomial in X, the cell's value) of each assertion whose value depends on cell (r, c)."""
    xs = rng.sample(range(P), 4)
    evals = []
    m = main.copy()
    for x in xs:
        m[r, c] = x
        evals.append(assertions(chip, m, r))
    # degree <= 3: equal at four points is constant
    return [(j, lagrange(xs, [e[j] for e in evals])) for j in range(len(evals[0])) if len({e[j] for e in evals}) > 1]


def alternatives_py(chip, main, seed=0):
    """[(row, column, x0, values, bus)] ascending by (row, column): every listed cell of one chip's main trace."""
    if AIRS[chip] is None:
        return []
    rng = random.Random(seed)
    h, w = main.shape
    out = []
    for r in range(h):
        row = [int(v) for v in main[r]]
        for c in range(w):
            S = [p for _, p in cell_polys(chip, main, r, c, rng)]
            if not S:
                continue
            g = S[0]
            for p in S[1:]:
                g = pgcd(g, p)
            x0 = int(main[r, c])
            vals = sorted(v for v in cantor_zassenhaus(distinct_roots_part(g), rng) if v != x0) if len(g) > 1 else []
            if vals:
                out.append((r, c, x0, tuple(vals), bus_pinned(chip, row, c)))
    return out


def per_column(cells, w):
    n = [[0, 0] for _ in range(w)]
    for _, c, _, _, bus in cells:
        n[c][0] += 1
        n[c][1] += not bus
    return [tuple(x) for x in n]


def _witness(name):
    import programs
    import valida_b200 as vb

    prog = {"fib25": lambda: vb.fib_program(25), "config5": lambda: programs.config5_program(30),
            "left_imm": lambda: programs.mixed_program(40)}[name]()
    return vb.run_program(prog, initial_fp=0x1000)


@pytest.mark.parametrize("chip", range(14))
def test_values_are_common_roots_on_random_traces(built, chip):
    """On random traces with some boolean-like cells (0 or 1), each value makes every assertion of S vanish, and the number of
    values is the number of distinct roots other than x0."""
    if AIRS[chip] is None:
        return
    rng = np.random.default_rng(900 + chip)
    for h in (1, 2, 8):
        main = rng.integers(0, P, (h, width(chip)), dtype=np.uint32)
        flags = rng.random(main.shape) < 0.5
        main[flags] = rng.integers(0, 2, int(flags.sum()))
        for r, c, x0, vals, _ in alternatives_py(chip, main, seed=chip):
            S = cell_polys(chip, main, r, c, random.Random(1))
            assert S
            for v in vals:
                m = main.copy()
                m[r, c] = v
                at_v = assertions(chip, m, r)
                assert all(at_v[j] == 0 for j, _ in S), (chip, r, c, v)
            g = S[0][1]
            for _, p in S[1:]:
                g = pgcd(g, p)
            n = len(distinct_roots_part(g)) - 1 - (1 if ev(g, x0) == 0 else 0)
            assert len(vals) == n, (chip, r, c, vals)


FINDINGS = {
    # program: {chip: (listed, bus-free, {column name: bus-free rows}) }; None: columns not pinned here
    "fib25": {0: (594, 252, {"is_imm_op": 71, "is_left_imm_op": 71, "is_beq": 52, "is_bne": 52, "is_imm32": 6}),
              3: (384, 69, None)},
    "config5": {0: (2793, 153, None), 8: (91, 16, None), 10: (408, 0, {})},
    "left_imm": {0: (1746, 424, None), 8: (332, 192, None)},
}
BUS_FREE_COLUMNS = {("fib25", 3): {"input_1[0]", "input_2[0]", "output[0]"}, ("config5", 8): {"is_lt", "is_lte", "is_sle", "is_slt"},
                    ("left_imm", 8): {"is_lt", "is_slt"}}


def _short(name):
    return name.rsplit(".", 1)[-1]


@pytest.mark.parametrize("name", sorted(FINDINGS))
def test_findings_on_the_reference_programs(built, name):
    import valida_b200 as vb

    t = _witness(name)
    for chip, (listed, free, cols) in FINDINGS[name].items():
        cells = alternatives_py(chip, t.main[chip])
        assert len(cells) == listed and sum(not b for *_, b in cells) == free, (name, chip, len(cells))
        assert all(len(v) == 1 for _, _, _, v, _ in cells)                   # exactly one other value each
        names = [_short(vb.column_name(chip, vb.TRACE_MAIN, c)) for c in range(width(chip))]
        got = {}
        for _, c, _, _, bus in cells:
            if not bus:
                got[names[c]] = got.get(names[c], 0) + 1
        if cols is not None:
            assert got == cols, (name, chip, got)
        if (name, chip) in BUS_FREE_COLUMNS:
            assert got and set(got) <= BUS_FREE_COLUMNS[(name, chip)], (name, chip, got)
        if chip == 0 and cols is None:
            assert all(n.startswith("is_") for n in got), got                 # opcode flags
