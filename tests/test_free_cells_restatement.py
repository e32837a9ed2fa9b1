"""The definition of a free cell (vgpu_free_cells, valida_b200/csrc/free.cu) written literally in plain Python, on the independent
texts of the AIRs (AIRS, test_quotient_restatement.py) and the interactions (CHIPS, test_perm_trace_restatement.py).

Main-trace cell (r, c) of one chip's witness is free when
  1. every Air::eval assertion keeps its value when the cell is set to x0 + 1, x0 + 2, x0 + 3 (and, here, to random values), on row r
     and on row (r - 1) mod h with that row's own selectors (on a one-row chip both are the one evaluation);
  2. no interaction's count gives column c a non-zero summed weight, and on a row where an interaction's count is not 0 none of its
     fields does.
The four values decide 1 exactly because every constraint has degree <= 3 in any single cell: the fourth finite difference of every
constraint in every main cell is pinned here to be zero.  And on the witnesses of vb.run_program the gaps the reference's text leaves
(memory and range AIRs empty, no program-bus interaction) come out as derived from that text.  CPU only."""
import ctypes as C

import numpy as np
import pytest

from test_perm_trace_restatement import CHIPS, P, apply
from test_quotient_restatement import AIRS

MEMORY_ALWAYS = ("diff", "diff_inv", "addr_not_equal", "counter", "counter_mult")
MEMORY_WHEN_UNUSED = ("addr", "value[0]", "value[1]", "value[2]", "value[3]", "clk", "is_static_initial")
MEMORY_COLUMNS = {"addr": 0, "value[0]": 1, "value[1]": 2, "value[2]": 3, "value[3]": 4, "clk": 5, "is_static_initial": 6, "is_read": 7,
                  "is_write": 8, "diff": 9, "diff_inv": 10, "addr_not_equal": 11, "counter": 12, "counter_mult": 13}


def width(chip):
    import valida_b200 as vb

    return C.cast(vb.lib().vgpu_basic_machine_chip(chip), C.POINTER(C.c_uint32))[1]


def weight(col, c):
    """The summed weight a VirtualPairCol gives main column c."""
    kind, v = col
    if kind == "main":
        return 1 if v == c else 0
    if kind == "const":
        return 0
    if kind == "weighted":
        return sum(w for cc, w in v if cc == c) % P
    return sum(1 for cc in v if cc == c) % P


def air_values(chip, main, r):
    """Every Air::eval assertion's value on row r (its next row (r + 1) mod h, its own selectors)."""
    if AIRS[chip] is None:
        return []
    h = main.shape[0]
    last = 1 if r == h - 1 else 0
    sel = {"first": 1 if r == 0 else 0, "last": last, "transition": 1 - last}
    return [x % P for x in AIRS[chip]([int(v) for v in main[r]], [int(v) for v in main[(r + 1) % h]], sel)]


def bus_pinned(chip, row, c):
    for _, _, fields, count in CHIPS.get(chip, []):
        if weight(count, c):
            return True
        if apply(count, row) and any(weight(f, c) for f in fields):
            return True
    return False


def air_pinned(chip, main, r, c, values):
    h = main.shape[0]
    rows = sorted({r, (r - 1) % h})
    base = [air_values(chip, main, q) for q in rows]
    m = main.copy()
    for v in values:
        m[r, c] = v % P
        if [air_values(chip, m, q) for q in rows] != base:
            return True
    return False


def free_py(chip, main, rows=None, random_values=0, seed=0):
    """The free cells of one chip's main trace, ascending by (row, column); rows: the rows judged (all by default)."""
    rng = np.random.default_rng(seed)
    h, w = main.shape
    out = []
    for r in (range(h) if rows is None else sorted(set(rows))):
        row = [int(v) for v in main[r]]
        for c in range(w):
            if bus_pinned(chip, row, c):
                continue
            x0 = int(main[r, c])
            values = [x0 + 1, x0 + 2, x0 + 3] + [int(x) for x in rng.integers(0, P, random_values)]
            if AIRS[chip] is not None and air_pinned(chip, main, r, c, values):
                continue
            out.append((r, c))
    return out


def per_column(cells, w):
    n = [0] * w
    for _, c in cells:
        n[c] += 1
    return n


@pytest.mark.parametrize("chip", range(14))
def test_every_constraint_has_degree_at_most_three_in_every_cell(built, chip):
    """The fourth finite difference of every AIR constraint in every single main cell (local and next row) is zero on random rows."""
    if AIRS[chip] is None:
        return
    rng = np.random.default_rng(700 + chip)
    w = width(chip)
    for _ in range(3):
        loc = [int(x) for x in rng.integers(0, P, w)]
        nxt = [int(x) for x in rng.integers(0, P, w)]
        for sel in ({"first": 1, "last": 0, "transition": 1}, {"first": 0, "last": 1, "transition": 0}, {"first": 0, "last": 0, "transition": 1}):
            for which in (0, 1):
                for c in range(w):
                    vals = []
                    for k in range(5):
                        a, b = list(loc), list(nxt)
                        (a if which == 0 else b)[c] = (loc[c] if which == 0 else nxt[c]) + k
                        vals.append([x % P for x in AIRS[chip](a, b, sel)])
                    d4 = [(f0 - 4 * f1 + 6 * f2 - 4 * f3 + f4) % P for f0, f1, f2, f3, f4 in zip(*vals)]
                    assert not any(d4), (chip, which, c)


@pytest.mark.parametrize("chip", range(14))
def test_the_four_values_decide_what_random_values_would(built, chip):
    """On random traces (h = 1, 2 and 8) the cells free under x0 + 1..3 are exactly those free under those and six random values."""
    for h in (1, 2, 8):
        main = np.random.default_rng(800 + 16 * chip + h).integers(0, P, (h, width(chip)), dtype=np.uint32)
        assert free_py(chip, main) == free_py(chip, main, random_values=6, seed=chip), (chip, h)


def test_known_gaps_on_a_fibonacci_witness(built):
    """Memory: diff, diff_inv, addr_not_equal, counter, counter_mult free on every row; addr, value, clk and is_static_initial exactly
    where is_read + is_write = 0; is_read and is_write never.  Range: counter exactly where mult = 0, mult never.  Program:
    multiplicity on every row."""
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(25), initial_fp=0x1000)
    mem = t.main[2]
    free = set(free_py(2, mem))
    unused = (mem[:, 7].astype(np.int64) + mem[:, 8]) % P == 0
    assert unused.any() and not unused.all()
    for r in range(mem.shape[0]):
        for name, c in MEMORY_COLUMNS.items():
            want = name in MEMORY_ALWAYS or (name in MEMORY_WHEN_UNUSED and unused[r])
            assert ((r, c) in free) == want, (r, name)
    rng = t.main[12]
    assert set(free_py(12, rng)) == {(r, 1) for r in range(rng.shape[0]) if rng[r, 0] == 0}
    assert (rng[:, 0] == 0).any()
    prog = t.main[1]
    assert free_py(1, prog) == [(r, 0) for r in range(prog.shape[0])]
