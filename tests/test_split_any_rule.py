"""The row rule of a split proof at any rank count 1..16 (csrc/ctx.h), through the library's own exports (no GPU): with P the next
power of two >= N and V = 8 P units, a vector of n >= 4096 P rows is cut into V units and rank r holds units
[r V // N, (r + 1) V // N).  At a power of two N that is today's even split; otherwise the runs differ by at most one unit."""
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RANKS = range(1, 17)
LENGTHS = [1 << k for k in range(0, 25)]
RES = r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)"


def _units(n):
    return 8 * (1 << (n - 1).bit_length())


def _is_pow2(n):
    return n & (n - 1) == 0


def _runs(share, length, n):
    return [share(length, n, r) for r in range(n)]


def _assert_partition(runs, length):
    at = 0
    for b, c, split in runs:
        assert split and b == at, runs
        at += c
    assert at == length, runs


def test_row_runs_partition_in_units(built):
    import valida_b200 as vb

    for n in RANKS:
        v = _units(n)
        for length in LENGTHS:
            runs = _runs(vb.row_share, length, n)
            split = n > 1 and length >= 4096 * (v // 8)
            if not split:
                assert runs == [(0, length, False)] * n, (n, length)
                continue
            _assert_partition(runs, length)
            unit = length // v
            assert all(b % unit == 0 and c % unit == 0 for b, c, _ in runs), (n, length)
            counts = [c // unit for _, c, _ in runs]
            assert max(counts) - min(counts) <= 1, (n, counts)
            assert [b // unit for b, _, _ in runs] == [r * v // n for r in range(n)]


def test_power_of_two_ranks_keep_the_even_split(built):
    import valida_b200 as vb

    for n in (1, 2, 4, 8, 16):
        for length in LENGTHS:
            rows = _runs(vb.row_share, length, n)
            if n > 1 and length >= 4096 * n:
                assert rows == [(r * length // n, length // n, True) for r in range(n)], (n, length)
            else:
                assert rows == [(0, length, False)] * n, (n, length)
            layers = _runs(vb.tree_share, length, n)
            if n > 1 and length >= n:
                assert layers == [(r * length // n, length // n, True) for r in range(n)], (n, length)
            else:
                assert layers == [(0, length, False)] * n, (n, length)


def test_uneven_ranks_examples_and_layer_rule(built):
    """N = 3 gives 10 / 11 / 11 of 32 units and N = 6 10 / 11 / 11 / 10 / 11 / 11 of 64; the largest run is 3.1 % above an even
    share at N = 3 and 6, 1.6 % at 5, 9.4 % at 7.  A tree layer stays split down to the V-node layer (whole units per rank), not below."""
    import valida_b200 as vb

    n_rows = 1 << 20
    for n, want in ((3, [10, 11, 11]), (6, [10, 11, 11, 10, 11, 11])):
        unit = n_rows // _units(n)
        assert [c // unit for _, c, _ in _runs(vb.row_share, n_rows, n)] == want
    for n, excess in ((3, 3.1), (5, 1.6), (6, 3.1), (7, 9.4)):
        runs = _runs(vb.row_share, n_rows, n)
        assert round(100 * (max(c for _, c, _ in runs) * n / n_rows - 1), 1) == excess, n
    for n in RANKS:
        if _is_pow2(n):
            continue
        v = _units(n)
        for length in LENGTHS:
            runs = _runs(vb.tree_share, length, n)
            if length < v:
                assert runs == [(0, length, False)] * n, (n, length)
            else:
                _assert_partition(runs, length)
                bounds = [r * v // n * (length // v) for r in range(n + 1)]
                assert runs == [(bounds[r], bounds[r + 1] - bounds[r], True) for r in range(n)], (n, length)


def test_column_plans_tile_every_width_at_any_rank_count(built):
    import valida_b200 as vb

    shapes = [(1 << 22, 51), (1 << 24, 14), (1 << 22, 3), (1 << 20, 1)]
    for n in RANKS:
        plan = vb.split_column_plan(n, shapes)
        for (_, w), pl in zip(shapes, plan):
            assert len(pl) == n + 1 and pl[0] == 0 and pl[-1] == w and all(pl[r] <= pl[r + 1] for r in range(n)), (n, pl)


def test_changed_kernels_stay_in_registers(built):
    """cols_to_rows_kernel (now given the run table) keeps no stack frame; the quotient kernel, launched once per run of units whose
    next rows one rank holds, keeps its 64-register ceiling and uses no local memory."""
    import re
    import shutil
    import subprocess

    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("needs cuobjdump")
    out = subprocess.run([cuobjdump, "-res-usage", os.path.join(ROOT, "valida_b200", "libvalida_b200.so")],
                         capture_output=True, text=True, check=True).stdout
    res = {m.group(1): tuple(int(m.group(i)) for i in range(2, 6)) for m in re.finditer(RES, out)}
    c2r = [v for k, v in res.items() if "cols_to_rows_kernel" in k]
    assert c2r and all(stack == 0 and local == 0 for _, stack, _, local in c2r), c2r
    q = {k: v for k, v in res.items() if "quotient_kernel" in k}
    assert len(q) == 14 and all(reg <= 64 and local == 0 for reg, _, _, local in q.values()), q
