"""cell_alternatives on the GPU (vgpu_cell_alternatives, valida_b200/csrc/alts.cu): every main-trace cell that the AIR would accept at
another value, with those values, on one GPU and over the row shards of a split context.

The list, the totals and the per-column counts are held to alternatives_py, the independent restatement in
test_cell_alternatives_restatement.py.  The values are shown to mean what the definition promises: bus-free values substituted into a
witness leave check_witness clean and check_buses empty and a proof of it verifies; a bus-read value leaves the chip's AIR clean and
unbalances a bus; a cell set to a random value is listed with its original value among its values."""
import ctypes as C

import numpy as np
import pytest

from test_cell_alternatives_restatement import alternatives_py, per_column
from test_check_constraints_restatement import PREP_CHIPS
from test_free_cells_restatement import width
from test_gpu_check_failures import _close, _ranks
from test_gpu_free_cells import PROGRAMS, _boundary_changed, _check, _changed, _prep_of, _witness
from test_gpu_local_shards import BORROW_LAYOUTS, _col_major, _local_tensors, _monty
from test_perm_trace_restatement import P

pytestmark = pytest.mark.gpu
CH = np.random.default_rng(5151).integers(0, P, 15, dtype=np.uint32)
BIG = 1 << 40


def _device(ctx, chip, main, prep, cap=BIG):
    import valida_b200 as vb

    dm = ctx.upload(main)
    dp = ctx.upload(prep) if prep is not None else None
    total = vb.cell_alternatives(ctx, chip, dm, dp, cap=0).total
    return vb.cell_alternatives(ctx, chip, dm, dp, cap=min(cap, total))


def _as_tuples(res):
    return [(c.row, c.column, c.value, c.values, c.bus) for c in res.cells]


def _agree(ctx, chip, main, prep):
    import valida_b200 as vb

    want = alternatives_py(chip, main)
    got = _device(ctx, chip, main, prep)
    assert _as_tuples(got) == want, chip
    assert got.total == len(want) and got.complete and got.bus_free == sum(not b for *_, b in want)
    names = [vb.column_name(chip, vb.TRACE_MAIN, c) for c in range(width(chip))]
    assert [got.per_column[n] for n in names] == per_column(want, width(chip))
    assert all(c.column_name == names[c.column] for c in got.cells)
    return want


@pytest.mark.parametrize("h", [1, 2, 8, 64])
@pytest.mark.parametrize("chip", range(14))
def test_random_traces_match_the_restatement(ctx, chip, h):
    rng = np.random.default_rng(4000 + 16 * chip + h)
    main = rng.integers(0, P, (h, width(chip)), dtype=np.uint32)
    # boolean-like cells, so that flags have another value and some counts are 0 (the bus flag takes both values)
    flags = rng.random(main.shape) < 0.4
    main[flags] = rng.integers(0, 2, int(flags.sum()))
    prep = rng.integers(0, P, (h, 7 if chip == 1 else 1), dtype=np.uint32) if chip in PREP_CHIPS else None
    _agree(ctx, chip, main, prep)


@pytest.mark.parametrize("name", sorted(PROGRAMS))
def test_program_witnesses_match_the_restatement(ctx, name):
    t, mats = _witness(name)
    for chip in range(14):
        _agree(ctx, chip, mats[chip], _prep_of(mats, chip))


def test_cap_gives_prefixes(ctx):
    import valida_b200 as vb

    _, mats = _witness("fib25")
    dm = ctx.upload(mats[0])
    full = vb.cell_alternatives(ctx, 0, dm, None, cap=BIG)
    total = full.total
    assert total > 500 and full.complete
    for cap in (0, 1, 200, total - 1, total, total + 1, 10 * total):
        got = vb.cell_alternatives(ctx, 0, dm, None, cap=cap)
        assert (got.total, got.bus_free, got.per_column) == (total, full.bus_free, full.per_column)
        assert got.cells == full.cells[:min(cap, total)] and got.complete == (cap >= total)


@pytest.mark.parametrize("name", sorted(PROGRAMS))
def test_bus_free_values_keep_the_witness_valid(ctx, oracle, name):
    """Every chip's bus-free values, substituted together on rows at least 2 apart (so no two share an assertion), leave what
    check_witness and check_buses say unchanged: on a clean witness they stay clean and empty, and a proof of that witness verifies."""
    import valida_b200 as vb

    t, mats = _witness(name)
    before = _check(ctx, mats)
    out = list(mats)
    changed = 0
    for chip in range(14):
        res = _device(ctx, chip, mats[chip], _prep_of(mats, chip))
        a = mats[chip].copy()
        h = a.shape[0]
        rows = []
        for c in res.cells:
            # no two changed cells in one evaluation: rows at least 2 apart, around the wrap too
            if not c.bus and all((c.row - q) % h not in (0, 1, h - 1) for q in rows):
                a[c.row, c.column] = c.values[-1]
                rows.append(c.row)
                changed += 1
        out[chip] = a
    assert changed
    assert _check(ctx, out) == before, name
    if before != (True, []):
        return
    cfg = vb.StarkConfig(ctx, oracle.rc480)
    dm = [ctx.upload(m) for m in out[:14]]
    dp = [ctx.upload(m) for m in out[14:]]
    proof = vb.prove_machine(cfg, t, device_resident=(dm, dp))
    vb.verify_machine(cfg, proof, t.preprocessed)


def test_bus_read_values_leave_the_air_and_unbalance_a_bus(ctx):
    import valida_b200 as vb

    _, mats = _witness("fib25")
    base = [ctx.upload(m) for m in mats]
    rng = np.random.default_rng(5)
    seen = 0
    for chip in range(14):
        res = _device(ctx, chip, mats[chip], _prep_of(mats, chip))
        bus = [c for c in res.cells if c.bus]
        for i in rng.choice(len(bus), min(4, len(bus)), replace=False) if bus else []:
            c = bus[i]
            bad = _changed(mats, chip, c.row, c.column, c.values[0])
            dm = list(base[:14])
            dm[chip] = ctx.upload(bad[chip])
            rep, _ = vb.check_witness(ctx, dm, base[14:], CH)
            assert rep[chip][0] == -1, (chip, c)
            assert vb.check_buses(ctx, dm, base[14:], CH).tuples, (chip, c)
            seen += 1
    assert seen


def test_repair(ctx):
    """A cell of a clean witness that some assertion depends on, set alone to a random value, is listed with its original value among
    its values."""
    import random

    from test_cell_alternatives_restatement import cell_polys

    rng = np.random.default_rng(9)
    _, mats = _witness("config5")
    for chip in (0, 3, 8, 10):
        main = mats[chip]
        h, w = main.shape
        tried = 0
        for _ in range(200):
            r, c = int(rng.integers(0, h)), int(rng.integers(0, w))
            v = int(rng.integers(0, P))
            bad = main.copy()
            bad[r, c] = v
            if not cell_polys(chip, bad, r, c, random.Random(0)):
                continue
            res = _device(ctx, chip, bad, _prep_of(mats, chip))
            cell = [x for x in res.cells if (x.row, x.column) == (r, c)]
            assert cell and int(main[r, c]) in cell[0].values, (chip, r, c)
            tried += 1
            if tried == 6:
                break
        assert tried, chip


@pytest.mark.parametrize("name", ["fib25", "config5", "left_imm"])
def test_disjoint_from_free_cells(ctx, name):
    import valida_b200 as vb

    _, mats = _witness(name)
    for chip in range(14):
        dm = ctx.upload(mats[chip])
        p = _prep_of(mats, chip)
        dp = ctx.upload(p) if p is not None else None
        free = {(c.row, c.column) for c in vb.free_cells(ctx, chip, dm, dp, cap=BIG).cells}
        listed = {(c.row, c.column) for c in vb.cell_alternatives(ctx, chip, dm, dp, cap=BIG).cells}
        assert not free & listed, chip


@pytest.fixture(scope="module")
def fib15(built):
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(((1 << 15) - 17) // 7), initial_fp=0x1000)
    assert t.main[0].shape[0] == 1 << 15
    return [np.array(m) for m in list(t.main) + list(t.preprocessed)]


def _key(res):
    return (_as_tuples(res), res.total, res.bus_free, res.per_column)


@pytest.mark.parametrize("nranks", [2, 3, 4, 8])
def test_split_every_route(ctx, fib15, nranks):
    import torch
    import valida_b200 as vb

    ctxs = _ranks(nranks)
    try:
        mats = _boundary_changed(fib15, ctxs, (0, 3, 8))
        chips = list(range(14))
        caps, want = {}, {}
        for chip in chips:
            res = _device(ctx, chip, mats[chip], _prep_of(mats, chip))
            want[chip] = _key(res)
            caps[chip] = res.total
        layout = "stride_rows_plus_3" if nranks % 2 else "base_plus_one_word"
        pad, off = BORROW_LAYOUTS[layout]

        def borrow(c, r):
            tens = _local_tensors(c, [_monty(a) for a in mats], lambda a, d: _col_major(a, d, pad, off))
            torch.cuda.synchronize()
            return [c.borrow_tensor_local(x, a.shape[0]) for x, a in zip(tens, mats)]

        routes = {"upload": lambda c, r: [c.upload(m) for m in mats],
                  "upload_rows": lambda c, r: [c.upload_rows(m) for m in mats],
                  "import_tensor_local": lambda c, r: [c.import_tensor_local(x, a.shape[0])
                                                       for x, a in zip(_local_tensors(c, mats, lambda a, d: _col_major(a, d)), mats)],
                  "borrow_" + layout: borrow}
        for name, make in routes.items():
            def rank(r, c):
                dm = make(c, r)
                out = {}
                for chip in chips:
                    c.comm_stats(reset=True)
                    res = vb.cell_alternatives(c, chip, dm[chip], _prep_of(dm, chip), cap=caps[chip])
                    out[chip] = (_key(res), c.comm_stats()["allgather"][0])
                return out

            for got in vb.run_ranks(rank, ctxs):
                for chip in chips:
                    split = ctxs[0].local_rows(mats[chip].shape[0])[1] < mats[chip].shape[0]
                    gathers = (3 if want[chip][1] else 2) if split else 0
                    assert got[chip] == (want[chip], gathers), (name, chip)
    finally:
        _close(ctxs)


def test_refusals_launch_nothing(ctx, fib15):
    import valida_b200 as vb

    def cases(c, dm):
        n, tot, bf = C.c_uint64(), C.c_uint64(), C.c_uint64()
        chip0 = vb.lib().vgpu_basic_machine_chip(0)

        def raw(cap, out, n_out, total, bus_free, chip=chip0):
            c.check(vb.lib().vgpu_cell_alternatives(c._h, chip, dm[0]._h, None, cap, out, n_out, total, bus_free, None))

        bad_chip = vb.api._ChipDesc()
        bad_chip.chip_id = 99
        return [("null output", lambda: raw(1, None, C.byref(n), C.byref(tot), C.byref(bf))),
                ("null output", lambda: raw(0, None, None, C.byref(tot), C.byref(bf))),
                ("null output", lambda: raw(0, None, C.byref(n), None, C.byref(bf))),
                ("null output", lambda: raw(0, None, C.byref(n), C.byref(tot), None)),
                ("unknown chip", lambda: raw(0, None, C.byref(n), C.byref(tot), C.byref(bf), C.pointer(bad_chip))),
                ("main width", lambda: vb.cell_alternatives(c, 3, dm[0], None)),
                ("needs its preprocessed trace", lambda: vb.cell_alternatives(c, 1, dm[1], None))]

    def run(c, dm):
        out = []
        for what, call in cases(c, dm):
            before = c.launch_count
            c.comm_stats(reset=True)
            with pytest.raises(vb.VgpuError) as e:
                call()
            out.append((what, what in str(e.value), c.launch_count == before, sum(k for k, _ in c.comm_stats().values())))
        return out

    lone = run(ctx, [ctx.upload(m) for m in fib15])
    assert all(named and no_launch and k == 0 for _, named, no_launch, k in lone), lone
    ctxs = _ranks(2)
    try:
        outs = vb.run_ranks(lambda r, c: run(c, [c.upload_rows(m) for m in fib15]), ctxs)
        assert outs[0] == outs[1] == lone, outs

        def wrong(r, c):
            dm = c.upload_rows(fib15[0])
            c.set_sharding(False)
            before = c.launch_count
            with pytest.raises(vb.VgpuError) as e:
                vb.cell_alternatives(c, 0, dm, None)
            return "not this context's run" in str(e.value) and c.launch_count == before

        assert vb.run_ranks(wrong, ctxs) == [True, True]
    finally:
        _close(ctxs)


@pytest.fixture(scope="module")
def fib22(built):
    import valida_b200 as vb

    return vb.run_program_log(vb.fib_program(((1 << 22) - 17) // 7))


def test_full_size(ctx, fib22):
    import valida_b200 as vb

    def sweep(c, dm, dp):
        return [_key(vb.cell_alternatives(c, chip, dm[chip], dp[PREP_CHIPS[chip]] if chip in PREP_CHIPS else None, cap=1 << 12))
                for chip in range(14)]

    dm, dp = fib22.witness_device(ctx)
    one = sweep(ctx, dm, dp)
    assert one[0][1] > 0
    del dm, dp
    t = fib22.traces()
    up = [ctx.upload(m) for m in t.main]
    upp = [ctx.upload(m) for m in t.preprocessed]
    assert sweep(ctx, up, upp) == one
    del up, upp
    for nranks in (2, 4):
        ctxs = _ranks(nranks)
        try:
            assert vb.run_ranks(lambda r, c: sweep(c, *fib22.witness_device(c)), ctxs) == [one] * nranks
        finally:
            _close(ctxs)
