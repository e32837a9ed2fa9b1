"""free_cells on the GPU (vgpu_free_cells, valida_b200/csrc/free.cu): every main-trace cell that no constraint and no bus event
depends on, on one GPU and over the row shards of a split context.

The list, the total and the per-column counts are held to free_py, the literal restatement of the definition in
test_free_cells_restatement.py.  Free cells are shown to mean what the definition promises: changed alone to a random value they leave
check_witness clean and check_buses empty, and a proof of such a witness verifies; pinned cells changed at random are caught.  The
reference's known gaps (memory, range and program chips) are checked against numpy on the traces."""
import ctypes as C

import numpy as np
import pytest

import programs
from test_check_constraints_restatement import PREP_CHIPS
from test_free_cells_restatement import MEMORY_ALWAYS, MEMORY_COLUMNS, MEMORY_WHEN_UNUSED, free_py, per_column, width
from test_gpu_check_failures import _close, _ranks
from test_gpu_local_shards import BORROW_LAYOUTS, _col_major, _local_tensors, _monty
from test_perm_trace_restatement import P

pytestmark = pytest.mark.gpu
CH = np.random.default_rng(5151).integers(0, P, 15, dtype=np.uint32)
BIG = 1 << 40

PROGRAMS = {
    "fib25": lambda: (__import__("valida_b200").fib_program(25), None),
    "left_imm": lambda: (programs.mixed_program(40), None),
    "signed_lt": lambda: (programs.lt_edge_operands_program(), None),
    "loads_stores": lambda: (programs.loads_stores_edge_program(), None),
    "config5": lambda: (programs.config5_program(30), None),
    "static_data": programs.static_data_program,
}


def _prep_of(mats, chip):
    return mats[14 + PREP_CHIPS[chip]] if chip in PREP_CHIPS else None


def _device(ctx, chip, main, prep, cap=BIG):
    import valida_b200 as vb

    dm = ctx.upload(main)
    dp = ctx.upload(prep) if prep is not None else None
    total = vb.free_cells(ctx, chip, dm, dp, cap=0).total
    return vb.free_cells(ctx, chip, dm, dp, cap=min(cap, total))


def _as_pairs(res):
    return [(c.row, c.column) for c in res.cells]


def _agree(ctx, chip, main, prep):
    import valida_b200 as vb

    want = free_py(chip, main)
    got = _device(ctx, chip, main, prep)
    assert _as_pairs(got) == want, chip
    assert got.total == len(want) and got.complete
    names = [vb.column_name(chip, vb.TRACE_MAIN, c) for c in range(width(chip))]
    assert [got.per_column[n] for n in names] == per_column(want, width(chip))
    assert all(c.column_name == names[c.column] for c in got.cells)
    return want


@pytest.mark.parametrize("h", [1, 2, 8, 64])
@pytest.mark.parametrize("chip", range(14))
def test_random_traces_match_the_restatement(ctx, chip, h):
    rng = np.random.default_rng(3000 + 16 * chip + h)
    main = rng.integers(0, P, (h, width(chip)), dtype=np.uint32)
    # rows whose counts are 0, so that fields come free there: the memory chip's is_read / is_write, the range chip's mult
    idle = rng.random(h) < 0.5
    for c in {2: (7, 8), 12: (0,)}.get(chip, ()):
        main[idle, c] = 0
    prep = rng.integers(0, P, (h, 7 if chip == 1 else 1), dtype=np.uint32) if chip in PREP_CHIPS else None
    _agree(ctx, chip, main, prep)


@pytest.mark.parametrize("name", sorted(PROGRAMS))
def test_program_witnesses_match_the_restatement(ctx, name):
    import valida_b200 as vb

    prog, cells = PROGRAMS[name]()
    t = vb.run_program(prog, initial_fp=0x1000, static_data=cells)
    mats = list(t.main) + list(t.preprocessed)
    for chip in range(14):
        _agree(ctx, chip, t.main[chip], _prep_of(mats, chip))


def test_cap_gives_prefixes(ctx):
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(25), initial_fp=0x1000)
    dm = ctx.upload(t.main[2])
    full = vb.free_cells(ctx, 2, dm, None, cap=BIG)
    total = full.total
    assert total > 1000 and full.complete
    for cap in (0, 1, 200, total - 1, total, total + 1, 10 * total):
        got = vb.free_cells(ctx, 2, dm, None, cap=cap)
        assert got.total == total and got.per_column == full.per_column
        assert got.cells == full.cells[:min(cap, total)] and got.complete == (cap >= total)


def _witness(name):
    import valida_b200 as vb

    prog, cells = PROGRAMS[name]()
    t = vb.run_program(prog, initial_fp=0x1000, static_data=cells)
    return t, [np.array(m) for m in list(t.main) + list(t.preprocessed)]


def _check(ctx, mats, base=None, chip=None):
    """(check_witness clean and the sums cancel, check_buses' tuples); base: the uploaded witness mats differs from in chip only."""
    import valida_b200 as vb

    dm = list(base[:14]) if base else [ctx.upload(m) for m in mats[:14]]
    dp = list(base[14:]) if base else [ctx.upload(m) for m in mats[14:]]
    if base:
        dm[chip] = ctx.upload(mats[chip])
    rep, cancel = vb.check_witness(ctx, dm, dp, CH)
    clean = cancel and all(r[0] == -1 for r in rep)
    return clean, vb.check_buses(ctx, dm, dp, CH).tuples


def _changed(mats, chip, row, col, value):
    out = list(mats)
    out[chip] = mats[chip].copy()
    out[chip][row, col] = value
    return out


@pytest.mark.parametrize("name", ["fib25", "config5"])
def test_free_cells_mean_what_they_say(ctx, oracle, name):
    """Free cells changed alone leave check_witness clean and check_buses empty; pinned ones are caught; a proof of a witness with
    a free cell changed verifies and differs from the original's."""
    import valida_b200 as vb

    t, mats = _witness(name)
    assert _check(ctx, mats) == (True, [])
    base = [ctx.upload(m) for m in mats]
    rng = np.random.default_rng(77)
    proved = False
    for chip in range(14):
        res = _device(ctx, chip, mats[chip], _prep_of(mats, chip))
        free = _as_pairs(res)
        h, w = mats[chip].shape
        picks = [free[0], free[-1]] + [free[i] for i in rng.choice(len(free), min(20, len(free)), replace=False)] if free else []
        for r, c in picks:
            v = (int(mats[chip][r, c]) + 1 + int(rng.integers(0, P - 1))) % P
            bad = _changed(mats, chip, r, c, v)
            assert _check(ctx, bad, base, chip) == (True, []), (chip, r, c)
            if not proved and chip == 2:
                cfg = vb.StarkConfig(ctx, oracle.rc480)
                dm = [ctx.upload(m) for m in bad[:14]]
                dp = [ctx.upload(m) for m in bad[14:]]
                proof = vb.prove_machine(cfg, t, device_resident=(dm, dp))
                vb.verify_machine(cfg, proof, t.preprocessed)
                assert proof != vb.prove_machine(cfg, t)
                proved = True
        pinned = sorted(set((r, c) for r in range(h) for c in range(w)) - set(free))
        for i in rng.choice(len(pinned), min(20, len(pinned)), replace=False):
            r, c = pinned[i]
            v = (int(mats[chip][r, c]) + 1 + int(rng.integers(0, P - 1))) % P
            clean, tuples = _check(ctx, _changed(mats, chip, r, c, v), base, chip)
            assert not clean, (chip, r, c)
    assert proved


def _gaps(mats):
    """The known gaps, from numpy on the traces: {chip: per-column free rows}."""
    mem, rc = mats[2], mats[12]
    unused = int(((mem[:, 7].astype(np.int64) + mem[:, 8]) % P == 0).sum())
    h = mem.shape[0]
    m = {n: (h if n in MEMORY_ALWAYS else unused if n in MEMORY_WHEN_UNUSED else 0) for n in MEMORY_COLUMNS}
    return {2: m, 12: {"mult": 0, "counter": int((rc[:, 0] == 0).sum())}, 1: {"multiplicity": mats[1].shape[0]}}


def test_known_gaps(ctx):
    _, mats = _witness("config5")
    for chip, want in _gaps(mats).items():
        assert _device(ctx, chip, mats[chip], _prep_of(mats, chip), cap=0).per_column == want, chip


@pytest.fixture(scope="module")
def fib15(built):
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(((1 << 15) - 17) // 7), initial_fp=0x1000)
    assert t.main[0].shape[0] == 1 << 15
    return [np.array(m) for m in list(t.main) + list(t.preprocessed)]


def _boundary_changed(mats, ctxs, chips):
    """Every rank boundary b of each chip's split: rows b - 1 and b (and global rows 0 and h - 1) changed in every column."""
    out = list(mats)
    for chip in chips:
        h = mats[chip].shape[0]
        a = mats[chip].copy()
        rows = {0, h - 1}
        for c in ctxs[1:]:
            b = c.local_rows(h)[0]
            rows |= {b - 1, b}
        for r in rows:
            a[r, r % a.shape[1]] = (int(a[r, r % a.shape[1]]) + 1) % P
        out[chip] = a
    return out


def _key(res):
    return ([(c.row, c.column) for c in res.cells], res.total, res.per_column)


@pytest.mark.parametrize("nranks", [2, 3, 4, 5, 6, 8])
def test_split_every_route(ctx, fib15, nranks):
    import torch
    import valida_b200 as vb

    ctxs = _ranks(nranks)
    try:
        mats = _boundary_changed(fib15, ctxs, (0, 2, 3))
        chips = list(range(14))
        caps = {}
        want = {}
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

        routes = {"upload_rows": lambda c, r: [c.upload_rows(m) for m in mats],
                  "import_tensor_local": lambda c, r: [c.import_tensor_local(x, a.shape[0])
                                                       for x, a in zip(_local_tensors(c, mats, lambda a, d: _col_major(a, d)), mats)],
                  "borrow_" + layout: borrow}
        for name, make in routes.items():
            def rank(r, c):
                dm = make(c, r)
                out = {}
                for chip in chips:
                    c.comm_stats(reset=True)
                    out[chip] = (_key(vb.free_cells(c, chip, dm[chip], _prep_of(dm, chip), cap=caps[chip])), c.comm_stats()["allgather"][0])
                return out

            for got in vb.run_ranks(rank, ctxs):
                for chip in chips:
                    split = ctxs[0].local_rows(mats[chip].shape[0])[1] < mats[chip].shape[0]
                    gathers = (3 if want[chip][1] else 2) if split else 0
                    assert got[chip] == (want[chip], gathers), (name, chip)
        # the device witness on the split context
        log = vb.run_program_log(vb.fib_program(((1 << 15) - 17) // 7))

        def device(r, c):
            dm, dp = log.witness_device(c)
            return [_key(vb.free_cells(c, chip, dm[chip], dp[PREP_CHIPS[chip]] if chip in PREP_CHIPS else None, cap=1 << 12)) for chip in chips]

        single = [_key(_device(ctx, chip, fib15[chip], _prep_of(fib15, chip), cap=1 << 12)) for chip in chips]
        assert vb.run_ranks(device, ctxs) == [single] * nranks
    finally:
        _close(ctxs)


def test_sharding_off_makes_no_collective(ctx, fib15):
    import valida_b200 as vb

    want = _key(_device(ctx, 0, fib15[0], None))
    ctxs = _ranks(2)
    try:
        for c in ctxs:
            c.set_sharding(False)
        c = ctxs[0]
        c.comm_stats(reset=True)
        got = vb.free_cells(c, 0, c.upload_rows(fib15[0]), None, cap=want[1])
        assert _key(got) == want and c.comm_stats()["allgather"][0] == 0
    finally:
        _close(ctxs)


def test_refusals_launch_nothing(ctx, fib15):
    import valida_b200 as vb

    def cases(c, dm):
        n, tot = C.c_uint64(), C.c_uint64()
        chip0 = vb.lib().vgpu_basic_machine_chip(0)

        def raw(cap, out, n_out, total, chip=chip0):
            c.check(vb.lib().vgpu_free_cells(c._h, chip, dm[0]._h, None, cap, out, n_out, total, None))

        bad_chip = vb.api._ChipDesc()
        bad_chip.chip_id = 99
        out = [("null output", lambda: raw(1, None, C.byref(n), C.byref(tot))),
               ("null output", lambda: raw(0, None, None, C.byref(tot))),
               ("null output", lambda: raw(0, None, C.byref(n), None)),
               ("unknown chip", lambda: raw(0, None, C.byref(n), C.byref(tot), C.pointer(bad_chip))),
               ("main width", lambda: vb.free_cells(c, 3, dm[0], None)),
               ("needs its preprocessed trace", lambda: vb.free_cells(c, 1, dm[1], None))]
        return out

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
        # a row shard that is not this context's run: sharding switched off after the upload
        def wrong(r, c):
            dm = c.upload_rows(fib15[0])
            c.set_sharding(False)
            before = c.launch_count
            with pytest.raises(vb.VgpuError) as e:
                vb.free_cells(c, 0, dm, None)
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
        return [_key(vb.free_cells(c, chip, dm[chip], dp[PREP_CHIPS[chip]] if chip in PREP_CHIPS else None, cap=1 << 12)) for chip in range(14)]

    dm, dp = fib22.witness_device(ctx)
    assert dm[0].shape[0] == 1 << 22 and dm[2].shape[0] == 1 << 24
    ctx.memory_stats(reset=True)
    base = ctx.memory_stats()["live"]
    one = sweep(ctx, dm, dp)
    peak = ctx.memory_stats()["peak"] - base
    assert peak <= 16 * (1 << 24) + 16 * (1 << 12) + (1 << 20), peak
    host = [dm[c].download() for c in (1, 2, 12)]
    mats = {1: host[0], 2: host[1], 12: host[2]}
    for chip, want in _gaps(mats).items():
        assert one[chip][2] == want, chip
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
