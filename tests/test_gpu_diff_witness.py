"""diff_witness on the GPU (vgpu_diff_witness, valida_b200/csrc/diff.cu): every cell of a witness that differs from what
Chip::generate_trace writes for a run, on one GPU and over the row shards of a split context.

The expected answer is a numpy comparison of the downloaded (or host-built) traces, sorted (chip, trace, row, column).  Clean
witnesses come from two generators: the device builder of the same log and the host builder (VmLog.traces()), uploaded."""
import ctypes as C

import numpy as np
import pytest

from generated_programs import REGIMES, generated_program
from test_gpu_check_constraints import CLEAN
from test_gpu_check_failures import _close, _ranks
from test_gpu_local_shards import BORROW_LAYOUTS, _col_major, _local_tensors, _monty
from test_perm_trace_restatement import P

pytestmark = pytest.mark.gpu
CH = np.random.default_rng(5151).integers(0, P, 15, dtype=np.uint32)


def _widths():
    import valida_b200 as vb

    d = [C.cast(vb.lib().vgpu_basic_machine_chip(c), C.POINTER(C.c_uint32)) for c in range(14)]   # chip_id, width, preprocessed_width
    return [int(x[1]) for x in d], [int(d[1][2]), int(d[12][2])]


def _column_base(chip, trace):
    main, prep = _widths()
    if trace == 0:
        return sum(main[:chip])
    return sum(main) + (prep[0] if chip == 12 else 0)


def _traces_of(chip):
    """(trace, index into the 16 matrices) of a chip: its main trace, and the program / range preprocessed trace of chips 1 / 12."""
    return [(0, chip)] + ([(1, 14 + (chip == 12))] if chip in (1, 12) else [])


def _expected(have, want):
    """numpy: (cells sorted (chip, trace, row, column) with both words, per-column counts, [(cells, first row) per chip]) of the
    16 row-major canonical matrices `have` against `want`; a chip whose heights differ is skipped."""
    import valida_b200 as vb

    cells, per, chips = [], np.zeros(vb.witness_column_count(), dtype=np.uint64), []
    for chip in range(14):
        n, first = 0, -1
        if have[chip].shape[0] == want[chip].shape[0]:
            for trace, k in _traces_of(chip):
                a, b = np.asarray(have[k]), np.asarray(want[k])
                rows, cols = np.nonzero(a != b)                   # row-major order: (row, column) ascending
                cells += [(chip, trace, int(r), int(c), int(a[r, c]), int(b[r, c])) for r, c in zip(rows, cols)]
                np.add.at(per, _column_base(chip, trace) + cols, 1)
                n += len(rows)
                if len(rows):
                    first = int(rows[0]) if first < 0 else min(first, int(rows[0]))
        chips.append((n, first))
    return cells, per, chips


def _as_list(res):
    return [(e.chip, e.trace, e.row, e.column, e.have, e.want) for e in res.cells]


def _whole(res):
    return _as_list(res), res.total, res.complete, [tuple(x) for x in res.chips], [int(x) for x in res.per_column]


def _check(res, have, want, heights=None):
    cells, per, chips = _expected(have, want)
    assert _as_list(res) == cells and res.total == len(cells) and res.complete
    assert [(x.cells, x.first_row) for x in res.chips] == chips
    assert np.array_equal(res.per_column, per)
    assert [(x.height_have, x.height_want) for x in res.chips] == (heights or [(m.shape[0], w.shape[0]) for m, w in zip(have[:14], want[:14])])


def _upload(ctx, mats):
    return [ctx.upload(np.asarray(m)) for m in mats[:14]], [ctx.upload(np.asarray(m)) for m in mats[14:]]


def _host(log):
    t = log.traces()
    return [np.array(m) for m in t.main + t.preprocessed]


def _assert_clean(ctx, log):
    import valida_b200 as vb

    for dm, dp in (log.witness_device(ctx), _upload(ctx, _host(log))):
        res = vb.diff_witness(ctx, log, dm, dp)
        assert res.cells == [] and res.total == 0 and res.complete and not res.per_column.any()
        assert all(x.cells == 0 and x.first_row == -1 and x.height_have == x.height_want for x in res.chips)


@pytest.mark.parametrize("name", sorted(CLEAN))
def test_clean_witnesses(ctx, name):
    """The device witness and the host traces of the same run report nothing, for Fibonacci, the reference's test programs and the
    static-data program."""
    import valida_b200 as vb

    prog, cells = CLEAN[name]()
    _assert_clean(ctx, vb.run_program_log(prog, initial_fp=0x1000, static_data=cells))


@pytest.mark.parametrize("regime", REGIMES)
def test_clean_generated_programs(ctx, regime):
    import valida_b200 as vb

    for seed in (31, 32):
        prog, fp = generated_program(seed, regime, 3000)
        _assert_clean(ctx, vb.run_program_log(prog, initial_fp=fp))


@pytest.fixture(scope="module")
def fib_small(built):
    import valida_b200 as vb

    log = vb.run_program_log(vb.fib_program(100))
    return log, _host(log)


def _tamper(mats, spots):
    out = [np.array(m) for m in mats]
    for i, (k, r, c) in enumerate(spots):
        out[k][r, c] = (int(out[k][r, c]) + 1 + i) % P
    return out


def test_tampered_cells_are_reported_exactly(ctx, fib_small):
    """k cells across the main and preprocessed traces (row 0, row h - 1, CPU column 27, a memory value byte, a range mult, the
    program and range preprocessed traces): exactly those cells, the tampered word as have and the original as want."""
    import valida_b200 as vb

    log, host = fib_small
    h0, h2 = host[0].shape[0], host[2].shape[0]
    spots = [(0, 0, 3), (0, h0 - 1, 10), (0, 40, 27), (0, 40, 28), (2, h2 // 3, 1), (2, h2 - 1, 0), (3, 7, 5), (12, 77, 0), (14, 3, 0),
             (14, 0, 6), (15, 5, 0)]
    bad = _tamper(host, spots)
    res = log.diff_witness(ctx, *_upload(ctx, bad))
    want = sorted((c, t, r, col, int(bad[k][r, col]), int(host[k][r, col]))
                  for k, r, col in spots for c, t in [(k if k < 14 else (1, 12)[k - 14], int(k >= 14))])
    assert _as_list(res) == want
    assert all(e.have != e.want for e in res.cells)
    _check(res, bad, host)
    assert [e.column_name for e in res.cells if e.chip == 12 and e.trace == 0] == [vb.column_name(12, 0, 0)]
    assert res.chips[0].first_row == 0 and res.chips[2].first_row == h2 // 3 and res.chips[1].cells == 2 and res.chips[12].cells == 2


def test_two_runs_agree_with_numpy_under_every_cap(ctx, fib_small):
    """A witness of another run with the same chip heights (Fibonacci at another frame pointer): the list is the numpy diff of the
    two host witnesses, and every cap gives the right prefix and count."""
    import valida_b200 as vb

    log, host = fib_small
    other = _host(vb.run_program_log(vb.fib_program(100), initial_fp=0x2000))
    assert [m.shape for m in other] == [m.shape for m in host]
    dm, dp = _upload(ctx, other)
    full = vb.diff_witness(ctx, log, dm, dp, cap=1 << 20)
    _check(full, other, host)
    total = full.total
    assert total > 100
    for cap in (0, 1, total - 1, total, total + 7):
        res = vb.diff_witness(ctx, log, dm, dp, cap=cap)
        assert len(res.cells) == min(cap, total) and res.total == total and res.complete == (cap >= total), cap
        assert _as_list(res) == _as_list(full)[:cap], cap
        assert [tuple(x) for x in res.chips] == [tuple(x) for x in full.chips] and np.array_equal(res.per_column, full.per_column)


def test_first_divergent_cycle(ctx):
    """Two programs that differ in one immediate: the first CPU entry is on the first cycle whose row differs, the first cycle that
    runs the changed instruction."""
    import valida_b200 as vb

    a, b = vb.fib_program(100), vb.fib_program(101)
    k = int(np.nonzero((a != b).any(axis=1))[0][0])
    assert (a != b).sum() == 1
    la, lb = vb.run_program_log(a), vb.run_program_log(b)
    ha, hb = _host(la), _host(lb)
    assert [m.shape for m in ha] == [m.shape for m in hb]
    res = vb.diff_witness(ctx, la, *_upload(ctx, hb))
    _check(res, hb, ha)
    first_cpu = next(e for e in res.cells if e.chip == 0)
    row = int(np.nonzero((ha[0] != hb[0]).any(axis=1))[0][0])
    pc = next(c for c in range(ha[0].shape[1]) if vb.column_name(0, 0, c) == "pc")
    assert first_cpu.row == row == res.chips[0].first_row and int(ha[0][row, pc]) == k
    assert (1, 1, k) in {(e.chip, e.trace, e.row) for e in res.cells}     # the program trace holds the immediate too


def test_height_mismatch_is_reported_and_skipped(ctx, fib_small):
    """The add chip padded to twice its height and the memory chip cut to half: both reported in their summaries and skipped; the
    other chips are still compared."""
    import valida_b200 as vb

    log, host = fib_small
    bad = _tamper(host, [(0, 5, 2)])
    bad[3] = np.vstack([bad[3], np.zeros_like(bad[3])])
    bad[2] = bad[2][: bad[2].shape[0] // 2]
    res = vb.diff_witness(ctx, log, *_upload(ctx, bad))
    _check(res, bad, host)
    assert _as_list(res) == [(0, 0, 5, 2, int(bad[0][5, 2]), int(host[0][5, 2]))]
    assert (res.chips[3].height_have, res.chips[3].height_want) == (2 * host[3].shape[0], host[3].shape[0])
    assert (res.chips[2].height_have, res.chips[2].height_want) == (host[2].shape[0] // 2, host[2].shape[0])
    assert res.chips[2].cells == res.chips[3].cells == 0 and res.chips[2].first_row == res.chips[3].first_row == -1


def test_refusals_launch_nothing(ctx, fib_small):
    """Each refusal names its problem, before any launch or collective, on a lone context and alike on every rank."""
    import valida_b200 as vb

    log, host = fib_small

    def run(c, upload):
        dm, dp = [upload(m) for m in host[:14]], [upload(m) for m in host[14:]]
        # quotient chunks of the add chip: rows stored bit-reversed
        pcs = vb.TwoAdicFriPcs(c)
        dq, cs = vb.generate_permutation_trace(c, 3, dm[3], None, CH)
        _, pdm = pcs.commit_batches([dm[3]])
        _, pdq = pcs.commit_batches([dq])
        chunks = vb.quotient(c, 3, dm[3].shape[0].bit_length() - 1, None, pcs.get_ldes(pdm)[0], pcs.get_ldes(pdq)[0], cs, CH, CH[:5])
        n, tot = C.c_uint64(), C.c_uint64()
        summ = np.zeros(14, dtype=vb.DIFF_SUMMARY_DTYPE)
        buf = np.zeros(4, dtype=vb.CELL_DIFF_DTYPE)

        def raw(main, prep, cap, out, n_out=C.byref(n), total=C.byref(tot), summary=summ.ctypes.data_as(C.c_void_p)):
            a = (C.c_void_p * 14)(*[m._h if m is not None else None for m in main])
            b = (C.c_void_p * 2)(*[m._h if m is not None else None for m in prep])
            c.check(vb.lib().vgpu_diff_witness(c._h, log._h, a, b, cap, out, n_out, total, summary, None))

        cases = [("null output", lambda: raw(dm, dp, 1, None)),
                 ("null output", lambda: raw(dm, dp, 0, None, n_out=None)),
                 ("null output", lambda: raw(dm, dp, 0, None, total=None)),
                 ("null output", lambda: raw(dm, dp, 0, None, summary=None)),
                 ("chip 5 has no trace", lambda: raw(dm[:5] + [None] + dm[6:], dp, 4, buf.ctypes.data_as(C.c_void_p))),
                 ("main width", lambda: vb.diff_witness(c, log, dm[:3] + [dm[5]] + dm[4:], dp)),
                 ("needs its preprocessed trace", lambda: raw(dm, [None, dp[1]], 0, None)),
                 ("preprocessed width", lambda: vb.diff_witness(c, log, dm, dp[::-1])),
                 ("bit-reversed", lambda: vb.diff_witness(c, log, dm[:3] + [chunks] + dm[4:], dp))]
        out = []
        for what, call in cases:
            before = c.launch_count
            c.comm_stats(reset=True)
            with pytest.raises(vb.VgpuError) as e:
                call()
            out.append((what, what in str(e.value), c.launch_count == before, sum(k for k, _ in c.comm_stats().values())))
        return out

    lone = run(ctx, ctx.upload)
    assert all(named and no_launch and k == 0 for _, named, no_launch, k in lone), lone
    ctxs = _ranks(2)
    try:
        outs = vb.run_ranks(lambda r, c: run(c, c.upload_rows), ctxs)
        assert outs[0] == outs[1] == lone, outs
    finally:
        _close(ctxs)


@pytest.fixture(scope="module")
def fib15(built):
    import valida_b200 as vb

    log = vb.run_program_log(vb.fib_program(((1 << 15) - 17) // 7))
    host = _host(log)
    assert host[0].shape[0] == 1 << 15 and host[2].shape[0] == 1 << 17
    return log, host


def test_a_shard_of_another_run_is_refused(fib15):
    """A row shard uploaded on a split context, passed once the context no longer splits: refused before anything is enqueued."""
    import valida_b200 as vb

    log, host = fib15
    ctxs = _ranks(2)
    try:
        dm = vb.run_ranks(lambda r, c: [c.upload_rows(m) for m in host], ctxs)
        for c in ctxs:
            c.set_sharding(False)
        c = ctxs[0]
        before = c.launch_count
        with pytest.raises(vb.VgpuError) as e:
            vb.diff_witness(c, log, dm[0][:14], dm[0][14:])
        assert "not this context's run" in str(e.value) and c.launch_count == before
    finally:
        _close(ctxs)


def _tampered_at_boundaries(mats, ctxs):
    """The CPU and memory chips at global row 0, the last row and both sides of every rank boundary (two columns each), the range
    chip's mult and a program-trace cell (chips every rank holds whole)."""
    spots = []
    for k, cols in ((0, (0, 27)), (2, (1, 13))):
        h = mats[k].shape[0]
        rows = {0, h - 1} | {x for c in ctxs[1:] for x in (c.local_rows(h)[0] - 1, c.local_rows(h)[0])}
        spots += [(k, r, col) for r in sorted(rows) for col in cols]
    return _tamper(mats, spots + [(12, 77, 0), (14, 2, 1)])


def _on_ranks(ctxs, log, make, cap=1 << 20):
    import valida_b200 as vb

    def rank(r, c):
        dm, dp = make(c, r)
        c.comm_stats(reset=True)
        res = vb.diff_witness(c, log, dm, dp, cap=cap)
        return _whole(res), c.comm_stats()["allgather"][0]

    return vb.run_ranks(rank, ctxs)


@pytest.mark.parametrize("nranks", [2, 3, 4, 5, 6, 8])
def test_split_every_route(ctx, fib15, nranks):
    """Fibonacci 2^15 changed on both sides of every rank boundary and in the whole short chips: every rank's output equals the
    single-GPU call's through upload_rows, import_tensor_local and borrow_tensor_local; the clean device witness reports nothing.
    The all-gathers are the counts and the listed cells (only the counts when nothing differs)."""
    import torch
    import valida_b200 as vb

    log, host = fib15
    ctxs = _ranks(nranks)
    try:
        h12 = host[12].shape[0]
        assert ctxs[0].local_rows(1 << 15)[1] < 1 << 15 and tuple(ctxs[0].local_rows(h12)) == (0, h12)
        mats = _tampered_at_boundaries(host, ctxs)
        single = vb.diff_witness(ctx, log, *_upload(ctx, mats))
        _check(single, mats, host)
        want = _whole(single)
        layout = "stride_rows_plus_3" if nranks % 2 else "base_plus_one_word"
        pad, off = BORROW_LAYOUTS[layout]

        def borrow(c, r):
            tens = _local_tensors(c, [_monty(a) for a in mats], lambda a, d: _col_major(a, d, pad, off))
            torch.cuda.synchronize()
            v = [c.borrow_tensor_local(x, a.shape[0]) for x, a in zip(tens, mats)]
            return v[:14], v[14:]

        def imported(c, r):
            v = [c.import_tensor_local(x, a.shape[0]) for x, a in zip(_local_tensors(c, mats, lambda a, d: _col_major(a, d)), mats)]
            return v[:14], v[14:]

        def rows(c, m):
            v = [c.upload_rows(x) for x in m]
            return v[:14], v[14:]

        routes = {"upload_rows": lambda c, r: rows(c, mats), "import_tensor_local": imported, "borrow_" + layout: borrow}
        for name, make in routes.items():
            for got in _on_ranks(ctxs, log, make):
                assert got == (want, 2), name
        empty = _whole(vb.diff_witness(ctx, log, *_upload(ctx, host)))
        assert empty[1] == 0
        assert _on_ranks(ctxs, log, lambda c, r: rows(c, host)) == [(empty, 1)] * nranks
        assert _on_ranks(ctxs, log, lambda c, r: log.witness_device(c)) == [(empty, 1)] * nranks
        # a cap below the total: the same prefix on every rank, equal to the single-GPU call's
        cap = single.total // 2
        part = _whole(vb.diff_witness(ctx, log, *_upload(ctx, mats), cap=cap))
        assert not part[2] and len(part[0]) == cap
        for got in _on_ranks(ctxs, log, lambda c, r: rows(c, mats), cap=cap):
            assert got == (part, 2)
    finally:
        _close(ctxs)


@pytest.fixture(scope="module")
def fib22(built):
    import valida_b200 as vb

    return vb.run_program_log(vb.fib_program(((1 << 22) - 17) // 7))


def test_full_size(ctx, fib22):
    """2^22 Fibonacci: the host traces, uploaded, against the log report nothing (generator parity at full size, with no download);
    one memory-chip value byte changed in the device witness gives exactly that cell; the call's extra device memory stays below
    one whole witness."""
    import torch
    import valida_b200 as vb

    host = _host(fib22)
    dm, dp = _upload(ctx, host)
    witness_bytes = sum(m.size * 4 for m in host)
    del host
    before = ctx.memory_stats(reset=True)
    res = vb.diff_witness(ctx, fib22, dm, dp)
    extra = ctx.memory_stats()["peak"] - before["live"]
    assert res.cells == [] and res.total == 0 and all(x.height_have == x.height_want for x in res.chips)
    assert 0 < extra < witness_bytes, (extra, witness_bytes)
    del dm, dp
    dm, dp = fib22.witness_device(ctx)
    h = dm[2].shape[0]
    assert h == 1 << 24
    mem = dm[2].to_tensor()
    r = h // 2 + 12345
    old = int(mem[r, 1])
    mem[r, 1] = (mem[r, 1].to(torch.int64) + 1) % P
    torch.cuda.synchronize()
    bad = ctx.import_tensor(mem)
    res = vb.diff_witness(ctx, fib22, dm[:2] + [bad] + dm[3:], dp)
    assert _as_list(res) == [(2, 0, r, 1, (old + 1) % P, old)] and res.total == 1
    assert res.cells[0].column_name == vb.column_name(2, 0, 1) and res.chips[2].first_row == r
    assert [x.cells for x in res.chips] == [0, 0, 1] + [0] * 11
