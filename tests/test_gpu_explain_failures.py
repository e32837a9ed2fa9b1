"""explain_failures on the GPU (vgpu_explain_failures, valida_b200/csrc/explain.cu): the values of the cells each failed constraint
reads, on the failing row and the next one, on one GPU and over the row shards of a split context.

Every value is held to the trace word at its (row or (row + 1) mod h, column), downloaded; a split context must give every rank the
single-GPU output with one all-gather; bus events of check_buses are explained from its inputs alone (no permutation trace) and
their cells must give back the event's tuple and multiplicity."""
import ctypes as C

import numpy as np
import pytest

from test_check_constraints_restatement import PREP_CHIPS
from test_gpu_check_failures import _close, _ranks
from test_gpu_local_shards import BORROW_LAYOUTS, _col_major, _local_tensors, _monty
from test_perm_trace_restatement import P

pytestmark = pytest.mark.gpu
CH = np.random.default_rng(6161).integers(0, P, 15, dtype=np.uint32)


def _desc(chip):
    import valida_b200 as vb
    from valida_b200.api import _ChipDesc

    return C.cast(vb.lib().vgpu_basic_machine_chip(chip), C.POINTER(_ChipDesc)).contents


def _pair_col(pc, cells):
    """VirtualPairCol::apply over explained cells {(trace, next, column): value} on the local row."""
    import valida_b200 as vb

    v = pc.constant
    for t in range(pc.n_terms):
        is_prep, col, w = pc.terms[3 * t], pc.terms[3 * t + 1], pc.terms[3 * t + 2]
        v += w * cells[(vb.TRACE_PREPROCESSED if is_prep else vb.TRACE_MAIN, False, col)]
    return v % P


def _check_values(ex, h, mats):
    """Every explained value equals the word of its trace at (row or (row + 1) mod h, column); mats[trace] None: absent."""
    import valida_b200 as vb

    for e in ex:
        for c in e.cells:
            m = mats[c.trace]
            row = (e.row + 1) % h if c.next else e.row
            assert c.value == (None if m is None else int(m[row, c.column])), (e.row, e.constraint, c)


@pytest.mark.parametrize("chip", range(14))
def test_random_traces_every_chip(ctx, chip):
    """check_failures' list (small cap) of random traces with a random permutation trace, and every constraint at row h - 1 (whose
    next row is row 0): values equal the downloaded words, counts equal constraint_cells, and without the permutation trace only
    its cells change, to None."""
    import valida_b200 as vb

    d = _desc(chip)
    h = 16
    rng = np.random.default_rng(8200 + chip)
    main = rng.integers(0, P, (h, d.width), dtype=np.uint32)
    prep = rng.integers(0, P, (h, d.preprocessed_width), dtype=np.uint32) if d.preprocessed_width else None
    perm = rng.integers(0, P, (h, 5 * (d.n_interactions + 1)), dtype=np.uint32)
    dm, dq = ctx.upload(main), ctx.upload(perm)
    dp = ctx.upload(prep) if prep is not None else None
    _, total = vb.constraint_count(chip)
    fails, n_fail, _ = vb.check_failures(ctx, chip, dm, dp, dq, CH, cap=40)
    assert n_fail > 0 and len(fails) == min(40, n_fail)
    for items in (fails, [(h - 1, c) for c in range(total)] + [(0, total - 1), (5, 0)]):
        ex = vb.explain_failures(ctx, chip, dm, dp, dq, items)
        pairs = [(int(r), int(c)) for r, c in (zip(items["row"], items["constraint"]) if isinstance(items, np.ndarray) else items)]
        assert [(e.row, e.constraint) for e in ex] == pairs
        for e in ex:
            label, cells = vb.constraint_cells(chip, e.constraint)
            assert e.label == label and [(c.trace, c.next, c.column, c.name) for c in e.cells] == [tuple(x) for x in cells]
        _check_values(ex, h, {vb.TRACE_MAIN: dm.download(), vb.TRACE_PREPROCESSED: prep, vb.TRACE_PERMUTATION: perm})
        bare = vb.explain_failures(ctx, chip, dm, dp, None, items)
        for e, b in zip(ex, bare):
            assert (b.row, b.constraint, b.label) == (e.row, e.constraint, e.label)
            assert [c._replace(value=None) if c.trace == vb.TRACE_PERMUTATION else c for c in e.cells] == b.cells
    ctx.comm_stats(reset=True)
    vb.explain_failures(ctx, chip, dm, dp, dq, fails)
    assert ctx.comm_stats()["allgather"][0] == 0


@pytest.fixture(scope="module")
def fib15_log(built):
    import valida_b200 as vb

    log = vb.run_program_log(vb.fib_program(((1 << 15) - 17) // 7))
    t = log.traces()
    assert t.main[0].shape[0] == 1 << 15 and t.main[2].shape[0] == 1 << 17
    return log, [np.array(m) for m in t.main + t.preprocessed]


SPLIT_CHIPS = (0, 2, 3, 12)      # cpu and memory (split on every rank count here), add, range (whole on every rank: rank 0 reports)


def _items(ctxs, h, total):
    """Every constraint at each rank's first and last row and at rows 0 and h - 1 (whose next row is row 0, on rank 0)."""
    rows = {0, h - 1}
    for c in ctxs:
        row0, n = c.local_rows(h)
        rows |= {row0, row0 + n - 1}
    return [(r, k) for r in sorted(rows) for k in range(total)]


def _explain_all(c, mats, items, with_perm=True):
    """Per chip: the explanation of its items, and the all-gathers of each call."""
    import valida_b200 as vb

    out = {}
    for chip in SPLIT_CHIPS:
        dp = mats[14 + PREP_CHIPS[chip]] if chip in PREP_CHIPS else None
        dq = vb.generate_permutation_trace(c, chip, mats[chip], dp, CH)[0] if with_perm else None
        c.comm_stats(reset=True)
        ex = vb.explain_failures(c, chip, mats[chip], dp, dq, items[chip])
        out[chip] = (ex, c.comm_stats()["allgather"][0])
    return out


@pytest.mark.parametrize("nranks", [2, 3, 4, 8])
def test_split_every_route(ctx, fib15_log, nranks):
    """Items at every rank's first and last row and at h - 1: every rank's output equals the single-GPU output, through upload_rows,
    import_tensor_local, borrow_tensor_local (column stride > rows) and the device witness, with one all-gather per call."""
    import torch
    import valida_b200 as vb

    log, mats = fib15_log
    ctxs = _ranks(nranks)
    try:
        assert ctxs[0].local_rows(1 << 15)[1] < 1 << 15 and tuple(ctxs[0].local_rows(mats[12].shape[0])) == (0, mats[12].shape[0])
        items = {chip: _items(ctxs, mats[chip].shape[0], vb.constraint_count(chip)[1]) for chip in SPLIT_CHIPS}
        single = _explain_all(ctx, [ctx.upload(m) for m in mats], items)
        for chip, (ex, gathers) in single.items():
            assert gathers == 0
            dp = mats[14 + PREP_CHIPS[chip]] if chip in PREP_CHIPS else None
            dq = vb.generate_permutation_trace(ctx, chip, ctx.upload(mats[chip]), ctx.upload(dp) if dp is not None else None, CH)[0]
            _check_values(ex, mats[chip].shape[0], {vb.TRACE_MAIN: mats[chip], vb.TRACE_PREPROCESSED: dp, vb.TRACE_PERMUTATION: dq.download()})
        want = {chip: (ex, 1) for chip, (ex, _) in single.items()}
        pad, off = BORROW_LAYOUTS["stride_rows_plus_3"]

        def borrow(c, r):
            tens = _local_tensors(c, [_monty(a) for a in mats], lambda a, d: _col_major(a, d, pad, off))
            torch.cuda.synchronize()
            return [c.borrow_tensor_local(x, a.shape[0]) for x, a in zip(tens, mats)]

        def imported(c, r):
            return [c.import_tensor_local(x, a.shape[0]) for x, a in zip(_local_tensors(c, mats, lambda a, d: _col_major(a, d)), mats)]

        def device(c, r):
            dm, dp = log.witness_device(c)
            return list(dm) + list(dp)

        routes = {"upload_rows": lambda c, r: [c.upload_rows(m) for m in mats], "import_tensor_local": imported, "borrow": borrow,
                  "device_witness": device}
        for name, make in routes.items():
            outs = vb.run_ranks(lambda r, c: _explain_all(c, make(c, r), items), ctxs)
            for got in outs:
                assert got == want, name
        # without the permutation trace: the same, permutation cells absent
        bare = vb.run_ranks(lambda r, c: _explain_all(c, [c.upload_rows(m) for m in mats], items, with_perm=False), ctxs)
        for chip in SPLIT_CHIPS:
            ex = [e._replace(cells=[x._replace(value=None) if x.trace == vb.TRACE_PERMUTATION else x for x in e.cells]) for e in want[chip][0]]
            assert all(got[chip] == (ex, 1) for got in bare), chip
    finally:
        _close(ctxs)


def test_refusals_launch_nothing(ctx, fib15_log):
    """Each refusal names its problem, before any launch or collective, on a lone context and alike on every rank."""
    import valida_b200 as vb

    _, mats = fib15_log

    def run(c, upload):
        dm = [upload(m) for m in mats]
        cpu = vb.lib().vgpu_basic_machine_chip(0)
        h0 = mats[0].shape[0]
        dq = vb.generate_permutation_trace(c, 0, dm[0], None, CH)[0]
        dq3 = vb.generate_permutation_trace(c, 3, dm[3], None, CH)[0]
        items = np.zeros(2, dtype=vb.CHECK_FAILURE_DTYPE)
        items["row"], items["constraint"] = (3, h0 - 1), (0, 57)
        need = sum(len(vb.constraint_cells(0, k)[1]) for k in (0, 57))
        first = (C.c_uint64 * 3)()
        vals = (C.c_uint32 * need)()
        nv = C.c_uint64()

        def raw(n, f, v, cap, perm=dq):
            c.check(vb.lib().vgpu_explain_failures(c._h, cpu, dm[0]._h, None, perm._h if perm is not None else None,
                                                   items.ctypes.data_as(C.c_void_p), n, f, v, cap, C.byref(nv)))

        cases = [("null output", lambda: raw(2, None, vals, need)),
                 ("null output", lambda: raw(2, first, None, need)),
                 ("more than cap", lambda: raw(2, first, vals, need - 1)),
                 ("item 1: row %d" % h0, lambda: vb.explain_failures(c, 0, dm[0], None, dq, [(0, 0), (h0, 0)])),
                 ("item 0: row -1", lambda: vb.explain_failures(c, 0, dm[0], None, dq, [(-1, 0)])),
                 ("item 2: constraint 60", lambda: vb.explain_failures(c, 0, dm[0], None, dq, [(0, 0), (1, 59), (2, 60)])),
                 ("main width", lambda: vb.explain_failures(c, 0, dm[3], None, None, [(0, 0)])),
                 ("permutation trace width", lambda: vb.explain_failures(c, 0, dm[0], None, dq3, [(0, 0)])),
                 ("needs its preprocessed trace", lambda: vb.explain_failures(c, 1, dm[1], None, None, [(0, 0)]))]
        out = []
        for what, call in cases:
            before = c.launch_count
            c.comm_stats(reset=True)
            with pytest.raises(vb.VgpuError) as e:
                call()
            out.append((what, what in str(e.value), c.launch_count == before, sum(k for k, _ in c.comm_stats().values())))
        raw(2, first, vals, need)                               # the same arguments, with room: accepted
        out.append(("ok", list(first) == [0, len(vb.constraint_cells(0, 0)[1]), need], nv.value == need, 0))
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
def fib22(built):
    import valida_b200 as vb

    return vb.run_program_log(vb.fib_program(((1 << 22) - 17) // 7))


def test_full_size_bus_events(ctx, fib22):
    """The 2^22 Fibonacci device witness with one memory value byte changed: every event of the tuples check_buses reports, explained
    without a permutation trace, gives back the tuple through the interaction's VirtualPairCols and the multiplicity through its count."""
    import torch
    import valida_b200 as vb

    dm, dp = fib22.witness_device(ctx)
    h = dm[2].shape[0]
    assert h == 1 << 24
    mem = dm[2].to_tensor()
    near = mem[h // 2:h // 2 + 4096].cpu().numpy().astype(np.int64)
    r = h // 2 + next(k for k in range(len(near)) if near[k, 7] + near[k, 8] == 1 and not near[k, 6])
    mem[r, 1] = (mem[r, 1].to(torch.int64) + 1) % P
    torch.cuda.synchronize()
    main = dm[:2] + [ctx.import_tensor(mem)] + dm[3:]
    res = vb.check_buses(ctx, main, dp, CH)
    assert res.complete and len(res.tuples) == 2
    n_events = 0
    for t in res.tuples:
        by_chip = {}
        for e in t.events:
            by_chip.setdefault(e.chip, []).append(e)
        for chip, evs in by_chip.items():
            air, _ = vb.constraint_count(chip)
            d = _desc(chip)
            k = d.n_interactions
            prep = dp[PREP_CHIPS[chip]] if chip in PREP_CHIPS else None
            # the interaction's constraint reads its fields; the LogUp first-row constraint every count on the row
            items = [x for e in evs for x in ((e.row, air + e.interaction), (e.row, air + k + 1))]
            ex = vb.explain_failures(ctx, chip, main[chip], prep, None, items)
            for e, fld, cnt in zip(evs, ex[0::2], ex[1::2]):
                assert fld.label == vb.constraint_label(chip, air + e.interaction) and cnt.label == "LogUp first row"
                cells = {(c.trace, c.next, c.column): c.value for x in (fld, cnt) for c in x.cells if c.trace != vb.TRACE_PERMUTATION}
                assert all(c.value is None for x in (fld, cnt) for c in x.cells if c.trace == vb.TRACE_PERMUTATION)
                it = d.interactions[e.interaction]
                fields = [_pair_col(it.fields[f], cells) for f in range(it.n_fields)]
                assert fields + [0] * (14 - len(fields)) == t.fields + [0] * (14 - len(t.fields)), (chip, e)
                assert _pair_col(it.count, cells) == e.multiplicity and bool(it.is_send) == e.send
                n_events += 1
    assert n_events == sum(len(t.events) for t in res.tuples) >= 3
