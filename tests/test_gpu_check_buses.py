"""check_buses on the GPU (vgpu_check_buses, valida_b200/csrc/buses.cu): every bus tuple a witness leaves unbalanced, with every event
that sends or receives it, on one GPU and over the row shards of a split context.

The output is held tuple for tuple and event for event to the plain-Python bus balance of test_bus_balance_restatement.py, and its
emptiness to check_witness' sums_cancel."""
import ctypes as C

import numpy as np
import pytest

from test_bus_balance_restatement import TAMPERS, fib_traces, unbalanced
from test_gpu_check_constraints import CLEAN
from test_gpu_check_failures import _close, _ranks, fib15  # noqa: F401
from test_gpu_local_shards import BORROW_LAYOUTS, _col_major, _local_tensors, _monty
from test_perm_trace_restatement import P

pytestmark = pytest.mark.gpu
CH = np.random.default_rng(5150).integers(0, P, 15, dtype=np.uint32)


def _as_list(res):
    return [(t.bus, tuple(t.fields), t.net, [(e.chip, e.row, e.interaction, e.multiplicity, e.send) for e in t.events]) for t in res.tuples]


def _upload(ctx, mats):
    return [ctx.upload(m) for m in mats[:14]], [ctx.upload(m) for m in mats[14:]]


def _device(ctx, mains, preps, cap=1 << 20):
    """check_buses of host traces on one context, and check_witness' sums_cancel of the same."""
    import valida_b200 as vb

    dm, dp = _upload(ctx, list(mains) + list(preps))
    res = vb.check_buses(ctx, dm, dp, CH, cap=cap)
    return res, vb.check_witness(ctx, dm, dp, CH)[1]


@pytest.mark.parametrize("name", sorted(CLEAN))
def test_clean_witnesses_are_balanced(ctx, name):
    import valida_b200 as vb

    prog, cells = CLEAN[name]()
    t = vb.run_program(prog, initial_fp=0x1000, static_data=cells)
    res, cancel = _device(ctx, t.main, t.preprocessed)
    assert res.tuples == [] and res.complete and res.unexamined == 0 and cancel


@pytest.mark.parametrize("name", sorted(TAMPERS))
def test_tampered_witnesses_match_the_restatement(ctx, name):
    import valida_b200 as vb

    t = fib_traces()
    mains, want, _ = TAMPERS[name](t)
    res, cancel = _device(ctx, mains, t.preprocessed)
    assert res.complete and not cancel
    assert _as_list(res) == unbalanced(mains)
    assert {(x.bus, tuple(x.fields), x.net) for x in res.tuples} == want
    assert all(x.bus_name == vb.BUS_NAMES[x.bus] and all(e.chip_name == vb.CHIP_NAMES[e.chip] for e in x.events) for x in res.tuples)


def _random_witness(h, seed):
    """Random traces of all 14 chips (every event a tuple of its own, whp) and of both preprocessed traces."""
    import valida_b200 as vb

    rng = np.random.default_rng(seed)
    mains = []
    for chip in range(14):
        d = C.cast(vb.lib().vgpu_basic_machine_chip(chip), C.POINTER(C.c_uint32))          # chip_id, width, preprocessed_width, ...
        mains.append(rng.integers(0, P, (h, d[1]), dtype=np.uint32))
    preps = [rng.integers(0, P, (h, C.cast(vb.lib().vgpu_basic_machine_chip(c), C.POINTER(C.c_uint32))[2]), dtype=np.uint32) for c in (1, 12)]
    return mains, preps


@pytest.mark.parametrize("h", [1, 4, 32])
def test_random_traces_match_the_restatement(ctx, h):
    mains, preps = _random_witness(h, 700 + h)
    want = unbalanced(mains)
    res, cancel = _device(ctx, mains, preps)
    assert want and res.complete and not cancel
    assert _as_list(res) == want
    # a small cap: what is listed is exact (net and every event) and the rest is counted as unexamined
    n_events = sum(len(e) for *_, e in want)
    for cap in (0, 1, n_events // 3):
        small, _ = _device(ctx, mains, preps, cap=cap)
        assert small.unexamined > 0 and not small.complete, cap
        got = _as_list(small)
        assert sum(len(e) for *_, e in got) <= cap and all(x in want for x in got), cap
    assert _device(ctx, mains, preps, cap=n_events)[0].complete


def test_refusals_launch_nothing(ctx, fib15):
    """Each refusal names its problem, before any launch or collective, on a lone context and alike on every rank."""
    import valida_b200 as vb

    def run(c, upload):
        dm, dp = [upload(m) for m in fib15[:14]], [upload(m) for m in fib15[14:]]
        ch = (C.c_uint32 * 15)(*[int(x) for x in CH])
        n1, n2, n3 = C.c_uint64(), C.c_uint64(), C.c_uint64()

        def raw(main, prep, cap, tup, ev, outs=(C.byref(n1), C.byref(n2), C.byref(n3))):
            a = (C.c_void_p * 14)(*[m._h if m is not None else None for m in main])
            b = (C.c_void_p * 2)(*[m._h if m is not None else None for m in prep])
            c.check(vb.lib().vgpu_check_buses(c._h, a, b, ch, cap, tup, outs[0], ev, outs[1], outs[2]))

        buf = (C.c_uint8 * 4096)()
        cases = [("null output", lambda: raw(dm, dp, 1, None, buf)),
                 ("null output", lambda: raw(dm, dp, 1, buf, None)),
                 ("null output", lambda: raw(dm, dp, 0, None, None, (C.byref(n1), None, C.byref(n3)))),
                 ("chip 5 has no trace", lambda: raw(dm[:5] + [None] + dm[6:], dp, 0, None, None)),
                 ("main width", lambda: vb.check_buses(c, dm[:3] + [dm[5]] + dm[4:], dp, CH)),
                 ("needs its preprocessed trace", lambda: raw(dm, [None, dp[1]], 0, None, None))]
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


def _tampered_at_boundaries(mats, ctxs):
    """The memory chip's is_read and the CPU's is_bus_op + 1 (each row then an event with a changed tuple or multiplicity) at global
    row 0, the last row and both sides of every rank boundary; and the range chip's mult, a chip every rank holds whole."""
    out = list(mats)
    for chip, col in ((2, 7), (0, 9)):
        a = mats[chip].copy()
        h = a.shape[0]
        rows = {0, h - 1} | {x for c in ctxs[1:] for x in (c.local_rows(h)[0] - 1, c.local_rows(h)[0])}
        for r in rows:
            a[r, col] = (int(a[r, col]) + 1) % P
        out[chip] = a
    a = mats[12].copy()
    a[77, 0] += 1
    out[12] = a
    return out


def _on_ranks(ctxs, make, cap=1 << 20):
    import valida_b200 as vb

    def rank(r, c):
        dm, dp = make(c, r)
        c.comm_stats(reset=True)
        res = vb.check_buses(c, dm, dp, CH, cap=cap)
        return _as_list(res), res.unexamined, c.comm_stats()["allgather"][0]

    return vb.run_ranks(rank, ctxs)


@pytest.fixture(scope="module")
def fib15_log(built):
    import valida_b200 as vb

    return vb.run_program_log(vb.fib_program(((1 << 15) - 17) // 7))


@pytest.mark.parametrize("nranks", [2, 3, 4, 5, 6, 8])
def test_split_every_route(ctx, fib15, fib15_log, nranks):
    """Fibonacci 2^15 tampered at and next to every rank boundary and in the range chip: every rank's output equals the single-GPU
    call's through upload_rows, import_tensor_local and borrow_tensor_local, each event counted once, and the clean device witness
    is balanced; the all-gathers are the
    bucket sums, the candidate counts and the examined events (only the first when the witness is clean)."""
    import torch
    import valida_b200 as vb

    ctxs = _ranks(nranks)
    try:
        h12 = fib15[12].shape[0]
        assert ctxs[0].local_rows(1 << 15)[1] < 1 << 15 and tuple(ctxs[0].local_rows(h12)) == (0, h12)
        mats = _tampered_at_boundaries(fib15, ctxs)
        dm, dp = _upload(ctx, mats)
        want = vb.check_buses(ctx, dm, dp, CH, cap=1 << 20)
        assert want.complete and want.tuples
        want = _as_list(want)
        events = [(e[0], e[1], e[2]) for *_, evs in want for e in evs]
        assert len(events) == len(set(events)) and sum(1 for e in events if e[:2] == (12, 77)) == 1
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

        routes = {"upload_rows": lambda c, r: _upload_rows(c, mats), "import_tensor_local": imported, "borrow_" + layout: borrow}
        for name, make in routes.items():
            for got in _on_ranks(ctxs, make):
                assert got == (want, 0, 3), name
        clean = _on_ranks(ctxs, lambda c, r: _upload_rows(c, fib15))
        assert clean == [([], 0, 1)] * nranks
        assert _on_ranks(ctxs, lambda c, r: fib15_log.witness_device(c)) == [([], 0, 1)] * nranks
        # a cap that examines part of the candidates: the same part on every rank, equal to the single-GPU call's
        cap = len(events) // 2
        single = vb.check_buses(ctx, dm, dp, CH, cap=cap)
        assert single.unexamined > 0
        for got in _on_ranks(ctxs, lambda c, r: _upload_rows(c, mats), cap=cap):
            assert got[:2] == (_as_list(single), single.unexamined)
    finally:
        _close(ctxs)


def _upload_rows(c, mats):
    v = [c.upload_rows(m) for m in mats]
    return v[:14], v[14:]


@pytest.fixture(scope="module")
def fib22(built):
    import valida_b200 as vb

    return vb.run_program_log(vb.fib_program(((1 << 22) - 17) // 7))


def test_full_size_device_witness(ctx, fib22):
    """The 2^22 Fibonacci device witness is balanced, on one GPU and split over 2 and 4 ranks; with one memory-chip value byte
    changed, exactly two tuples: the operation the CPU sends, now received once less (+1), and the changed tuple received (-1),
    with their rows."""
    import torch
    import valida_b200 as vb

    dm, dp = fib22.witness_device(ctx)
    res = vb.check_buses(ctx, dm, dp, CH)
    assert res.tuples == [] and res.complete
    for nranks in (2, 4):
        ctxs = _ranks(nranks)
        try:
            for got in vb.run_ranks(lambda r, c: vb.check_buses(c, *fib22.witness_device(c), CH), ctxs):
                assert got.tuples == [] and got.complete
        finally:
            _close(ctxs)
    h = dm[2].shape[0]
    assert h == 1 << 24
    mem = dm[2].to_tensor()
    near = mem[h // 2:h // 2 + 4096].cpu().numpy().astype(np.int64)
    r = h // 2 + next(k for k in range(len(near)) if near[k, 7] + near[k, 8] == 1 and not near[k, 6])
    row = [int(x) for x in near[r - h // 2]]
    mem[r, 1] = (mem[r, 1].to(torch.int64) + 1) % P
    torch.cuda.synchronize()
    bad = ctx.import_tensor(mem)
    res = vb.check_buses(ctx, dm[:2] + [bad] + dm[3:], dp, CH)
    old = [row[7], row[5], row[0], row[6]] + row[1:5]
    new = list(old)
    new[4] = (new[4] + 1) % P
    trim = lambda f: f[:max([i + 1 for i, x in enumerate(f) if x] or [0])]
    assert res.complete and [(t.bus, t.fields, t.net) for t in res.tuples] == sorted([(2, trim(old), 1), (2, trim(new), -1)],
                                                                                    key=lambda t: (t[0], t[1] + [0] * (14 - len(t[1]))))
    ev = {t.net: t.events for t in res.tuples}
    assert [(e.chip, e.row, e.interaction, e.send) for e in ev[-1]] == [(2, r, 0, False)]
    # the old tuple: the CPU channels that access the cell in that cycle (a cycle may read one address on two channels), and the
    # memory rows that still receive it, one fewer
    sends, receives = [e for e in ev[1] if e.send], [e for e in ev[1] if not e.send]
    assert sends and len(sends) == len(receives) + 1 and all(e.chip == 2 and e.row != r for e in receives)
    cpu = dm[0].to_tensor()
    for e in sends:
        ch = 29 + 7 * e.interaction
        assert e.chip == 0 and int(cpu[e.row, 0]) == row[5] and int(cpu[e.row, ch]) == 1 and int(cpu[e.row, ch + 2]) == row[0]
