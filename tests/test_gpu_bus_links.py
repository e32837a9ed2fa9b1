"""bus_links and cycles_of on the GPU (vgpu_bus_links, valida_b200/csrc/links.cu): every event that carries each item's bus tuple, and
the cycles behind a row, on one GPU and over the row shards of a split context.

The raw output (links, events, their order and the unlisted count) is held byte for byte to the plain-Python restatement of
test_bus_links_restatement.py, to check_buses where both report a tuple, and at full size to a numpy join of the CPU and add columns."""
import ctypes as C

import numpy as np
import pytest

from test_bus_balance_restatement import TAMPERS, fib_traces
from test_bus_links_restatement import CHIPS, P, Witness
from test_gpu_check_buses import CH, _random_witness
from test_gpu_check_constraints import CLEAN
from test_gpu_check_failures import _close, _ranks, fib15  # noqa: F401
from test_gpu_local_shards import _col_major, _local_tensors, _monty

pytestmark = pytest.mark.gpu
BIG = 1 << 20


def _array(items):
    import valida_b200 as vb

    arr = np.zeros(len(items), dtype=vb.BUS_EVENT_DTYPE)
    for i, (chip, m, row) in enumerate(items):
        arr[i]["chip"], arr[i]["interaction"], arr[i]["row"] = chip, m, row
    return arr


def _raw(ctx, dm, dp, items, cap):
    """vgpu_bus_links' output as bytes: (links, events, unlisted)."""
    import valida_b200 as vb

    arr = _array(items)
    n = len(arr)
    links = np.zeros(max(n, 1), dtype=vb.BUS_LINK_DTYPE)
    ev = np.zeros(max(cap, 1), dtype=vb.BUS_EVENT_DTYPE)
    ne, un = C.c_uint64(), C.c_uint64()
    a, b = (C.c_void_p * 14)(*[m._h for m in dm]), (C.c_void_p * 2)(*[m._h for m in dp])
    ctx.check(vb.lib().vgpu_bus_links(ctx._h, a, b, arr.ctypes.data_as(C.c_void_p) if n else None, n, links.ctypes.data_as(C.c_void_p), cap,
                                      ev.ctypes.data_as(C.c_void_p) if cap else None, C.byref(ne), C.byref(un)))
    return links[:n].tobytes(), ev[:ne.value].tobytes(), int(un.value)


def _want(w, items, cap):
    """The restatement's answer in the same bytes."""
    import valida_b200 as vb

    links, events, un = w.links(items, cap)
    la = np.zeros(len(links), dtype=vb.BUS_LINK_DTYPE)
    for i, x in enumerate(links):
        la[i] = x
    ea = np.zeros(len(events), dtype=vb.BUS_EVENT_DTYPE)
    for i, (chip, m, row, mult, send) in enumerate(events):
        ea[i] = (chip, m, row, mult, send)
    return la.tobytes(), ea.tobytes(), un


def _sample(w, seed, k=6):
    """Every interaction of k sampled rows (and the first and last row) of every chip with interactions, then a quarter of them again."""
    rng = np.random.default_rng(seed)
    out = []
    for chip in range(14):
        h = w.mains[chip].shape[0]
        rows = sorted(set(rng.integers(0, h, k).tolist()) | {0, h - 1})
        out += [(chip, m, r) for r in rows for m in range(len(CHIPS[chip]))]
    return out + [out[i] for i in rng.permutation(len(out))[:len(out) // 4]]


def _upload(ctx, mains, preps):
    return [ctx.upload(m) for m in mains], [ctx.upload(m) for m in preps]


@pytest.mark.parametrize("name", sorted(CLEAN))
def test_reference_programs_host_and_device_witnesses(ctx, name):
    import valida_b200 as vb

    prog, cells = CLEAN[name]()
    t = vb.run_program(prog, initial_fp=0x1000, static_data=cells)
    w = Witness(t.main)
    items = _sample(w, len(name))
    want = _want(w, items, BIG)
    assert _raw(ctx, *_upload(ctx, t.main, t.preprocessed), items, BIG) == want
    assert any(w.item(*x)[2] == 0 for x in items) and want[2] == 0
    log = vb.run_program_log(prog, static_data=cells)
    assert _raw(ctx, *log.witness_device(ctx), items, BIG) == want


@pytest.mark.parametrize("h", [1, 4, 32])
def test_random_traces_match_the_restatement(ctx, h):
    mains, preps = _random_witness(h, 900 + h)
    w = Witness(mains)
    dm, dp = _upload(ctx, mains, preps)
    items = _sample(w, h)
    full = _want(w, items, BIG)
    assert _raw(ctx, dm, dp, items, BIG) == full
    n_events = len(full[1]) // 24
    for cap in range(n_events + 1):
        assert _raw(ctx, dm, dp, items, cap) == _want(w, items, cap), cap


@pytest.mark.parametrize("name", ["add_output", "memory_value", "range_mult"])
def test_tampered_witnesses_agree_with_check_buses(ctx, name):
    """check_buses' events are items as they are; for each tuple it reports, the events are its events and sends - receives its net.
    Every cap gives the stated prefix with exact totals."""
    import valida_b200 as vb

    t = fib_traces()
    mains, _, _ = TAMPERS[name](t)
    w = Witness(mains)
    dm, dp = _upload(ctx, mains, t.preprocessed)
    bad = vb.check_buses(ctx, dm, dp, CH)
    assert bad.tuples and bad.complete
    evs = [e for x in bad.tuples for e in x.events]
    items = [(e.chip, e.interaction, e.row) for e in evs] + _sample(w, 3)
    full = _want(w, items, BIG)
    assert _raw(ctx, dm, dp, items, BIG) == full
    res = vb.bus_links(ctx, dm, dp, evs, BIG)
    assert res.complete and len(res.links) == len(evs)
    for x in bad.tuples:
        for e in x.events:
            link = res.links[evs.index(e)]
            assert (link.bus, link.bus_name, link.fields) == (x.bus, x.bus_name, x.fields)
            assert link.events == x.events and (link.sends - link.receives) % P == x.net % P and link.n_events == len(x.events)
    n_events = len(full[1]) // 24
    for cap in range(n_events + 1):
        assert _raw(ctx, dm, dp, items, cap) == _want(w, items, cap), cap


@pytest.mark.parametrize("name", ["fib", "config5", "static_data"])
def test_cycles_of_equals_the_search(ctx, name):
    import programs
    import valida_b200 as vb

    prog, cells = {"fib": (vb.fib_program(3), None), "config5": (programs.config5_program(10), None),
                   "static_data": programs.static_data_program()}[name]
    t = vb.run_program(prog, initial_fp=0x1000, static_data=cells)
    w = Witness(t.main)
    dm, dp = _upload(ctx, t.main, t.preprocessed)
    for chip in range(14):
        rows = list(range(w.mains[chip].shape[0]))
        got = vb.cycles_of(ctx, dm, dp, chip, rows)
        assert got.complete and got.cycles == [w.cycles(chip, r) for r in rows], chip
    if name == "fib":
        add = w.mains[3]
        real = [r for r in range(add.shape[0]) if add[r, 15]]
        cycles = vb.cycles_of(ctx, dm, dp, 3, real).cycles
        assert real and all(c and all(int(w.mains[0][r, 3]) == 100 for r in c) for c in cycles)
    # a cap too small for a range byte's adds: the answer says so
    assert not vb.cycles_of(ctx, dm, dp, 12, [int(np.argmax(w.mains[12][:, 0]))], cap=1).complete or name == "static_data"


def test_refusals_launch_nothing(ctx, fib15):
    """Each refusal names its problem, before any launch or collective, on a lone context and alike on every rank."""
    import valida_b200 as vb

    def run(c, upload):
        dm, dp = [upload(m) for m in fib15[:14]], [upload(m) for m in fib15[14:]]
        n1, n2 = C.c_uint64(), C.c_uint64()
        buf = (C.c_uint8 * 4096)()

        def raw(main, prep, items, links, cap, events, outs=(C.byref(n1), C.byref(n2))):
            a = (C.c_void_p * 14)(*[m._h if m is not None else None for m in main])
            b = (C.c_void_p * 2)(*[m._h if m is not None else None for m in prep])
            arr = _array(items)
            c.check(vb.lib().vgpu_bus_links(c._h, a, b, arr.ctypes.data_as(C.c_void_p), len(items), links, cap, events, outs[0], outs[1]))

        ok = [(0, 3, 5)]
        cases = [("null output", lambda: raw(dm, dp, ok, None, 0, None)),
                 ("null output", lambda: raw(dm, dp, ok, buf, 1, None)),
                 ("null output", lambda: raw(dm, dp, ok, buf, 0, None, (None, C.byref(n2)))),
                 ("item 1: chip 14", lambda: raw(dm, dp, ok + [(14, 0, 0)], buf, 0, None)),
                 ("item 0: interaction 0 is not below chip 1's 0", lambda: raw(dm, dp, [(1, 0, 0)], buf, 0, None)),
                 ("item 1: interaction 5 is not below chip 3's 5", lambda: raw(dm, dp, ok + [(3, 5, 0)], buf, 0, None)),
                 ("item 0: row 32768 is outside chip 0's trace", lambda: raw(dm, dp, [(0, 0, 1 << 15)], buf, 0, None)),
                 ("item 0: row -1", lambda: raw(dm, dp, [(2, 0, -1)], buf, 0, None)),
                 ("chip 5 has no trace", lambda: raw(dm[:5] + [None] + dm[6:], dp, ok, buf, 0, None)),
                 ("main width", lambda: vb.bus_links(c, dm[:3] + [dm[5]] + dm[4:], dp, ok)),
                 ("needs its preprocessed trace", lambda: raw(dm, [None, dp[1]], ok, buf, 0, None))]
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


def _boundary_items(mats, ctxs):
    """Every interaction of the rows at and next to every rank boundary, the first and the last row of every chip, and range rows."""
    rows = {}
    for chip in range(14):
        h = mats[chip].shape[0]
        rows[chip] = {0, h - 1} | {x for c in ctxs[1:] for b in (c.local_rows(h)[0],) for x in (b - 1, b) if 0 < b < h}
    rows[12] |= {5, 77, 200}
    return [(chip, m, r) for chip in range(14) for r in sorted(rows[chip]) for m in range(len(CHIPS[chip]))]


@pytest.mark.parametrize("nranks", [2, 3, 4, 8])
def test_split_every_route(ctx, fib15, nranks):
    """Fibonacci 2^15 with items on every rank boundary: every rank's output is the single-GPU output byte for byte, through
    upload_rows, import_tensor_rows, import_tensor_local and borrow_tensor_local, with the three all-gathers the header states (two
    when nothing is listed)."""
    import torch
    import valida_b200 as vb

    ctxs = _ranks(nranks)
    try:
        assert ctxs[0].local_rows(1 << 15)[1] < 1 << 15
        items = _boundary_items(fib15, ctxs)
        single = {cap: _raw(ctx, *_upload(ctx, fib15[:14], fib15[14:]), items, cap) for cap in (0, 1000, BIG)}
        assert single[BIG][2] == 0 and single[1000][2] > 0 and single[0][1] == b""

        def rows(c, r):
            v = [c.upload_rows(a) for a in fib15]
            return v[:14], v[14:]

        def imported_rows(c, r):
            v = [c.import_tensor_rows(torch.from_numpy(a.view(np.int32)).to("cuda:%d" % c.device)) for a in fib15]
            return v[:14], v[14:]

        def imported_local(c, r):
            v = [c.import_tensor_local(x, a.shape[0]) for x, a in zip(_local_tensors(c, fib15, lambda a, d: _col_major(a, d)), fib15)]
            return v[:14], v[14:]

        def borrowed(c, r):
            tens = _local_tensors(c, [_monty(a) for a in fib15], lambda a, d: _col_major(a, d, 3, 0))
            torch.cuda.synchronize()
            v = [c.borrow_tensor_local(x, a.shape[0]) for x, a in zip(tens, fib15)]
            return v[:14], v[14:]

        for name, make in {"upload_rows": rows, "import_tensor_rows": imported_rows, "import_tensor_local": imported_local,
                           "borrow_tensor_local": borrowed}.items():
            def rank(r, c):
                dm, dp = make(c, r)
                out = []
                for cap in (0, 1000, BIG):
                    c.comm_stats(reset=True)
                    got = _raw(c, dm, dp, items, cap)
                    out.append((got, c.comm_stats()["allgather"][0]))
                return out

            for got in vb.run_ranks(rank, ctxs):
                assert got == [(single[0], 2), (single[1000], 3), (single[BIG], 3)], name
    finally:
        _close(ctxs)


@pytest.fixture(scope="module")
def fib22(built):
    import valida_b200 as vb

    return vb.run_program_log(vb.fib_program(((1 << 22) - 17) // 7))


def _keys(a):
    a = np.ascontiguousarray(a, dtype=np.uint32)
    return a.view(np.dtype((np.void, a.shape[1] * 4))).ravel()


def test_full_size_device_witness(ctx, fib22):
    """The 2^22 Fibonacci device witness: 2^16 add-row items and the CPU-row items of one cycle, on one GPU and over 2 ranks, against a
    numpy join of the downloaded CPU and add columns."""
    import valida_b200 as vb

    dm, dp = fib22.witness_device(ctx)
    cpu = dm[0].to_tensor()
    add = dm[3].to_tensor()
    cpu_cols = [3] + list(range(32, 36)) + list(range(39, 43)) + list(range(46, 50)) + [50]
    send_mask = (cpu[:, 9] != 0).cpu().numpy()
    sends = cpu[:, cpu_cols].cpu().numpy().view(np.uint32)[send_mask]
    a = add.cpu().numpy().view(np.uint32)
    del cpu, add
    real = a[:, 15] != 0
    tup = np.concatenate([np.full((a.shape[0], 1), 100, np.uint32), a[:, 0:8], a[:, 11:15], np.zeros((a.shape[0], 1), np.uint32)], axis=1)
    rng = np.random.default_rng(22)
    add_rows = np.sort(rng.choice(np.nonzero(real)[0], 1 << 16, replace=False))
    s_keys, s_counts = np.unique(_keys(sends), return_counts=True)
    r_keys, r_counts = np.unique(_keys(tup[real]), return_counts=True)
    ik = _keys(tup[add_rows])

    def count(keys, counts):
        i = np.minimum(np.searchsorted(keys, ik), len(keys) - 1)
        return np.where(keys[i] == ik, counts[i], 0)

    n_send, n_recv = count(s_keys, s_counts), count(r_keys, r_counts)
    assert (n_send > 0).all()
    cycle = 12345
    items = [(3, 4, int(r)) for r in add_rows] + [(0, m, cycle) for m in range(4)]
    res = vb.bus_links(ctx, dm, dp, items, cap=1 << 22)
    assert res.complete
    for k, link in enumerate(res.links[:1 << 16]):
        assert (link.multiplicity, link.sends, link.receives, link.n_events) == (1, n_send[k], n_recv[k], n_send[k] + n_recv[k]), k
        assert link.fields == [int(x) for x in tup[add_rows[k]]][:len(link.fields)]
    for k in rng.choice(1 << 16, 32, replace=False):
        cyc = [e.row for e in res.links[k].events if e.chip == 0]
        assert cyc and all(np.array_equal(sends[np.searchsorted(np.nonzero(send_mask)[0], r)], tup[add_rows[k]]) for r in cyc)
    assert all(e.chip != 0 or e.row == cycle for x in res.links[-4:-1] if x.multiplicity for e in x.events)   # the memory channels
    single = _raw(ctx, dm, dp, items, 1 << 22)
    ctxs = _ranks(2)
    try:
        for got in vb.run_ranks(lambda r, c: _raw(c, *fib22.witness_device(c), items, 1 << 22), ctxs):
            assert got == single
    finally:
        _close(ctxs)
