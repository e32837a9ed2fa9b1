"""The witness check of a split proof: check_constraints_local on each rank's row shards and check_witness over a whole machine
witness (valida_b200/csrc/check.cu).

Ranks are threads of this process (comm_init_local, all on device 0 when the box has one GPU); Fibonacci with 2^15 CPU rows splits
the CPU and memory traces at 2, 4 and 8 ranks.  Every rank must report what the single-GPU check of the whole traces reports
(check_constraints on one context) and, on the rows a change can reach, what the plain-Python check_py computes.  The process-per-GPU
launch (NCCL) is checked at the end when the box has two GPUs."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from test_check_constraints_restatement import PREP_CHIPS, check_py
from test_gpu_check_constraints import CLEAN, _check_rows
from test_gpu_local_shards import BORROW_LAYOUTS, _col_major, _local_tensors, _monty
from test_quotient_restatement import AIRS

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 2013265921
NRANKS = [2, 4, 8]
CH = np.random.default_rng(2024).integers(0, P, 15, dtype=np.uint32)
SPLIT_CHIPS = (0, 2, 3)            # cpu, memory, add: split at 2 and 4 ranks (add is whole at 8)


def _ranks(n):
    import torch
    import valida_b200 as vb

    k = torch.cuda.device_count()
    ctxs = [vb.Context(i % k) for i in range(n)]
    vb.comm_init_local(ctxs)
    return ctxs


def _close(ctxs):
    for c in ctxs:
        c.close()


def _prep(mats, chip):
    return mats[14 + PREP_CHIPS[chip]] if chip in PREP_CHIPS else None


def _single(ctx, mats, ch=CH, perms=None):
    """Per chip on one context, whole traces: (check_constraints result, cumulative sum) — the expected values."""
    import valida_b200 as vb

    out = []
    for chip in range(14):
        dm = ctx.upload(mats[chip])
        dp = ctx.upload(_prep(mats, chip)) if chip in PREP_CHIPS else None
        dq, cs = vb.generate_permutation_trace(ctx, chip, dm, dp, ch)
        if perms is not None:
            perms[chip] = dq.download()
        out.append((vb.check_constraints(ctx, chip, dm, dp, dq, ch), [int(x) for x in cs]))
    return out


def _cancel(sums):
    return all(sum(s[l] for s in sums) % P == 0 for l in range(5))


def _assert_reports(reports, cancel, expected):
    for chip, (rep, (res, cs)) in enumerate(zip(reports, expected)):
        assert rep[:3] == res, (chip, rep[:3], res)
        assert [int(x) for x in rep[3]] == cs, chip
    assert cancel == _cancel([cs for _, cs in expected])


@pytest.fixture(scope="module")
def fib15(built):
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(((1 << 15) - 17) // 7), initial_fp=0x1000)
    assert t.main[0].shape[0] == 1 << 15 and t.main[2].shape[0] == 1 << 17
    return [np.array(m) for m in t.main + t.preprocessed]


@pytest.fixture(scope="module")
def fib15_single(ctx, fib15):
    perms = {}
    return _single(ctx, fib15, perms=perms), perms


def _tampered(mats, chip, row, col=0):
    out = list(mats)
    out[chip] = mats[chip].copy()
    out[chip][row, col] = (int(out[chip][row, col]) + 1) % P
    return out


def _boundary_rows(h, n, r):
    """The last row of rank r, the first row of rank r + 1, global row 0 and global row h - 1."""
    return sorted({(r + 1) * (h // n) - 1, (r + 1) * (h // n), 0, h - 1})


def _witness_on_ranks(ctxs, mats):
    import valida_b200 as vb

    def rank(r, c):
        dm = [c.upload_rows(m) for m in mats]
        return vb.check_witness(c, dm[:14], dm[14:], CH)

    return vb.run_ranks(rank, ctxs)


@pytest.mark.parametrize("nranks", NRANKS)
def test_clean_witnesses(ctx, fib15, fib15_single, nranks):
    """The CLEAN programs (every chip whole) and Fibonacci at 2^15 CPU rows (tall chips split): every chip clean on every rank, the
    sums cancel and equal vgpu_perm_trace's."""
    import valida_b200 as vb

    cases = {"fib15": (fib15, fib15_single[0])}
    for name, make in CLEAN.items():
        prog, cells = make()
        t = vb.run_program(prog, initial_fp=0x1000, static_data=cells)
        mats = [np.array(m) for m in t.main + t.preprocessed]
        cases[name] = (mats, _single(ctx, mats))
    ctxs = _ranks(nranks)
    try:
        assert ctxs[0].local_rows(1 << 17)[1] < 1 << 17 and ctxs[0].local_rows(1 << 15)[1] < 1 << 15
        for name, (mats, expected) in cases.items():
            assert all(res == (-1, 0, 0) for res, _ in expected), name
            for reports, cancel in _witness_on_ranks(ctxs, mats):
                _assert_reports(reports, cancel, expected)
                assert cancel, name
    finally:
        _close(ctxs)


@pytest.mark.parametrize("nranks", NRANKS)
def test_boundary_tampering(ctx, fib15, fib15_single, nranks):
    """A cpu, memory or add cell changed at the last row of rank r, the first row of rank r + 1, global row 0 and global row h - 1:
    every rank reports the single-GPU check's first row, constraint and count (and check_py's on the rows the change reaches), and
    the cancel flag follows the sums.  A word of the permutation trace's last running sum is located the same way."""
    import valida_b200 as vb

    ctxs = _ranks(nranks)
    r = nranks // 2 - 1
    try:
        for chip in SPLIT_CHIPS:
            h = fib15[chip].shape[0]
            for row in _boundary_rows(h, nranks, r):
                mats, perms = _tampered(fib15, chip, row), {}
                expected = _single(ctx, mats, perms=perms)
                res, perm = expected[chip][0], perms[chip]
                idx = sorted({(row - 1) % h, row, (row + 1) % h, h - 1})     # the rows that rows row - 1 and row read, and the last row
                first, failing = _check_rows(chip, mats[chip], mats[chip][idx], perm[idx], idx, CH, [(row - 1) % h, row])
                assert res == ((-1, 0, 0) if first is None else (first[0], first[1], failing)), (chip, row)
                if chip == 0:
                    assert res[0] in ((row - 1) % h, row), (row, res)       # clk is constrained on every row
                for reports, cancel in _witness_on_ranks(ctxs, mats):
                    _assert_reports(reports, cancel, expected)
        # the permutation trace's last running sum (the cumulative sum) changed: rows h - 2 and h - 1 read it
        chip = 0
        h, perm = fib15[chip].shape[0], fib15_single[1][chip].copy()
        k5 = perm.shape[1] - 5
        perm[h - 1, k5] = (int(perm[h - 1, k5]) + 1) % P
        want = vb.check_constraints(ctx, chip, ctx.upload(fib15[chip]), None, ctx.upload(perm), CH)
        first, failing = check_py(chip, fib15[chip], perm, CH, rows=[h - 2, h - 1])
        assert want == (first[0], first[1], failing) and want[0] == h - 2

        def rank(r_, c):
            return vb.check_constraints_local(c, chip, c.upload_rows(fib15[chip]), None, c.upload_rows(perm), CH)

        assert vb.run_ranks(rank, ctxs) == [want] * nranks
    finally:
        _close(ctxs)


@pytest.mark.parametrize("nranks", NRANKS)
def test_random_traces_every_chip(ctx, nranks):
    """Random main (and preprocessed) traces of 2^14 rows, split at every rank count, with honest permutation traces: every
    constraint fails somewhere; the first row, constraint and count equal the single-GPU result."""
    import valida_b200 as vb

    h = 1 << 14
    cases = []
    for chip in range(14):
        rng = np.random.default_rng(900 + chip)
        desc = C.cast(vb.lib().vgpu_basic_machine_chip(chip), C.POINTER(C.c_uint32))      # chip_id, width, preprocessed_width, ...
        main = rng.integers(0, P, (h, desc[1]), dtype=np.uint32)
        prep = rng.integers(0, P, (h, desc[2]), dtype=np.uint32) if desc[2] else None
        dm, dp = ctx.upload(main), ctx.upload(prep) if prep is not None else None
        dq, _ = vb.generate_permutation_trace(ctx, chip, dm, dp, CH)
        want = vb.check_constraints(ctx, chip, dm, dp, dq, CH)
        if AIRS[chip] is not None:                # a chip with AIR constraints fails on random rows
            assert want[0] >= 0 and want[2] > 0, (chip, want)
        cases.append((chip, main, prep, dq.download(), want))
    ctxs = _ranks(nranks)
    try:
        assert ctxs[0].local_rows(h)[1] == h // nranks

        def rank(r, c):
            return [vb.check_constraints_local(c, chip, c.upload_rows(m), c.upload_rows(p) if p is not None else None, c.upload_rows(q), CH)
                    for chip, m, p, q, _ in cases]

        for got in vb.run_ranks(rank, ctxs):
            assert got == [w for *_, w in cases]
    finally:
        _close(ctxs)


@pytest.mark.parametrize("nranks", [2, 8])
def test_every_input_route(ctx, fib15, fib15_single, nranks):
    """upload_rows, import_tensor_local, borrow_tensor_local at every BORROW_LAYOUTS layout, witness_device on the split context, and
    tall traces passed whole with upload (their failing rows count once, not once per rank): the same reports."""
    import torch
    import valida_b200 as vb

    h = fib15[0].shape[0]
    mats = _tampered(fib15, 0, h // nranks)              # the first row of rank 1: rows h / N - 1 and h / N fail
    expected = _single(ctx, mats)
    assert expected[0][0][2] == 2
    ctxs = _ranks(nranks)
    try:
        routes = {"upload_rows": lambda c, r: [c.upload_rows(m) for m in mats],
                  "upload_whole": lambda c, r: [c.upload(m) for m in mats],
                  "import_tensor_local": lambda c, r: [c.import_tensor_local(x, a.shape[0])
                                                       for x, a in zip(_local_tensors(c, mats, lambda a, d: _col_major(a, d)), mats)]}
        for layout, (pad, off) in BORROW_LAYOUTS.items():
            def borrow(c, r, pad=pad, off=off):
                tens = _local_tensors(c, [_monty(a) for a in mats], lambda a, d: _col_major(a, d, pad, off))
                torch.cuda.synchronize()
                return [c.borrow_tensor_local(x, a.shape[0]) for x, a in zip(tens, mats)]
            routes["borrow_" + layout] = borrow
        for name, make in routes.items():
            def rank(r, c):
                dm = make(c, r)
                return vb.check_witness(c, dm[:14], dm[14:], CH)

            for reports, cancel in vb.run_ranks(rank, ctxs):
                _assert_reports(reports, cancel, expected)
        log = vb.run_program_log(vb.fib_program(((1 << 15) - 17) // 7))

        def device(r, c):
            dm, dp = log.witness_device(c)
            assert dm[0].local_rows()[1] == h // nranks
            return vb.check_witness(c, dm, dp, CH)

        for reports, cancel in vb.run_ranks(device, ctxs):
            _assert_reports(reports, cancel, fib15_single[0])
    finally:
        _close(ctxs)


def test_lone_context_and_sharding_off(ctx, fib15, fib15_single):
    """On a lone context check_constraints_local IS check_constraints and check_witness is 14 x (generate_permutation_trace +
    check_constraints) with the summed sums; a split group with sharding off behaves as lone contexts (no collective)."""
    import valida_b200 as vb

    h = fib15[0].shape[0]
    for mats in (fib15, _tampered(fib15, 0, h // 2), _tampered(fib15, 2, 5)):
        expected = _single(ctx, mats)
        dm = [ctx.upload(m) for m in mats]
        for chip in range(14):
            dp = dm[14 + PREP_CHIPS[chip]] if chip in PREP_CHIPS else None
            dq, _ = vb.generate_permutation_trace(ctx, chip, dm[chip], dp, CH)
            assert vb.check_constraints_local(ctx, chip, dm[chip], dp, dq, CH) == vb.check_constraints(ctx, chip, dm[chip], dp, dq, CH)
        reports, cancel = vb.check_witness(ctx, dm[:14], dm[14:], CH)
        _assert_reports(reports, cancel, expected)
    ctxs = _ranks(2)
    try:
        for c in ctxs:
            c.set_sharding(False)
        c = ctxs[0]
        c.comm_stats(reset=True)
        dm = [c.upload_rows(m) for m in fib15]
        assert dm[0].local_rows() == (0, h)
        _assert_reports(*vb.check_witness(c, dm[:14], dm[14:], CH), fib15_single[0])
        assert c.comm_stats()["allgather"][0] == 0
    finally:
        _close(ctxs)


def test_collectives_of_each_call(fib15):
    """Two all-gathers for check_constraints_local of a split chip; for check_witness two besides the LogUp traces' (one per split
    chip)."""
    import valida_b200 as vb

    ctxs = _ranks(4)
    try:
        def rank(r, c):
            dm = [c.upload_rows(m) for m in fib15]
            dq, _ = vb.generate_permutation_trace(c, 0, dm[0], None, CH)
            c.comm_stats(reset=True)
            vb.check_constraints_local(c, 0, dm[0], None, dq, CH)
            local = c.comm_stats()["allgather"][0]
            split = sum(c.local_rows(m.shape[0])[1] < m.shape[0] for m in fib15[:14])
            vb.check_witness(c, dm[:14], dm[14:], CH)
            return local, c.comm_stats()["allgather"][0], split

        for local, witness, split in vb.run_ranks(rank, ctxs):
            assert local == 2
            assert split >= 2 and witness == 2 + split
    finally:
        _close(ctxs)


def _chip_desc_copy(chip, chip_id):
    """A copy of a BasicMachine chip descriptor with another chip id (the public calls only hand out the 14 known ones)."""
    import valida_b200 as vb

    pair_col = 4 * (2 + 3 * 4)
    size = 16 + 5 * (4 + 14 * pair_col + pair_col + 8)      # vgpu_chip_desc: 4 words, then 5 interactions
    buf = C.create_string_buffer(size)
    C.memmove(buf, vb.lib().vgpu_basic_machine_chip(chip), size)
    C.cast(buf, C.POINTER(C.c_uint32))[0] = chip_id
    return buf


def test_refusals_launch_nothing(fib15):
    """Each refusal names its problem on every rank alike, before any launch or collective."""
    import valida_b200 as vb

    ctxs = _ranks(2)
    try:
        def rank(r, c):
            dm = [c.upload_rows(m) for m in fib15]
            dq = {chip: vb.generate_permutation_trace(c, chip, dm[chip], None, CH)[0] for chip in (0, 3)}
            odd = c.upload(np.zeros((3, fib15[3].shape[1]), dtype=np.uint32))
            odd_q = c.upload(np.zeros((3, dq[3].shape[1]), dtype=np.uint32))
            short_q = c.upload(np.zeros((8, dq[0].shape[1]), dtype=np.uint32))
            unknown = _chip_desc_copy(0, 99)

            def raw_unknown():
                row, con, n = C.c_int64(), C.c_uint32(), C.c_uint64()
                c.check(vb.lib().vgpu_check_constraints_local(c._h, C.cast(unknown, C.c_void_p), dm[0]._h, None, dq[0]._h,
                                                              (C.c_uint32 * 15)(*[int(x) for x in CH]),
                                                              C.byref(row), C.byref(con), C.byref(n)))

            cases = [("unknown chip", raw_unknown),
                     ("main width", lambda: vb.check_constraints_local(c, 3, dm[0], None, dq[0], CH)),
                     ("differ in height", lambda: vb.check_constraints_local(c, 0, dm[0], None, short_q, CH)),
                     ("not a power of two", lambda: vb.check_constraints_local(c, 3, odd, None, odd_q, CH))]
            out = []
            for what, call in cases:
                before = c.launch_count
                c.comm_stats(reset=True)
                with pytest.raises(vb.VgpuError) as e:
                    call()
                out.append((what, what in str(e.value), c.launch_count == before, sum(n for n, _ in c.comm_stats().values())))
            c.set_sharding(False)                         # the shards no longer are this context's run
            before = c.launch_count
            with pytest.raises(vb.VgpuError) as e:
                vb.check_constraints_local(c, 0, dm[0], None, dq[0], CH)
            out.append(("run", "not this context's run" in str(e.value), c.launch_count == before, 0))
            with pytest.raises(vb.VgpuError) as e:
                vb.check_witness(c, dm[:14], dm[14:], CH)
            out.append(("run (witness)", "not this context's run" in str(e.value), c.launch_count == before, 0))
            return out

        for out in vb.run_ranks(rank, ctxs):
            for what, named, no_launch, collectives in out:
                assert named and no_launch and collectives == 0, (what, named, no_launch, collectives)
    finally:
        _close(ctxs)


def test_bit_reversed_rows_are_refused(ctx, fib15):
    """Quotient chunks store their rows bit-reversed: not a trace, refused by name before any launch (a rule of the shapes alone, so
    alike on every rank)."""
    import valida_b200 as vb

    pcs = vb.TwoAdicFriPcs(ctx)
    dm = ctx.upload(fib15[3])
    dq, cs = vb.generate_permutation_trace(ctx, 3, dm, None, CH)
    _, pdm = pcs.commit_batches([dm])
    _, pdq = pcs.commit_batches([dq])
    log_h = fib15[3].shape[0].bit_length() - 1
    chunks = vb.quotient(ctx, 3, log_h, None, pcs.get_ldes(pdm)[0], pcs.get_ldes(pdq)[0], cs, CH, CH[:5])
    before = ctx.launch_count
    with pytest.raises(vb.VgpuError, match="bit-reversed"):
        vb.check_constraints_local(ctx, 3, chunks, None, dq, CH)
    assert ctx.launch_count == before


@pytest.fixture(scope="module")
def fib22(built):
    import valida_b200 as vb

    return vb.run_program_log(vb.fib_program(((1 << 22) - 17) // 7))


def test_full_size_memory_on_one_gpu(fib22):
    """check_witness of the Fibonacci 2^22 device witness on one GPU holds the traces, the largest permutation trace and < 64 MB
    more, and reports a clean witness."""
    import valida_b200 as vb

    c = vb.Context(0)
    try:
        dm, dp = fib22.witness_device(c)
        c.synchronize()
        live = c.memory_stats(reset=True)["live"]
        reports, cancel = vb.check_witness(c, dm, dp, CH)
        peak = c.memory_stats()["peak"]
        assert cancel and all(r[:3] == (-1, 0, 0) for r in reports)
        largest_perm = max(m.shape[0] * 5 * (C.cast(vb.lib().vgpu_basic_machine_chip(i), C.POINTER(C.c_uint32))[3] + 1) * 4
                           for i, m in enumerate(dm))
        assert peak - live < largest_perm + (64 << 20), (peak - live, largest_perm)
    finally:
        c.close()


@pytest.mark.parametrize("nranks", NRANKS)
def test_full_size_split(ctx, fib22, nranks):
    """Fibonacci 2^22 from witness_device split over the ranks is clean; with one CPU cell changed at a rank boundary it is located
    exactly as the single-GPU check locates it."""
    import torch
    import valida_b200 as vb

    dm1, dp1 = fib22.witness_device(ctx)
    h = dm1[0].shape[0]
    row = h // nranks                                # the first row of rank 1
    cpu = dm1[0].to_tensor()
    cpu[row, 0] += 1                                 # clk: canonical words below p - 1
    d = ctx.import_tensor(cpu)
    dq, _ = vb.generate_permutation_trace(ctx, 0, d, None, CH)
    want = vb.check_constraints(ctx, 0, d, None, dq, CH)
    assert want[0] == row - 1 and want[2] == 2
    del dm1, dp1, d, dq, cpu
    ctxs = _ranks(nranks)
    try:
        def rank(r, c):
            dm, dp = fib22.witness_device(c)
            clean = vb.check_witness(c, dm, dp, CH)
            row0, rows = dm[0].local_rows()
            x = dm[0].local_to_tensor()
            if row0 <= row < row0 + rows:
                x[row - row0, 0] += 1
            torch.cuda.synchronize()
            dm[0] = c.import_tensor_local(x, h)
            return clean, vb.check_witness(c, dm, dp, CH)[0][0][:3]

        for (reports, cancel), got in vb.run_ranks(rank, ctxs):
            assert cancel and all(r[:3] == (-1, 0, 0) for r in reports)
            assert got == want
    finally:
        _close(ctxs)


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist

    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import valida_b200 as vb

    ctx = vb.Context(rank)
    t = vb.run_program(vb.fib_program(((1 << 15) - 17) // 7), initial_fp=0x1000)
    mats = _tampered([np.array(m) for m in t.main + t.preprocessed], 0, (1 << 15) // world)
    dm = [ctx.upload(m) for m in mats]
    single = vb.check_witness(ctx, dm[:14], dm[14:], CH)
    del dm
    ctx.comm_init_from_torch()
    tens = _local_tensors(ctx, [_monty(a) for a in mats], lambda a, d: _col_major(a, d, pad=1))
    torch.cuda.synchronize()
    dm = [ctx.borrow_tensor_local(x, a.shape[0]) for x, a in zip(tens, mats)]
    reports, cancel = vb.check_witness(ctx, dm[:14], dm[14:], CH)
    out[rank] = {"split": dm[0].local_rows()[1] < 1 << 15,
                 "located": reports[0][:3] == ((1 << 15) // world - 1, single[0][0][1], 2),
                 "equal": all(a[:3] == b[:3] and list(a[3]) == list(b[3]) for a, b in zip(reports, single[0])) and cancel == single[1]}
    for m in dm:
        m.free()
    ctx.close()
    dist.destroy_process_group()


def test_processes_check_only_their_rows(built):
    import torch
    import torch.multiprocessing as mp

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs: one process per GPU")
    mgr = mp.Manager()
    out = mgr.dict()
    port = 36500 + (os.getpid() % 2000)
    mp.spawn(_worker, args=(2, port, out), nprocs=2, join=True)
    for rank in range(2):
        assert all(out[rank].values()), (rank, dict(out[rank]))
