"""check_failures on the GPU (vgpu_check_failures, valida_b200/csrc/check.cu): every (row, constraint, value) on which a chip's
check does not vanish, the total and the failing rows per constraint, on one GPU and over the row shards of a split context.

The list is held value for value to failures_py below, a plain-Python restatement of the whole check text (the AIRS of
test_quotient_restatement.py with the debug selectors, then eval_permutation_constraints' LogUp constraints, in eval order), and to
check_constraints: its first entry is check_constraints' first failure, its distinct rows are check_constraints' failing rows and
the per-constraint counts add up to the total."""
import collections
import ctypes as C

import numpy as np
import pytest

import programs
from test_check_constraints_restatement import PREP_CHIPS, fib_traces, random_case, tamper_cases, tampered
from test_gpu_check_constraints import CLEAN
from test_gpu_local_shards import BORROW_LAYOUTS, _col_major, _local_tensors, _monty
from test_perm_trace_restatement import CHIPS, P, SEND, apply, e_add, e_from, e_mul, e_sub
from test_quotient_restatement import AIRS, e_scale

pytestmark = pytest.mark.gpu
CH = np.random.default_rng(4242).integers(0, P, 15, dtype=np.uint32)
BIG = 1 << 40                                  # a cap above every total here


def failures_py(chip, main, perm, ch, rows=None):
    """Every (row, constraint, value[5]) of one chip on which the check does not vanish, ascending by row then constraint; values
    canonical (a base-field constraint has limbs 1..4 = 0).  rows: the rows to check (all by default); they read rows i and
    (i + 1) mod h of main and perm, and the cumulative sum from perm's last row."""
    h, inter = main.shape[0], CHIPS[chip]
    k = len(inter)
    r1, r2 = [int(x) for x in ch[5:10]], [int(x) for x in ch[10:15]]
    alphas_global, acc = [], e_from(1)
    for _ in range(4):
        acc = e_mul(acc, r1)
        alphas_global.append(acc)
    cumsum = [int(v) for v in perm[h - 1, 5 * k:5 * k + 5]]
    out = []
    for i in sorted({r % h for r in (range(h) if rows is None else rows)}):
        j = (i + 1) % h
        loc, nxt = [int(v) for v in main[i]], [int(v) for v in main[j]]
        pl = [[int(v) for v in perm[i, 5 * m:5 * m + 5]] for m in range(k + 1)]
        pn = [[int(v) for v in perm[j, 5 * m:5 * m + 5]] for m in range(k + 1)]
        last = 1 if i == h - 1 else 0
        sel = {"first": 1 if i == 0 else 0, "last": last, "transition": 1 - last}
        cons = [e_from(c) for c in AIRS[chip](loc, nxt, sel)] if AIRS[chip] else []
        phi_local, phi_next = pl[k], pn[k]
        rhs, phi0 = e_from(0), e_from(0)
        for m, (sign, bus, fields, count) in enumerate(inter):
            rlc, beta = e_from(0), e_from(1)
            for f in fields:
                rlc = e_add(rlc, e_scale(beta, apply(f, loc)))
                beta = e_mul(beta, r2)
            rlc = e_add(rlc, alphas_global[bus])
            cons.append(e_sub(e_mul(rlc, pl[m]), e_from(1)))
            t_loc, t_nxt = e_scale(pl[m], apply(count, loc)), e_scale(pn[m], apply(count, nxt))
            if sign == SEND:
                phi0, rhs = e_add(phi0, t_loc), e_add(rhs, t_nxt)
            else:
                phi0, rhs = e_sub(phi0, t_loc), e_sub(rhs, t_nxt)
        cons.append(e_scale(e_sub(e_sub(phi_next, phi_local), rhs), sel["transition"]))
        cons.append(e_scale(e_sub(phi_local, phi0), sel["first"]))
        cons.append(e_scale(e_sub(phi_local, cumsum), sel["last"]))
        out += [(i, c, tuple(x % P for x in v)) for c, v in enumerate(cons) if any(x % P for x in v)]
    return out


def _per_constraint(fails, chip):
    import valida_b200 as vb

    n = collections.Counter(c for _, c, _ in fails)
    return [n[c] for c in range(vb.constraint_count(chip)[1])]


def _as_list(arr):
    return [(int(r["row"]), int(r["constraint"]), tuple(int(v) for v in r["value"])) for r in arr]


def _agree(fails, total, per, check):
    """The complete list against check_constraints' (first row, first constraint, failing rows)."""
    assert len(fails) == total and sum(per) == total
    first = (fails[0][0], fails[0][1]) if fails else (-1, 0)
    assert check == first + (len({r for r, _, _ in fails}),), (check, first)


def _device(ctx, chip, main, prep, ch, perm=None, cap=BIG):
    """Uploads the traces (the honest permutation trace built on the device unless one is given) and returns (check_failures'
    list, total, per-constraint counts, check_constraints' result)."""
    import valida_b200 as vb

    dm = ctx.upload(main)
    dp = ctx.upload(prep) if prep is not None else None
    dq = ctx.upload(perm) if perm is not None else vb.generate_permutation_trace(ctx, chip, dm, dp, ch)[0]
    total = vb.check_failures(ctx, chip, dm, dp, dq, ch, cap=0)[1]
    arr, total, per = vb.check_failures(ctx, chip, dm, dp, dq, ch, cap=min(cap, total))
    return _as_list(arr), total, [int(x) for x in per], vb.check_constraints(ctx, chip, dm, dp, dq, ch)


def _prep_of(traces, chip):
    return traces.preprocessed[PREP_CHIPS[chip]] if chip in PREP_CHIPS else None


@pytest.mark.parametrize("h", [1, 2, 16, 256])
@pytest.mark.parametrize("chip", sorted(CHIPS))
def test_random_traces_match_the_restatement(ctx, oracle, chip, h):
    """Random traces with honest permutation traces: every AIR constraint's value on every row, and the LogUp constraints'."""
    main, prep, perm, ch = random_case(oracle, chip, h, 9100 + 16 * chip + h)
    want = failures_py(chip, main, perm, ch)
    fails, total, per, check = _device(ctx, chip, main, prep, ch, perm)
    assert fails == want
    assert per == _per_constraint(want, chip)
    _agree(fails, total, per, check)
    if AIRS[chip] is not None and h > 1:
        assert total > 0


@pytest.mark.parametrize("name", sorted(CLEAN))
def test_clean_witnesses_have_no_failures(ctx, oracle, name):
    import valida_b200 as vb

    prog, cells = CLEAN[name]()
    t = vb.run_program(prog, initial_fp=0x1000, static_data=cells)
    ch = oracle.prove(t.main, t.preprocessed, debug_checks=False).transcript()["perm_challenges"]
    for chip in range(14):
        fails, total, per, check = _device(ctx, chip, t.main[chip], _prep_of(t, chip), ch)
        assert fails == [] and total == 0 and per == [0] * len(per), chip
        _agree(fails, total, per, check)


@pytest.mark.parametrize("name", ["lt_edges", "loads_stores"])
def test_rejected_programs_match_the_restatement(ctx, oracle, name):
    import valida_b200 as vb

    prog = programs.lt_edge_operands_program() if name == "lt_edges" else programs.loads_stores_edge_program()
    t = vb.run_program(prog, initial_fp=0x1000)
    ref = oracle.prove(t.main, t.preprocessed, debug_checks=True)
    ch = ref.transcript()["perm_challenges"]
    seen = 0
    for chip in range(14):
        perm = ref.perm_trace(chip)
        want = failures_py(chip, t.main[chip], perm, ch)
        fails, total, per, check = _device(ctx, chip, t.main[chip], _prep_of(t, chip), ch, perm)
        assert fails == want, chip
        assert per == _per_constraint(want, chip), chip
        _agree(fails, total, per, check)
        seen += total
    assert seen > 0


@pytest.mark.parametrize("chip", sorted(CHIPS))
def test_tampered_permutation_traces_match_the_restatement(ctx, oracle, chip):
    t = fib_traces()
    main, prep = t.main[chip], _prep_of(t, chip)
    ch = np.random.default_rng(60 + chip).integers(0, P, 15, dtype=np.uint32)
    perm, _ = oracle.perm_trace(chip, main, prep, ch)
    for row, col in tamper_cases(main.shape[0], perm.shape[1]):
        bad = tampered(perm, row, col)
        want = failures_py(chip, main, bad, ch)
        fails, total, per, check = _device(ctx, chip, main, prep, ch, bad)
        assert want and fails == want, (row, col)
        assert per == _per_constraint(want, chip), (row, col)
        _agree(fails, total, per, check)


def test_cap(ctx, oracle):
    """cap = 0 writes nothing and still counts; a cap below the total writes the list's prefix; a cap above writes all of it."""
    import valida_b200 as vb

    chip, h = 0, 256
    main, prep, perm, ch = random_case(oracle, chip, h, 9300)
    dm, dq = ctx.upload(main), ctx.upload(perm)
    full, total, per = vb.check_failures(ctx, chip, dm, None, dq, ch, cap=h * 256)
    assert len(full) == total > 1000
    full = _as_list(full)
    for cap in (0, 1, 2, 127, total // 3, total - 1, total, total + 1, 10 * total):
        arr, t, p = vb.check_failures(ctx, chip, dm, None, dq, ch, cap=cap)
        assert t == total and list(p) == list(per), cap
        assert _as_list(arr) == full[:min(cap, total)], cap


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


@pytest.fixture(scope="module")
def fib15(built):
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(((1 << 15) - 17) // 7), initial_fp=0x1000)
    assert t.main[0].shape[0] == 1 << 15 and t.main[2].shape[0] == 1 << 17
    return [np.array(m) for m in t.main + t.preprocessed]


def _boundary_tampered(mats, ctxs, chips):
    """Every rank boundary b of each chip's split: rows b - 1 and b (and global row 0 and the last row) changed in column 0."""
    out = list(mats)
    for chip in chips:
        h = mats[chip].shape[0]
        a = mats[chip].copy()
        rows = {0, h - 1}
        for c in ctxs[1:]:
            b = c.local_rows(h)[0]
            rows |= {b - 1, b}
        for r in rows:
            a[r, 0] = (int(a[r, 0]) + 1) % P
        out[chip] = a
    return out


def _single_all(ctx, mats, chips):
    """Per chip on one context: (list as bytes, total, per-constraint counts) of the whole traces, and the list agrees with
    check_constraints."""
    import valida_b200 as vb

    out = {}
    for chip in chips:
        dm = ctx.upload(mats[chip])
        dp = ctx.upload(mats[14 + PREP_CHIPS[chip]]) if chip in PREP_CHIPS else None
        dq, _ = vb.generate_permutation_trace(ctx, chip, dm, dp, CH)
        check = vb.check_constraints(ctx, chip, dm, dp, dq, CH)
        total = vb.check_failures(ctx, chip, dm, dp, dq, CH, cap=0)[1]
        arr, total, per = vb.check_failures(ctx, chip, dm, dp, dq, CH, cap=total)
        first = (int(arr[0]["row"]), int(arr[0]["constraint"])) if total else (-1, 0)
        assert check == first + (len(np.unique(arr["row"])),) and int(per.sum()) == total == len(arr), (chip, check)
        out[chip] = (arr.tobytes(), total, [int(x) for x in per])
    return out


def _on_ranks(ctxs, mats, chips, make, caps):
    """Every rank's check_failures of its own matrices (make(ctx, rank)), per chip (list as bytes, total, per-constraint counts)."""
    import valida_b200 as vb

    def rank(r, c):
        dm = make(c, r)
        res = {}
        for chip in chips:
            dp = dm[14 + PREP_CHIPS[chip]] if chip in PREP_CHIPS else None
            dq, _ = vb.generate_permutation_trace(c, chip, dm[chip], dp, CH)
            arr, total, per = vb.check_failures(c, chip, dm[chip], dp, dq, CH, cap=caps[chip])
            res[chip] = (arr.tobytes(), total, [int(x) for x in per])
        return res

    return vb.run_ranks(rank, ctxs)


@pytest.mark.parametrize("nranks", [2, 3, 4, 5, 8])
def test_split_boundaries_every_route(ctx, fib15, nranks):
    """Fibonacci 2^15 with the cpu and memory traces changed at and next to every rank boundary: every rank's list, total and counts
    equal the single-GPU call's, through upload_rows, import_tensor_local and borrow_tensor_local; capped lists are its prefixes.
    The memory chip's permutation trace changed at the same places reaches the LogUp constraints across the boundaries."""
    import torch
    import valida_b200 as vb

    ctxs = _ranks(nranks)
    try:
        assert ctxs[0].local_rows(1 << 15)[1] < 1 << 15
        mats = _boundary_tampered(fib15, ctxs, (0, 3))
        chips = list(range(14))
        want = _single_all(ctx, mats, chips)
        assert want[0][1] > 0 and want[3][1] > 0
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
        caps = {chip: want[chip][1] for chip in chips}
        for name, make in routes.items():
            for got in _on_ranks(ctxs, mats, chips, make, caps):
                assert got == want, name
        for cap in (0, 1, want[0][1] // 2):
            for got in _on_ranks(ctxs, mats, (0,), routes["upload_rows"], {0: cap}):
                assert got[0] == (want[0][0][:32 * cap], want[0][1], want[0][2]), cap
        # the LogUp constraints across the boundaries: the memory chip's permutation trace changed at and next to each one
        chip, h = 2, fib15[2].shape[0]
        dm = ctx.upload(fib15[chip])
        perm = vb.generate_permutation_trace(ctx, chip, dm, None, CH)[0].download()
        rows = {0, h - 1} | {x for c in ctxs[1:] for x in (c.local_rows(h)[0] - 1, c.local_rows(h)[0])}
        for r in rows:
            perm = tampered(perm, r, (3 * r) % perm.shape[1])
        fails, total, per, check = _device(ctx, chip, fib15[chip], None, CH, perm)
        _agree(fails, total, per, check)
        assert total > 0

        def logup(r, c):
            arr, t, p = vb.check_failures(c, chip, c.upload_rows(fib15[chip]), None, c.upload_rows(perm), CH, cap=total)
            return _as_list(arr), t, [int(x) for x in p]

        assert vb.run_ranks(logup, ctxs) == [(fails, total, per)] * nranks
    finally:
        _close(ctxs)


@pytest.mark.parametrize("nranks", [2, 3, 4, 5, 8])
def test_split_random_traces(ctx, nranks):
    """Random 2^14-row traces of every chip (split at every rank count here), honest permutation traces: every rank's output is the
    single-GPU call's."""
    import valida_b200 as vb

    h = 1 << 14
    mats = []
    for chip in range(14):
        d = C.cast(vb.lib().vgpu_basic_machine_chip(chip), C.POINTER(C.c_uint32))      # chip_id, width, preprocessed_width, ...
        mats.append(np.random.default_rng(950 + chip).integers(0, P, (h, d[1]), dtype=np.uint32))
    for chip in sorted(PREP_CHIPS, key=PREP_CHIPS.get):
        d = C.cast(vb.lib().vgpu_basic_machine_chip(chip), C.POINTER(C.c_uint32))
        mats.append(np.random.default_rng(990 + chip).integers(0, P, (h, d[2]), dtype=np.uint32))
    want = _single_all(ctx, mats, range(14))
    ctxs = _ranks(nranks)
    try:
        assert ctxs[0].local_rows(h)[1] < h
        for got in _on_ranks(ctxs, mats, range(14), lambda c, r: [c.upload_rows(m) for m in mats], {c: want[c][1] for c in range(14)}):
            assert got == want
    finally:
        _close(ctxs)


def test_sharding_off_is_a_lone_context(ctx, fib15):
    import valida_b200 as vb

    mats = _tampered_cpu(fib15, 5000)
    want = _single_all(ctx, mats, (0, 2))
    ctxs = _ranks(2)
    try:
        for c in ctxs:
            c.set_sharding(False)
        c = ctxs[0]
        c.comm_stats(reset=True)
        dm = [c.upload_rows(m) for m in mats]
        assert dm[0].local_rows() == (0, mats[0].shape[0])
        for chip in (0, 2):
            dq, _ = vb.generate_permutation_trace(c, chip, dm[chip], None, CH)
            arr, total, per = vb.check_failures(c, chip, dm[chip], None, dq, CH, cap=want[chip][1] + 1)
            assert (arr.tobytes(), total, [int(x) for x in per]) == want[chip]
        assert c.comm_stats()["allgather"][0] == 0
    finally:
        _close(ctxs)


def _tampered_cpu(mats, row):
    out = list(mats)
    out[0] = mats[0].copy()
    out[0][row, 0] = (int(out[0][row, 0]) + 1) % P
    return out


def test_refusals_launch_nothing(ctx, fib15):
    """Each refusal names its problem, on a lone context and alike on every rank, before any launch or collective."""
    import valida_b200 as vb

    def cases(c, dm, dq):
        ch = (C.c_uint32 * 15)(*[int(x) for x in CH])
        n, tot = C.c_uint64(), C.c_uint64()
        chip0 = vb.lib().vgpu_basic_machine_chip(0)
        odd = c.upload(np.zeros((3, fib15[3].shape[1]), dtype=np.uint32))
        air3, total3 = vb.constraint_count(3)
        odd_q = c.upload(np.zeros((3, 5 * (total3 - air3 - 2)), dtype=np.uint32))
        short_q = c.upload(np.zeros((8, dq[0].shape[1]), dtype=np.uint32))

        def raw(cap, out, n_out, total):
            c.check(vb.lib().vgpu_check_failures(c._h, chip0, dm[0]._h, None, dq[0]._h, ch, cap, out, n_out, total, None))

        return [("null output", lambda: raw(1, None, C.byref(n), C.byref(tot))),
                ("null output", lambda: raw(0, None, None, C.byref(tot))),
                ("null output", lambda: raw(0, None, C.byref(n), None)),
                ("main width", lambda: vb.check_failures(c, 3, dm[0], None, dq[0], CH)),
                ("differ in height", lambda: vb.check_failures(c, 0, dm[0], None, short_q, CH)),
                ("not a power of two", lambda: vb.check_failures(c, 3, odd, None, odd_q, CH)),
                ("needs its preprocessed trace", lambda: vb.check_failures(c, 1, dm[1], None, dq[1], CH))]

    def run(c, dm, dq):
        out = []
        for what, call in cases(c, dm, dq):
            before = c.launch_count
            c.comm_stats(reset=True)
            with pytest.raises(vb.VgpuError) as e:
                call()
            out.append((what, what in str(e.value), c.launch_count == before, sum(k for k, _ in c.comm_stats().values())))
        return out

    def prepared(c, upload):
        dm = [upload(m) for m in fib15]
        dq = {chip: vb.generate_permutation_trace(c, chip, dm[chip], dm[14] if chip == 1 else None, CH)[0] for chip in (0, 1)}
        return dm, dq

    lone = run(ctx, *prepared(ctx, ctx.upload))
    assert all(named and no_launch and k == 0 for _, named, no_launch, k in lone), lone
    assert vb.lib().vgpu_chip_constraint_count(None, None, None) != 0
    with pytest.raises(vb.VgpuError):
        vb.constraint_label(0, vb.constraint_count(0)[1])
    ctxs = _ranks(2)
    try:
        outs = vb.run_ranks(lambda r, c: run(c, *prepared(c, c.upload_rows)), ctxs)
        assert outs[0] == outs[1] == lone, outs
    finally:
        _close(ctxs)


def test_constraint_labels():
    import valida_b200 as vb

    air, total = vb.constraint_count(0)
    assert (air, total) == (53, 60)
    assert vb.constraint_label(0, 0) == "Air::eval assertion 0"
    assert vb.constraint_label(0, 53) == "interaction 0 (bus 2, send)"
    assert [vb.constraint_label(0, i) for i in (57, 58, 59)] == ["LogUp transition", "LogUp first row", "LogUp last row"]
    assert vb.constraint_label(2, 0) == "interaction 0 (bus 2, receive)"
    for chip, inter in CHIPS.items():
        a, t = vb.constraint_count(chip)
        w = C.cast(vb.lib().vgpu_basic_machine_chip(chip), C.POINTER(C.c_uint32))[1]
        row = [0] * w
        assert t == a + len(inter) + 3 and a == (len(AIRS[chip](row, row, {"first": 0, "last": 0, "transition": 1})) if AIRS[chip] else 0)


@pytest.fixture(scope="module")
def fib22(built):
    import valida_b200 as vb

    return vb.run_program_log(vb.fib_program(((1 << 22) - 17) // 7))


def _witness_failures(c, fib22, chips=range(14)):
    import valida_b200 as vb

    dm, dp = fib22.witness_device(c)
    out = []
    for chip in chips:
        pr = dp[PREP_CHIPS[chip]] if chip in PREP_CHIPS else None
        dq, _ = vb.generate_permutation_trace(c, chip, dm[chip], pr, CH)
        arr, total, per = vb.check_failures(c, chip, dm[chip], pr, dq, CH)
        out.append((len(arr), total, int(per.sum())))
        del dq
    return out


def test_full_size_clean_one_gpu_and_split(ctx, fib22):
    import valida_b200 as vb

    assert _witness_failures(ctx, fib22) == [(0, 0, 0)] * 14
    for nranks in (2, 4):
        ctxs = _ranks(nranks)
        try:
            for got in vb.run_ranks(lambda r, c: _witness_failures(c, fib22), ctxs):
                assert got == [(0, 0, 0)] * 14
        finally:
            _close(ctxs)


def test_full_size_tampered_memory_chip(ctx, fib22):
    """Ten words of the 2^24-row memory chip's permutation trace changed (row 0, the last row and its cumulative-sum cell among them):
    the list is failures_py on the rows those words reach, and the totals agree with check_constraints."""
    import torch
    import valida_b200 as vb

    chip = 2
    dm, dp = fib22.witness_device(ctx)
    h = dm[chip].shape[0]
    assert h == 1 << 24
    dq, _ = vb.generate_permutation_trace(ctx, chip, dm[chip], None, CH)
    q = dq.to_tensor()
    del dq
    w = q.shape[1]
    words = [(0, 3), (1, 0), (h // 3, 7), (h // 2, 5), (h // 2 + 1, 9), ((1 << 20) + 17, 2), (h - 5, 4), (h - 2, 8), (h - 1, 1), (h - 1, w - 1)]
    for r, col in words:
        q[r, col] = (q[r, col].to(torch.int64) + 1) % P
    torch.cuda.synchronize()
    bad = ctx.import_tensor(q)
    reach = sorted({x % h for r, _ in words for x in (r - 1, r)} | {h - 2, h - 1})        # rows that read a changed word
    idx = sorted(set(reach) | {(x + 1) % h for x in reach} | {h - 1})
    main = dm[chip].to_tensor()[idx].cpu().numpy().astype(np.uint32)
    perm = q[idx].cpu().numpy().astype(np.uint32)
    pos = {i: k for k, i in enumerate(idx)}

    class Rows:
        def __init__(self, sub):
            self.sub, self.shape = sub, (h,) + sub.shape[1:]

        def __getitem__(self, key):
            if isinstance(key, tuple):
                return self.sub[(pos[key[0]],) + key[1:]]
            return self.sub[pos[key]]

    want = failures_py(chip, Rows(main), Rows(perm), CH, rows=reach)
    arr, total, per = vb.check_failures(ctx, chip, dm[chip], None, bad, CH)
    fails = _as_list(arr)
    assert 10 <= len(want) and fails == want
    assert list(per) == _per_constraint(want, chip)
    _agree(fails, total, [int(x) for x in per], vb.check_constraints(ctx, chip, dm[chip], None, bad, CH))
