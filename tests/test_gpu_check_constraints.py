"""check_constraints on the GPU (valida_b200/csrc/check.cu) and the debug mode of prove_machine.

The device sweep is held to two texts of the reference's debug-build check: the plain-Python per-row checker of
test_check_constraints_restatement.py (first failing row and constraint, and the count of failing rows) and the oracle's
check_constraints.  Clean witnesses report nothing, the witnesses the CPU AIR rejects are located exactly, random and tampered
traces agree row for row, and the debug mode leaves the proof bytes alone."""
import os
import sys

import numpy as np
import pytest

import programs
from test_check_constraints_restatement import (PREP_CHIPS, as_oracle_code, check_py, fib_traces, oracle_check,  # noqa: F401
                                                random_case, tamper_cases, tampered)
from test_perm_trace_restatement import CHIPS, P

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_large_proof_digests import assert_matches_golden  # noqa: E402

pytestmark = pytest.mark.gpu


def _lt_edges_without_double_immediate():
    prog = programs.lt_edge_operands_program()
    assert prog[-2].tolist() == [115, -104, 7, 7, 1, 1]
    return np.concatenate([prog[:-2], prog[-1:]])


CLEAN = {
    "fib25": lambda: (__import__("valida_b200").fib_program(25), None),
    "fib0": lambda: (__import__("valida_b200").fib_program(0), None),
    "lone_stop": lambda: (np.array([[8, 0, 0, 0, 0, 0]], dtype=np.int32), None),
    "single_address": lambda: (programs.single_address_program(5), None),
    "lt_edges": lambda: (_lt_edges_without_double_immediate(), None),
    "mixed": lambda: (programs.mixed_program(100), None),
    "config5": lambda: (programs.config5_program(60), None),
    "static_data": programs.static_data_program,
}


def _prep(traces, chip):
    return traces.preprocessed[PREP_CHIPS[chip]] if chip in PREP_CHIPS else None


def _device_check(ctx, chip, main, prep, ch, perm=None):
    """Uploads the traces, builds the permutation trace on the device unless one is given, and checks the chip there."""
    import valida_b200 as vb

    dm = ctx.upload(main)
    dp = ctx.upload(prep) if prep is not None else None
    cs = None
    if perm is None:
        dq, cs = vb.generate_permutation_trace(ctx, chip, dm, dp, ch)
    else:
        dq = ctx.upload(perm)
    return vb.check_constraints(ctx, chip, dm, dp, dq, ch), cs


def _expect(first, failing):
    return (-1, 0, 0) if first is None else (first[0], first[1], failing)


@pytest.mark.parametrize("name", sorted(CLEAN))
def test_clean_witnesses_pass_on_every_chip(ctx, oracle, name):
    import valida_b200 as vb

    prog, cells = CLEAN[name]()
    t = vb.run_program(prog, initial_fp=0x1000, static_data=cells)
    ch = oracle.prove(t.main, t.preprocessed, debug_checks=False).transcript()["perm_challenges"]
    total = [0] * 5
    for chip in range(14):
        res, cs = _device_check(ctx, chip, t.main[chip], _prep(t, chip), ch)
        assert res == (-1, 0, 0), (chip, res)
        total = [(a + int(b)) % P for a, b in zip(total, cs)]
    assert total == [0] * 5


@pytest.mark.parametrize("name", ["lt_edges", "loads_stores"])
def test_rejected_witnesses_are_located(ctx, oracle, name):
    import valida_b200 as vb

    prog = programs.lt_edge_operands_program() if name == "lt_edges" else programs.loads_stores_edge_program()
    t = vb.run_program(prog, initial_fp=0x1000)
    ref = oracle.prove(t.main, t.preprocessed, debug_checks=True)
    ch = ref.transcript()["perm_challenges"]
    want = ref.constraint_failures()
    for chip in range(14):
        (row, con, failing), _ = _device_check(ctx, chip, t.main[chip], _prep(t, chip), ch)
        assert (-1 if row < 0 else row * 4096 + con) == want[chip], chip
        assert failing == check_py(chip, t.main[chip], ref.perm_trace(chip), ch)[1], chip
    cfg = vb.StarkConfig(ctx, oracle.rc480)
    ctx.set_debug_checks(True)
    try:
        with pytest.raises(vb.VgpuError) as e:
            vb.prove_machine(cfg, t)
    finally:
        ctx.set_debug_checks(False)
    row, con = divmod(want[0], 4096)
    assert "chip 0 (cpu): constraint %d does not vanish on row %d" % (con, row) in str(e.value)


@pytest.mark.parametrize("h", [1, 2, 16])
@pytest.mark.parametrize("chip", sorted(CHIPS))
def test_random_traces_match_both_texts(ctx, oracle, oracle_check, chip, h):
    main, prep, perm, ch = random_case(oracle, chip, h, 7000 + 16 * chip + h)
    first, failing = check_py(chip, main, perm, ch)
    assert as_oracle_code(first) == oracle_check.check_constraints(chip, main, prep, perm, ch)
    res, _ = _device_check(ctx, chip, main, prep, ch)
    assert res == _expect(first, failing)


@pytest.mark.parametrize("chip", sorted(CHIPS))
def test_tampered_permutation_traces_match_both_texts(ctx, oracle, oracle_check, chip):
    """The LogUp constraints fail only on a permutation trace that is not the honest one: uploaded here word by word."""
    t = fib_traces()
    main, prep = t.main[chip], _prep(t, chip)
    ch = np.random.default_rng(50 + chip).integers(0, P, 15, dtype=np.uint32)
    perm, _ = oracle.perm_trace(chip, main, prep, ch)
    assert _device_check(ctx, chip, main, prep, ch, perm)[0] == (-1, 0, 0)
    for row, col in tamper_cases(main.shape[0], perm.shape[1]):
        bad = tampered(perm, row, col)
        first, failing = check_py(chip, main, bad, ch)
        assert as_oracle_code(first) == oracle_check.check_constraints(chip, main, prep, bad, ch)
        assert _device_check(ctx, chip, main, prep, ch, bad)[0] == _expect(first, failing), (row, col)


def _phase_names(ctx):
    import valida_b200 as vb

    return [n for n, _ in vb.last_prove_phases(ctx)]


@pytest.mark.parametrize("device_resident", [False, True])
def test_debug_mode_keeps_the_proof_bytes(ctx, oracle, device_resident):
    import valida_b200 as vb

    t = vb.run_program(programs.config5_program(60), initial_fp=0x1000)
    cfg = vb.StarkConfig(ctx, oracle.rc480)
    dev = ([ctx.upload(m) for m in t.main], [ctx.upload(m) for m in t.preprocessed]) if device_resident else None
    off = vb.prove_machine(cfg, t, device_resident=dev)
    assert "check constraints" not in _phase_names(ctx)
    ctx.set_debug_checks(True)
    try:
        on = vb.prove_machine(cfg, t, device_resident=dev)
        assert "check constraints" in _phase_names(ctx)
    finally:
        ctx.set_debug_checks(False)
    assert on == off == oracle.prove(t.main, t.preprocessed, debug_checks=False).cbor()


def test_argument_errors_launch_nothing(ctx, oracle):
    import valida_b200 as vb

    t = fib_traces()
    ch = np.arange(15, dtype=np.uint32)
    dm = [ctx.upload(m) for m in t.main]
    dp = [ctx.upload(m) for m in t.preprocessed]
    perm = {c: vb.generate_permutation_trace(ctx, c, dm[c], dp[PREP_CHIPS[c]] if c in PREP_CHIPS else None, ch)[0] for c in (0, 1, 3)}
    short = ctx.upload(t.main[3][: t.main[3].shape[0] // 2])
    cases = [
        ("width", lambda: vb.check_constraints(ctx, 3, dm[0], None, perm[3], ch)),
        ("permutation trace width", lambda: vb.check_constraints(ctx, 3, dm[3], None, perm[0], ch)),
        ("height", lambda: vb.check_constraints(ctx, 3, short, None, perm[3], ch)),
        ("preprocessed", lambda: vb.check_constraints(ctx, 1, dm[1], None, perm[1], ch)),
    ]
    for what, call in cases:
        before = ctx.launch_count
        with pytest.raises(vb.VgpuError) as e:
            call()
        assert ctx.launch_count == before, what
        assert what in str(e.value), (what, str(e.value))


def test_split_contexts_refuse_the_debug_mode(oracle):
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(((1 << 13) - 17) // 7), initial_fp=0x1000)
    ranks = [vb.Context(0), vb.Context(0)]
    try:
        vb.comm_init_local(ranks)
        cfgs = [vb.StarkConfig(c, oracle.rc480) for c in ranks]

        def work(r, c):
            c.set_debug_checks(True)
            try:
                vb.prove_machine(cfgs[r], t)
            except vb.VgpuError as e:
                msg = str(e)
            else:
                msg = None
            # a row shard cannot be checked: its last row's next row lives on the other rank
            dm = c.upload_rows(t.main[0])
            assert dm.local_rows()[1] < t.main[0].shape[0]
            dq = c.upload_rows(np.zeros((t.main[0].shape[0], 25), dtype=np.uint32))
            with pytest.raises(vb.VgpuError, match="row shards"):
                vb.check_constraints(c, 0, dm, None, dq, np.zeros(15, dtype=np.uint32))
            return msg

        msgs = vb.run_ranks(work, ranks)
        assert all(m is not None and "debug checks" in m for m in msgs), msgs
    finally:
        for c in ranks:
            c.close()


def test_full_size_fibonacci(ctx, oracle):
    """Fibonacci with 2^22 CPU rows (memory chip 2^24) from the device witness: the bytes are the recorded oracle proof's; the debug
    mode passes and leaves the bytes alone; one CPU cell changed at a row r is found on rows r - 1 and r only, as the Python checker
    computes on those rows, and the cumulative sums no longer cancel when row r sends on the memory bus (the last row is padding and
    sends nothing)."""
    import valida_b200 as vb

    n = ((1 << 22) - 17) // 7
    log = vb.run_program_log(vb.fib_program(n))
    cfg = vb.StarkConfig(ctx, oracle.rc480)
    dm, dp = log.witness_device(ctx)
    h = dm[0].shape[0]
    assert h == 1 << 22
    off = vb.prove_machine(cfg, None, device_resident=(dm, dp))
    assert_matches_golden(off, "fib_2p22")
    ctx.set_debug_checks(True)
    try:
        on = vb.prove_machine(cfg, None, device_resident=(dm, dp))
    finally:
        ctx.set_debug_checks(False)
    assert on == off
    del dm, dp
    t = log.traces()
    ch = np.random.default_rng(22).integers(0, P, 15, dtype=np.uint32)
    sums = {}
    dmain = {}
    for chip in range(1, 14):
        dmain[chip] = ctx.upload(t.main[chip])
        dprep = ctx.upload(_prep(t, chip)) if chip in PREP_CHIPS else None
        _, sums[chip] = vb.generate_permutation_trace(ctx, chip, dmain[chip], dprep, ch)
        del dprep
    for r in (0, h // 2 + 5, h - 1):
        cpu = t.main[0].copy()
        cpu[r, 0] = (int(cpu[r, 0]) + 1) % P          # clk
        dcpu = ctx.upload(cpu)
        dq, cs = vb.generate_permutation_trace(ctx, 0, dcpu, None, ch)
        got = vb.check_constraints(ctx, 0, dcpu, None, dq, ch)
        idx = sorted({(r - 1) % h, r, (r + 1) % h, h - 1})     # the rows that rows r - 1 and r read, and the last row
        perm = dq.download()
        sub_main, sub_perm = cpu[idx], perm[idx]
        del perm
        first, failing = _check_rows(0, cpu, sub_main, sub_perm, idx, ch, [(r - 1) % h, r])
        assert got == _expect(first, failing), r
        # a row that uses a memory channel sends its clk on the memory bus: the sums move; a padding row sends nothing
        total = [(sum(int(s[l]) for s in sums.values()) + int(cs[l])) % P for l in range(5)]
        sends = any(int(cpu[r, c]) for c in (29, 36, 43))
        assert (total != [0] * 5) == sends, r
        assert sends or r == h - 1
        del dcpu, dq


def _check_rows(chip, full_main, sub_main, sub_perm, idx, ch, rows):
    """check_py on the rows `rows` of a tall trace, given only the rows `idx` (which hold every row those rows read and the last row)."""
    h = full_main.shape[0]
    pos = {i: k for k, i in enumerate(idx)}

    class Rows:
        def __init__(self, sub):
            self.sub, self.shape = sub, (h,) + sub.shape[1:]

        def __getitem__(self, key):
            if isinstance(key, tuple):
                return self.sub[(pos[key[0]],) + key[1:]]
            return self.sub[pos[key]]

    return check_py(chip, Rows(sub_main), Rows(sub_perm), ch, rows=rows)
