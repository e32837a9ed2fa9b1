"""Bus balance of a machine witness in plain Python: every EVENT (a row of a chip and one of its interactions whose multiplicity is not
zero) with its bus, its tuple (the interaction's fields on the row, zero-padded to 14) and its sign, and per (bus, padded tuple) the
net multiplicity, sends minus receives mod p.  Built on the interaction tables and `apply` of test_perm_trace_restatement.py, the
same text the LogUp restatement is pinned to, so this is what vgpu_check_buses (tests/test_gpu_check_buses.py) is held to.

CPU only.  Honest witnesses balance; hand-derived tampered witnesses leave exactly the expected tuples unbalanced; and on every case
"nothing unbalanced" agrees with the oracle's cumulative sums cancelling."""
import collections
import json
import os

import numpy as np
import pytest

import programs
from generated_programs import counted_program, generated_program
from test_perm_trace_restatement import CHIPS, GENERAL, MEM, P, RANGE, SEND, apply

MAX_FIELDS = 14
GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "programs.json")))


def trim(fields):
    fields = list(fields)
    while fields and fields[-1] == 0:
        fields.pop()
    return tuple(fields)


def signed(net):
    return net - P if net > P // 2 else net


def bus_events(mains):
    """Every event of the 14 main traces: (bus, padded tuple, chip, row, interaction, multiplicity, is_send)."""
    out = []
    for chip in range(14):
        inter = CHIPS[chip]
        for row, vals in enumerate(np.asarray(mains[chip]).tolist()):
            for m, (sign, bus, fields, count) in enumerate(inter):
                mult = apply(count, vals) % P
                if mult:
                    tup = tuple(apply(f, vals) % P for f in fields) + (0,) * (MAX_FIELDS - len(fields))
                    out.append((bus, tup, chip, row, m, mult, sign == SEND))
    return out


def unbalanced(mains):
    """The unbalanced tuples, ascending by (bus, padded tuple): (bus, tuple trimmed of trailing zeros, signed net, events), the events
    (chip, row, interaction, multiplicity, is_send) ascending by (chip, row, interaction) — the form check_buses returns."""
    net = collections.Counter()
    evs = collections.defaultdict(list)
    for bus, tup, chip, row, m, mult, send in bus_events(mains):
        net[(bus, tup)] = (net[(bus, tup)] + (mult if send else P - mult)) % P
        evs[(bus, tup)].append((chip, row, m, mult, send))
    return [(bus, trim(tup), signed(net[(bus, tup)]), sorted(evs[(bus, tup)], key=lambda e: (e[0], e[1], e[2])))
            for bus, tup in sorted(net) if net[(bus, tup)]]


def sums_cancel(oracle, mains, preps, seed=5):
    """The oracle's cumulative sums of the 14 chips (LogUp under random challenges) add to zero."""
    ch = np.random.default_rng(seed).integers(0, P, 15, dtype=np.uint32)
    total = [0] * 5
    for chip in range(14):
        prep = preps[0] if chip == 1 else preps[1] if chip == 12 else None
        _, cs = oracle.perm_trace(chip, np.ascontiguousarray(mains[chip]), prep, ch)
        total = [(a + int(b)) % P for a, b in zip(total, cs)]
    return total == [0] * 5


def fib_traces():
    import valida_b200 as vb

    return vb.run_program(vb.fib_program(3), initial_fp=0x1000)


def _changed(t, chip, row, col, value):
    mains = [np.array(m) for m in t.main]
    mains[chip][row, col] = value % P
    return mains


# ---- hand-derived tampered witnesses: (mains, the expected (bus, trimmed tuple, net) set) --------------------------------------
def _memory_value(t):
    """A memory-chip value byte + 1 on a row that receives an operation: the CPU's send is left unmatched (+1) and the changed
    tuple received with nothing sent (-1)."""
    mem = t.main[2]
    row = next(r for r in range(mem.shape[0]) if int(mem[r, 7]) + int(mem[r, 8]) == 1 and not mem[r, 6])
    old = [int(x) for x in (mem[row, 7], mem[row, 5], mem[row, 0], mem[row, 6], *mem[row, 1:5])]
    new = list(old)
    new[4] = (new[4] + 1) % P
    return _changed(t, 2, row, 1, int(mem[row, 1]) + 1), {(MEM, trim(old), 1), (MEM, trim(new), -1)}, (2, row)


def _range_mult(t):
    rng_ = t.main[12]
    row = next(r for r in range(rng_.shape[0]) if rng_[r, 0] and rng_[r, 1])
    return _changed(t, 12, row, 0, int(rng_[row, 0]) + 1), {(RANGE, (int(rng_[row, 1]),), -1)}, (12, row)


def _cpu_used(t):
    """A CPU memory channel's `used` flag cleared: the memory chip's receive of that operation is left unmatched (-1)."""
    cpu = t.main[0]
    row, ch = next((r, c) for r in range(cpu.shape[0]) for c in (29, 36, 43) if cpu[r, c])
    tup = [int(cpu[row, ch + 1]), int(cpu[row, 0]), int(cpu[row, ch + 2]), 0] + [int(x) for x in cpu[row, ch + 3:ch + 7]]
    return _changed(t, 0, row, ch, 0), {(MEM, trim(tup), -1)}, (2, None)     # the CPU row is no event any more


def _add_output(t):
    """An add output byte b + 1: its range send moves from b (-1) to b + 1 (+1), and the add's general-bus receive moves from the
    CPU's tuple (+1) to the changed one (-1)."""
    add = t.main[3]
    row = next(r for r in range(add.shape[0]) if add[r, 15] and add[r, 11] < 255)
    b = int(add[row, 11])
    old = [100] + [int(x) for x in add[row, 0:8]] + [int(x) for x in add[row, 11:15]]
    new = list(old)
    new[9] = b + 1
    want = {(RANGE, trim([b]), -1), (RANGE, (b + 1,), 1), (GENERAL, trim(old), 1), (GENERAL, trim(new), -1)}
    return _changed(t, 3, row, 11, b + 1), want, (3, row)


def _alu_clk(t):
    """clk_or_zero (CPU column 50) set on an add: the CPU's 14-field send no longer meets the add chip's 13-field receive, which
    it does while that field is zero."""
    cpu = t.main[0]
    row = next(r for r in range(cpu.shape[0]) if cpu[r, 9] and cpu[r, 3] == 100)
    assert cpu[row, 50] == 0
    old = [int(cpu[row, 3])] + [int(x) for c in (32, 39, 46) for x in cpu[row, c:c + 4]]
    return _changed(t, 0, row, 50, 7), {(GENERAL, trim(old + [7]), 1), (GENERAL, trim(old), -1)}, (0, row)


TAMPERS = {"memory_value": _memory_value, "range_mult": _range_mult, "cpu_used": _cpu_used, "add_output": _add_output, "alu_clk": _alu_clk}


LT_FAMILY = {104, 115, 117, 118}


def _programs():
    """Every program of tests/golden/programs.json, generated straight-line programs of every ALU family, and the multi-chip mixes."""
    out = {name: (np.array(g["program"], dtype=np.int32), 0x1000, None) for name, g in GOLDEN.items()}
    for seed in (1, 2):
        prog, cells, fp = counted_program(seed, adds=12, subs=10, lts=12, bits=10, cycles=120, n_static=4 * seed)
        out["counted_%d" % seed] = (prog, fp, cells)
    out["generated_e"] = (*generated_program(1, "e", 300), None)
    out["mixed"] = (programs.mixed_program(20), 0x1000, None)
    out["config5"] = (programs.config5_program(10), 0x1000, None)
    prog, cells = programs.static_data_program()
    out["static_data"] = (prog, 0x1000, cells)
    return out


@pytest.mark.parametrize("name", sorted(_programs()))
def test_honest_witnesses_balance(built, oracle, name):
    import valida_b200 as vb

    prog, fp, cells = _programs()[name]
    t = vb.run_program(prog, initial_fp=fp, static_data=cells)
    events = bus_events(t.main)
    assert events and unbalanced(t.main) == []
    assert sums_cancel(oracle, t.main, t.preprocessed)


@pytest.mark.parametrize("regime", "abcde")
def test_generated_programs_agree_with_the_oracle(built, oracle, regime):
    """The generated loops of tests/generated_programs.py include lt-family operations with both operands immediate.  The witness
    of such an operation leaves the CPU's general-bus send and the lt chip's receive apart, as the oracle's witness does: its
    cumulative sums do not cancel either.  Whatever the program, the tuples are empty exactly when the oracle's sums cancel, and
    every unbalanced tuple is an lt-family operation on the general bus."""
    import valida_b200 as vb

    prog, fp = generated_program(1, regime, 300)
    t = vb.run_program(prog, initial_fp=fp)
    got = unbalanced(t.main)
    assert (got == []) == sums_cancel(oracle, t.main, t.preprocessed)
    assert all(bus == GENERAL and tup[0] in LT_FAMILY for bus, tup, _, _ in got), got
    assert sum(net for _, _, net, _ in got) == 0


def test_trailing_zero_fields_do_not_tell_tuples_apart(built):
    """The CPU's general-bus send has 14 fields, the ALU chips' receives 13; they meet because the 14th is zero."""
    t = fib_traces()
    sends = {(b, tup) for b, tup, chip, *_ in bus_events(t.main) if chip == 0 and b == GENERAL}
    receives = {(b, tup) for b, tup, chip, *_ in bus_events(t.main) if chip == 3 and b == GENERAL}
    assert receives and receives <= sends
    assert len(CHIPS[0][3][2]) == 14 and len(CHIPS[3][4][2]) == 13


@pytest.mark.parametrize("name", sorted(TAMPERS))
def test_tampered_witnesses_report_the_expected_tuples(built, oracle, name):
    t = fib_traces()
    mains, want, (chip, row) = TAMPERS[name](t)
    got = unbalanced(mains)
    assert {(bus, tup, net) for bus, tup, net, _ in got} == want
    # the changed row (or, when it no longer sends, the chip left unmatched) is an event of one of them, and each net is the sum
    # of its tuple's events
    assert any(e[0] == chip and row in (None, e[1]) for *_, evs in got for e in evs)
    for bus, tup, net, evs in got:
        assert signed(sum(m if s else P - m for _, _, _, m, s in evs) % P) == net
    assert not sums_cancel(oracle, mains, t.preprocessed)
