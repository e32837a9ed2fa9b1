"""Bus links of a machine witness in plain Python: for each item (chip, interaction, row), its tuple on its row, its own count, and every
event of the witness that carries the tuple; and the cycles behind a row, by breadth-first search in the graph whose nodes are
(chip, row) and whose edges join two nodes that each carry an event of the same tuple.  Built on bus_events of
test_bus_balance_restatement.py, so this is what vgpu_bus_links and cycles_of (tests/test_gpu_bus_links.py) are held to.

CPU only.  On the witnesses of fib_program and of the programs of tests/programs.py: every ALU row is sent its tuple, by a CPU row
whose opcode and operand words are that tuple unless the shift chip sends it; every memory operation links to the one CPU row whose
clk its tuple carries, and a static-initial row to none; every counted range byte reaches its cycles through add and sub rows only."""
import collections

import numpy as np
import pytest

import programs
from test_bus_balance_restatement import MAX_FIELDS, bus_events
from test_perm_trace_restatement import CHIPS, GENERAL, MEM, P, RANGE, SEND, apply

UNLISTED = 0xFFFFFFFFFFFFFFFF
ALU_CHIPS = (3, 4, 5, 6, 7, 8, 9, 10)


class Witness:
    """The events of 14 main traces grouped by (bus, padded tuple), each group ascending by (chip, row, interaction)."""

    def __init__(self, mains):
        self.mains = [np.array(m) for m in mains]
        self.groups = collections.defaultdict(list)
        for bus, tup, chip, row, m, mult, send in bus_events(self.mains):
            self.groups[(bus, tup)].append((chip, m, row, mult, send))
        for g in self.groups.values():
            g.sort(key=lambda e: (e[0], e[2], e[1]))

    def item(self, chip, m, row):
        """(bus, padded tuple, count) of interaction m of the chip on the row."""
        sign, bus, fields, count = CHIPS[chip][m]
        vals = self.mains[chip][row].tolist()
        return bus, tuple(apply(f, vals) % P for f in fields) + (0,) * (MAX_FIELDS - len(fields)), apply(count, vals) % P

    def links(self, items, cap):
        """vgpu_bus_links' output: per item (bus, padded fields, multiplicity, sends, receives, n_events, first_event), the listed
        events (chip, interaction, row, multiplicity, is_send) and the number of unlisted tuples."""
        its = [self.item(*x) for x in items]
        keys = sorted({(bus, tup) for bus, tup, _ in its})
        first, events = {}, []
        for k in keys:
            g = self.groups.get(k, [])
            if len(events) + len(g) > cap:
                break
            first[k] = len(events)
            events += g
        out = []
        for bus, tup, mult in its:
            g = self.groups.get((bus, tup), [])
            sends = sum(e[3] for e in g if e[4]) % P
            receives = sum(e[3] for e in g if not e[4]) % P
            out.append((bus, tup, mult, sends, receives, len(g), first.get((bus, tup), UNLISTED)))
        return out, events, len(keys) - len(first)

    def neighbours(self, chip, row):
        """The nodes that carry an event of a tuple the node carries an event of, the node itself left out."""
        out = set()
        for m in range(len(CHIPS[chip])):
            bus, tup, mult = self.item(chip, m, row)
            if mult:
                out |= {(c, r) for c, _, r, _, _ in self.groups[(bus, tup)]}
        out.discard((chip, row))
        return out

    def cycles(self, chip, row):
        """The CPU rows at the least distance from (chip, row), up to distance 2."""
        if chip == 0:
            return [row]
        near = self.neighbours(chip, row)
        hit = sorted(r for c, r in near if c == 0)
        if hit:
            return hit
        return sorted({r for node in near for c, r in self.neighbours(*node) if c == 0})


def witnesses():
    import valida_b200 as vb

    out = {"fib": vb.run_program(vb.fib_program(3), initial_fp=0x1000),
           "config5": vb.run_program(programs.config5_program(10), initial_fp=0x1000),
           "mixed": vb.run_program(programs.mixed_program(20), initial_fp=0x1000)}
    prog, cells = programs.static_data_program()
    out["static_data"] = vb.run_program(prog, initial_fp=0x1000, static_data=cells)
    return out


NAMES = ("config5", "fib", "mixed", "static_data")


@pytest.fixture(scope="module")
def wits(built):
    return {name: Witness(t.main) for name, t in witnesses().items()}


def _receive(chip):
    return next(m for m, (sign, bus, _, _) in enumerate(CHIPS[chip]) if sign != SEND and bus == GENERAL)


@pytest.mark.parametrize("name", NAMES)
def test_alu_rows_are_sent_by_their_cycle(wits, name):
    """Every ALU row with a non-zero count is sent its tuple: by a CPU row whose opcode and operand words are the tuple, or, for the
    multiplies and divides a shift makes, by the shift chip, whose row is then sent by a CPU row."""
    w = wits[name]
    cpu = w.mains[0]
    seen = 0
    for chip in ALU_CHIPS:
        m = _receive(chip)
        for row in range(w.mains[chip].shape[0]):
            bus, tup, mult = w.item(chip, m, row)
            if not mult:
                continue
            seen += 1
            senders = [e for e in w.groups[(bus, tup)] if e[4]]
            cpu_senders = [e for e in senders if e[0] == 0]
            assert senders, (chip, row)
            for c, _, r, _, _ in cpu_senders:
                assert int(cpu[r, 3]) == tup[0] and [int(x) for c0 in (32, 39, 46) for x in cpu[r, c0:c0 + 4]] == list(tup[1:13])
            if cpu_senders:
                assert w.cycles(chip, row) == sorted(r for _, _, r, _, _ in cpu_senders)
            else:
                assert {e[0] for e in senders} == {7} and w.cycles(chip, row)
    assert seen or name == "static_data"


@pytest.mark.parametrize("name", NAMES)
def test_memory_rows_link_to_the_cycle_of_their_clk(wits, name):
    w = wits[name]
    mem, cpu = w.mains[2], w.mains[0]
    static = 0
    for row in range(mem.shape[0]):
        if not (int(mem[row, 7]) + int(mem[row, 8])) % P:
            continue
        if mem[row, 6]:
            static += 1
            assert w.cycles(2, row) == [], row
            continue
        bus, tup, _ = w.item(2, 0, row)
        assert bus == MEM and tup[1] == int(mem[row, 5])
        assert w.cycles(2, row) == [r for r in range(cpu.shape[0]) if int(cpu[r, 0]) == tup[1]], row
    assert static > 0 or name != "static_data"


@pytest.mark.parametrize("name", NAMES)
def test_range_rows_reach_cycles_through_add_and_sub(wits, name):
    w = wits[name]
    rng = w.mains[12]
    counted = 0
    for row in range(rng.shape[0]):
        if not rng[row, 0]:
            continue
        counted += 1
        near = w.neighbours(12, row)
        assert near and {c for c, _ in near} <= {3, 4}, row
        want = sorted({r for node in near for c, r in w.neighbours(*node) if c == 0})
        assert want and w.cycles(12, row) == want
    assert counted or name == "static_data"


def test_links_follow_the_definition(wits):
    """Shared tuples share one range, tuples are listed ascending while they fit, and the totals do not depend on cap."""
    w = wits["fib"]
    items = [(3, 4, 1), (0, 3, 0), (3, 4, 1), (12, 0, 5), (2, 0, 0), (3, 0, w.mains[3].shape[0] - 1)]
    full, events, unlisted = w.links(items, 1 << 30)
    assert unlisted == 0 and full[0] == full[2]
    by_key = {(x[0], x[1]): x for x in full}
    keys = sorted(by_key)
    assert [by_key[k][6] for k in keys] == sorted(by_key[k][6] for k in keys)
    assert sum(x[5] for x in by_key.values()) == len(events)
    assert all(events[x[6]:x[6] + x[5]] == w.groups.get(k, []) for k, x in by_key.items())
    for cap in range(len(events) + 1):
        got, ev, un = w.links(items, cap)
        assert [x[:6] for x in got] == [x[:6] for x in full]
        assert ev == events[:len(ev)]
        listed = {(x[0], x[1]) for x in got if x[6] != UNLISTED}
        assert listed == set(keys[:len(keys) - un]) and len(ev) == sum(len(w.groups.get(k, [])) for k in listed) <= cap
