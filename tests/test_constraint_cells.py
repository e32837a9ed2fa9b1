"""The constraint catalogue (vgpu_chip_constraint_cells, vgpu_chip_column_name; valida_b200/csrc/explain.cu) held to an independent
text: the plain-Python AIRs of test_quotient_restatement.py and the LogUp constraints of test_check_constraints_restatement.py,
evaluated here per row into EVERY constraint's value.  On random traces of all 14 chips, at row 0, a middle row and row h-1, each cell
of the main, preprocessed and permutation traces on the local and the next row is changed to a random value, one at a time:
  - a cell outside constraint c's list never changes c's value;
  - every listed cell changes it on at least one of those rows (except the LogUp last-row constraint, which compares the running sum
    on row h-1 with itself, the cumulative sum the check reads from that same cell).
Also: labels cover every index in eval order, the AIR sections come in eval order, and every trace's columns are named, uniquely.
CPU only (the catalogue is host code)."""
import ctypes as C

import numpy as np
import pytest

from test_perm_trace_restatement import CHIPS, P, SEND, apply, e_add, e_from, e_mul, e_sub
from test_quotient_restatement import AIRS, e_scale

H = 8
ROWS = (0, 3, H - 1)

# the blocks of each chip's eval, in eval order (empty: no Air::eval assertions)
SECTIONS = {
    0: ["CpuChip::eval_pc", "CpuChip::eval_fp", "CpuChip::eval_equality", "CpuChip::eval_memory_channels", "CpuChip::eval clock",
        "CpuChip::eval immediates", "CpuChip::eval stop"],
    1: [], 2: [], 6: [], 12: [],
    3: ["Add32Chip::eval limbs", "Add32Chip::eval carries"],
    4: ["Sub32Chip::eval"],
    5: ["Mul32Chip::eval congruences", "Mul32Chip::eval counter"],
    7: ["Shift32Chip::eval bits_2", "Shift32Chip::eval power_of_two", "Shift32Chip::eval opcode flags"],
    8: ["Lt32Chip::eval byte_flag", "Lt32Chip::eval top bits", "Lt32Chip::eval different_signs", "Lt32Chip::eval opcode flags",
        "Lt32Chip::eval output", "Lt32Chip::eval bits booleans"],
    9: ["Com32Chip::eval"],
    10: ["Bitwise32Chip::eval bytes", "Bitwise32Chip::eval opcode flags"],
    11: ["OutputChip::eval range check", "OutputChip::eval bus opcode"],
    13: ["StaticDataChip::eval_main"],
}


def _desc(chip):
    import valida_b200 as vb
    from valida_b200.api import _ChipDesc

    return C.cast(vb.lib().vgpu_basic_machine_chip(chip), C.POINTER(_ChipDesc)).contents


def all_constraints(chip, main, prep, perm, ch15, i):
    """Every constraint's value (5 limbs) on row i of one chip, in eval order: the check of check_py, without stopping at the
    first failure.  prep is not read: no BasicMachine AIR or interaction reads a preprocessed column."""
    h, inter = main.shape[0], CHIPS[chip]
    k = len(inter)
    r1, r2 = [int(x) for x in ch15[5:10]], [int(x) for x in ch15[10:15]]
    alphas_global, acc = [], e_from(1)
    for _ in range(4):
        acc = e_mul(acc, r1)
        alphas_global.append(acc)
    cumsum = [int(v) for v in perm[h - 1, 5 * k:5 * k + 5]]
    j = (i + 1) % h
    loc, nxt = [int(v) for v in main[i]], [int(v) for v in main[j]]
    pl = [[int(v) for v in perm[i, 5 * m:5 * m + 5]] for m in range(k + 1)]
    pn = [[int(v) for v in perm[j, 5 * m:5 * m + 5]] for m in range(k + 1)]
    last = 1 if i == h - 1 else 0
    sel = {"first": 1 if i == 0 else 0, "last": last, "transition": 1 - last}
    cons = [e_from(c) for c in AIRS[chip](loc, nxt, sel)] if AIRS[chip] else []
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
    cons.append(e_scale(e_sub(e_sub(pn[k], pl[k]), rhs), sel["transition"]))
    cons.append(e_scale(e_sub(pl[k], phi0), sel["first"]))
    cons.append(e_scale(e_sub(pl[k], cumsum), sel["last"]))
    return cons


def _random_traces(chip, seed):
    d = _desc(chip)
    rng = np.random.default_rng(seed)
    main = rng.integers(0, P, (H, d.width), dtype=np.uint32)
    prep = rng.integers(0, P, (H, d.preprocessed_width), dtype=np.uint32)
    perm = rng.integers(0, P, (H, 5 * (d.n_interactions + 1)), dtype=np.uint32)
    return main, prep, perm, rng.integers(0, P, 15, dtype=np.uint32), rng


@pytest.mark.parametrize("chip", range(14))
def test_listed_cells_are_exactly_the_cells_a_constraint_reads(built, chip):
    import valida_b200 as vb

    main, prep, perm, ch, rng = _random_traces(chip, 9100 + chip)
    air, total = vb.constraint_count(chip)
    listed = [{(c.trace, c.next, c.column) for c in vb.constraint_cells(chip, c)[1]} for c in range(total)]
    mats = {vb.TRACE_MAIN: main, vb.TRACE_PREPROCESSED: prep, vb.TRACE_PERMUTATION: perm}
    moved = [set() for _ in range(total)]
    for i in ROWS:
        base = all_constraints(chip, main, prep, perm, ch, i)
        assert len(base) == total
        for trace, m in mats.items():
            for nxt in (False, True):
                for col in range(m.shape[1]):
                    row = (i + 1) % H if nxt else i
                    old = m[row, col]
                    m[row, col] = (int(old) + 1 + int(rng.integers(0, P - 1))) % P
                    now = all_constraints(chip, main, prep, perm, ch, i)
                    m[row, col] = old
                    for c in range(total):
                        if now[c] != base[c]:
                            assert (trace, nxt, col) in listed[c], (chip, c, i, trace, nxt, col)
                            moved[c].add((trace, nxt, col))
    for c in range(total):
        if c == total - 1:           # LogUp last row: the running sum on row h-1 against itself
            assert moved[c] == set() and listed[c] == {(vb.TRACE_PERMUTATION, False, 5 * (total - air - 3) + l) for l in range(5)}
        else:
            assert moved[c] == listed[c], (chip, c, listed[c] - moved[c])


@pytest.mark.parametrize("chip", range(14))
def test_labels_follow_eval_order(built, chip):
    import valida_b200 as vb

    air, total = vb.constraint_count(chip)
    labels = [vb.constraint_cells(chip, c)[0] for c in range(total)]
    assert labels[air:] == [vb.constraint_label(chip, c) for c in range(air, total)]
    runs = [s for j, s in enumerate(labels[:air]) if j == 0 or labels[j - 1] != s]
    assert runs == SECTIONS[chip]                     # each block once, contiguous, in eval order
    assert air == (len(AIRS[chip]([0] * 80, [0] * 80, {"first": 0, "last": 0, "transition": 1})) if AIRS[chip] else 0)
    for bad in (-1, total):
        with pytest.raises(vb.VgpuError):
            vb.constraint_cells(chip, bad)
    for c in range(total):                            # ascending (trace, next, column), named
        cells = vb.constraint_cells(chip, c)[1]
        assert [(x.trace, x.next, x.column) for x in cells] == sorted({(x.trace, x.next, x.column) for x in cells})
        assert all(x.name == vb.column_name(chip, x.trace, x.column) is not None for x in cells)


@pytest.mark.parametrize("chip", range(14))
def test_every_column_is_named_once(built, chip):
    import valida_b200 as vb

    d = _desc(chip)
    assert d.n_interactions == len(CHIPS[chip])
    for trace, w in ((vb.TRACE_MAIN, d.width), (vb.TRACE_PREPROCESSED, d.preprocessed_width), (vb.TRACE_PERMUTATION, 5 * (d.n_interactions + 1))):
        names = [vb.column_name(chip, trace, c) for c in range(w)]
        assert all(names) and len(set(names)) == w, (trace, names)
        assert vb.column_name(chip, trace, w) is None
    assert vb.column_name(chip, 3, 0) is None
    k = d.n_interactions
    assert vb.column_name(chip, vb.TRACE_PERMUTATION, 5 * k + 2) == "running_sum[2]"
    if k:
        assert vb.column_name(chip, vb.TRACE_PERMUTATION, 5 * (k - 1) + 4) == "interactions[%d].reciprocal[4]" % (k - 1)


def test_column_names_follow_the_layout(built):
    import valida_b200 as vb

    assert [vb.column_name(0, vb.TRACE_MAIN, c) for c in (0, 1, 2, 3, 4, 9, 25, 26, 29, 38, 41, 50)] == [
        "clk", "pc", "fp", "instruction.opcode", "instruction.operands.a", "opcode_flags.is_bus_op", "opcode_flags.is_loadfp", "diff",
        "mem_channels[0].used", "mem_channels[1].addr", "mem_channels[1].value[2]", "chip_channel.clk_or_zero"]
    assert [vb.column_name(1, vb.TRACE_PREPROCESSED, c) for c in range(7)] == [
        "pc", "opcode", "operands.a", "operands.b", "operands.c", "operands.d", "operands.e"]
    assert vb.column_name(10, vb.TRACE_MAIN, 8 + 8 * 2 + 5) == "bits_1[2][5]"
    assert vb.column_name(8, vb.TRACE_MAIN, 44) == "different_signs"
    assert [vb.column_name(12, t, 0) for t in (vb.TRACE_MAIN, vb.TRACE_PREPROCESSED)] == ["mult", "counter"]
