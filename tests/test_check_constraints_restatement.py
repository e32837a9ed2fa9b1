"""check_constraints (machine/src/check_constraints.rs:14-84; the reference's debug-build witness check) restated per row in plain
Python: the AIRS of test_quotient_restatement.py with the debug selectors is_first_row = [i == 0], is_last_row = [i == h-1],
is_transition = 1 - is_last_row, then the LogUp constraints of eval_permutation_constraints (machine/src/chip.rs:210-289) on the
natural rows i and (i + 1) mod h, the cumulative sum read from the permutation trace's last row and last column.  Constraints are
numbered in eval order: the chip's assertions, one per interaction, then the transition, first-row and last-row constraints.

It is compared with the oracle's check (oracle/machine.h) on random traces with honest permutation traces, on honest Fibonacci
traces with one permutation-trace word changed, and on the two edge programs the CPU AIR rejects.  The device sweep
(valida_b200/csrc/check.cu, tests/test_gpu_check_constraints.py) is held to both.  CPU only."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import programs
from test_perm_trace_restatement import CHIPS, P, SEND, apply, e_add, e_from, e_mul, e_sub
from test_quotient_restatement import AIRS, e_scale

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
PREP_CHIPS = {1: 0, 12: 1}          # chip -> index of its preprocessed trace (program, range)


def check_py(chip, main, perm, ch15, rows=None):
    """Per-row check of one chip: returns ((row, constraint) of the first failure or None, number of failing rows).
    rows: the rows to check (all by default); they read rows i and (i + 1) mod h of main and perm."""
    h, inter = main.shape[0], CHIPS[chip]
    k = len(inter)
    r1, r2 = [int(x) for x in ch15[5:10]], [int(x) for x in ch15[10:15]]
    alphas_global, acc = [], e_from(1)
    for _ in range(4):
        acc = e_mul(acc, r1)
        alphas_global.append(acc)
    cumsum = [int(v) for v in perm[h - 1, 5 * k:5 * k + 5]]
    first, failing = None, 0
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
        bad = next((c for c, v in enumerate(cons) if any(v)), None)
        if bad is not None:
            failing += 1
            if first is None:
                first = (i, bad)
    return first, failing


def as_oracle_code(first):
    """(row, constraint) / None in the oracle's encoding: row * 4096 + constraint / -1."""
    return -1 if first is None else first[0] * 4096 + first[1]


class OracleCheck:
    """orc_check_constraints of tests/c/oracle_check.cc: the oracle's check_constraints on a given permutation trace."""

    def __init__(self, path):
        self.L = C.CDLL(path)
        self.L.orc_check_constraints.restype = C.c_int64

    def check_constraints(self, chip, main, prep, perm_flat, challenges15):
        u32p = C.POINTER(C.c_uint32)
        arr = lambda a: np.ascontiguousarray(a, dtype=np.uint32)
        main, perm, ch = arr(main), arr(perm_flat), arr(challenges15)
        prep = arr(prep) if prep is not None else None
        return int(self.L.orc_check_constraints(C.c_uint32(chip), main.ctypes.data_as(u32p), C.c_uint64(main.shape[0]),
                                                prep.ctypes.data_as(u32p) if prep is not None else None, perm.ctypes.data_as(u32p),
                                                ch.ctypes.data_as(u32p)))


_oracle_check = None


@pytest.fixture(scope="session")
def oracle_check(built, tmp_path_factory):
    global _oracle_check
    if _oracle_check is None:
        out = str(tmp_path_factory.mktemp("oracle_check") / "liboracle_check.so")
        subprocess.run([CXX, "-O2", "-std=c++17", "-fPIC", "-fopenmp", "-shared", "-I", os.path.join(ROOT, "oracle"),
                        os.path.join(ROOT, "tests", "c", "oracle_check.cc"), "-o", out], check=True)
        _oracle_check = OracleCheck(out)
    return _oracle_check


def random_case(oracle, chip, h, seed):
    """Random main (and preprocessed) trace of one chip with its honest permutation trace, and the challenges."""
    rng = np.random.default_rng(seed)
    main = rng.integers(0, P, (h, oracle.chip_width(chip)), dtype=np.uint32)
    pw = oracle.chip_prep_width(chip)
    prep = rng.integers(0, P, (h, pw), dtype=np.uint32) if pw else None
    ch = rng.integers(0, P, 15, dtype=np.uint32)
    perm, _ = oracle.perm_trace(chip, main, prep, ch)
    return main, prep, perm, ch


def fib_traces():
    import valida_b200 as vb

    return vb.run_program(vb.fib_program(3), initial_fp=0x1000)


def tamper_cases(h, width):
    """(row, column) of the permutation-trace words changed: row 0, a middle row and the last row, and the cumulative-sum cell."""
    cases = [(0, 1 % width), (h // 2, (h // 2 + 3) % width), (h - 1, 0), (h - 1, width - 1)]
    return list(dict.fromkeys(cases))


def tampered(perm, row, col):
    p = perm.copy()
    p[row, col] = (int(p[row, col]) + 1) % P
    return p


@pytest.mark.parametrize("h", [1, 2, 16])
@pytest.mark.parametrize("chip", sorted(CHIPS))
def test_checker_matches_oracle_on_random_traces(oracle, oracle_check, chip, h):
    main, prep, perm, ch = random_case(oracle, chip, h, 7000 + 16 * chip + h)
    first, failing = check_py(chip, main, perm, ch)
    assert as_oracle_code(first) == oracle_check.check_constraints(chip, main, prep, perm, ch)
    if AIRS[chip] is None:
        assert first is None and failing == 0        # an honest permutation trace satisfies the LogUp constraints


@pytest.mark.parametrize("chip", sorted(CHIPS))
def test_checker_matches_oracle_on_tampered_permutation_traces(oracle, oracle_check, chip):
    t = fib_traces()
    main = t.main[chip]
    prep = t.preprocessed[PREP_CHIPS[chip]] if chip in PREP_CHIPS else None
    ch = np.random.default_rng(50 + chip).integers(0, P, 15, dtype=np.uint32)
    perm, _ = oracle.perm_trace(chip, main, prep, ch)
    assert check_py(chip, main, perm, ch) == (None, 0)
    assert oracle_check.check_constraints(chip, main, prep, perm, ch) == -1
    for row, col in tamper_cases(main.shape[0], perm.shape[1]):
        bad = tampered(perm, row, col)
        first, failing = check_py(chip, main, bad, ch)
        assert first is not None and failing >= 1, (row, col)
        assert as_oracle_code(first) == oracle_check.check_constraints(chip, main, prep, bad, ch), (row, col)


@pytest.mark.parametrize("name", ["lt_edges", "loads_stores"])
def test_checker_matches_the_oracle_prover_on_the_rejected_edge_programs(oracle, name):
    import valida_b200 as vb

    prog = programs.lt_edge_operands_program() if name == "lt_edges" else programs.loads_stores_edge_program()
    t = vb.run_program(prog, initial_fp=0x1000)
    ref = oracle.prove(t.main, t.preprocessed, debug_checks=True)
    ch = ref.transcript()["perm_challenges"]
    got = [as_oracle_code(check_py(chip, t.main[chip], ref.perm_trace(chip), ch)[0]) for chip in range(14)]
    assert got == ref.constraint_failures()
    assert got[0] >= 0
