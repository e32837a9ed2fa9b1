"""The host witness builder (csrc/host/tracegen.cc) against the plain restatement (tracegen_restated.py) on seeded generated programs
(generated_programs.py) in every address regime, and at frame pointers, addresses and static cells at or above p, where both must
reduce mod p as the reference's from_canonical_u32 does.  Every word of every host trace must be below p.  No GPU."""
import numpy as np
import pytest

from generated_programs import REGIMES, counted_program, generated_program, with_dead_rows
from tracegen_restated import P, Vm, all_traces, assert_canonical, assert_traces_equal


def check(program, fp, static_data=None):
    import valida_b200 as vb

    got = vb.run_program(program, initial_fp=fp, static_data=static_data)
    vm = Vm(program, fp, static_data).run()
    assert_canonical(got.main + got.preprocessed, "host")
    assert_traces_equal(got.main, got.preprocessed, *all_traces(vm), "host", "restatement")
    return vm, got


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_generated_program_traces(built, regime, seed):
    prog, fp = generated_program(seed, regime, cycles=[300, 1500, 4000, 3000][seed - 1])
    vm, _ = check(prog, fp)
    assert vm.clock <= 1 << 12
    addrs = {a for ops in vm.mem_ops.values() for _, a, _ in ops}
    var = np.bitwise_or.reduce(list(addrs)) ^ np.bitwise_and.reduce(list(addrs))
    if regime == "b":
        assert var >> 24 and not var & 0xFFFFFF, hex(var)              # only the top byte varies
    elif regime == "c":
        assert var == 0x180, hex(var)                                  # only bits 7 and 8 vary
    elif regime == "a":
        assert all((var >> s) & 255 for s in (0, 8, 16, 24)) and max(addrs) >= 0xFFFF0000 and any(a >= P for a in addrs)
    iters = max(c for pc, c in enumerate(vm.counts) if pc != vm.pc)   # loop iterations (the final pc's count includes the padding)
    pointers = len(addrs) - {"a": 12 + 7, "b": 12, "c": 4, "d": 12, "e": 13}[regime]
    if regime in "bd":                                                 # 64 top bytes, 32 low bits: revisited
        assert pointers >= min({"b": 64, "d": 32}[regime], iters) // 3, (pointers, iters)
    elif regime in "ae":
        assert pointers >= iters * 3 // 4, (pointers, iters)           # about one new pointer per iteration
    assert vm.registers[-1][1] != fp                                   # stops in another frame


@pytest.mark.parametrize("fp", [0x78000000, 0x80000000, 0xFFFFF000, P, P - 4])
def test_fibonacci_frame_at_or_above_p(built, fp):
    import valida_b200 as vb

    vm, got = check(vb.fib_program(25), fp)
    assert vm.clock == 192 and got.main[0][0, 2] == fp % P
    assert got.main[0][-1, 2] == fp % P                                # a STOP padding row: the last fp, reduced


def test_static_cells_at_or_above_p(built):
    prog, static, fp = counted_program(7, adds=5, lts=5, bits=5, cycles=200, n_static=37, fp=0xFFFFFF00)
    assert any(a >= P for a in static) and any(a < P for a in static)
    check(prog, fp, static)


def test_counted_program_counts(built):
    # the counts counted_program promises, which the GPU padding tests rely on
    vm, _ = check(*counted_program(3, adds=17, subs=1, lts=0, bits=33, cycles=1 << 9)[::2])
    assert (vm.clock, len(vm.adds), len(vm.subs), len(vm.lts), len(vm.bits)) == (1 << 9, 17, 1, 0, 33)
    prog, static, fp = counted_program(4, lts=5, mem=(1 << 10) + 1, n_static=20)
    vm, _ = check(prog, fp, static)
    assert len(static) + sum(len(v) for v in vm.mem_ops.values()) == (1 << 10) + 21


def test_rows_that_never_run_with_opcodes_at_or_above_p(built):
    # the program chip's preprocessed trace holds every row of the program, executed or not (machine/src/program.rs:44)
    prog, fp = generated_program(5, "a", 500)
    vm, got = check(with_dead_rows(prog), fp)
    assert got.preprocessed[0][len(prog), 1] == 0 and got.preprocessed[0][len(prog) + 2, 1] == 0xFFFFFFFF % P
