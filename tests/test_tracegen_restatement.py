"""A second reading, in plain Python and written from the Rust text, of the INPUT side of the proving path: `Machine::run`
(basic/src/lib.rs:127-145, 1063-1188) and `Chip::generate_trace` of the chips a Fibonacci-class program reaches —

    instruction semantics     cpu/src/lib.rs:440-872 (load32, store32, jal, jalv, beq, bne, imm32, stop, loadfp),
                              alu_u32/src/add/mod.rs:138-169, alu_u32/src/sub/mod.rs:126-166
    CPU rows                  cpu/src/lib.rs:79-97 (generate_trace), 163-236 (op_to_row), 244-284 (memory channels),
                              286-321 (word diffs), 323-362 (STOP padding), 364-381 (immediates); columns cpu/src/columns.rs:8-75
    memory rows               memory/src/lib.rs:143-194, 237-263; columns memory/src/columns.rs:8-41
    add / sub rows            alu_u32/src/add/mod.rs:38-129, alu_u32/src/sub/mod.rs:90-117
    lt family                 alu_u32/src/lt/mod.rs:87-165 (rows), 167-216 (operands incl. LEFT immediates), 232-309; Word ordering machine/src/core.rs:321-330
    and / or / xor            alu_u32/src/bitwise/mod.rs:84-131 (rows), 140-254
    mul floor                 alu_u32/src/mul/mod.rs:38-64 (2^10 counter rows)
    static data               static_data/src/lib.rs:26-33 (initialize_memory), 59-79 (rows); memory/src/lib.rs:132-135, 163-169, 265-283
    range / program           range/src/lib.rs:32-72, range/src/stark.rs:22-25, program/src/lib.rs:38-48, 73-80, program/src/stark.rs:22-40

— compared WORD FOR WORD with the product's host witness generator (valida_b200/csrc/host/tracegen.cc via vgpu_machine_run).
The trace digests of tests/golden/trace_hashes.json pin the generator against itself; the restatement (tests/tracegen_restated.py,
data structures of its own: a dict of cells, per-clock operation lists, Python's stable sort) is the independent text, like
test_perm_trace_restatement.py and test_quotient_restatement.py are for the LogUp and quotient code.  No GPU."""
import numpy as np
import pytest

from programs import loads_stores_edge_program, lt_edge_operands_program, single_address_program
from tracegen_restated import ADD32, IMM32, LOAD32, LOADFP, M32, STOP, STORE32, Vm, all_traces, assert_traces_equal, u32, word


def check(program, fp=0x1000, static_data=None):
    import valida_b200 as vb

    got = vb.run_program(program, initial_fp=fp, static_data=static_data)
    vm = Vm(program, fp, static_data).run()
    assert_traces_equal(got.main, got.preprocessed, *all_traces(vm), "generator", "restatement")
    return vm, got


@pytest.mark.parametrize("n", [0, 1, 3, 25, 582, 2339, 9359])       # 9359: 2^16 CPU rows, 2^18 memory rows — the sizes at which the generator uses all threads
def test_fibonacci_traces_word_for_word(built, n):
    import valida_b200 as vb

    vm, got = check(vb.fib_program(n))
    if n == 25:                                                        # the reference test's own figures (basic/tests/test_prover.rs:479-486)
        assert (vm.clock, sum(len(v) for v in vm.mem_ops.values()), len(vm.adds)) == (192, 401, 105)
        assert vm.cells[(0x1000 + 4) & M32] == (0, 1, 37, 17)          # Word([0, 1, 37, 17]) = fib(25) = 75025


def _ins(op, a=0, b=0, c=0, d=0, e=0):
    return [op, a, b, c, d, e]


def test_loads_stores_loadfp_sub_and_signed_immediates(built):
    # every instruction of the restated subset that the Fibonacci program does not reach (tests/programs.py; the device witness
    # and the GPU proof are checked on the same program in test_gpu_witness.py / test_gpu_prove.py)
    vm, got = check(loads_stores_edge_program())
    assert vm.cells[(0x1000 - 36) & M32] == word(254) and vm.pc == 13 and vm.fp == 0x1000
    assert len(vm.subs) == 2 and len(vm.adds) == 1


def test_degenerate_memory_logs(built):
    # a lone STOP (no memory operation at all) and a log whose every operation is at one address
    vm, got = check(np.array([_ins(STOP)], dtype=np.int32))
    assert vm.clock == 1 and not vm.mem_ops
    vm, got = check(single_address_program(5))
    assert {addr for ops in vm.mem_ops.values() for _, addr, _ in ops} == {(0x1000 - 4) & M32}


def test_the_references_other_test_programs_and_the_multi_chip_mixes(built):
    # basic/tests/test_prover.rs:490-625 (left immediates, signed inequalities, loadfp) as recorded in tests/golden/programs.json,
    # and the synthetic programs of tests/programs.py (add, sub, lt family incl. left immediates, and / or / xor, bne back-edge)
    import json
    import os

    from programs import config5_program, mixed_program

    golden = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "programs.json")))
    for name in ("left_imm_ops_program", "signed_inequality_program", "loadfp_program"):
        vm, _ = check(np.array(golden[name]["program"], dtype=np.int32))
        for addr, value in golden[name]["expected_cells"]:                 # the reference tests' own assertions on mem().cells
            assert u32(vm.cells[addr & M32]) == value & M32, (name, hex(addr))
    vm, _ = check(mixed_program(37))
    assert len(vm.lts) == 4 * 37 and len(vm.adds) == 3 * 37
    vm, _ = check(config5_program(40))
    assert len(vm.bits) == 6 * 40 and len(vm.subs) == 2 * 40 and len(vm.lts) == 4 * 40
    big = ((1 << 16) - 8) // 15                                                # 2^16 CPU rows: every chip's multi-threaded row fill
    vm, _ = check(config5_program(big))
    assert vm.clock == 3 + 15 * big + 1 and len(vm.bits) == 6 * big


def test_lt_family_edge_operands(built):
    # equal operands (no differing byte: flags, bits and diff_inv stay zero), operands that differ in the TOP byte only, sign
    # boundaries, both immediates at once (the recorded immediate is the right one, written through the LEFT-immediate path)
    vm, _ = check(lt_edge_operands_program())
    assert u32(vm.cells[(0x1000 - 100) & M32]) == 1 and u32(vm.cells[(0x1000 - 104) & M32]) == 1


def test_static_data_program(built):
    # prove_static_data (basic/tests/test_static_data.rs:30-113): two static cells, one of them loaded through a pointer
    from programs import static_data_program

    prog, cells = static_data_program()
    vm, got = check(prog, static_data=cells)
    assert vm.clock == 4 and u32(vm.cells[(0x1000 - 4) & M32]) == 0x25
    # more cells than a power of two, out of address order on the way in, one of them overwritten by the program later
    prog2 = np.array([_ins(IMM32, 0, 0, 0, 0, 0x20), _ins(LOAD32, -4, 0, 0), _ins(ADD32, -8, -4, 5, 0, 1), _ins(LOADFP, -12, -8),
                      _ins(IMM32, -16, 0, 0, 0, 0x18), _ins(STORE32, 0, -16, -8), _ins(STOP)], dtype=np.int32)
    vm, got = check(prog2, static_data={0x20: 1000, 0x10: 7, 0x18: 9})
    assert u32(vm.cells[0x18]) == 1005 and got.main[13].shape == (4, 6) and got.main[2][:3, 6].tolist() == [1, 1, 1]
