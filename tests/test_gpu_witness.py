"""Witness generation on the device (SURVEY.md 8(f)1): the traces vgpu_witness_device builds from the interpreter's logs equal
the host builder's word for word — every chip, every program family the reference can prove — and proving from them gives the
same proof bytes."""
import json
import os

import numpy as np
import pytest

from programs import (config5_program, loads_stores_edge_program, lt_edge_operands_program, mixed_program,
                      single_address_program, static_data_program)

pytestmark = pytest.mark.gpu
GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "programs.json")))


def _check(ctx, program, static_data=None):
    import valida_b200 as vb

    log = vb.run_program_log(program, initial_fp=0x1000, static_data=static_data)
    host = log.traces()
    again = vb.run_program(program, initial_fp=0x1000, static_data=static_data)      # the one-call host path
    dm, dp = log.witness_device(ctx)
    for i in range(14):
        assert np.array_equal(host.main[i], again.main[i]), vb.MachineTraces.CHIPS[i]
        assert dm[i].shape == host.main[i].shape, vb.MachineTraces.CHIPS[i]
        assert np.array_equal(dm[i].download(), host.main[i]), vb.MachineTraces.CHIPS[i]
    for i in range(2):
        assert np.array_equal(dp[i].download(), host.preprocessed[i])
    return log, host, dm, dp


@pytest.mark.parametrize("n", [25, 0, 582])
def test_fibonacci_witness(ctx, n):
    import valida_b200 as vb

    log, host, _, _ = _check(ctx, vb.fib_program(n))
    if n == 25:
        assert (log.clock, log.mem_ops, log.add_ops) == (192, 401, 105)          # basic/tests/test_prover.rs:479-482


@pytest.mark.parametrize("name", ["left_imm_ops_program", "signed_inequality_program", "loadfp_program"])
def test_reference_test_programs_witness(ctx, name):
    _check(ctx, np.array(GOLDEN[name]["program"], dtype=np.int32))


def test_multichip_and_static_data_witness(ctx):
    _check(ctx, mixed_program(300))
    _check(ctx, config5_program(700))
    prog, cells = static_data_program()
    _check(ctx, prog, static_data=cells)


def test_memory_log_sort_with_wide_addresses(ctx):
    """load32 / store32 through pointers spread the addresses over several radix digits (every digit pass of the device sort runs)."""
    B = 24
    prog = np.array([
        [7, -4, 0x00, 0x12, 0x34, 0x50],        # p = 0x00123450
        [7, -8, 0, 0, 0, 0],                     # i = 0
        [2, 0, -4, -8, 0, 0],                    # store32: mem[p] = i            <- loop
        [1, -12, 0, -4, 0, 0],                   # load32 : t = mem[p]
        [100, -4, -4, 0x01010104, 0, 1],         # p += 0x01010104 (every byte of the address moves)
        [100, -8, -8, 1, 0, 1],                  # i += 1
        [6, 2 * B, -8, 40, 0, 1],                # bne loop, i, 40
        [8, 0, 0, 0, 0, 0],
    ], dtype=np.int32)
    _check(ctx, prog)


def test_edge_operand_programs_witness(ctx):
    """The programs built to reach the builders' edges: equal operands and a difference in the top byte only (the device's
    lt_rows_kernel finds the first differing byte on its own), sign boundaries, immediates on both sides, negative immediates,
    borrows, jal / jalv frame changes (the device's CPU diff_inv is a per-row Fermat inverse, the host's a table)."""
    _check(ctx, lt_edge_operands_program())
    _check(ctx, loads_stores_edge_program())


def test_degenerate_memory_logs_witness(ctx):
    """A lone STOP (an empty memory log) and a log whose every operation has the same address (the device radix sort has
    nothing to order)."""
    _check(ctx, np.array([[8, 0, 0, 0, 0, 0]], dtype=np.int32))
    _check(ctx, single_address_program(1))
    _check(ctx, single_address_program(40))


def test_prove_from_device_witness(ctx, oracle):
    import valida_b200 as vb

    cfg = vb.StarkConfig(ctx, oracle.rc480)
    log, host, dm, dp = _check(ctx, vb.fib_program(582))
    assert vb.prove_machine(cfg, host, device_resident=(dm, dp)) == vb.prove_machine(cfg, host)


def test_split_proof_from_device_witness(ctx, oracle):
    """Every rank expands the logs into ITS rows of the tall chips and proves: the single-GPU bytes."""
    import torch
    import valida_b200 as vb

    prog = vb.fib_program(((1 << 15) - 17) // 7)
    log = vb.run_program_log(prog)
    host = log.traces()
    single = vb.prove_machine(vb.StarkConfig(ctx, oracle.rc480), host)
    k = torch.cuda.device_count()
    ctxs = [vb.Context(i % k) for i in range(4)]
    try:
        vb.comm_init_local(ctxs)
        cfgs = [vb.StarkConfig(c, oracle.rc480) for c in ctxs]

        def go(r, c):
            dm, dp = log.witness_device(c)
            assert dm[0].local_rows() == (r * (1 << 13), 1 << 13) and dm[0].shape == (1 << 15, 51)
            r0, n = dm[2].local_rows()
            assert np.array_equal(dm[2].download()[r0:r0 + n], host.main[2][r0:r0 + n])
            return vb.prove_machine(cfgs[r], host, device_resident=(dm, dp))

        assert all(p == single for p in vb.run_ranks(go, ctxs))
    finally:
        for c in ctxs:
            c.close()
