"""valida_b200 — GPU-native (H100, sm_90a) STARK prover backend for Valida's Machine::prove() hot path.

Host-side mirror of the reference's prover-facing interface (StarkConfig / UnivariatePcsWithLde /
Machine::prove) over the C ABI in include/valida_b200.h.  There is no CPU fallback: constructing a
Context without a CUDA device raises.
"""
from .api import (  # noqa: F401
    BABYBEAR_P,
    MERKLE_KECCAK256,
    MERKLE_POSEIDON16,
    REPR_CANONICAL,
    REPR_MONTY_R32,
    Context,
    DeviceMatrix,
    ProverData,
    Radix2Dft,
    TwoAdicFriPcs,
    MachineTraces,
    VgpuError,
    StarkConfig,
    prove_machine,
    verify_machine,
    VerificationError,
    last_prove_phases,
    fib_program,
    generate_permutation_trace,
    quotient,
    check_constraints,
    check_constraints_local,
    check_witness,
    lib,
    lib_path,
    run_program,
    run_program_log,
    VmLog,
    comm_unique_id,
    comm_init_local,
    run_ranks,
    shard_range,
    split_column_plan,
    tree_share,
    row_share,
)
