"""GPU Machine::prove parity: proof bytes identical to the oracle's, accepted by the oracle verifier,
tampering rejected; plus size-independent properties on a larger trace."""
import os
import sys

import cbor2
import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_large_proof_digests import assert_matches_golden  # noqa: E402

P = 2013265921
pytestmark = pytest.mark.gpu


def gpu_prove(ctx, oracle, traces):
    import valida_b200 as vb

    cfg = vb.StarkConfig(ctx, oracle.rc480)
    return vb.prove_machine(cfg, traces)


@pytest.mark.parametrize("n", [25, 0, 3])
def test_prove_fibonacci_bytes_equal_oracle(ctx, oracle, n):
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(n), initial_fp=0x1000)
    proof = gpu_prove(ctx, oracle, t)
    ref = oracle.prove(t.main, t.preprocessed, debug_checks=False)
    ref_bytes = ref.cbor()
    if proof != ref_bytes:   # localise the first divergence for the report
        a, b = cbor2.loads(proof), cbor2.loads(ref_bytes)
        assert a["commitments"] == b["commitments"], "commitments differ"
        for i, (x, y) in enumerate(zip(a["chip_proofs"], b["chip_proofs"])):
            assert x == y, "chip proof %d differs" % i
        assert a["opening_proof"]["fri_proof"]["commit_phase_commits"] == b["opening_proof"]["fri_proof"]["commit_phase_commits"], "FRI commits differ"
        assert a["opening_proof"]["fri_proof"]["final_poly"] == b["opening_proof"]["fri_proof"]["final_poly"]
        assert a["opening_proof"]["fri_proof"]["pow_witness"] == b["opening_proof"]["fri_proof"]["pow_witness"]
        assert a["opening_proof"]["fri_proof"]["query_proofs"] == b["opening_proof"]["fri_proof"]["query_proofs"], "FRI query proofs differ"
        assert a["opening_proof"]["query_openings"] == b["opening_proof"]["query_openings"], "input openings differ"
    assert proof == ref_bytes
    assert oracle.verify(proof, t.preprocessed) == 0


def test_prove_device_resident_entry_matches_host_entry(ctx, oracle):
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(25), initial_fp=0x1000)
    cfg = vb.StarkConfig(ctx, oracle.rc480)
    dm = [ctx.upload(m) for m in t.main]
    dp = [ctx.upload(m) for m in t.preprocessed]
    assert vb.prove_machine(cfg, t, device_resident=(dm, dp)) == vb.prove_machine(cfg, t)
    phases = vb.last_prove_phases(ctx)
    assert phases[0][0].startswith("upload traces") and phases[1][0] == "commit preprocessed"


def test_gpu_proof_tampering_rejected(ctx, oracle):
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(25), initial_fp=0x1000)
    proof = gpu_prove(ctx, oracle, t)
    d = cbor2.loads(proof)
    d["chip_proofs"][0]["opened_values"]["trace_local"][7]["value"][0]["value"] ^= 1
    assert oracle.verify(cbor2.dumps(d), t.preprocessed) != 0
    # a corrupted witness must not yield an accepting proof (either the prover refuses or the verifier rejects)
    bad = vb.run_program(vb.fib_program(25), initial_fp=0x1000)
    bad.main[0][17, 1] = (int(bad.main[0][17, 1]) + 1) % P   # pc of one CPU row
    try:
        p2 = gpu_prove(ctx, oracle, bad)
    except vb.VgpuError as e:
        assert "low degree" in str(e)
    else:
        assert oracle.verify(p2, bad.preprocessed) != 0


def test_prove_larger_trace_verifies_and_matches(ctx, oracle):
    """2^12-row CPU trace (n = 582, BASELINE config 1's nominal size): bytes equal + verifier accepts."""
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(582), initial_fp=0x1000)
    assert t.main[0].shape[0] == 4096 and t.main[2].shape[0] == 1 << 14
    proof = gpu_prove(ctx, oracle, t)
    assert oracle.verify(proof, t.preprocessed) == 0
    assert proof == oracle.prove(t.main, t.preprocessed, debug_checks=False).cbor()


def test_prove_2_16_rows_verifies(ctx, oracle):
    """65537 cycles (2^17 CPU rows): the verifier accepts, and the bytes are the recorded oracle proof's."""
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(9360), initial_fp=0x1000)   # 65537 cycles -> 2^17 CPU rows
    proof = gpu_prove(ctx, oracle, t)
    assert oracle.verify(proof, t.preprocessed) == 0
    assert_matches_golden(proof, "fib_2p17")


import json
import os

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "programs.json")))


@pytest.mark.parametrize("name", ["left_imm_ops_program", "signed_inequality_program", "loadfp_program"])
def test_prove_reference_test_programs_bytes_equal(ctx, oracle, name):
    """prove_left_imm_ops / prove_signed_inequality / prove_loadfp of basic/tests/test_prover.rs:490-625."""
    import valida_b200 as vb

    t = vb.run_program(np.array(GOLDEN[name]["program"], dtype=np.int32), initial_fp=0x1000)
    for addr, value in GOLDEN[name]["expected_cells"]:
        assert t.mem_cell(addr) == value
    proof = gpu_prove(ctx, oracle, t)
    assert proof == oracle.prove(t.main, t.preprocessed, debug_checks=False).cbor()
    assert oracle.verify(proof, t.preprocessed) == 0


from programs import (config5_program, loads_stores_edge_program, lt_edge_operands_program, mixed_program,  # noqa: E402
                      single_address_program)


def _lt_edges_without_double_immediate():
    prog = lt_edge_operands_program()
    assert prog[-2].tolist() == [115, -104, 7, 7, 1, 1]
    return np.concatenate([prog[:-2], prog[-1:]])


@pytest.mark.parametrize("name", ["lt_edges", "lone_stop", "single_address"])
def test_prove_edge_programs_bytes_equal(ctx, oracle, name):
    """Proofs of traces at the witness builders' edges: the lt family on equal operands, on a difference in the top byte only and
    at the sign boundaries (the lt edge program without its both-immediates instruction, see below); a lone STOP; a memory log
    at one address.  Bytes equal to the oracle's, and the oracle verifier accepts."""
    import valida_b200 as vb

    prog = {"lt_edges": _lt_edges_without_double_immediate, "lone_stop": lambda: np.array([[8, 0, 0, 0, 0, 0]], dtype=np.int32),
            "single_address": lambda: single_address_program(5)}[name]()
    t = vb.run_program(prog, initial_fp=0x1000)
    ref = oracle.prove(t.main, t.preprocessed, debug_checks=True)
    assert ref.constraint_failures() == [-1] * 14 and ref.cumulative_sum_zero()
    proof = gpu_prove(ctx, oracle, t)
    assert proof == ref.cbor()
    assert oracle.verify(proof, t.preprocessed) == 0


@pytest.mark.parametrize("name", ["lt_edges", "loads_stores"])
def test_edge_programs_the_cpu_air_rejects(ctx, oracle, name):
    """The two edge programs unchanged are not provable, in the reference either.  A store32 reads the pointer at fp + b on its
    first memory channel (cpu/src/lib.rs:615-631) where the CPU AIR asks for fp + c, and an lte32 with both operands immediate
    reads its second operand at an address the AIR's read-address constraint does not accept.  Every stage up to the quotient is
    still compared bit for bit with the oracle on these traces, and so are the proof bytes; both verifiers reject them."""
    import valida_b200 as vb

    prog = lt_edge_operands_program() if name == "lt_edges" else loads_stores_edge_program()
    t = vb.run_program(prog, initial_fp=0x1000)
    ref = oracle.prove(t.main, t.preprocessed, debug_checks=True)
    assert ref.constraint_failures()[0] >= 0 and ref.constraint_failures()[1:] == [-1] * 13
    tr = ref.transcript()
    pcs = vb.TwoAdicFriPcs(ctx)
    for chip in range(14):
        prep = t.preprocessed[0] if chip == 1 else t.preprocessed[1] if chip == 12 else None
        perm, cs = vb.generate_permutation_trace(ctx, chip, ctx.upload(t.main[chip]), ctx.upload(prep) if prep is not None else None,
                                                 tr["perm_challenges"])
        assert np.array_equal(perm.download(), ref.perm_trace(chip)), chip
        assert np.array_equal(cs, ref.cumulative_sum(chip)), chip
        _, main_pd = pcs.commit_batches([t.main[chip]])
        _, perm_pd = pcs.commit_batches([perm])
        prep_lde = None
        if prep is not None:
            _, prep_pd = pcs.commit_batches([prep])
            prep_lde = pcs.get_ldes(prep_pd)[0]
        log_degree = t.main[chip].shape[0].bit_length() - 1
        q = vb.quotient(ctx, chip, log_degree, prep_lde, pcs.get_ldes(main_pd)[0], pcs.get_ldes(perm_pd)[0], cs, tr["perm_challenges"], tr["alpha"])
        assert np.array_equal(q.download(), ref.quotient_chunks(chip)), chip
    proof = gpu_prove(ctx, oracle, t)
    assert proof == ref.cbor()
    assert oracle.verify(proof, t.preprocessed) != 0
    with pytest.raises(vb.VerificationError):
        vb.verify_machine(vb.StarkConfig(ctx, oracle.rc480), proof, t.preprocessed)


def test_prove_mixed_chip_program(ctx, oracle):
    import valida_b200 as vb

    t = vb.run_program(mixed_program(100), initial_fp=0x1000)
    assert t.main[8].shape[0] == 512 and t.main[3].shape[0] == 512    # 400 lt ops, 300 add ops
    ref = oracle.prove(t.main, t.preprocessed, debug_checks=True)
    assert ref.constraint_failures() == [-1] * 14 and ref.cumulative_sum_zero()
    proof = gpu_prove(ctx, oracle, t)
    assert proof == ref.cbor()
    assert oracle.verify(proof, t.preprocessed) == 0
    # larger instance: verifier accepts, bytes equal to the recorded oracle proof
    t2 = vb.run_program(mixed_program(20000), initial_fp=0x1000)
    assert t2.main[0].shape[0] == 1 << 18
    p2 = gpu_prove(ctx, oracle, t2)
    assert oracle.verify(p2, t2.preprocessed) == 0
    assert_matches_golden(p2, "mixed_20000")


def test_prove_config5_program(ctx, oracle):
    """BASELINE config 5 shape at test size: add, sub, lt family, and/or/xor chips all carry real rows."""
    import valida_b200 as vb

    t = vb.run_program(config5_program(60), initial_fp=0x1000)
    assert t.main[4].shape[0] == 128 and t.main[10].shape[0] == 512 and t.main[8].shape[0] == 256
    ref = oracle.prove(t.main, t.preprocessed, debug_checks=True)
    assert ref.constraint_failures() == [-1] * 14 and ref.cumulative_sum_zero()
    proof = gpu_prove(ctx, oracle, t)
    assert proof == ref.cbor()
    vb.verify_machine(vb.StarkConfig(ctx, oracle.rc480), proof, t.preprocessed)
    t2 = vb.run_program(config5_program(16000), initial_fp=0x1000)
    assert t2.main[0].shape[0] == 1 << 18
    p2 = gpu_prove(ctx, oracle, t2)
    assert oracle.verify(p2, t2.preprocessed) == 0
    assert_matches_golden(p2, "config5_16000")


def test_prove_full_size_2p22_verifies(ctx, oracle):
    """BASELINE config 3 at full size (Fibonacci, 2^22 CPU rows, 2^24 memory rows): both verifiers accept the proof, its
    bytes are the recorded oracle proof's, and a second run yields the same bytes (the proof is a pure function of the traces
    and the challenger)."""
    import valida_b200 as vb

    n = ((1 << 22) - 17) // 7
    t = vb.run_program(vb.fib_program(n), initial_fp=0x1000)
    assert t.main[0].shape[0] == 1 << 22 and t.main[2].shape[0] == 1 << 24
    cfg = vb.StarkConfig(ctx, oracle.rc480)
    proof = vb.prove_machine(cfg, t)
    assert oracle.verify(proof, t.preprocessed) == 0
    vb.verify_machine(cfg, proof, t.preprocessed)
    assert_matches_golden(proof, "fib_2p22")
    assert vb.prove_machine(cfg, t) == proof


def test_prove_config4_2p24_rows_on_one_gpu(ctx, oracle):
    """BASELINE config 4's trace (Fibonacci, 2^24 CPU rows; memory chip 2^26 rows, LDE 2^27 = BabyBear's two-adicity) on a
    single H100 (80 GB): both verifiers accept."""
    import valida_b200 as vb

    n = ((1 << 24) - 17) // 7
    t = vb.run_program(vb.fib_program(n), initial_fp=0x1000)
    assert t.main[0].shape[0] == 1 << 24 and t.main[2].shape[0] == 1 << 26
    cfg = vb.StarkConfig(ctx, oracle.rc480)
    try:
        proof = vb.prove_machine(cfg, t)
        vb.verify_machine(cfg, proof, t.preprocessed)
    finally:
        ctx.release_cached()      # the proof filled most of the 80 GB: later tests open contexts of their own
    assert oracle.verify(proof, t.preprocessed) == 0
