"""The oracle prover's output bytes are pinned (tests/golden/oracle_proof_hashes.json): refactors of oracle/ — e.g. performance work
on the CPU baseline — must reproduce them exactly, for every thread count."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))


def test_oracle_proofs_match_recorded_digests(built):
    import make_oracle_proof_hashes

    want = json.load(open(os.path.join(HERE, "golden", "oracle_proof_hashes.json")))
    assert make_oracle_proof_hashes.compute() == want


def test_oracle_large_proofs_match_recorded_digests(built):
    """The Keccak entries of tests/golden/large_proof_digests.json up to 2^18 rows, recomputed from the oracle (the 2^20 and 2^22
    entries and the Poseidon-16 ones only by their generator), and the stage comparison agrees with the recorded stage values."""
    import oracle_binding

    import make_large_proof_digests as g

    want = g.load()
    assert set(g.CPU_CASES) < set(want) == set(g.CASES)
    got = g.compute(g.CPU_CASES)
    for name in g.CPU_CASES:
        assert got[name] == want[name], name
    t = g.traces("fib_2p17")
    proof = oracle_binding.Oracle().prove(t.main, t.preprocessed, debug_checks=False).cbor()
    g.assert_matches_golden(proof, "fib_2p17")
    assert g.stage_difference(proof, want["fib_2p17"]) is None
    # a changed stage value is named, the earliest first
    import cbor2
    import pytest

    d = cbor2.loads(proof)
    d["opening_proof"]["fri_proof"]["pow_witness"]["value"] ^= 1
    with pytest.raises(AssertionError, match="fri.pow_witness"):
        g.assert_matches_golden(cbor2.dumps(d), "fib_2p17")
    d["chip_proofs"][3]["cumulative_sum"]["value"][0]["value"] ^= 1
    assert g.stage_difference(cbor2.dumps(d), want["fib_2p17"]) == "chip 3 cumulative_sum"


def test_oracle_proof_independent_of_thread_count(built, oracle):
    import hashlib
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(582), initial_fp=0x1000)
    want = json.load(open(os.path.join(HERE, "golden", "oracle_proof_hashes.json")))["fib_582"]["sha256"]
    top = oracle.max_threads()
    try:
        for th in (1, 3, top):
            oracle.set_threads(th)
            assert hashlib.sha256(oracle.prove(t.main, t.preprocessed, debug_checks=False).cbor()).hexdigest() == want, th
    finally:
        oracle.set_threads(top)
