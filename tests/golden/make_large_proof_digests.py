"""Digests of oracle proofs at sizes where the GPU suite otherwise checks only that a verifier accepts: Fibonacci at 2^17,
2^20 and 2^22 CPU rows, the 2^18-row mixed and config-5 programs, and Fibonacci at 2^17 and 2^20 with Poseidon-16 trees.

Each entry holds the proof's length and SHA-256, and the stage values that locate a mismatch without the oracle: the
transcript (permutation challenges, alpha, zeta, the four commitments), the FRI commit-phase commitments, final polynomial
and proof-of-work witness, and per chip the digests of the permutation trace and the quotient chunks and the cumulative sum.
A matrix digest is `matrix_digest`: SHA-256 of the row-major canonical words as little-endian uint32.

    python tests/golden/make_large_proof_digests.py   -> tests/golden/large_proof_digests.json
(about 7 minutes on 8 cores; the 2^22 proof peaks at 28 GB of host memory)"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

PATH = os.path.join(HERE, "large_proof_digests.json")
N_CHIPS = 14


def matrix_digest(m):
    return hashlib.sha256(np.ascontiguousarray(m, dtype="<u4").tobytes()).hexdigest()


def fib_n(log_rows):
    """The Fibonacci argument whose CPU trace has 2^log_rows rows (2^17 is the 65537-cycle run of test_gpu_prove)."""
    return 9360 if log_rows == 17 else ((1 << log_rows) - 17) // 7


# name -> (Merkle hash, program, program argument); the Keccak entries up to 2^18 rows are recomputed by the CPU suite
CASES = {
    "fib_2p17": ("keccak", "fib", fib_n(17)),
    "fib_2p20": ("keccak", "fib", fib_n(20)),
    "fib_2p22": ("keccak", "fib", fib_n(22)),
    "mixed_20000": ("keccak", "mixed", 20000),
    "config5_16000": ("keccak", "config5", 16000),
    "p16_fib_2p17": ("poseidon16", "fib", fib_n(17)),
    "p16_fib_2p20": ("poseidon16", "fib", fib_n(20)),
}
CPU_CASES = ("fib_2p17", "mixed_20000", "config5_16000")


def traces(name):
    import valida_b200 as vb
    import programs

    _, prog, n = CASES[name]
    p = {"fib": vb.fib_program, "mixed": programs.mixed_program, "config5": programs.config5_program}[prog](n)
    return vb.run_program(p, initial_fp=0x1000)


def _plain(x):
    """The decoded CBOR with its {"value": v} wrappers removed."""
    if isinstance(x, dict):
        return _plain(x["value"]) if set(x) == {"value"} else {k: _plain(v) for k, v in x.items()}
    if isinstance(x, list):
        return [_plain(v) for v in x]
    return x


def proof_entry(proof, cbor):
    """The golden entry of one oracle proof (an oracle_binding.OracleProof and its CBOR bytes)."""
    import cbor2

    tr = proof.transcript()
    fri = _plain(cbor2.loads(cbor)["opening_proof"]["fri_proof"])
    return {
        "bytes": len(cbor),
        "sha256": hashlib.sha256(cbor).hexdigest(),
        "transcript": {k: [int(w) for w in v] for k, v in sorted(tr.items())},
        "fri": {k: fri[k] for k in ("commit_phase_commits", "final_poly", "pow_witness")},
        "chips": [{"perm_trace": matrix_digest(proof.perm_trace(c)), "quotient_chunks": matrix_digest(proof.quotient_chunks(c)),
                   "cumulative_sum": [int(w) for w in proof.cumulative_sum(c)]} for c in range(N_CHIPS)],
    }


def compute(names=tuple(CASES)):
    import oracle_binding

    orcs = {}
    res = {}
    for name in names:
        mmcs = CASES[name][0]
        if mmcs not in orcs:
            if mmcs == "keccak":
                orcs[mmcs] = oracle_binding.Oracle()
            else:
                import poseidon_mmcs

                orcs[mmcs] = poseidon_mmcs.PoseidonOracle()
        t = traces(name)
        proof = orcs[mmcs].prove(t.main, t.preprocessed, debug_checks=False)
        res[name] = proof_entry(proof, proof.cbor())
        del proof, t
    return res


def load():
    return json.load(open(PATH))


P = 2013265921
R_INV = pow(1 << 32, P - 2, P)


def _canonical(words):
    """Field words as the CBOR stores them (Montgomery form, x * 2^32 mod p) -> canonical, as the transcript records them."""
    return [w * R_INV % P for w in words]


def stage_difference(cbor, entry):
    """The first recorded stage value that the decoded proof does not carry, in protocol order, or None."""
    import cbor2

    d = _plain(cbor2.loads(cbor))
    tr = entry["transcript"]
    for key, golden in (("main_trace", "main_commit"), ("perm_trace", "perm_commit")):
        if _canonical(d["commitments"][key]) != tr[golden]:
            return "commitments.%s" % key
    for c, chip in enumerate(entry["chips"]):
        if _canonical(d["chip_proofs"][c]["cumulative_sum"]) != chip["cumulative_sum"]:
            return "chip %d cumulative_sum" % c
    if _canonical(d["commitments"]["quotient_chunks"]) != tr["quotient_commit"]:
        return "commitments.quotient_chunks"
    fri = d["opening_proof"]["fri_proof"]
    for key in ("commit_phase_commits", "final_poly", "pow_witness"):
        if fri[key] != entry["fri"][key]:
            return "fri.%s" % key
    return None


def assert_matches_golden(cbor, name):
    """The proof's bytes are the recorded oracle proof's; otherwise the assertion names the first stage that departs."""
    entry = load()[name]
    if len(cbor) == entry["bytes"] and hashlib.sha256(cbor).hexdigest() == entry["sha256"]:
        return
    at = stage_difference(cbor, entry) or "the query proofs or opened values (every recorded stage value is equal)"
    raise AssertionError("%s: the proof departs from the oracle's at %s" % (name, at))


if __name__ == "__main__":
    res = compute()
    with open(PATH, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote large_proof_digests.json")
