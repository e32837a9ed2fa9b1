"""The product's proof codec (valida_b200/csrc/host/proof.cc) on the CPU, built with g++ and the address / undefined-behaviour
sanitizers: the oracle's proofs and openings decode and re-encode byte for byte, and malformed bytes are refused cleanly,
with no sanitizer report and no allocation larger than the input warrants.  The GPU tests compare the prover's bytes with
the oracle's and feed the verifier tampered proofs; this pins the one codec both of them share, without a device."""
import os
import random
import subprocess

import numpy as np
import pytest

import programs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 2013265921
FELT = b"\xa1\x65value"
# any single allocation above 64 MB is a sanitizer error: a hostile length must not reach an allocation
ENV = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:allocator_may_return_null=0:max_allocation_size_mb=64",
           UBSAN_OPTIONS="print_stacktrace=1:halt_on_error=1")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("codec") / "proof_codec_check")
    csrc = os.path.join(ROOT, "valida_b200", "csrc")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                    "-I", csrc, "-I", "/usr/local/cuda/include", os.path.join(ROOT, "tests", "c", "proof_codec_check.cc"),
                    os.path.join(csrc, "host", "proof.cc"), "-o", out], check=True)
    return out


def codec(exe, kind, data):
    """encode(decode(data)), or None when the decoder rejects it."""
    r = subprocess.run([exe], input=kind.encode() + b"\n" + bytes(data), capture_output=True, env=ENV)
    assert r.stderr == b"", r.stderr.decode(errors="replace")[-3000:]
    assert r.returncode in (0, 3), r.returncode
    return r.stdout if r.returncode == 0 else None


def machine_proof(oracle, program, **run):
    import valida_b200 as vb

    t = vb.run_program(program, initial_fp=0x1000, **run)
    return oracle.prove(t.main, t.preprocessed, debug_checks=False).cbor()


@pytest.fixture(scope="module")
def fib25_proof(built, oracle):
    import valida_b200 as vb

    return machine_proof(oracle, vb.fib_program(25))


PROGRAMS = {
    "fib582": lambda vb: (vb.fib_program(582), {}),
    "mixed": lambda vb: (programs.mixed_program(100), {}),
    "config5": lambda vb: (programs.config5_program(60), {}),
    "static_data": lambda vb: (programs.static_data_program()[0], {"static_data": programs.static_data_program()[1]}),
}


def test_oracle_proofs_round_trip(exe, fib25_proof, oracle):
    import valida_b200 as vb

    assert codec(exe, "proof", fib25_proof) == fib25_proof
    for name, make in PROGRAMS.items():
        program, run = make(vb)
        proof = machine_proof(oracle, program, **run)
        assert codec(exe, "proof", proof) == proof, name


def test_oracle_openings_round_trip(exe, oracle):
    """The shapes of vgpu_open: mixed heights, a one-row matrix, one and two points, per-matrix shifts."""
    rng = np.random.default_rng(77)

    def mat(log_h, w):
        return rng.integers(0, P, (1 << log_h, w), dtype=np.uint32)

    def point():
        return [int(v) for v in rng.integers(0, P, 5)]

    def gen(log_h):
        return pow(0x1A427A41, 1 << (27 - log_h), P)

    z, z2 = point(), point()
    r0 = [mat(9, 6), mat(11, 3), mat(0, 4)]
    r1 = [mat(9, 10), mat(11, 10)]
    cases = [
        ([r0, r1], [[z, [v * gen(9) % P for v in z]], [z, [v * gen(11) % P for v in z]], [z], [z2], [z2]], [1, 1, 1, 961, 961]),
        ([[mat(4, 2)]], [[z]], None),
        ([[mat(0, 1)], [mat(3, 5)]], [[z, z2], [z2]], None),
    ]
    for rounds, points, shifts in cases:
        opening = oracle.open(rounds, points, np.arange(8, dtype=np.uint32), shifts=shifts)
        assert codec(exe, "opening", opening) == opening


def test_malformed_bytes_are_rejected(exe, fib25_proof):
    pf = fib25_proof
    rejected = lambda data, kind="proof": codec(exe, kind, data) is None  # noqa: E731
    assert rejected(b"") and rejected(b"", "opening")
    rng = random.Random(2026)
    for cut in list(range(len(pf) - 64, len(pf))) + rng.sample(range(len(pf)), 64):
        assert rejected(pf[:cut]), cut
    assert rejected(pf + b"\x00")
    # a felt equal to p is refused; p - 1 is the largest accepted
    at = pf.index(FELT + b"\x1a") + len(FELT) + 1
    assert rejected(pf[:at] + P.to_bytes(4, "big") + pf[at + 4:])
    top = pf[:at] + (P - 1).to_bytes(4, "big") + pf[at + 4:]
    assert codec(exe, "proof", top) == top
    for key in [b"commitments", b"commit_phase_commits", b"sibling_value", b"pow_witness", b"opened_values", b"cumulative_sum", b"value"]:
        at = pf.index(key)
        assert rejected(pf[:at] + key[:-1] + b"_" + pf[at + len(key):]), key
    # map sizes: the top-level map of 3 and a chip's opened values, a map of 7
    assert pf[0] == 0xA3 and rejected(b"\xa2" + pf[1:]) and rejected(b"\xa4" + pf[1:])
    at = pf.index(b"\x6dopened_values\xa7") + 14
    assert rejected(pf[:at] + b"\xa6" + pf[at + 1:]) and rejected(pf[:at] + b"\xa8" + pf[at + 1:])
    # array heads claiming 2^32 and 2^63 elements, in place of the 14 chip proofs and of the rows of a query's batch opening
    for head in [b"\x6bchip_proofs\x8e", b"\x6dopened_values\x8e"]:
        at = pf.index(head) + len(head) - 1
        for n in [1 << 32, 1 << 63]:
            assert rejected(pf[:at] + b"\x9b" + n.to_bytes(8, "big") + pf[at + 1:]), (head, n)
