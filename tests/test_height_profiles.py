"""The chip-height profiles of tests/height_profiles.py cover what they are there for, and on the small ones (preprocessed traces of
at most 2^8 rows) the oracle's verifier and Machine::verify restated in plain Python (test_verifier_restatement.py) reach the same
verdict: on random traces, on honest witnesses, and on an honest witness with any one chip's trace replaced by random rows.
tests/test_gpu_height_profiles.py proves and verifies the same profiles on the GPU."""
import os
import re

import numpy as np
import pytest

from height_profiles import (ADD, ALL_PROFILES, BITWISE, CHIP_WIDTHS, CPU, EDGE_WORDS, HONEST, MAX_LOG, MEMORY, NUM_CHIPS, P, PREP_WIDTHS,
                             PROFILES, PROGRAM, RANDOM_PROFILES, RANGE, ROUTE_PROFILE, SMALL_HONEST, first_difference, log_heights,
                             random_traces, small, to_monty, with_chip_replaced)

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "valida_b200", "csrc")
LOG_BLOWUP = 1


def _staging_constants():
    src = open(os.path.join(CSRC, "staging.cu")).read()
    m = re.search(r"constexpr size_t STAGE_CHUNK = (\d+)u << (\d+), STAGE_MIN = (\d+)u << (\d+);", src)
    return int(m.group(1)) << int(m.group(2)), int(m.group(3)) << int(m.group(4))


# ---- coverage -------------------------------------------------------------------------------------------------------------
def test_every_log_height_occurs():
    assert {lh for p in ALL_PROFILES.values() for lh in p} == set(range(MAX_LOG + 1))
    assert all(len(p) == NUM_CHIPS and all(0 <= lh <= MAX_LOG for lh in p) for p in ALL_PROFILES.values())
    assert len(RANDOM_PROFILES) == 24 and len(set(map(tuple, ALL_PROFILES.values()))) == len(ALL_PROFILES)


def test_every_chip_is_the_one_tallest_chip_somewhere():
    leaders = {p.index(max(p)) for p in ALL_PROFILES.values() if p.count(max(p)) == 1}
    assert leaders == set(range(NUM_CHIPS))


def test_some_profiles_tie_at_the_maximum_height():
    tied = {n for n, p in ALL_PROFILES.items() if p.count(max(p)) > 1}
    assert {"flat12", "gaps", "twin_tallest"} <= tied and tied & set(RANDOM_PROFILES)


def test_named_profiles_are_what_their_names_say():
    one_row = PROFILES["one_row"]
    assert max(one_row) + LOG_BLOWUP == LOG_BLOWUP                         # log_max == LOG_BLOWUP: no FRI layer
    assert sorted(PROFILES["staircase"]) == list(range(NUM_CHIPS)) == PROFILES["reverse_staircase"][::-1]
    assert set(PROFILES["gaps"]) == {0, 5, 11}
    twin = PROFILES["twin_tallest"]
    a, b = [c for c in range(NUM_CHIPS) if twin[c] == max(twin)]
    assert b - a > 1 and all(twin[c] < max(twin) for c in range(a + 1, b))
    one_tall = PROFILES["one_tall"]
    assert one_tall[BITWISE] == MAX_LOG and CHIP_WIDTHS[BITWISE] == max(CHIP_WIDTHS) and sum(one_tall) == MAX_LOG
    prog = PROFILES["program_tallest"]
    assert prog[PROGRAM] == MAX_LOG and max(lh for c, lh in enumerate(prog) if c != PROGRAM) <= 10
    rng = PROFILES["range_tallest"]
    assert rng[RANGE] == MAX_LOG and rng.count(MAX_LOG) == 1
    assert prog.index(MAX_LOG) != 0 and rng.index(MAX_LOG) != 0               # the tallest chip is not the CPU


def test_route_profile_crosses_the_staging_threshold():
    """The host routes' profile has a matrix staged in a whole chunk and a partial one, a matrix exactly at the threshold (staged),
    and one just below it (one direct copy)."""
    chunk, stage_min = _staging_constants()
    sizes = {c: (1 << lh) * CHIP_WIDTHS[c] * 4 for c, lh in enumerate(ROUTE_PROFILE)}
    staged = [s for s in sizes.values() if s >= stage_min]
    assert stage_min in staged
    assert any(s > chunk and s % chunk for s in staged)
    assert any(stage_min / 2 < s < stage_min for s in sizes.values())
    assert (sizes[CPU], sizes[ADD], sizes[MEMORY]) == (51 << 19, 8 << 20, 7 << 20)


def test_honest_profiles_differ_from_the_fibonacci_shape(built):
    """The honest witnesses reach heights Fibonacci does not: the program ROM tallest, the lt and bitwise chips tall."""
    import valida_b200 as vb

    hs = {n: log_heights(f(vb).main) for n, f in HONEST.items()}
    assert hs["fib_tall_rom"][PROGRAM] > max(lh for c, lh in enumerate(hs["fib_tall_rom"]) if c != PROGRAM)
    assert hs["counted_5000"][0] == MAX_LOG and min(hs["counted_5000"][8], hs["counted_5000"][BITWISE]) >= 10
    assert small(hs[SMALL_HONEST])


# ---- the helpers ----------------------------------------------------------------------------------------------------------
def test_random_traces_and_montgomery_images():
    main, prep = random_traces(PROFILES["twin_tallest"], 1)
    assert log_heights(main) == PROFILES["twin_tallest"] and [m.shape[1] for m in main] == CHIP_WIDTHS
    assert [m.shape for m in prep] == [(1 << PROFILES["twin_tallest"][c], w) for c, w in PREP_WIDTHS.items()]
    words = np.concatenate([m.ravel() for m in main + prep])
    assert words.max() < P and 0.05 < np.isin(words, EDGE_WORDS).mean() < 0.15
    assert set(EDGE_WORDS) <= set(words.tolist())
    assert [int(v) for v in to_monty(np.array(EDGE_WORDS[-2:], dtype=np.uint32))] == [1, P - 1]
    sample = words[:1000]
    assert [int(v) for v in to_monty(sample)] == [int(x) * (1 << 32) % P for x in sample]
    changed = with_chip_replaced(main, 5)
    assert all(changed[c] is main[c] for c in range(NUM_CHIPS) if c != 5) and changed[5].shape == main[5].shape
    assert not np.array_equal(changed[5], main[5])


def test_first_difference_names_the_path():
    import cbor2

    d = {"a": [1, {"b": [5, 6]}], "c": 2}
    e = {"a": [1, {"b": [5, 7]}], "c": 2}
    assert first_difference(cbor2.dumps(d), cbor2.dumps(d)) == ""
    assert first_difference(cbor2.dumps(d), cbor2.dumps(e)) == "a[1].b[1]"
    assert first_difference(cbor2.dumps(d), cbor2.dumps({"a": [1], "c": 2})) == "a (length 2 != 1)"
    assert first_difference(cbor2.dumps(d)[:-1], cbor2.dumps(d)) == "undecodable"


# ---- verifier agreement on the small profiles ------------------------------------------------------------------------------
def _py_verdict(oracle, proof, prep):
    from test_quotient_restatement import CHIPS
    from test_verifier_restatement import Reject, machine_verify_py

    try:
        machine_verify_py(proof, prep, [int(x) for x in oracle.rc480], [len(CHIPS[i]) for i in range(NUM_CHIPS)])
        return "accept"
    except Reject as e:
        return str(e)


def _oracle_verdict(code):
    from test_verifier_restatement import STAGE_OF_CODE

    return "accept" if code == 0 else STAGE_OF_CODE.get(code, "constraints chip %d" % (-100 - code))


@pytest.mark.parametrize("name", ["one_row", "gaps", "one_tall", "twin_tallest"])
def test_random_traces_same_verdict(built, oracle, name):
    assert small(PROFILES[name])
    main, prep = random_traces(PROFILES[name], 1)
    proof = oracle.prove(main, prep, debug_checks=False).cbor()
    code = oracle.verify(proof, prep)
    assert code != 0
    assert _py_verdict(oracle, proof, prep) == _oracle_verdict(code)


@pytest.fixture(scope="module")
def honest_small(built):
    import valida_b200 as vb

    t = HONEST[SMALL_HONEST](vb)
    assert small(log_heights(t.main))
    return t


def test_honest_small_witness_accepted_by_both(oracle, honest_small):
    t = honest_small
    proof = oracle.prove(t.main, t.preprocessed, debug_checks=True).cbor()
    assert oracle.verify(proof, t.preprocessed) == 0
    assert _py_verdict(oracle, proof, t.preprocessed) == "accept"


# The oracle's verdict with chip c's trace replaced by random rows is its first failed check: the chip's own constraints (-100 - c),
# or for memory, div, range and static data the sum of the cumulative sums (-20).  The program chip (1) has no AIR constraints and
# no interactions in the reference, so nothing binds its multiplicity column and the proof is ACCEPTED: a soundness gap of the
# reference, pinned here as its behaviour.
REPLACED_VERDICTS = [-100, 0, -20, -103, -104, -105, -20, -107, -108, -109, -110, -111, -20, -20]


@pytest.mark.parametrize("chip", range(NUM_CHIPS))
def test_one_chip_replaced_same_verdict(oracle, honest_small, chip):
    t = honest_small
    main = with_chip_replaced(t.main, chip)
    proof = oracle.prove(main, t.preprocessed, debug_checks=False).cbor()
    code = oracle.verify(proof, t.preprocessed)
    assert code == REPLACED_VERDICTS[chip]
    assert _py_verdict(oracle, proof, t.preprocessed) == _oracle_verdict(code)
