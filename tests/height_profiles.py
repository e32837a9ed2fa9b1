"""Chip-height profiles for whole-proof parity: which of the 14 chips is tall, which is short, and how the trace words arrive.

Much of the prover around the stage kernels depends on the profile of log heights rather than on the words: the alpha offset of
each reduced opening is counted per height, a FRI fold adds the reduced openings of the next height only where that height exists,
each round's query leaf is shifted by that round's tallest matrix, equal heights keep their order in the mixed-height trees, and a
split proof splits each chip or not by its own height.  A profile is the list of the 14 chips' log heights; the preprocessed
traces (program ROM of chip 1, range table of chip 12) follow their chips' heights.

    PROFILES          named profiles: one row everywhere (no FRI layers), every height at once, the tallest chip first, last,
                      twice or alone, the program ROM and the range table as the tallest traces, heights with gaps
    RANDOM_PROFILES   seeded ones, each chip's log height uniform in [0, 13]; the first 14 make chip k the one tallest chip
    ROUTE_PROFILE     CPU, memory and add at 2^17 rows: host matrices on both sides of the staged-upload threshold
    HONEST            honest witnesses (proofs that verify) with other profiles: straight-line programs of adds, lts and bits,
                      Fibonacci under a program ROM taller than every other trace, config5

random_traces() makes the words of a profile (uniform below p with edge words mixed in), to_monty() their Montgomery images,
and first_difference() names the first field in which two proofs differ, so that a failing parity check names its stage."""
import cbor2
import numpy as np

from generated_programs import counted_program

P = 2013265921
NUM_CHIPS = 14
MAX_LOG = 13
CPU, PROGRAM, MEMORY, ADD, BITWISE, RANGE = 0, 1, 2, 3, 10, 12
CHIP_WIDTHS = [51, 1, 14, 16, 16, 18, 14, 28, 45, 14, 79, 7, 2, 6]
PREP_WIDTHS = {PROGRAM: 7, RANGE: 1}                   # the preprocessed traces, in the order the prover takes them
MONTY_ONE = pow(2, -32, P)                             # canonical words whose Montgomery images are 1 and p - 1
EDGE_WORDS = [0, 1, P - 1, P - 2, (P - 1) // 2, 1 << 30, MONTY_ONE, P - MONTY_ONE]

PROFILES = {
    "one_row": [0] * NUM_CHIPS,
    "staircase": list(range(NUM_CHIPS)),
    "reverse_staircase": [MAX_LOG - c for c in range(NUM_CHIPS)],
    "flat12": [12] * NUM_CHIPS,
    "gaps": [11, 0, 5, 11, 0, 5, 5, 0, 11, 0, 5, 11, 0, 5],
    "twin_tallest": [9, 4, 11, 13, 2, 7, 0, 12, 5, 1, 13, 3, 8, 6],          # chips 3 and 10, shorter chips between them
    "one_tall": [13 if c == BITWISE else 0 for c in range(NUM_CHIPS)],       # the widest chip (79 columns) alone
    "program_tallest": [10, 13, 9, 8, 3, 10, 0, 2, 7, 1, 6, 0, 8, 4],
    "range_tallest": [12, 5, 11, 9, 0, 10, 3, 7, 12, 2, 8, 1, 13, 6],
}


def _random_profile(k):
    logs = np.random.default_rng([20, k]).integers(0, MAX_LOG + 1, NUM_CHIPS)
    if k < NUM_CHIPS:                  # chip k alone at the tallest height drawn (a tie at it is lowered by one)
        top = max(int(logs.max()), 1)
        logs[logs == top] = top - 1
        logs[k] = top
    return [int(v) for v in logs]


RANDOM_PROFILES = {"random%02d" % k: _random_profile(k) for k in range(24)}
ALL_PROFILES = {**PROFILES, **RANDOM_PROFILES}

# CPU (51 columns: 25.5 MiB, a whole staging chunk and a partial one), add (16: exactly the 8 MiB threshold, staged) and memory
# (14: 7 MiB, copied directly) at 2^17 rows; the others short
ROUTE_PROFILE = [17, 6, 17, 17, 0, 10, 3, 0, 8, 1, 5, 0, 8, 2]


def small(profile, max_prep_log=8):
    """Preprocessed traces of at most 2^max_prep_log rows: the plain-Python verifier re-commits them in reasonable time."""
    return profile[PROGRAM] <= max_prep_log and profile[RANGE] <= max_prep_log


def random_words(rng, shape):
    """Uniform words below p of the given shape, about 10 % of them EDGE_WORDS."""
    w = rng.integers(0, P, shape, dtype=np.uint32)
    edge = rng.random(shape) < 0.1
    w[edge] = rng.choice(np.array(EDGE_WORDS, dtype=np.uint32), int(edge.sum()))
    return w


def random_traces(profile, seed):
    """(14 main traces, 2 preprocessed traces) of the profile's heights: uniform words below p, about 10 % of them edge words."""
    rng = np.random.default_rng([seed] + list(profile))
    main = [random_words(rng, (1 << lh, CHIP_WIDTHS[c])) for c, lh in enumerate(profile)]
    prep = [random_words(rng, (1 << profile[c], w)) for c, w in PREP_WIDTHS.items()]
    return main, prep


def with_chip_replaced(main, chip, seed=0):
    """The main traces with chip `chip`'s trace replaced by random rows of the same height."""
    out = list(main)
    out[chip] = random_words(np.random.default_rng([seed, chip]), main[chip].shape)
    return out


def to_monty(m):
    """The Montgomery images x * 2^32 mod p of canonical words."""
    return ((np.asarray(m, dtype=np.uint64) << np.uint64(32)) % np.uint64(P)).astype(np.uint32)


def _fib_tall_rom(vb):
    """Fibonacci (25) with its program zero-padded to 2^11 rows that never run: the program ROM is the tallest trace."""
    prog = vb.fib_program(25)
    prog = np.concatenate([prog, np.zeros(((1 << 11) - len(prog), prog.shape[1]), dtype=prog.dtype)])
    return vb.run_program(prog, initial_fp=0x1000)


def _counted(seed, **kw):
    # adds, lts and bits only: a sub that borrows is unprovable in the reference, and static cells at random addresses fail the
    # static-data chip
    def run(vb):
        prog, static, fp = counted_program(seed, **kw)
        return vb.run_program(prog, initial_fp=fp)
    return run


def _config5(vb):
    import programs

    return vb.run_program(programs.config5_program(6), initial_fp=0x1000)


# name -> function of the valida_b200 module returning the MachineTraces of an honest run
HONEST = {
    "counted_200": _counted(3, adds=3, lts=3, bits=3, cycles=200),
    "counted_1500": _counted(5, adds=400, lts=200, bits=100, cycles=1500),
    "counted_5000": _counted(8, adds=40, lts=900, bits=1200, cycles=5000),
    "fib_tall_rom": _fib_tall_rom,
    "config5": _config5,
}
SMALL_HONEST = "counted_200"


def log_heights(main):
    return [m.shape[0].bit_length() - 1 for m in main]


def first_difference(a, b):
    """The path of the first field in which the CBOR proofs a and b differ (e.g. "opening_proof.fri_proof.commit_phase_commits[3]
    [0].value"), "" when the documents are equal, "undecodable" when one of them is not CBOR."""
    try:
        da, db = cbor2.loads(a), cbor2.loads(b)
    except (ValueError, cbor2.CBORDecodeError):
        return "undecodable"

    def walk(x, y, path):
        if type(x) is not type(y):
            return path
        if isinstance(x, dict):
            for k in x:
                if k not in y:
                    return "%s.%s" % (path, k)
                d = walk(x[k], y[k], "%s.%s" % (path, k))
                if d is not None:
                    return d
            return None if x.keys() == y.keys() else path
        if isinstance(x, list):
            for i, (u, v) in enumerate(zip(x, y)):
                d = walk(u, v, "%s[%d]" % (path, i))
                if d is not None:
                    return d
            return None if len(x) == len(y) else "%s (length %d != %d)" % (path, len(x), len(y))
        return None if x == y else path

    d = walk(da, db, "")
    return "" if d is None else d.lstrip(".") or "(root)"
