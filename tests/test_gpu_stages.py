"""GPU parity, stage by stage, against the oracle: permutation trace (K5) and quotient chunks (K6/K7)."""
import numpy as np
import pytest

P = 2013265921
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fib(built):
    import valida_b200 as vb

    return vb.run_program(vb.fib_program(25), initial_fp=0x1000)


@pytest.fixture(scope="module")
def oracle_run(fib, oracle):
    return oracle.prove(fib.main, fib.preprocessed, debug_checks=False)


def prep_of(fib, chip):
    return fib.preprocessed[0] if chip == 1 else fib.preprocessed[1] if chip == 12 else None


@pytest.mark.parametrize("chip", list(range(14)))
def test_perm_trace_bit_exact(ctx, oracle, fib, oracle_run, chip):
    import valida_b200 as vb

    tr = oracle_run.transcript()
    main = ctx.upload(fib.main[chip])
    prep = prep_of(fib, chip)
    dprep = ctx.upload(prep) if prep is not None else None
    perm, cs = vb.generate_permutation_trace(ctx, chip, main, dprep, tr["perm_challenges"])
    exp = oracle_run.perm_trace(chip)
    assert perm.shape == exp.shape
    assert np.array_equal(perm.download(), exp)
    assert np.array_equal(cs, oracle_run.cumulative_sum(chip))


def test_perm_trace_random_traces_and_zero_denominators(ctx, oracle):
    """Random (non-witness) traces across heights incl. scan chunk boundaries, and a row whose
    denominator is exactly zero (batch inverse must leave it zero: util/src/lib.rs:21-43)."""
    import valida_b200 as vb

    rng = np.random.default_rng(5)
    ch = rng.integers(0, P, size=15, dtype=np.uint32)
    for chip, h in [(2, 1), (2, 2), (3, 2048), (0, 4096), (2, 8192), (12, 256)]:
        w = oracle.chip_width(chip)
        m = rng.integers(0, P, size=(h, w), dtype=np.uint32)
        pw = oracle.chip_prep_width(chip)
        prep = rng.integers(0, P, size=(h, pw), dtype=np.uint32) if pw else None
        exp, ecs = oracle.perm_trace(chip, m, prep, ch)
        got, cs = vb.generate_permutation_trace(ctx, chip, ctx.upload(m), ctx.upload(prep) if pw else None, ch)
        assert np.array_equal(got.download(), exp), (chip, h)
        assert np.array_equal(cs, ecs)
    # range chip: denominator = r1^4 + counter; choose counter = -r1^4 when r1 is a base-field element
    ch2 = np.zeros(15, dtype=np.uint32)
    ch2[5] = 3  # r1 = 3 (base field), alphas_global[3] = 3^4 = 81
    ch2[10] = 7
    m = np.zeros((4, 2), dtype=np.uint32)
    m[:, 0] = [1, 2, 3, 4]
    m[:, 1] = [5, P - 81, 6, 7]  # row 1: 81 + (p - 81) = 0
    exp, ecs = oracle.perm_trace(12, m, np.zeros((4, 1), dtype=np.uint32), ch2)
    assert not exp[1, :5].any()
    got, cs = vb.generate_permutation_trace(ctx, 12, ctx.upload(m), ctx.upload(np.zeros((4, 1), dtype=np.uint32)), ch2)
    assert np.array_equal(got.download(), exp) and np.array_equal(cs, ecs)


@pytest.mark.parametrize("chip", list(range(14)))
def test_quotient_chunks_bit_exact(ctx, oracle, fib, oracle_run, chip):
    import valida_b200 as vb

    tr = oracle_run.transcript()
    pcs = vb.TwoAdicFriPcs(ctx)
    h = fib.main[chip].shape[0]
    log_degree = h.bit_length() - 1
    _, main_pd = pcs.commit_batches([fib.main[chip]])
    _, perm_pd = pcs.commit_batches([oracle_run.perm_trace(chip)])
    prep = prep_of(fib, chip)
    prep_lde = None
    if prep is not None:
        _, prep_pd = pcs.commit_batches([prep])
        prep_lde = pcs.get_ldes(prep_pd)[0]
    q = vb.quotient(ctx, chip, log_degree, prep_lde, pcs.get_ldes(main_pd)[0], pcs.get_ldes(perm_pd)[0],
                    oracle_run.cumulative_sum(chip), tr["perm_challenges"], tr["alpha"])
    assert np.array_equal(q.download(), oracle_run.quotient_chunks(chip))


@pytest.mark.parametrize("chip", list(range(14)))
def test_quotient_random_traces_exercise_every_constraint(ctx, oracle, chip):
    """On random (constraint-violating) traces every constraint contributes a non-zero term, so a wrong
    column index, sign or constraint order anywhere in the device AIR shows up as a mismatch.  The program and range chips
    read a random preprocessed matrix."""
    quotient_random_traces(ctx, oracle, chip, 4, 40 + chip)


@pytest.mark.parametrize("chip,log_degree", [(c, d) for c in range(14) for d in (0, 1)] + [(0, 15), (10, 15)])
def test_quotient_random_traces_one_two_and_2p15_rows(ctx, oracle, chip, log_degree):
    """The same at one row, two rows (first and last row coincide or are neighbours), and 2^15 rows, where the domain exponents
    of the kernel reach the low half of the two-level root table."""
    quotient_random_traces(ctx, oracle, chip, log_degree, 40 + 100 * log_degree + chip)


def quotient_random_traces(ctx, oracle, chip, log_degree, seed):
    import valida_b200 as vb

    rng = np.random.default_rng(seed)
    h = 1 << log_degree
    w, pwid, prw = oracle.chip_width(chip), oracle.chip_perm_width(chip), oracle.chip_prep_width(chip)
    assert (prw > 0) == (chip in (1, 12))
    main = rng.integers(0, P, size=(h, w), dtype=np.uint32)
    perm = rng.integers(0, P, size=(h, pwid), dtype=np.uint32)
    ch = rng.integers(0, P, size=15, dtype=np.uint32)
    alpha = rng.integers(0, P, size=5, dtype=np.uint32)
    cs = rng.integers(0, P, size=5, dtype=np.uint32)
    pcs = vb.TwoAdicFriPcs(ctx)
    _, mpd = pcs.commit_batches([main])
    _, ppd = pcs.commit_batches([perm])
    ml, pl = pcs.get_ldes(mpd)[0], pcs.get_ldes(ppd)[0]
    prl = None
    if prw:
        _, rpd = pcs.commit_batches([rng.integers(0, P, size=(h, prw), dtype=np.uint32)])
        prl = pcs.get_ldes(rpd)[0]
    exp = oracle.quotient(chip, log_degree, prl.download() if prw else None, ml.download(), pl.download(), cs, ch, alpha)
    got = vb.quotient(ctx, chip, log_degree, prl, ml, pl, cs, ch, alpha).download()
    assert np.array_equal(got, exp)


def test_open_multi_batches_stand_alone(ctx, oracle):
    """vgpu_open = pcs.open_multi_batches on its own: two commitments (mixed heights, one with per-matrix shifts),
    one- and two-point openings, transcript seeded with the two roots — bytes equal to the oracle's."""
    import ctypes as C
    import valida_b200 as vb

    rng = np.random.default_rng(77)
    P = 2013265921
    r0 = [rng.integers(0, P, (1 << 9, 6), dtype=np.uint32), rng.integers(0, P, (1 << 11, 3), dtype=np.uint32), rng.integers(0, P, (1, 4), dtype=np.uint32)]
    r1 = [rng.integers(0, P, (1 << 9, 10), dtype=np.uint32), rng.integers(0, P, (1 << 11, 10), dtype=np.uint32)]
    shifts1 = [961, 961]
    cfg = vb.StarkConfig(ctx, oracle.rc480)
    pcs = cfg.pcs()
    root0, pd0 = pcs.commit_batches(r0)
    root1, pd1 = pcs.commit_shifted_batches(r1, shifts1)
    assert np.array_equal(root0, oracle.commit_batches(r0)) and np.array_equal(root1, oracle.commit_batches(r1, coset_shifts=shifts1))
    L = vb.lib()
    ctx.check(L.vgpu_challenger_reset(ctx._h))
    obs = np.concatenate([root0, root1]).astype(np.uint32)
    ctx.check(L.vgpu_challenger_observe(ctx._h, obs.ctypes.data_as(C.POINTER(C.c_uint32)), obs.size))
    zeta = (C.c_uint32 * 5)()
    ctx.check(L.vgpu_challenger_sample_ext(ctx._h, zeta))
    z = [int(v) for v in zeta]

    def ext_mul_base(e, b):
        return [int(v) * b % P for v in e]

    def gen(log_h):
        return pow(0x1A427A41, 1 << (27 - log_h), P)

    pts0 = [[z, ext_mul_base(z, gen(9))], [z, ext_mul_base(z, gen(11))], [z]]
    z2 = [int(v) for v in oracle.ext_mul(z, z)]
    pts1 = [[z2], [z2]]
    got = pcs.open_multi_batches([(pd0, pts0), (pd1, pts1)])
    # the oracle's challenger: same observations, then the same sample (its value is checked through the opening)
    want = oracle.open([r0, r1], pts0 + pts1, obs, shifts=[1, 1, 1] + shifts1, sample_ext_first=True)
    assert got == want
    pd0.free(); pd1.free()
