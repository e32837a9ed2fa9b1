"""Each stage of a proof split across 2, 4 and 8 ranks, word for word against the oracle on random inputs.

A split proof runs stage code a single GPU never does: the LogUp scan adds the totals of the earlier ranks to a rank's own
prefix sums; the quotient of a rank's shard reads its "next" rows from a peer's shard; the barycentric sums of an opening are
divided by coset between the two halves of the ranks; the inverse denominators cover one rank's run of rows; the FRI layers stay
in row shards until the first one too short to split, which is all-gathered; and each query answer comes from the rank that holds
it.  Whole witness proofs reach these paths only for a few chips and opening shapes, and a wrong byte there does not say which
stage, chip or rank went wrong.  So here every chip's permutation trace and quotient, and openings of every width, of a
base-field point, of a point shared by several rounds and of mixed heights, are compared rank by rank.

The ranks are threads of this process (vb.comm_init_local), several to a GPU when the box has fewer.  Every oracle value is
computed before the ranks start.  Commits, permutation traces and openings are collective on a split context: every rank makes
the same calls in the same order, and frees in the same order, so that the first-fit symmetric heap stays alike on all ranks.

The first part restates the host-side rules that decide what is split (the size model) and checks, without a GPU, that every GPU
case crosses the threshold it is there for."""
import ctypes as C
import os
import re
import time

import numpy as np
import pytest

from test_gpu_large_parity import SCAN_CHUNK, scan_passes
from test_gpu_open_edges import WIDTHS, ext, off_coset

P = 2013265921
CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "valida_b200", "csrc")
RANKS = [2, 4, 8]
NUM_CHIPS = 14
PREP_CHIPS = (1, 12)
RANGE_CHIP = 12


def _src(name):
    return open(os.path.join(CSRC, name)).read()


# ---- the host-side rules, restated ---------------------------------------------------------------------------------------
SPLIT_MIN = int(re.search(r"inline bool vg_split_rows\(const vgpu_ctx\* ctx, uint64_t n\) \{ return vg_sharded\(ctx\) && "
                          r"n >= \(uint64_t\)ctx->comm_size \* (\d+); \}", _src("ctx.h")).group(1))
TRACE_FACTOR = int(re.search(r"inline VgRun vg_trace_run\(const vgpu_ctx\* ctx, uint64_t h\) \{ return vg_run\(h, ctx->comm_size, "
                             r"ctx->comm_rank, vg_split_rows\(ctx, (\d+) \* h\)\); \}", _src("ctx.h")).group(1))
RO_MAXW = int(re.search(r"\bRO_MAXW = (\d+);", _src("open.cu")).group(1))


def split_rows(n, nranks):
    """vg_split_rows: a matrix or vector of n stored rows is cut into row shards when every rank keeps at least SPLIT_MIN."""
    return nranks > 1 and n >= SPLIT_MIN * nranks


def trace_split(h, nranks):
    """A trace of h rows is split (upload_rows, the LogUp sweep) when its LDE of 2h rows is."""
    return split_rows(2 * h, nranks)


def first_coset_columns(w):
    """vg_eval_columns_first_coset: the columns the first-half ranks sum; the second-half ranks sum the rest."""
    return (w + 1) // 2


def columns_summed(w, lde_h, nranks, rank):
    if not split_rows(lde_h, nranks):
        return w
    return first_coset_columns(w) if rank < nranks // 2 else w - first_coset_columns(w)


def reverse_bits(x, bits):
    x = np.asarray(x, dtype=np.int64)
    r = np.zeros_like(x)
    for b in range(bits):
        r |= ((x >> b) & 1) << (bits - 1 - b)
    return r


def shard_natural_rows(gh, nranks, rank):
    """The natural rows a rank's row shard of a gh-row matrix stored bit-reversed holds: stored rows [rank gh/N, (rank+1) gh/N)."""
    n = gh // nranks
    return reverse_bits(np.arange(rank * n, (rank + 1) * n), gh.bit_length() - 1)


def fri_whole_from(log_max, nranks):
    """The length of the first FRI layer (folding down from 2^log_max) too short to split: it is all-gathered, and the reduced
    openings of LDEs of that height join it there."""
    n = 1 << log_max
    while split_rows(n, nranks):
        n //= 2
    return n


def test_model_matches_the_single_definition():
    assert SPLIT_MIN == 4096 and TRACE_FACTOR == 2 and RO_MAXW == 96
    # rank r holds stored rows [r n/N, (r+1) n/N) of a split matrix (shard_natural_rows), all n of a whole one
    assert "return split ? VgRun{rank * (n / nranks), n / nranks, true} : VgRun{0, n, false};" in _src("ctx.h")
    # the rule is defined in ctx.h alone: every other site asks it, and no column-share distribution is left
    for d, _, files in os.walk(CSRC):
        for f in files:
            path = os.path.join(d, f)
            if os.path.relpath(path, CSRC) != "ctx.h":
                src = open(path).read()
                for name in ("vg_split_rows(", "VG_COLS", "col0", "vg_dmat_alloc_dist"):
                    assert name not in src, (path, name)
    assert "uint32_t vg_eval_columns_first_coset(uint32_t w) { return (w + 1) / 2; }" in _src("open.cu")
    assert "const VgRun run = vg_trace_run(ctx, main->gh);" in _src("perm.cu")
    assert "if (!vg_trace_run(ctx, host->height).split) return vgpu_dmat_upload(ctx, host, repr, out);" in _src("api.cu")
    assert "if (vg_trace_run(ctx, mats[i]->gh).split) tall.push_back(i);" in _src("api.cu")       # commit: LDEs of 2h rows
    assert "const bool split = main_lde->dist == VG_ROWS;" in _src("quotient.cu")
    assert "VG_TRY(vg_dmat_alloc_run(ctx, h, 10, split, false, &out));" in _src("quotient.cu")
    assert "out->bitrev_rows = true;" in _src("quotient.cu")
    prover = _src(os.path.join("host", "prover.cc"))
    assert "int32_t rowvec_alloc(vgpu_ctx* ctx, uint64_t n, RowVec* v) {\n    const VgRun run = vg_row_run(ctx, n);" in prover
    assert "if (cur.shard() && !next.shard()) {" in prover


# ---- the GPU cases --------------------------------------------------------------------------------------------------------
PERM_PER_RANK = [1024, 2048, 4096]              # trace rows per rank
QUOTIENT_PER_RANK = [2048, 4096]
OPEN_LDE_PER_RANK = [4096, 8192]                # LDE rows per rank of the width cases
TALL_LOG_H, TALL_RANKS = 23, 2                  # the range chip's LogUp scan past 1024 chunks on each rank


def zero_rows(h, nranks):
    """Rows on both sides of every rank boundary, and the last row."""
    rows = set()
    for r in range(nranks):
        row0 = r * h // nranks
        rows |= {row0, row0 + 1} | ({row0 - 1} if r else set())
    return sorted(rows | {h - 1})


def mixed_heights(nranks):
    """(trace rows, width) of the mixed-height opening: LDEs of 8192 N, 4096 N (split, the last split FRI layer) and 2048 N rows
    (replicated, joins the first whole layer), and short ones."""
    return [(4096 * nranks, 3), (2048 * nranks, 7), (1024 * nranks, 5), (1024 * nranks, 1), (512, 2), (1, 4)]


def test_logup_cases_cross_the_split():
    for n in RANKS:
        hs = [k * n for k in PERM_PER_RANK]
        assert [trace_split(h, n) for h in hs] == [False, True, True]
        # a rank scans exactly one chunk at 2048 N rows, several at 4096 N
        assert [-(-(h // n) // SCAN_CHUNK) for h in hs[1:]] == [1, 2]
        zr = zero_rows(4096 * n, n)
        assert len(zr) == 3 * n and max(zr) == 4096 * n - 1
    # the tall case: each rank's run of chunk sums takes two passes of scan_small_kernel before the rank offset is added
    assert trace_split(1 << TALL_LOG_H, TALL_RANKS) and scan_passes((1 << TALL_LOG_H) // TALL_RANKS) == (2048, 2)


def test_quotient_cases_are_split():
    for n in RANKS:
        assert all(trace_split(k * n, n) for k in QUOTIENT_PER_RANK)


def test_shard_natural_rows_cover_the_matrix():
    """A rank's shard of a bit-reversed matrix is not a run of natural rows: rank r holds the rows i with i mod N = brev(r)."""
    for n in RANKS:
        gh = 2048 * n
        rows = [shard_natural_rows(gh, n, r) for r in range(n)]
        assert np.array_equal(np.sort(np.concatenate(rows)), np.arange(gh))
        for r in range(n):
            assert set((rows[r] % n).tolist()) == {int(reverse_bits(r, n.bit_length() - 1))}


def test_opening_cases_cross_the_split():
    for n in RANKS:
        for per_rank in OPEN_LDE_PER_RANK:
            lde_h = per_rank * n
            assert split_rows(lde_h, n)
            # w = 1 leaves the second-half ranks without a column; every other width gives both halves some
            assert [columns_summed(1, lde_h, n, r) for r in range(n)] == [1] * (n // 2) + [0] * (n // 2)
            assert all(columns_summed(w, lde_h, n, n - 1) > 0 for w in WIDTHS if w > 1)
        assert any(w > RO_MAXW for w in WIDTHS) and 1 in WIDTHS
        # mixed heights: the FRI layer turns whole at 2048 N, where the replicated 2048 N reduced openings join it
        ldes = [2 * h for h, _ in mixed_heights(n)]
        assert 4096 * n in ldes and 2048 * n in ldes
        assert split_rows(4096 * n, n) and not split_rows(2048 * n, n)
        assert fri_whole_from(max(ldes).bit_length() - 1, n) == 2048 * n
        # the base-field point lies on none of the cosets of its split (4096 N, 8192 N) and replicated (2048 N) LDEs
        assert all(off_coset(7, (m * n).bit_length() - 1) for m in (2048, 4096, 8192))


# ---- ranks ---------------------------------------------------------------------------------------------------------------
def _ranks(nranks, oracle, *fns, merkle=None):
    """Each fn(rank, ctx, cfg) in turn on every rank of a fresh split group; the results of each, in rank order."""
    import valida_b200 as vb
    from test_gpu_split_local import _close, _group

    ctxs, cfgs = _group(nranks, oracle)
    try:
        if merkle is not None:
            vb.run_ranks(lambda r, c: c.set_merkle_hash(merkle), ctxs)
        return [vb.run_ranks(lambda r, c: fn(r, c, cfgs[r]), ctxs) for fn in fns]
    finally:
        _close(ctxs)


# ---- LogUp traces --------------------------------------------------------------------------------------------------------
def _perm_cases(oracle, rng, h, chips):
    ch = rng.integers(0, P, size=15, dtype=np.uint32)
    cases = []
    for chip in chips:
        main = rng.integers(0, P, size=(h, oracle.chip_width(chip)), dtype=np.uint32)
        pw = oracle.chip_prep_width(chip)
        prep = rng.integers(0, P, size=(h, pw), dtype=np.uint32) if pw else None
        cases.append((chip, main, prep, ch))
    return cases


def _perm_on_ranks(oracle, nranks, cases):
    """Every case on every rank; the preprocessed trace goes in both as a row shard and as a whole matrix.  Returns the
    differences as (chip, rank, preprocessed as, what)."""
    import valida_b200 as vb

    want = [oracle.perm_trace(chip, main, prep, ch) for chip, main, prep, ch in cases]
    h = cases[0][1].shape[0]

    def go(r, c, cfg):
        out = []
        for k, (chip, main, prep, ch) in enumerate(cases):
            for prep_as in (("rows", "whole") if prep is not None else (None,)):
                dm = c.upload_rows(main)
                dp = None if prep is None else c.upload_rows(prep) if prep_as == "rows" else c.upload(prep)
                perm, cs = vb.generate_permutation_trace(c, chip, dm, dp, ch)
                row0, rows = perm.local_rows()
                got = perm.download()[row0:row0 + rows].copy()
                for m in (perm, dp, dm):
                    if m is not None:
                        m.free()
                out.append((k, prep_as, row0, rows, got, cs))
            c.release_cached()
        return out

    bad = []
    for r, out in enumerate(_ranks(nranks, oracle, go)[0]):
        for k, prep_as, row0, rows, got, cs in out:
            chip, (exp, ecs) = cases[k][0], want[k]
            split = trace_split(h, nranks)
            if (row0, rows) != ((r * h // nranks, h // nranks) if split else (0, h)):
                bad.append((chip, r, prep_as, "rows held", row0, rows))
                continue
            diff = np.flatnonzero((got != exp[row0:row0 + rows]).any(axis=1))
            if diff.size:
                bad.append((chip, r, prep_as, "perm trace rows", (row0 + diff[:4]).tolist(), diff.size))
            if not np.array_equal(cs, ecs):
                bad.append((chip, r, prep_as, "cumulative sum"))
    return bad


@pytest.mark.gpu
@pytest.mark.parametrize("per_rank", PERM_PER_RANK)
@pytest.mark.parametrize("nranks", RANKS)
def test_split_perm_trace_every_chip(oracle, nranks, per_rank):
    """All 14 chips on random traces: at 1024 N rows every rank sweeps the whole trace, at 2048 N one scan chunk of its own
    rows and at 4096 N two, to which it adds the totals of the ranks before it."""
    rng = np.random.default_rng(1000 * nranks + per_rank)
    assert _perm_on_ranks(oracle, nranks, _perm_cases(oracle, rng, per_rank * nranks, range(NUM_CHIPS))) == []


@pytest.mark.gpu
@pytest.mark.parametrize("nranks", RANKS)
def test_split_perm_trace_zero_denominators_at_rank_boundaries(oracle, nranks):
    """The range chip's denominator r1^4 + counter is zero for r1 = 3 and a counter of p - 81 (test_gpu_stages.py).  Such rows
    on both sides of every rank boundary and at the last row must stay zero through each rank's batch inverse and scan."""
    rng = np.random.default_rng(7 + nranks)
    h = 4096 * nranks
    ch = np.zeros(15, dtype=np.uint32)
    ch[5], ch[10] = 3, 7
    main = rng.integers(0, P, size=(h, 2), dtype=np.uint32)
    main[:, 1] = rng.integers(0, P - 81, size=h, dtype=np.uint32)
    zr = zero_rows(h, nranks)
    main[zr, 1] = P - 81
    prep = rng.integers(0, P, size=(h, 1), dtype=np.uint32)
    exp, _ = oracle.perm_trace(RANGE_CHIP, main, prep, ch)
    assert not exp[zr, :5].any()
    assert exp[np.setdiff1d(np.arange(h), zr), :5].any(axis=1).all()
    assert _perm_on_ranks(oracle, nranks, [(RANGE_CHIP, main, prep, ch)]) == []


@pytest.mark.gpu
def test_split_perm_trace_scan_past_1024_chunks_per_rank(oracle):
    """The range chip at 2^23 rows over two ranks: each rank's 2048 chunk sums take two passes of scan_small_kernel, and only
    then is the first rank's total added to the second's rows."""
    rng = np.random.default_rng(23)
    cases = _perm_cases(oracle, rng, 1 << TALL_LOG_H, [RANGE_CHIP])
    t0 = time.perf_counter()
    bad = _perm_on_ranks(oracle, TALL_RANKS, cases)
    print("\n2^%d-row range chip over %d ranks: %.1f s, the oracle's permutation trace included" % (TALL_LOG_H, TALL_RANKS, time.perf_counter() - t0))
    assert bad == []


# ---- quotients -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("per_rank", QUOTIENT_PER_RANK)
@pytest.mark.parametrize("nranks", RANKS)
def test_split_quotient_every_chip(oracle, nranks, per_rank):
    """All 14 chips on random main, permutation and preprocessed traces, with random challenges, alpha and cumulative sum, so
    every constraint contributes.  The LDEs are committed on the split context (row shards in the symmetric heap); from N = 4 on
    a rank's "next" rows lie in a peer's shard.  Each rank's chunk rows are compared at their natural rows, and the ranks together
    must write every row exactly once."""
    import valida_b200 as vb

    h = per_rank * nranks
    log_degree = h.bit_length() - 1
    rng = np.random.default_rng(2000 * nranks + per_rank)
    cases = []
    for chip in range(NUM_CHIPS):
        prw = oracle.chip_prep_width(chip)
        assert (prw > 0) == (chip in PREP_CHIPS)
        mats = [rng.integers(0, P, size=(h, w), dtype=np.uint32) for w in (oracle.chip_width(chip), oracle.chip_perm_width(chip), prw) if w]
        ch = rng.integers(0, P, size=15, dtype=np.uint32)
        alpha = rng.integers(0, P, size=5, dtype=np.uint32)
        cs = rng.integers(0, P, size=5, dtype=np.uint32)
        root, ldes = oracle.commit_batches(mats, want_ldes=True)
        exp = oracle.quotient(chip, log_degree, ldes[2] if prw else None, ldes[0], ldes[1], cs, ch, alpha)
        cases.append((chip, mats, ch, alpha, cs, root, exp))
    pds = {}

    def go(r, c, cfg):
        pcs = vb.TwoAdicFriPcs(c)
        pds[r] = []
        out = []
        for chip, mats, ch, alpha, cs, _, _ in cases:
            root, pd = pcs.commit_batches(mats)
            pds[r].append(pd)
            ldes = pcs.get_ldes(pd)
            q = vb.quotient(c, chip, log_degree, ldes[2] if len(ldes) > 2 else None, ldes[0], ldes[1], cs, ch, alpha)
            got = np.full((h, 10), P, dtype=np.uint32)           # P is no field word: it marks the rows left untouched
            q.download(out=got)
            out.append((root, [m.local_rows() for m in ldes], q.local_rows(), got))
            q.free()
        return out

    def free(r, c, cfg):                                          # only now: a peer read these LDEs
        for pd in pds[r]:
            pd.free()

    results, _ = _ranks(nranks, oracle, go, free)

    bad = []
    for k, (chip, mats, _, _, _, root, exp) in enumerate(cases):
        written = np.zeros(h, dtype=np.int64)
        for r in range(nranks):
            groot, lde_rows, q_rows, got = results[r][k]
            if not np.array_equal(groot, root):
                bad.append((chip, r, "commitment"))
            if any(lr != (r * 2 * h // nranks, 2 * h // nranks) for lr in lde_rows) or q_rows != (r * h // nranks, h // nranks):
                bad.append((chip, r, "rows held", lde_rows, q_rows))
                continue
            nat = shard_natural_rows(h, nranks, r)
            held = (got != P).all(axis=1)
            if not np.array_equal(np.flatnonzero(held), np.sort(nat)) or (got[~held] != P).any():
                bad.append((chip, r, "rows written", np.flatnonzero(held)[:4].tolist()))
            diff = nat[(got[nat] != exp[nat]).any(axis=1)]
            if diff.size:
                bad.append((chip, r, "quotient rows", np.sort(diff)[:4].tolist(), diff.size))
            written += held
        if not (written == 1).all():
            bad.append((chip, "rows not written exactly once", np.flatnonzero(written != 1)[:4].tolist()))
    assert bad == []


# ---- openings ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mmcs(built):
    from poseidon_mmcs import PoseidonOracle

    return PoseidonOracle()


def open_split_and_compare(oracle, nranks, rounds, merkle=None):
    """rounds: [(matrices, [points of each matrix])].  Every rank commits every round, seeds the challenger with the roots and
    opens; each rank's roots and bytes must be the oracle's (computed first)."""
    import valida_b200 as vb

    roots = [oracle.commit_batches(mats) for mats, _ in rounds]
    obs = np.concatenate(roots).astype(np.uint32)
    want = oracle.open([mats for mats, _ in rounds], [p for _, pts in rounds for p in pts], obs)

    def go(r, c, cfg):
        pcs = cfg.pcs()
        committed = [pcs.commit_batches(mats) for mats, _ in rounds]
        L = vb.lib()
        c.check(L.vgpu_challenger_reset(c._h))
        c.check(L.vgpu_challenger_observe(c._h, obs.ctypes.data_as(C.POINTER(C.c_uint32)), obs.size))
        got = pcs.open_multi_batches([(pd, pts) for (_, pd), (_, pts) in zip(committed, rounds)])
        for _, pd in committed:
            pd.free()
        c.release_cached()
        return [root for root, _ in committed], got

    results, = _ranks(nranks, oracle, go, merkle=merkle)
    bad = [r for r, (got_roots, _) in enumerate(results) if not all(np.array_equal(a, b) for a, b in zip(got_roots, roots))]
    assert bad == [], ("ranks whose roots differ", bad)
    bad = [r for r, (_, got) in enumerate(results) if got != want]
    assert bad == [], ("ranks whose opening differs", bad)


@pytest.mark.gpu
@pytest.mark.parametrize("npoints", [1, 2])
@pytest.mark.parametrize("lde_per_rank", OPEN_LDE_PER_RANK)
@pytest.mark.parametrize("nranks", RANKS)
def test_split_open_every_width(oracle, nranks, lde_per_rank, npoints):
    """The widths of test_gpu_open_edges.py on split LDEs: odd widths divide unevenly between the cosets, w = 1 leaves the
    second-half ranks without a column, and widths above RO_MAXW take several reduced-opening launches on every rank."""
    rng = np.random.default_rng(3000 + 100 * nranks + lde_per_rank // 1024 + npoints)
    h = lde_per_rank * nranks // 2
    mats = [rng.integers(0, P, (h, w), dtype=np.uint32) for w in WIDTHS]
    z = ext(rng)
    open_split_and_compare(oracle, nranks, [(mats, [[z] if npoints == 1 else [z, ext(rng)] for _ in mats])])


def _base_point_rounds(rng, nranks):
    """The shape of test_open_base_field_point with split (4096 N, 8192 N rows) and replicated (2048 N rows) LDEs."""
    zb, ze = [7, 0, 0, 0, 0], ext(rng)
    n = nranks
    r0 = [rng.integers(0, P, (2048 * n, 7), dtype=np.uint32), rng.integers(0, P, (2048 * n, 40), dtype=np.uint32),
          rng.integers(0, P, (1024 * n, 3), dtype=np.uint32)]
    r1 = [rng.integers(0, P, (4096 * n, 97), dtype=np.uint32), rng.integers(0, P, (4096 * n, 5), dtype=np.uint32)]
    return [(r0, [[zb, ze], [ze], [zb]]), (r1, [[zb], [ze, zb]])]


@pytest.mark.gpu
@pytest.mark.parametrize("nranks", RANKS)
def test_split_open_base_field_point(oracle, nranks):
    """A base-field point takes coset_minus_point_kernel and the ext5 batch inverse over each rank's own run of rows; it shares
    a height with an extension point, and one matrix is opened at both."""
    open_split_and_compare(oracle, nranks, _base_point_rounds(np.random.default_rng(4000 + nranks), nranks))


@pytest.mark.gpu
@pytest.mark.parametrize("nranks", RANKS)
def test_split_open_shared_point_across_rounds(oracle, nranks):
    """One point in three rounds of split matrices: each round's reduced openings continue the alpha powers where the previous
    round of that height stopped, on every rank's shard."""
    rng = np.random.default_rng(5000 + nranks)
    z, z2 = ext(rng), ext(rng)
    rounds = []
    for widths in ([97, 5], [64], [3, 33]):
        mats = [rng.integers(0, P, (2048 * nranks, w), dtype=np.uint32) for w in widths] + [rng.integers(0, P, (4096 * nranks, 2), dtype=np.uint32)]
        rounds.append((mats, [[z] for _ in widths] + [[z, z2]]))
    open_split_and_compare(oracle, nranks, rounds)


def _mixed_round(rng, nranks):
    z = ext(rng)
    mats = [rng.integers(0, P, (h, w), dtype=np.uint32) for h, w in mixed_heights(nranks)]
    return [(mats, [[z, ext(rng)] if i % 2 else [z] for i in range(len(mats))])]


@pytest.mark.gpu
@pytest.mark.parametrize("nranks", RANKS)
def test_split_open_mixed_heights(oracle, nranks):
    """LDEs of 8192 N and 4096 N rows (split) and of 2048 N rows (replicated) in one round: the reduced openings of the
    2048 N matrices join the FRI layer where it is all-gathered and turns whole."""
    open_split_and_compare(oracle, nranks, _mixed_round(np.random.default_rng(6000 + nranks), nranks))


@pytest.mark.gpu
@pytest.mark.parametrize("nranks", RANKS)
def test_split_open_mixed_heights_poseidon16(mmcs, nranks):
    """The mixed-height opening with Poseidon-16 Merkle trees: the split sub-trees and the FRI layer trees hash field-natively."""
    import valida_b200 as vb

    open_split_and_compare(mmcs, nranks, _mixed_round(np.random.default_rng(7000 + nranks), nranks), merkle=vb.MERKLE_POSEIDON16)
