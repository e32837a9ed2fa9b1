"""The stages of large proofs, word for word against the oracle, on the kernel paths that only tall inputs reach.

A verifier that accepts a proof does not show that the prover computed what it should: a wrong digest in a sub-tree that no
query opens, or a wrong value at an LDE row no query touches, leaves every opened path consistent.  So the sizes below are
compared exactly, either with the live oracle or with the recorded digests of oracle proofs (tests/golden/
large_proof_digests.json, written by tests/golden/make_large_proof_digests.py):

  * the LogUp prefix scan past 1024 chunks, where scan_small_kernel carries its running sum from one pass to the next;
  * barycentric sums over several tiles per CTA (bary_kernel's cp.async double buffer), also on a column grid;
  * the quotient of every chip at 2^17 rows and of three chips at 2^20;
  * Keccak and Poseidon-16 trees above 2^18 leaves, with shorter matrices injected in the per-layer launches and in the fused
    tail, and an opening whose query paths are rebuilt over a tall tree;
  * whole proofs at 2^17 to 2^22 rows, on one GPU and split over several ranks, each stage of the 2^22 proof on its own.

The first part restates the host-side launch choices in plain Python (the size model) and checks, without a GPU, that every
GPU case crosses the threshold of the path it is there for.  SM_COUNT is the H100 SXM's; a GPU test checks it."""
import os
import re
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

from make_large_proof_digests import assert_matches_golden, fib_n, load, matrix_digest  # noqa: E402

P = 2013265921
GEN = 31
CSRC = os.path.join(HERE, "..", "valida_b200", "csrc")
SM_COUNT = 132


def _src(name):
    return open(os.path.join(CSRC, name)).read()


def _const(src, name):
    return int(re.search(r"\b%s = (\d+)\b" % name, src).group(1))


# ---- the host-side choices, restated ------------------------------------------------------------------------------------
SCAN_THREADS, SCAN_PER_THREAD = 256, 8
SCAN_CHUNK = SCAN_THREADS * SCAN_PER_THREAD
SCAN_SMALL_BLOCK = 1024                       # chunk sums scanned per pass of scan_small_kernel
BARY_COLS, BARY_WARPS, BARY_TILE = 2, 16, 1024
BARY_CHUNKS = BARY_TILE // 128
TAIL_FUSE = 1 << 15
VG_TREE_DROP = 8


def scan_passes(h):
    """(chunks, passes of scan_small_kernel) of vg_prefix_sum_columns over h rows."""
    chunks = -(-h // SCAN_CHUNK)
    return chunks, -(-chunks // SCAN_SMALL_BLOCK) if chunks > 1 else 0


def bary_grid(w, h, sm=SM_COUNT):
    """bary_kernel's launch for w columns of an LDE whose first coset has h rows: (by, cpg, rs, bx, ntiles)."""
    by = (w + 31) // 32
    cpg = 2 * (((w + by - 1) // by + 1) // 2)
    rs = min(BARY_CHUNKS, BARY_WARPS // (cpg // BARY_COLS))
    ntiles = h // BARY_TILE
    bx = min(ntiles, max(1, sm // by))
    return by, cpg, rs, bx, ntiles


def tree_joins(log_lde, shorter_logs):
    """Where each shorter matrix (log LDE height) joins a tree whose tallest LDE has 2^log_lde rows: (layer, kernel), with kernel
    "layer" for a compress_layer_kernel / p16_layer_kernel launch and "tail" inside the fused tail."""
    return [(log_lde - s, "layer" if (1 << s) > TAIL_FUSE else "tail") for s in shorter_logs]


def test_model_constants_match_the_source():
    perm, opn, mrk = _src("perm.cu"), _src("open.cu"), _src("merkle.cu")
    assert (_const(perm, "SCAN_THREADS"), _const(perm, "SCAN_PER_THREAD")) == (SCAN_THREADS, SCAN_PER_THREAD)
    assert "SCAN_CHUNK = SCAN_THREADS * SCAN_PER_THREAD" in perm
    assert "__launch_bounds__(1024) scan_small_kernel" in perm and "base += 1024" in perm
    assert "scan_small_kernel<<<dim3(1, ncols), 1024" in perm
    for name, v in (("BARY_COLS", BARY_COLS), ("BARY_WARPS", BARY_WARPS), ("BARY_TILE", BARY_TILE)):
        assert _const(opn, name) == v, name
    assert "BARY_CHUNKS = BARY_TILE / 128" in opn
    for line in ("const unsigned by = (w + 31) / 32;", "p.cpg = 2 * (((w + by - 1) / by + 1) / 2);",
                 "p.rs = std::min<uint32_t>(BARY_CHUNKS, BARY_WARPS / (p.cpg / BARY_COLS));", "const uint64_t ntiles = rows / BARY_TILE;",
                 "std::min<uint64_t>(ntiles, std::max<uint64_t>(1, (uint64_t)ctx->sm_count / by));"):
        assert line in opn, line
    assert "constexpr uint64_t TAIL_FUSE = 1u << %d;" % (TAIL_FUSE.bit_length() - 1) in mrk
    assert "if (p.ccount <= TAIL_FUSE) {" in mrk
    assert _const(_src("merkle.h"), "VG_TREE_DROP") == VG_TREE_DROP


# ---- the GPU cases --------------------------------------------------------------------------------------------------------
RANGE_CHIP, MEMORY_CHIP = 12, 2
SCAN_CASES = [(RANGE_CHIP, 21), (RANGE_CHIP, 22), (MEMORY_CHIP, 24)]
ZERO_ROWS = [SCAN_CHUNK - 1, SCAN_CHUNK, SCAN_CHUNK * SCAN_SMALL_BLOCK - 1, SCAN_CHUNK * SCAN_SMALL_BLOCK]
ZERO_LOG_H = 22
# (log height of the opened matrices, widths, points per matrix: 1, 2, or "base" for one base-field point)
OPEN_CASES = [(15, (200, 130), 1), (15, (200, 130), 2), (18, (1, 14, 33), 1), (18, (1, 14, 33), 2), (18, (5,), "base")]
QUOTIENT_CASES = [(c, 17) for c in range(14)] + [(0, 20), (2, 20), (10, 20)]
# tallest log LDE height -> [(log LDE height, width)] of the shorter matrices
KECCAK_TREES = {
    20: [(18, 2), (16, 1), (15, 3), (9, 2)],
    25: [(24, 1), (16, 2), (15, 1), (4, 3)],
}
KECCAK_OPEN_TREE = (23, [(21, 3), (17, 1), (12, 2)])      # an opening: its paths are rebuilt below layer VG_TREE_DROP
POSEIDON_TREES = {20: [(18, 2), (16, 1), (15, 3), (9, 2)]}
SPLIT_RANKS = [2, 4, 8]


def test_scan_cases_run_past_one_pass():
    assert [scan_passes(1 << lh) for _, lh in SCAN_CASES] == [(1024, 1), (2048, 2), (8192, 8)]
    # the zero rows sit on both sides of a chunk boundary and of the first pass boundary of the chunk sums
    chunks = [r // SCAN_CHUNK for r in ZERO_ROWS]
    assert chunks == [0, 1, SCAN_SMALL_BLOCK - 1, SCAN_SMALL_BLOCK]
    assert max(ZERO_ROWS) < 1 << ZERO_LOG_H and scan_passes(1 << ZERO_LOG_H)[1] == 2


def test_open_cases_run_several_tiles_per_cta():
    for log_h, widths, _ in OPEN_CASES:
        for w in widths:
            by, cpg, rs, bx, ntiles = bary_grid(w, 1 << log_h)
            assert ntiles > bx, (log_h, w, bx, ntiles)       # a CTA's second tile: the double buffer's other half
    assert {bary_grid(w, 1 << 15)[0] for w in (200, 130)} == {7, 5}
    assert bary_grid(33, 1 << 18)[0] == 2 and bary_grid(14, 1 << 18)[:3] == (1, 14, 2)
    # the largest exact comparison before this file: 2^17 rows at <= 32 columns, 2^14 at 200 columns, one tile per CTA
    assert bary_grid(32, 1 << 17)[3:] == (128, 128) and bary_grid(200, 1 << 14)[3:] == (16, 16)


def test_tree_cases_inject_in_layer_launches_and_in_the_tail():
    for log_lde, shorter in list(KECCAK_TREES.items()) + [KECCAK_OPEN_TREE] + list(POSEIDON_TREES.items()):
        assert log_lde > 18
        kinds = {k for _, k in tree_joins(log_lde, [s for s, _ in shorter])}
        assert kinds == {"layer", "tail"}, log_lde
        # the last per-layer launch (2 * TAIL_FUSE nodes) and the first fused layer (TAIL_FUSE nodes) both take an injection,
        # except in the opening case, which injects into the dropped layers instead
        if log_lde != KECCAK_OPEN_TREE[0]:
            assert {16, 15} <= {s for s, _ in shorter}
    log_lde, shorter = KECCAK_OPEN_TREE
    assert any(j < VG_TREE_DROP and k == "layer" for j, k in tree_joins(log_lde, [s for s, _ in shorter]))
    assert any(j >= VG_TREE_DROP and k == "tail" for j, k in tree_joins(log_lde, [s for s, _ in shorter]))


def test_golden_proofs_reach_tall_trees_and_scans(built):
    """Fibonacci with 2^k CPU rows has a memory chip of 2^(k+2) rows: the 2^20 proofs (Keccak and Poseidon) commit 2^23 LDE
    leaves, and the 2^22 proof's memory chip scans 2^24 rows (eight passes)."""
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(fib_n(20)), initial_fp=0x1000)
    assert t.main[0].shape[0] == 1 << 20 and t.main[MEMORY_CHIP].shape[0] == 1 << 22
    assert max(m.shape[0] for m in t.main) * 2 == 1 << 23
    assert scan_passes(1 << 24)[1] == 8 and scan_passes(1 << 22)[1] == 2
    assert set(load()) == {"fib_2p17", "fib_2p20", "fib_2p22", "mixed_20000", "config5_16000", "p16_fib_2p17", "p16_fib_2p20"}


@pytest.mark.gpu
def test_sm_count_is_the_modelled_one():
    import torch

    assert torch.cuda.get_device_properties(0).multi_processor_count == SM_COUNT


# ---- LogUp scans --------------------------------------------------------------------------------------------------------
def _prep_random(oracle, rng, chip, h):
    pw = oracle.chip_prep_width(chip)
    return rng.integers(0, P, size=(h, pw), dtype=np.uint32) if pw else None


def _perm_compare(ctx, oracle, chip, main, prep, ch):
    import valida_b200 as vb

    exp, ecs = oracle.perm_trace(chip, main, prep, ch)
    dm = ctx.upload(main)
    dp = ctx.upload(prep) if prep is not None else None
    got, cs = vb.generate_permutation_trace(ctx, chip, dm, dp, ch)
    g = got.download()
    for m in (dm, dp, got):
        if m is not None:
            m.free()
    ctx.release_cached()
    bad = np.flatnonzero((g != exp).any(axis=1))
    assert bad.size == 0, ("first differing rows", bad[:8], bad.size)
    assert np.array_equal(cs, ecs)
    return exp


@pytest.mark.gpu
@pytest.mark.parametrize("chip,log_h", SCAN_CASES)
def test_perm_trace_scan_past_1024_chunks(ctx, oracle, chip, log_h):
    rng = np.random.default_rng(100 + log_h)
    h = 1 << log_h
    ch = rng.integers(0, P, size=15, dtype=np.uint32)
    main = rng.integers(0, P, size=(h, oracle.chip_width(chip)), dtype=np.uint32)
    _perm_compare(ctx, oracle, chip, main, _prep_random(oracle, rng, chip, h), ch)


@pytest.mark.gpu
def test_perm_trace_zero_denominators_at_chunk_and_pass_boundaries(ctx, oracle):
    """The range chip's denominator is r1^4 + counter: with r1 = 3 a counter of p - 81 makes it zero, and the batch inverse must
    leave it zero.  Such rows sit on both sides of a chunk boundary and of the first pass boundary of the chunk sums."""
    rng = np.random.default_rng(7)
    h = 1 << ZERO_LOG_H
    ch = np.zeros(15, dtype=np.uint32)
    ch[5], ch[10] = 3, 7
    main = rng.integers(0, P, size=(h, 2), dtype=np.uint32)
    main[:, 1] = rng.integers(0, P - 81, size=h, dtype=np.uint32)
    main[ZERO_ROWS, 1] = P - 81
    exp = _perm_compare(ctx, oracle, RANGE_CHIP, main, np.zeros((h, 1), dtype=np.uint32), ch)
    assert not exp[ZERO_ROWS, :5].any()
    assert exp[[r - 1 for r in ZERO_ROWS if r - 1 not in ZERO_ROWS], :5].any(axis=1).all()


# ---- barycentric sums ---------------------------------------------------------------------------------------------------
def _off_coset(z, log_lde):
    return pow(z * pow(GEN, P - 2, P) % P, 1 << log_lde, P) != 1


@pytest.mark.gpu
@pytest.mark.parametrize("log_h,widths,points", OPEN_CASES)
def test_open_multi_tile_barycentric_sums(ctx, oracle, log_h, widths, points):
    from test_gpu_open_edges import open_and_compare

    rng = np.random.default_rng(200 + log_h + sum(widths))
    mats = [rng.integers(0, P, (1 << log_h, w), dtype=np.uint32) for w in widths]
    ext = lambda: [int(v) for v in rng.integers(0, P, 5)]                  # noqa: E731
    if points == "base":
        zb = [7, 0, 0, 0, 0]
        assert _off_coset(7, log_h + 1)
        pts = [[zb]] * len(mats)
    else:
        z = ext()
        pts = [[z] if points == 1 else [z, ext()] for _ in mats]
    open_and_compare(ctx, oracle, [(mats, pts)])
    ctx.release_cached()


# ---- quotients ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("chip,log_degree", QUOTIENT_CASES)
def test_quotient_random_traces_tall(ctx, oracle, chip, log_degree):
    from test_gpu_stages import quotient_random_traces

    quotient_random_traces(ctx, oracle, chip, log_degree, 300 + 100 * log_degree + chip)
    ctx.release_cached()


# ---- tall trees -----------------------------------------------------------------------------------------------------------
def _tree_mats(log_lde, shorter, seed):
    """Trace matrices whose LDEs have the given heights; a shorter matrix sits between two of the tallest."""
    rng = np.random.default_rng(seed)
    tall = [rng.integers(0, P, (1 << (log_lde - 1), 1), dtype=np.uint32) for _ in range(2)]
    short = [rng.integers(0, P, (1 << (s - 1), w), dtype=np.uint32) for s, w in shorter]
    return tall[:1] + short + tall[1:]


@pytest.mark.gpu
@pytest.mark.parametrize("log_lde", sorted(KECCAK_TREES))
def test_keccak_tall_tree_roots(ctx, oracle, log_lde):
    import valida_b200 as vb

    mats = _tree_mats(log_lde, KECCAK_TREES[log_lde], log_lde)
    root, pd = vb.TwoAdicFriPcs(ctx).commit_batches(mats)
    pd.free()
    ctx.release_cached()
    assert np.array_equal(root, oracle.commit_batches(mats))


@pytest.mark.gpu
def test_keccak_tall_tree_opening(ctx, oracle):
    """Root and opening of a 2^23-leaf tree: the 40 query paths are rebuilt below the kept layers, through an injection there."""
    from test_gpu_open_edges import open_and_compare

    log_lde, shorter = KECCAK_OPEN_TREE
    mats = _tree_mats(log_lde, shorter, log_lde)
    z = [int(v) for v in np.random.default_rng(23).integers(0, P, 5)]
    open_and_compare(ctx, oracle, [(mats, [[z]] * len(mats))])
    ctx.release_cached()


@pytest.fixture(scope="module")
def mmcs(built):
    from poseidon_mmcs import PoseidonOracle

    return PoseidonOracle()


@pytest.fixture(scope="module")
def p16(built, oracle):
    """A context of its own in Poseidon-16 mode, and its StarkConfig."""
    import valida_b200 as vb

    ctx = vb.Context(0)
    cfg = vb.StarkConfig(ctx, oracle.rc480)
    ctx.set_merkle_hash(vb.MERKLE_POSEIDON16)
    yield ctx, cfg
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("log_lde", sorted(POSEIDON_TREES))
def test_poseidon_tall_tree_roots(p16, mmcs, log_lde):
    ctx, cfg = p16
    mats = _tree_mats(log_lde, POSEIDON_TREES[log_lde], 1000 + log_lde)
    root, pd = cfg.pcs().commit_batches(mats)
    pd.free()
    ctx.release_cached()
    assert np.array_equal(root, mmcs.commit_batches(mats))


# ---- whole proofs against the recorded oracle proofs -------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("log_rows", [17, 20])
def test_poseidon_fibonacci_proof_equals_golden(p16, log_rows):
    import valida_b200 as vb

    ctx, cfg = p16
    t = vb.run_program(vb.fib_program(fib_n(log_rows)), initial_fp=0x1000)
    assert t.main[0].shape[0] == 1 << log_rows
    try:
        proof = vb.prove_machine(cfg, t)
    finally:
        ctx.release_cached()
    assert_matches_golden(proof, "p16_fib_2p%d" % log_rows)


@pytest.fixture(scope="module")
def fib20(built):
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(fib_n(20)), initial_fp=0x1000)
    assert t.main[0].shape[0] == 1 << 20
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("nranks", SPLIT_RANKS)
def test_split_fibonacci_2p20_equals_golden(oracle, fib20, nranks):
    """One proof over 2, 4 or 8 thread ranks: every rank sweeps many scan chunks, barycentric tiles and tree layers of its
    shard, and every rank returns the oracle's bytes."""
    import valida_b200 as vb
    from test_gpu_split_local import _close, _group

    ctxs, cfgs = _group(nranks, oracle)
    try:
        proofs = vb.run_ranks(lambda r, c: vb.prove_machine(cfgs[r], fib20), ctxs)
    finally:
        _close(ctxs)
    for p in proofs:
        assert_matches_golden(p, "fib_2p20")


@pytest.mark.gpu
def test_fibonacci_2p22_stages_equal_golden(ctx, oracle):
    """Each stage of the 2^22 proof recomputed from the recorded transcript: the main commitment, and per chip the permutation
    trace, the cumulative sum and the quotient chunks.  A wrong proof names its stage and chip here."""
    import valida_b200 as vb

    g = load()["fib_2p22"]
    tr = {k: np.array(v, dtype=np.uint32) for k, v in g["transcript"].items()}
    t = vb.run_program(vb.fib_program(fib_n(22)), initial_fp=0x1000)
    pcs = vb.TwoAdicFriPcs(ctx)
    main_root, main_pd = pcs.commit_batches(t.main)
    assert np.array_equal(main_root, tr["main_commit"]), "main commitment"
    main_ldes = pcs.get_ldes(main_pd)
    bad = []
    try:
        for chip in range(14):
            want = g["chips"][chip]
            prep = t.preprocessed[0] if chip == 1 else t.preprocessed[1] if chip == 12 else None
            dm = ctx.upload(t.main[chip])
            dp = ctx.upload(prep) if prep is not None else None
            perm, cs = vb.generate_permutation_trace(ctx, chip, dm, dp, tr["perm_challenges"])
            if matrix_digest(perm.download()) != want["perm_trace"]:
                bad.append((chip, "perm_trace"))
            if [int(v) for v in cs] != want["cumulative_sum"]:
                bad.append((chip, "cumulative_sum"))
            _, perm_pd = pcs.commit_batches([perm])
            prep_pd = pcs.commit_batches([prep])[1] if prep is not None else None
            q = vb.quotient(ctx, chip, t.main[chip].shape[0].bit_length() - 1, pcs.get_ldes(prep_pd)[0] if prep is not None else None,
                            main_ldes[chip], pcs.get_ldes(perm_pd)[0], np.array(want["cumulative_sum"], dtype=np.uint32),
                            tr["perm_challenges"], tr["alpha"])
            if matrix_digest(q.download()) != want["quotient_chunks"]:
                bad.append((chip, "quotient_chunks"))
            for m in (dm, dp, perm, q, perm_pd, prep_pd):
                if m is not None:
                    m.free()
            ctx.release_cached()
    finally:
        main_pd.free()
        ctx.release_cached()
    assert bad == []
