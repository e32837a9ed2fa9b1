"""Merkle trees that keep only their upper layers (VG_TREE_DROP = 8 in valida_b200/csrc/merkle.h): the query phase rebuilds
the lower levels of every authentication path on the device from the leaves.  Checked here where the other tests do not reach:
trees of depth just below, at and just above the dropped layers, shorter matrices joining below, at and above them, FRI layers
shorter than one rebuilt sub-tree, the smallest split of a proof over 2 / 4 / 8 ranks, Fibonacci 2^24 (BASELINE config 4) proven
from traces the caller holds on the device, and the context's memory counters."""
import ctypes as C

import numpy as np
import pytest

P = 2013265921
DROP = 8                                      # VG_TREE_DROP
pytestmark = pytest.mark.gpu


def ext(rng):
    return [int(v) for v in rng.integers(0, P, 5)]


def open_and_compare(ctx, oracle, rounds, rc):
    """rounds: [(matrices, [points of each matrix])].  Commits every round, seeds a challenger built from the round constants `rc`
    with the roots and opens: the bytes must equal the oracle's opening."""
    import valida_b200 as vb

    pcs = vb.StarkConfig(ctx, rc).pcs()
    pds, roots = [], []
    for mats, _ in rounds:
        root, pd = pcs.commit_batches(mats)
        assert np.array_equal(root, oracle.commit_batches(mats)), [m.shape for m in mats]
        pds.append(pd)
        roots.append(root)
    obs = np.concatenate(roots).astype(np.uint32)
    L = vb.lib()
    ctx.check(L.vgpu_challenger_reset(ctx._h))
    ctx.check(L.vgpu_challenger_observe(ctx._h, obs.ctypes.data_as(C.POINTER(C.c_uint32)), obs.size))
    try:
        got = pcs.open_multi_batches([(pd, pts) for pd, (_, pts) in zip(pds, rounds)])
    finally:
        for pd in pds:
            pd.free()
    want = oracle.open([mats for mats, _ in rounds], [p for _, pts in rounds for p in pts], obs, rc=rc)
    assert got == want


def round_constants(seed):
    """A challenger of its own per seed: other query indices, so other leaves and sub-trees are rebuilt."""
    return np.random.default_rng(seed).integers(0, P, 480, dtype=np.uint32)


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("log_lde", [DROP - 1, DROP, DROP + 1])
def test_open_tree_depth_around_the_dropped_layers(ctx, oracle, log_lde, seed):
    """One tree of depth DROP - 1 (nothing but the root is kept), DROP (the same) and DROP + 1 (the root and the layer below);
    its FRI layers are all shorter than one rebuilt sub-tree.  The leaves are rows of two sponge blocks (45 words)."""
    rng = np.random.default_rng(100 * log_lde + seed)
    h = 1 << (log_lde - 1)                    # the committed LDE doubles the height
    mats = [rng.integers(0, P, (h, 40), dtype=np.uint32), rng.integers(0, P, (h, 5), dtype=np.uint32)]
    z = ext(rng)
    open_and_compare(ctx, oracle, [(mats, [[z], [z, ext(rng)]])], round_constants(seed))


@pytest.mark.parametrize("seed", [4, 5, 6])
def test_open_mixed_heights_inject_below_at_and_above_the_dropped_layers(ctx, oracle, seed):
    """A tree of depth 12 whose shorter matrices join at levels 1, 7 (rebuilt), 8 (the first kept layer) and 10, one of them with
    rows of two sponge blocks; a second round of depth 9 with a matrix joining at level 2.  The main tree's FRI layers run from
    2^11 pairs down, through every depth the rebuild handles."""
    rng = np.random.default_rng(seed)
    lde = 1 << 12
    heights_widths = [(lde, 3), (lde, 70), (lde >> 1, 2), (lde >> 7, 40), (lde >> 8, 1), (lde >> 10, 6)]
    mats = [rng.integers(0, P, (h // 2, w), dtype=np.uint32) for h, w in heights_widths]
    r2 = [rng.integers(0, P, (1 << 8, 9), dtype=np.uint32), rng.integers(0, P, (1 << 6, 4), dtype=np.uint32)]
    z = ext(rng)
    open_and_compare(ctx, oracle, [(mats, [[z]] * len(mats)), (r2, [[z, ext(rng)], [ext(rng)]])], round_constants(seed))


@pytest.mark.parametrize("nranks", [2, 4, 8])
def test_split_proof_at_the_smallest_split(ctx, oracle, nranks):
    """A Fibonacci run whose tallest chip (memory) has exactly 4096 * nranks LDE rows: the smallest trees that are split, with 4096
    leaves per rank, and a first FRI layer split into runs of 2048 pairs.  Every rank rebuilds the paths of the leaves in its run
    and returns the single-GPU bytes."""
    import torch
    import valida_b200 as vb

    log_cpu = 9 + nranks.bit_length() - 1
    t = vb.run_program(vb.fib_program(((1 << log_cpu) - 17) // 7), initial_fp=0x1000)
    assert t.main[2].shape[0] * 2 == 4096 * nranks and max(m.shape[0] for m in t.main) == t.main[2].shape[0]
    single = vb.prove_machine(vb.StarkConfig(ctx, oracle.rc480), t)
    assert single == oracle.prove(t.main, t.preprocessed, debug_checks=False).cbor()
    k = torch.cuda.device_count()
    ctxs = [vb.Context(i % k) for i in range(nranks)]
    try:
        vb.comm_init_local(ctxs)
        cfgs = [vb.StarkConfig(c, oracle.rc480) for c in ctxs]
        assert all(p == single for p in vb.run_ranks(lambda r, c: vb.prove_machine(cfgs[r], t), ctxs))
    finally:
        for c in ctxs:
            c.close()


def test_prove_config4_from_device_memory_on_one_gpu(ctx, oracle):
    """BASELINE config 4 (Fibonacci, 2^24 CPU rows; memory chip 2^26 rows, LDE 2^27) through vgpu_prove_device, from traces
    uploaded by the caller and from the device witness: the bytes of vgpu_prove on the same traces, accepted by both verifiers."""
    import valida_b200 as vb

    log = vb.run_program_log(vb.fib_program(((1 << 24) - 17) // 7))
    t = log.traces()
    assert t.main[0].shape[0] == 1 << 24 and t.main[2].shape[0] == 1 << 26
    cfg = vb.StarkConfig(ctx, oracle.rc480)
    ctx.release_cached()
    try:
        proof = vb.prove_machine(cfg, t)
        ctx.release_cached()
        dm = [ctx.upload(m) for m in t.main]
        dp = [ctx.upload(m) for m in t.preprocessed]
        assert vb.prove_machine(cfg, t, device_resident=(dm, dp)) == proof
        for m in dm + dp:
            m.free()
        ctx.release_cached()
        dm, dp = log.witness_device(ctx)
        assert vb.prove_machine(cfg, t, device_resident=(dm, dp)) == proof
        for m in dm + dp:
            m.free()
        vb.verify_machine(cfg, proof, t.preprocessed)
    finally:
        ctx.release_cached()      # the proofs filled most of the 80 GB: later tests open contexts of their own
    assert oracle.verify(proof, t.preprocessed) == 0


def test_memory_stats_after_a_proof(ctx, oracle):
    """Live bytes return to their value from before a proof; release_cached() empties the cache and leaves live bytes alone."""
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(((1 << 14) - 17) // 7), initial_fp=0x1000)
    cfg = vb.StarkConfig(ctx, oracle.rc480)
    dm = [ctx.upload(m) for m in t.main]
    dp = [ctx.upload(m) for m in t.preprocessed]
    first = vb.prove_machine(cfg, t, device_resident=(dm, dp))    # tables a context builds once are made here
    ctx.memory_stats(reset=True)                                  # returns the counts from before the reset
    before = ctx.memory_stats()
    assert before["peak"] == before["live"]
    assert vb.prove_machine(cfg, t, device_resident=(dm, dp)) == first
    after = ctx.memory_stats()
    assert after["live"] == before["live"]
    assert after["peak"] > after["live"] and after["cached"] > 0
    ctx.release_cached()
    released = ctx.memory_stats()
    assert released["cached"] == 0 and released["live"] == before["live"]


def test_peak_memory_of_a_2p22_device_proof(ctx, oracle):
    """Fibonacci 2^22 (BASELINE config 3) through vgpu_prove_device: the peak live bytes stay within the caller's traces, the
    LDEs of the four commitments and a scratch allowance."""
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(((1 << 22) - 17) // 7), initial_fp=0x1000)
    assert t.main[0].shape[0] == 1 << 22 and t.main[2].shape[0] == 1 << 24
    cfg = vb.StarkConfig(ctx, oracle.rc480)
    ctx.release_cached()
    dm = [ctx.upload(m) for m in t.main]
    dp = [ctx.upload(m) for m in t.preprocessed]
    try:
        ctx.memory_stats(reset=True)
        proof = vb.prove_machine(cfg, t, device_resident=(dm, dp))
        peak = ctx.memory_stats()["peak"]
    finally:
        for m in dm + dp:
            m.free()
        ctx.release_cached()
    assert oracle.verify(proof, t.preprocessed) == 0
    traces = sum(m.nbytes for m in t.main) + sum(m.nbytes for m in t.preprocessed)
    # committed LDEs (blowup 2): preprocessed, main, permutation (oracle.chip_perm_width base columns) and quotient chunks
    # (10 columns) of every chip
    ldes = sum(2 * m.nbytes for m in t.preprocessed)
    for i, m in enumerate(t.main):
        ldes += 2 * m.shape[0] * 4 * (m.shape[1] + oracle.chip_perm_width(i) + 10)
    print("2^22 device proof: peak live %.3f GB = traces %.3f GB + LDEs %.3f GB + %.3f GB"
          % (peak / 1e9, traces / 1e9, ldes / 1e9, (peak - traces - ldes) / 1e9))
    # Allowance: 4.5 GiB (4.83 GB).  Measured on an H100 80GB HBM3: 4.05 GB above traces + LDEs at the peak.  The scratch is not
    # itemised; its largest parts by size are the ext5 vectors of the opening (20 B per LDE row: the inverse denominators of the
    # three opening points at the memory chip's 2^25 rows are 2.0 GB) and the transient lower layers of a tree while it is built
    # (2 x 2^25 x 32 B = 2.1 GB).  Keeping every tree layer (8.6 GB at this size) would not fit.
    assert peak <= traces + ldes + (9 << 29), (peak, traces, ldes)
