"""Poseidon-16 Merkle trees on the device (vgpu_ctx_set_merkle_hash(VGPU_MERKLE_POSEIDON16)): commits, openings, proofs from
host and device traces and split over 2 / 4 / 8 ranks, all byte for byte against the oracle's Poseidon MMCS
(tests/poseidon_mmcs.py, tests/c/poseidon_mmcs_oracle.cc); both verifiers accept the proofs; the two hashes do not mix on one context; Fibonacci 2^22 proves in
the same device memory as with Keccak."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

P = 2013265921
DROP = 8                                      # VG_TREE_DROP
WIDTHS = [1, 7, 8, 9, 16, 17, 67]


def ext(rng):
    return [int(v) for v in rng.integers(0, P, 5)]


@pytest.fixture(scope="module")
def mmcs(oracle):
    from poseidon_mmcs import PoseidonOracle

    return PoseidonOracle()


@pytest.fixture(scope="module")
def p16(built, oracle):
    """A context of its own in Poseidon mode, and its StarkConfig."""
    import valida_b200 as vb

    ctx = vb.Context(0)
    cfg = vb.StarkConfig(ctx, oracle.rc480)
    ctx.set_merkle_hash(vb.MERKLE_POSEIDON16)
    yield ctx, cfg
    ctx.close()


def open_and_compare(ctx, cfg, mmcs, rounds):
    """rounds: [(matrices, [points of each matrix])]: roots, then the opening after observing them, equal to the oracle's."""
    import valida_b200 as vb

    pcs = cfg.pcs()
    pds, roots = [], []
    try:
        for mats, _ in rounds:
            root, pd = pcs.commit_batches(mats)
            pds.append(pd)
            roots.append(root)
            assert np.array_equal(root, mmcs.commit_batches(mats)), [m.shape for m in mats]
        obs = np.concatenate(roots).astype(np.uint32)
        L = vb.lib()
        ctx.check(L.vgpu_challenger_reset(ctx._h))
        ctx.check(L.vgpu_challenger_observe(ctx._h, obs.ctypes.data_as(C.POINTER(C.c_uint32)), obs.size))
        got = pcs.open_multi_batches([(pd, pts) for pd, (_, pts) in zip(pds, rounds)])
    finally:
        for pd in pds:
            pd.free()
    assert got == mmcs.open([mats for mats, _ in rounds], [p for _, pts in rounds for p in pts], obs)


# tallest LDE height 2^k; (level, width) of the shorter matrices: level j joins where the layer has 2^(k - j) nodes
COMMITS = {
    1: [], 2: [(1, 9)], 5: [(2, 67), (4, 1)],
    8: [(1, 17), (7, 8)],                                 # depth 8: only the root kept; joins below and at the top
    9: [(1, 16), (8, 7)],                                 # the first kept layer
    12: [(3, 67), (7, 1), (8, 9), (10, 17)],             # below, at and above the dropped layers
    15: [(5, 7)],                                         # a first layer of 2^14 nodes: the whole tree is one fused tail run
    16: [(1, 8), (2, 9)],                                 # first layer 2^15: the tail-fusion boundary
    17: [(1, 1), (9, 67), (16, 16)],
}


@pytest.mark.parametrize("log_lde", sorted(COMMITS))
def test_commit_roots(p16, mmcs, log_lde):
    ctx, cfg = p16
    rng = np.random.default_rng(log_lde)
    h = 1 << (log_lde - 1)
    tall = [rng.integers(0, P, (h, w), dtype=np.uint32) for w in (WIDTHS if log_lde <= 12 else [3, 9])]
    short = [rng.integers(0, P, (h >> j, w), dtype=np.uint32) for j, w in COMMITS[log_lde]]
    mats = tall[:2] + short + tall[2:]                     # a shorter matrix between two of the tallest: the stable order
    root, pd = cfg.pcs().commit_batches(mats)
    pd.free()
    assert np.array_equal(root, mmcs.commit_batches(mats))


@pytest.mark.parametrize("log_h", [9, 13])
def test_open_every_width(p16, mmcs, log_h):
    ctx, cfg = p16
    rng = np.random.default_rng(50 + log_h)
    mats = [rng.integers(0, P, (1 << log_h, w), dtype=np.uint32) for w in [1, 2, 31, 32, 33, 63, 64, 65, 97, 130, 200]]
    z = ext(rng)
    open_and_compare(ctx, cfg, mmcs, [(mats, [[z] if i % 2 else [z, ext(rng)] for i in range(len(mats))])])


def test_open_base_field_point_and_shared_point_across_rounds(p16, mmcs):
    ctx, cfg = p16
    rng = np.random.default_rng(2024)
    zb, ze = [7, 0, 0, 0, 0], ext(rng)
    r0 = [rng.integers(0, P, (1 << 10, 7), dtype=np.uint32), rng.integers(0, P, (1 << 10, 40), dtype=np.uint32),
          rng.integers(0, P, (1 << 9, 3), dtype=np.uint32)]
    r1 = [rng.integers(0, P, (1 << 12, 97), dtype=np.uint32), rng.integers(0, P, (1 << 12, 5), dtype=np.uint32)]
    r2 = [rng.integers(0, P, (1 << 10, 64), dtype=np.uint32)]
    open_and_compare(ctx, cfg, mmcs, [(r0, [[zb, ze], [ze], [zb]]), (r1, [[zb], [ze, zb]]), (r2, [[ze]])])


def _programs():
    import programs
    import valida_b200 as vb

    prog, cells = programs.static_data_program()
    return {
        "fib25": lambda: vb.run_program(vb.fib_program(25), initial_fp=0x1000),
        "fib582": lambda: vb.run_program(vb.fib_program(582), initial_fp=0x1000),
        "mixed": lambda: vb.run_program(programs.mixed_program(100), initial_fp=0x1000),
        "config5": lambda: vb.run_program(programs.config5_program(60), initial_fp=0x1000),
        "static_data": lambda: vb.run_program(prog, initial_fp=0x1000, static_data=cells),
    }


@pytest.mark.parametrize("name", ["fib25", "fib582", "mixed", "config5", "static_data"])
def test_prove_bytes_equal_oracle(p16, mmcs, name):
    import valida_b200 as vb

    ctx, cfg = p16
    t = _programs()[name]()
    want = mmcs.prove(t.main, t.preprocessed).cbor()
    assert vb.prove_machine(cfg, t) == want
    dm = [ctx.upload(m) for m in t.main]
    dp = [ctx.upload(m) for m in t.preprocessed]
    try:
        assert vb.prove_machine(cfg, t, device_resident=(dm, dp)) == want
    finally:
        for m in dm + dp:
            m.free()
    vb.verify_machine(cfg, want, t.preprocessed)
    assert mmcs.verify(want, t.preprocessed) == 0


def test_prove_from_the_device_witness(p16, mmcs):
    import valida_b200 as vb

    ctx, cfg = p16
    log = vb.run_program_log(vb.fib_program(((1 << 12) - 17) // 7))
    t = log.traces()
    want = mmcs.prove(t.main, t.preprocessed).cbor()
    dm, dp = log.witness_device(ctx)
    try:
        assert vb.prove_machine(cfg, t, device_resident=(dm, dp)) == want
    finally:
        for m in dm + dp:
            m.free()


@pytest.mark.parametrize("nranks", [2, 4, 8])
def test_split_proof_bytes_equal_single_gpu(p16, mmcs, oracle, nranks):
    """The tallest chip has 2 * 4096 * nranks LDE rows: every tree of the proof is split, the rebuilt paths of each rank included."""
    import torch
    import valida_b200 as vb

    ctx, cfg = p16
    log_cpu = 10 + nranks.bit_length() - 1
    t = vb.run_program(vb.fib_program(((1 << log_cpu) - 17) // 7), initial_fp=0x1000)
    assert t.main[2].shape[0] * 2 == 8192 * nranks
    single = vb.prove_machine(cfg, t)
    k = torch.cuda.device_count()
    ctxs = [vb.Context(i % k) for i in range(nranks)]
    try:
        vb.comm_init_local(ctxs)
        cfgs = [vb.StarkConfig(c, oracle.rc480) for c in ctxs]
        for c in ctxs:
            c.set_merkle_hash(vb.MERKLE_POSEIDON16)
        assert all(p == single for p in vb.run_ranks(lambda r, c: vb.prove_machine(cfgs[r], t), ctxs))
    finally:
        for c in ctxs:
            c.close()
    assert mmcs.verify(single, t.preprocessed) == 0


def test_modes_do_not_mix(built, oracle, mmcs):
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(25), initial_fp=0x1000)
    keccak_ref = oracle.prove(t.main, t.preprocessed, debug_checks=False).cbor()
    ctx = vb.Context(0)
    try:
        with pytest.raises(vb.VgpuError, match="unknown hash"):
            ctx.set_merkle_hash(2)
        ctx.set_merkle_hash(vb.MERKLE_POSEIDON16)
        with pytest.raises(vb.VgpuError, match="vgpu_set_challenger"):       # a Poseidon commit needs the challenger's permutation
            vb.TwoAdicFriPcs(ctx).commit_batches([np.ones((8, 3), dtype=np.uint32)])
        cfg = vb.StarkConfig(ctx, oracle.rc480)
        pos = vb.prove_machine(cfg, t)
        assert pos == mmcs.prove(t.main, t.preprocessed).cbor()
        _, pos_pd = cfg.pcs().commit_batches(t.main)
        ctx.set_merkle_hash(vb.MERKLE_KECCAK256)
        assert vb.prove_machine(cfg, t) == keccak_ref                       # Keccak after Poseidon on one context: the fresh bytes
        with pytest.raises(vb.VerificationError) as e:
            vb.verify_machine(cfg, pos, t.preprocessed)
        assert e.value.verdict < 0
        with pytest.raises(vb.VgpuError, match="another Merkle hash"):
            cfg.pcs().open_multi_batches([(pos_pd, [[ext(np.random.default_rng(1))]] * 14)])
        pos_pd.free()
        ctx.set_merkle_hash(vb.MERKLE_POSEIDON16)
        with pytest.raises(vb.VerificationError):
            vb.verify_machine(cfg, keccak_ref, t.preprocessed)
        vb.verify_machine(cfg, pos, t.preprocessed)
    finally:
        ctx.close()


def test_fibonacci_2p22_peak_memory_as_keccak(built, oracle):
    """BASELINE config 3 through vgpu_prove_device: the Poseidon proof is accepted, and its peak live bytes are within 1 % of the
    Keccak proof's (digests are 32 bytes under either hash)."""
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(((1 << 22) - 17) // 7), initial_fp=0x1000)
    ctx = vb.Context(0)
    try:
        cfg = vb.StarkConfig(ctx, oracle.rc480)
        dm = [ctx.upload(m) for m in t.main]
        dp = [ctx.upload(m) for m in t.preprocessed]
        peaks = {}
        for hash in (vb.MERKLE_KECCAK256, vb.MERKLE_POSEIDON16):
            ctx.set_merkle_hash(hash)
            ctx.memory_stats(reset=True)
            proof = vb.prove_machine(cfg, t, device_resident=(dm, dp))
            peaks[hash] = ctx.memory_stats()["peak"]
        vb.verify_machine(cfg, proof, t.preprocessed)
        for m in dm + dp:
            m.free()
    finally:
        ctx.close()
    print("2^22 device proof peak live bytes: Keccak %.3f GB, Poseidon-16 %.3f GB" % (peaks[0] / 1e9, peaks[1] / 1e9))
    assert abs(peaks[1] - peaks[0]) <= 0.01 * peaks[0], peaks
