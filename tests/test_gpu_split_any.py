"""ONE proof split over a rank count that is not a power of two (3, 5, 6, 7, 12): the ranks hold uneven runs of whole units
(csrc/ctx.h), the tree's gathered layer is the V-node one, a rank may straddle the middle row of an LDE, and the quotient's next rows
of one rank's run lie on several ranks.  Proof bytes equal the single-GPU proof (the oracle's) through every input route, and both
verifiers accept them.  The ranks are threads of this process (vgpu_comm_init_local), several on one device when the box has fewer
GPUs; a process per rank (NCCL + CUDA IPC) runs where the box has three GPUs."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 2013265921
UNEVEN = [3, 5, 6, 7, 12]
CH = np.random.default_rng(77).integers(0, P, 15, dtype=np.uint32)


def _units(n):
    return 8 * (1 << (n - 1).bit_length())


def _ranks(n):
    import torch
    import valida_b200 as vb

    k = torch.cuda.device_count()
    ctxs = [vb.Context(i % k) for i in range(n)]
    vb.comm_init_local(ctxs)
    return ctxs


def _close(ctxs):
    for c in ctxs:
        c.close()


def _monty(a):
    return ((np.asarray(a, dtype=np.uint64) << np.uint64(32)) % np.uint64(P)).astype(np.uint32)


def _host(t):
    return t.cpu().numpy().view(np.uint32)


def _row_major(a, device):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).to(device)


def _col_major(a, device, pad=0):
    """A (h, w) column-major CUDA view of `a` with column stride h + pad."""
    import torch

    h, w = a.shape
    buf = torch.full((w * (h + pad),), -1, dtype=torch.int32, device=device)
    buf.view(w, h + pad)[:, :h] = _row_major(np.ascontiguousarray(a.T), device)
    return torch.as_strided(buf, (h, w), (1, h + pad))


@pytest.fixture(scope="module")
def fib15(built, ctx, oracle):
    """Fibonacci with a 2^15-row CPU trace and a 2^17-row memory trace (LDE 2^18 rows: split at every N <= 16), and its single-GPU
    proof, which is the oracle's."""
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(((1 << 15) - 17) // 7), initial_fp=0x1000)
    assert t.main[0].shape[0] == 1 << 15 and t.main[2].shape[0] == 1 << 17
    proof = vb.prove_machine(vb.StarkConfig(ctx, oracle.rc480), t)
    assert proof == oracle.prove(t.main, t.preprocessed, debug_checks=False).cbor()
    return t, proof


@pytest.mark.parametrize("nranks", UNEVEN)
def test_uneven_split_proof_bytes(ctx, oracle, fib15, nranks):
    """vgpu_prove from host traces: the tallest LDE is split into uneven runs and every rank returns the single-GPU bytes, which the
    oracle's verifier and the library's own accept."""
    import valida_b200 as vb

    t, single = fib15
    ctxs = _ranks(nranks)
    try:
        h = 2 * t.main[2].shape[0]
        runs = [c.local_rows(h // 2) for c in ctxs]
        assert len({n for _, n in runs}) == 2                       # uneven: two run lengths
        cfgs = [vb.StarkConfig(c, oracle.rc480) for c in ctxs]
        proofs = vb.run_ranks(lambda r, c: vb.prove_machine(cfgs[r], t), ctxs)
        assert all(p == single for p in proofs)
        stats = ctxs[0].comm_stats()
        assert stats["exchange"][0] > 0 and stats["allgather"][0] > 0
    finally:
        _close(ctxs)
    assert oracle.verify(single, t.preprocessed) == 0
    vb.verify_machine(vb.StarkConfig(ctx, oracle.rc480), single, t.preprocessed)


@pytest.mark.parametrize("nranks", [3, 6])
def test_uneven_split_poseidon_mode(built, oracle, fib15, nranks):
    """The Poseidon-16 Merkle mode: the same uneven runs, the single-GPU Poseidon proof's bytes, accepted by both verifiers."""
    import valida_b200 as vb
    from poseidon_mmcs import PoseidonOracle

    t, _ = fib15
    one = vb.Context(0)
    try:
        cfg = vb.StarkConfig(one, oracle.rc480)
        one.set_merkle_hash(vb.MERKLE_POSEIDON16)
        single = vb.prove_machine(cfg, t)
        vb.verify_machine(cfg, single, t.preprocessed)
    finally:
        one.close()
    ctxs = _ranks(nranks)
    try:
        cfgs = [vb.StarkConfig(c, oracle.rc480) for c in ctxs]
        for c in ctxs:
            c.set_merkle_hash(vb.MERKLE_POSEIDON16)
        assert all(p == single for p in vb.run_ranks(lambda r, c: vb.prove_machine(cfgs[r], t), ctxs))
    finally:
        _close(ctxs)
    assert PoseidonOracle().verify(single, t.preprocessed) == 0


@pytest.mark.parametrize("nranks", [3, 7])
def test_uneven_split_input_routes(ctx, oracle, fib15, nranks):
    """upload_rows, import_tensor_local, borrow_tensor_local (a column stride above the rows) and the device witness: each rank holds
    its own uneven run of every tall trace and proves the single-GPU bytes."""
    import valida_b200 as vb

    t, single = fib15
    mats = [np.array(m) for m in t.main + t.preprocessed]
    monty = [_monty(a) for a in mats]
    ctxs = _ranks(nranks)
    try:
        cfgs = [vb.StarkConfig(c, oracle.rc480) for c in ctxs]

        def prove(r, dm):
            return vb.prove_machine(cfgs[r], None, device_resident=(dm[:14], dm[14:]))

        def local(c, a, make):
            row0, rows = c.local_rows(a.shape[0])
            return make(a[row0:row0 + rows], "cuda:%d" % c.device)

        def routes(r, c):
            out = {}
            dm = [c.upload_rows(a) for a in mats]
            assert dm[2].local_rows() == c.local_rows(mats[2].shape[0])
            out["upload_rows"] = prove(r, dm)
            dm = [c.import_tensor_local(local(c, a, _row_major), a.shape[0], vb.REPR_CANONICAL) for a in mats]
            out["import_local"] = prove(r, dm)
            tens = [local(c, a, lambda x, d: _col_major(x, d, pad=3)) for a in monty]
            dm = [c.borrow_tensor_local(x, a.shape[0]) for x, a in zip(tens, monty)]
            out["borrow_local"] = prove(r, dm)
            return out

        for res in vb.run_ranks(routes, ctxs):
            assert all(p == single for p in res.values()), [k for k, p in res.items() if p != single]
        log = vb.run_program_log(vb.fib_program(((1 << 15) - 17) // 7))
        host = log.traces()
        host_single = vb.prove_machine(vb.StarkConfig(ctx, oracle.rc480), host)

        def witness(r, c):
            wm, wp = log.witness_device(c)
            return vb.prove_machine(cfgs[r], host, device_resident=(wm, wp))

        assert all(p == host_single for p in vb.run_ranks(witness, ctxs))
    finally:
        _close(ctxs)


@pytest.mark.parametrize("nranks", [3, 7])
def test_uneven_local_rows_partition_and_round_trip(oracle, fib15, nranks):
    """local_rows of all ranks partitions [0, H) in rank order for every trace height; local_to_tensor gives back a rank's rows."""
    import valida_b200 as vb

    t, _ = fib15
    mats = [np.array(m) for m in t.main]
    ctxs = _ranks(nranks)
    try:
        for a in mats:
            h = a.shape[0]
            runs = [c.local_rows(h) for c in ctxs]
            if runs[0][1] == h:
                assert runs == [(0, h)] * nranks
                continue
            assert runs[0][0] == 0 and all(runs[r][0] + runs[r][1] == runs[r + 1][0] for r in range(nranks - 1))
            assert runs[-1][0] + runs[-1][1] == h
            assert all(b % (h // _units(nranks)) == 0 for b, _ in runs)

        def rank(r, c):
            ok = []
            for a in mats:
                row0, rows = c.local_rows(a.shape[0])
                m = c.import_tensor_local(_col_major(a[row0:row0 + rows], "cuda:%d" % c.device, pad=1), a.shape[0], vb.REPR_CANONICAL)
                ok.append(m.local_rows() == (row0, rows) and np.array_equal(_host(m.local_to_tensor()), a[row0:row0 + rows]))
                m.free()
            return all(ok)

        assert all(vb.run_ranks(rank, ctxs))
    finally:
        _close(ctxs)


@pytest.mark.parametrize("nranks", [3, 6, 7])
def test_uneven_witness_checks_at_every_boundary(ctx, fib15, nranks):
    """A cell of the CPU trace (its clock, constrained on every row) changed on each side of every rank boundary, in one tampered
    witness: check_witness and check_constraints_local report on every rank what the single-GPU check reports."""
    import valida_b200 as vb

    t, _ = fib15
    mats = [np.array(m) for m in t.main + t.preprocessed]
    ctxs = _ranks(nranks)
    try:
        for chip in (0,):
            h = mats[chip].shape[0]
            starts = [c.local_rows(h)[0] for c in ctxs]
            assert len(set(b - a for a, b in zip(starts, starts[1:] + [h]))) == 2, (chip, starts)
            bad = [m.copy() for m in mats]
            for b in starts[1:]:
                for row in (b - 1, b):
                    bad[chip][row, 0] = (int(bad[chip][row, 0]) + 1) % P
            dm = ctx.upload(bad[chip])
            dq, _ = vb.generate_permutation_trace(ctx, chip, dm, None, CH)
            want = vb.check_constraints(ctx, chip, dm, None, dq, CH)
            assert want[0] >= 0, (chip, want)
            perm = dq.download()

            def local(r, c):
                return vb.check_constraints_local(c, chip, c.upload_rows(bad[chip]), None, c.upload_rows(perm), CH)

            assert vb.run_ranks(local, ctxs) == [want] * nranks

            def whole(r, c):
                dmr = [c.upload_rows(m) for m in bad]
                return vb.check_witness(c, dmr[:14], dmr[14:], CH)

            for reports, _cancel in vb.run_ranks(whole, ctxs):
                assert tuple(reports[chip][:3]) == tuple(want), (chip, reports[chip], want)
    finally:
        _close(ctxs)


@pytest.mark.parametrize("nranks", [6, 7])
def test_uneven_split_fibonacci_2p22_memory_rows(oracle, nranks):
    """Fibonacci with 2^20 CPU rows and a 2^22-row memory trace over 6 and 7 thread ranks: the single-GPU (oracle) bytes."""
    import valida_b200 as vb

    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_large_proof_digests import assert_matches_golden, fib_n

    t = vb.run_program(vb.fib_program(fib_n(20)), initial_fp=0x1000)
    assert t.main[2].shape[0] == 1 << 22
    ctxs = _ranks(nranks)
    try:
        cfgs = [vb.StarkConfig(c, oracle.rc480) for c in ctxs]
        proofs = vb.run_ranks(lambda r, c: vb.prove_machine(cfgs[r], t), ctxs)
    finally:
        _close(ctxs)
    for p in proofs:
        assert_matches_golden(p, "fib_2p20")


def test_rank_counts_outside_1_to_16_are_refused(built):
    import ctypes as C

    import valida_b200 as vb

    ctxs = [vb.Context(0) for _ in range(17)]
    try:
        with pytest.raises(vb.VgpuError, match="1..16"):
            vb.comm_init_local(ctxs)
        one = (C.c_void_p * 1)(ctxs[0]._h)
        assert vb.lib().vgpu_comm_init_local(one, 0) == -1
        assert all(c.local_rows(1 << 20) == (0, 1 << 20) for c in ctxs)      # nothing was set up
        with pytest.raises(vb.VgpuError, match="1..16"):
            ctxs[0].comm_init(0, 17, bytes(128))
        with pytest.raises(vb.VgpuError, match="bad rank"):
            ctxs[0].comm_init(0, 0, bytes(128))
    finally:
        _close(ctxs)


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist

    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import oracle_binding
    import valida_b200 as vb

    orc = oracle_binding.Oracle()
    ctx = vb.Context(rank)
    cfg = vb.StarkConfig(ctx, orc.rc480)
    t = vb.run_program(vb.fib_program(((1 << 15) - 17) // 7), initial_fp=0x1000)
    single = vb.prove_machine(cfg, t)
    ctx.comm_init_from_torch()
    out[rank] = {"uneven": ctx.local_rows(1 << 17)[1] != (1 << 17) // world or (1 << 17) % world != 0,
                 "proof_equal": vb.prove_machine(cfg, t) == single,
                 "oracle": single == orc.prove(t.main, t.preprocessed, debug_checks=False).cbor()}
    ctx.close()
    dist.destroy_process_group()


def test_processes_three_ranks(built):
    """A process per GPU at N = 3 (NCCL broadcasts gather the uneven runs, CUDA IPC maps the heaps): the single-GPU bytes."""
    import torch
    import torch.multiprocessing as mp

    if torch.cuda.device_count() < 3:
        pytest.skip("needs 3 GPUs: one process per GPU")
    mgr = mp.Manager()
    out = mgr.dict()
    port = 36500 + (os.getpid() % 2000)
    mp.spawn(_worker, args=(3, port, out), nprocs=3, join=True)
    for rank in range(3):
        assert all(out[rank].values()), (rank, dict(out[rank]))
