"""Split proofs from traces each rank holds only its own rows of, in its own GPU memory: import_tensor_local (a copy),
borrow_tensor_local (proven from in place) and local_to_tensor (the rows a rank holds, out).  Every rank gets tensors of only
local_rows(H) rows of each trace; the proof bytes equal the single-GPU proof and the oracle's.

Ranks are threads of this process (comm_init_local, all on device 0 when the box has one GPU), so the whole data path runs on a
one-GPU box; the process-per-GPU launch (NCCL + CUDA IPC) is checked at the end when the box has two GPUs."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from test_gpu_split_local import _close, _group

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_large_proof_digests import assert_matches_golden, fib_n  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 2013265921


def _torch():
    import torch

    return torch


def _monty(a):
    return ((np.asarray(a, dtype=np.uint64) << np.uint64(32)) % np.uint64(P)).astype(np.uint32)


def _host(t):
    return t.cpu().numpy().view(np.uint32)


def _row_major(a, device):
    return _torch().from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).to(device)


def _col_major(a, device, pad=0, off=0):
    """A (h, w) column-major CUDA view of `a`: stride(1) == h + pad, `off` words past the start of its buffer."""
    torch = _torch()
    h, w = a.shape
    buf = torch.full((off + w * (h + pad),), -1, dtype=torch.int32, device=device)
    buf[off:].view(w, h + pad)[:, :h] = _row_major(np.ascontiguousarray(a.T), device)
    return torch.as_strided(buf, (h, w), (1, h + pad), off)


def _local_tensors(c, mats, make):
    """This rank's rows of every matrix, as tensors on its device built by make(rows of the host matrix, device)."""
    out = []
    for a in mats:
        row0, rows = c.local_rows(a.shape[0])
        out.append(make(a[row0:row0 + rows], "cuda:%d" % c.device))
    return out


def _prove(cfg, mats):
    import valida_b200 as vb

    return vb.prove_machine(cfg, None, device_resident=(mats[:14], mats[14:]))


@pytest.fixture(scope="module")
def fib15(built, ctx, oracle):
    """Fibonacci with a 2^15-row CPU trace and a 2^17-row memory trace, and its single-GPU proof (the oracle's bytes)."""
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(((1 << 15) - 17) // 7), initial_fp=0x1000)
    assert t.main[0].shape[0] == 1 << 15 and t.main[2].shape[0] == 1 << 17
    proof = vb.prove_machine(vb.StarkConfig(ctx, oracle.rc480), t)
    assert proof == oracle.prove(t.main, t.preprocessed, debug_checks=False).cbor()
    return t, proof


@pytest.mark.parametrize("nranks", [2, 4, 8])
def test_import_local_proves_the_single_gpu_bytes(oracle, fib15, nranks):
    """Each rank imports tensors of its own rows only, in both reprs, row-major and column-major."""
    import valida_b200 as vb

    t, single = fib15
    mats = t.main + t.preprocessed
    ctxs, cfgs = _group(nranks, oracle)
    try:
        for r, c in enumerate(ctxs):
            rows = (1 << 17) // nranks
            assert c.local_rows(1 << 17) == (r * rows, rows)                   # the memory chip is split
            assert c.local_rows(t.main[13].shape[0]) == (0, t.main[13].shape[0])   # a short trace is whole
        for repr_, conv in ((vb.REPR_CANONICAL, lambda a: a), (vb.REPR_MONTY_R32, _monty)):
            for make in (_row_major, _col_major):
                def rank(r, c):
                    tens = _local_tensors(c, [conv(a) for a in mats], make)
                    dm = [c.import_tensor_local(x, a.shape[0], repr_) for x, a in zip(tens, mats)]
                    assert dm[2].local_rows() == c.local_rows(1 << 17) and dm[2].shape == t.main[2].shape
                    return _prove(cfgs[r], dm)

                assert all(p == single for p in vb.run_ranks(rank, ctxs)), (repr_, make.__name__)
    finally:
        _close(ctxs)


BORROW_LAYOUTS = {"stride_rows": (0, 0), "stride_rows_plus_1": (1, 0), "stride_rows_plus_3": (3, 0), "base_plus_one_word": (0, 1)}


@pytest.mark.parametrize("layout", list(BORROW_LAYOUTS))
@pytest.mark.parametrize("nranks", [2, 4, 8])
def test_borrow_local_proves_in_place(oracle, fib15, nranks, layout):
    """Column-major Montgomery shards at column stride rows, rows + 1 and rows + 3, and at a base one word past 16-byte alignment:
    the odd strides and the offset base reach the word-at-a-time exchange.  Nothing is copied and the tensors are untouched."""
    import valida_b200 as vb

    torch = _torch()
    t, single = fib15
    mats = [_monty(a) for a in t.main + t.preprocessed]
    pad, off = BORROW_LAYOUTS[layout]
    ctxs, cfgs = _group(nranks, oracle)
    try:
        tens = [_local_tensors(c, mats, lambda a, d: _col_major(a, d, pad, off)) for c in ctxs]
        before = [[x.clone() for x in ts] for ts in tens]
        torch.cuda.synchronize()

        def rank(r, c):
            live = c.memory_stats()["live"]
            dm = [c.borrow_tensor_local(x, a.shape[0]) for x, a in zip(tens[r], mats)]
            assert c.memory_stats()["live"] == live
            proof = _prove(cfgs[r], dm)
            for m in dm:
                m.free()
            return proof

        assert all(p == single for p in vb.run_ranks(rank, ctxs))
        torch.cuda.synchronize()
        assert all(torch.equal(x, y) for ts, bs in zip(tens, before) for x, y in zip(ts, bs))
    finally:
        _close(ctxs)


@pytest.mark.parametrize("nranks", [2, 4])
def test_import_local_equals_import_rows(oracle, nranks):
    """Per rank, importing the rank's slice equals importing the whole tensor with import_tensor_rows, tall and short."""
    import valida_b200 as vb

    rng = np.random.default_rng(nranks)
    ctxs, _ = _group(nranks, oracle)
    try:
        for h, w in ((1 << 14, 5), (1 << 15, 129), (1 << 10, 3)):
            a = rng.integers(0, P, size=(h, w), dtype=np.uint32)
            for k, c in enumerate(ctxs):
                dev = "cuda:%d" % c.device
                row0, rows = c.local_rows(h)
                assert (row0, rows) == ((k * h // nranks, h // nranks) if 2 * h >= nranks * 4096 else (0, h))
                for r in (vb.REPR_CANONICAL, vb.REPR_MONTY_R32):
                    whole = c.import_tensor_rows(_row_major(a, dev), r)
                    local = c.import_tensor_local(_col_major(a[row0:row0 + rows], dev, pad=2), h, r)
                    assert local.local_rows() == whole.local_rows() == (row0, rows)
                    assert local.shape == whole.shape == (h, w)
                    assert np.array_equal(_host(local.local_to_tensor(vb.REPR_MONTY_R32)), _host(whole.local_to_tensor(vb.REPR_MONTY_R32)))
                    assert np.array_equal(_host(local.local_to_tensor(r)), a[row0:row0 + rows])
                    whole.free()
                    local.free()
    finally:
        _close(ctxs)


def test_device_witness_local_rows_out_and_borrowed_back(oracle, fib15):
    """On a split context the device witness is held as row shards: local_to_tensor gives each rank its rows of the host traces, and
    borrowing those tensors back proves to the single-GPU bytes."""
    import valida_b200 as vb

    torch = _torch()
    t, single = fib15
    log = vb.run_program_log(vb.fib_program(((1 << 15) - 17) // 7))
    mats = t.main + t.preprocessed
    ctxs, cfgs = _group(4, oracle)
    try:
        def rank(r, c):
            wm, wp = log.witness_device(c)
            tens = []
            for m, a in zip(wm + wp, mats):
                row0, rows = m.local_rows()
                assert (row0, rows) == c.local_rows(a.shape[0])
                assert np.array_equal(_host(m.local_to_tensor()), a[row0:row0 + rows])
                x = m.local_to_tensor(vb.REPR_MONTY_R32, out=torch.empty((a.shape[1], rows), dtype=torch.int32, device="cuda:%d" % c.device).t())
                tens.append(x)
            for m in wm + wp:
                m.free()
            dm = [c.borrow_tensor_local(x, a.shape[0]) for x, a in zip(tens, mats)]
            return _prove(cfgs[r], dm)

        assert all(p == single for p in vb.run_ranks(rank, ctxs))
    finally:
        _close(ctxs)


@pytest.mark.parametrize("sharding", [True, False])
def test_refusals(oracle, sharding):
    """Host-side refusals name the numbers and launch nothing; a word not below p fails on the ranks that hold it only, naming its
    row in the whole matrix."""
    import valida_b200 as vb
    from valida_b200.api import _DevMatrix, lib

    torch = _torch()
    H, W = 1 << 14, 3
    ctxs, _ = _group(2, oracle)
    try:
        for c in ctxs:
            c.set_sharding(sharding)
        a = np.random.default_rng(3).integers(0, P, size=(H, W), dtype=np.uint32)
        for k, c in enumerate(ctxs):
            dev = "cuda:%d" % c.device
            row0, rows = c.local_rows(H)
            assert (row0, rows) == ((k * H // 2, H // 2) if sharding else (0, H))
            n = c.launch_count
            wrong = _row_major(a[:rows - 4], dev)
            with pytest.raises(vb.VgpuError, match=r"rows = %d starting at row0 = %d" % (rows, row0)):
                c.import_tensor_local(wrong, H)
            with pytest.raises(ValueError, match=r"rows = %d starting at row0 = %d" % (rows, row0)):
                c.borrow_tensor_local(_col_major(a[:rows - 4], dev), H)
            buf = torch.zeros((W, rows), dtype=torch.int32, device=dev)

            def refused(call, pattern):
                out = C.c_void_p()
                assert call(out) != 0
                assert pattern in lib().vgpu_last_error(c._h).decode(), lib().vgpu_last_error(c._h).decode()
                assert not out.value

            refused(lambda o: lib().vgpu_dmat_borrow_local(c._h, buf.data_ptr(), H, W, rows - 1, C.byref(o)), "below the height")
            refused(lambda o: lib().vgpu_dmat_borrow_local(c._h, buf.data_ptr() + 2, H, W, rows, C.byref(o)), "4-byte aligned")
            host = np.zeros((W, rows), dtype=np.uint32)
            refused(lambda o: lib().vgpu_dmat_borrow_local(c._h, host.ctypes.data, H, W, rows, C.byref(o)), "not device memory")
            hv = _DevMatrix(host.ctypes.data, rows, W, 1, rows)
            refused(lambda o: lib().vgpu_dmat_import_local(c._h, C.byref(hv), H, 0, C.byref(o)), "not device memory")
            if torch.cuda.device_count() > 1:
                other = torch.zeros((W, rows), dtype=torch.int32, device="cuda:%d" % ((c.device + 1) % torch.cuda.device_count()))
                refused(lambda o: lib().vgpu_dmat_borrow_local(c._h, other.data_ptr(), H, W, rows, C.byref(o)), "not device memory")
            assert c.launch_count == n
            m = c.import_tensor_local(_row_major(a[row0:row0 + rows], dev), H)
            n = c.launch_count
            with pytest.raises(vb.VgpuError, match=r"rows = %d starting at row0 = %d" % (rows, row0)):
                m.local_to_tensor(out=torch.empty((rows + 4, W), dtype=torch.int32, device=dev))
            with pytest.raises(vb.VgpuError, match="not device memory"):
                lib_out = _DevMatrix(host.ctypes.data, rows, W, 1, rows)
                c.check(lib().vgpu_dmat_export_local(c._h, m._h, 0, C.byref(lib_out)))
            assert c.launch_count == n
            m.free()
        # a word >= p at global row g: the ranks that hold row g fail naming it, the others import their rows
        for g, col in ((H // 2 + 5, 2), (7, 0)):
            b = a.copy()
            b[g, col] = P
            for k, c in enumerate(ctxs):
                dev = "cuda:%d" % c.device
                row0, rows = c.local_rows(H)
                part = b[row0:row0 + rows]
                calls = [lambda: c.import_tensor_local(_row_major(part, dev), H, vb.REPR_CANONICAL),
                         lambda: c.import_tensor_local(_col_major(part, dev, pad=1), H, vb.REPR_MONTY_R32),
                         lambda: c.borrow_tensor_local(_col_major(part, dev, pad=3), H)]
                for call in calls:
                    if row0 <= g < row0 + rows:
                        with pytest.raises(vb.VgpuError, match=r"row %d, column %d\b" % (g, col)):
                            call()
                    else:
                        call().free()
    finally:
        _close(ctxs)


def test_lone_context_and_sharding_off_match_the_whole_matrix_calls(ctx, oracle):
    """Without a split the local calls are import_tensor / borrow_tensor / to_tensor."""
    import valida_b200 as vb

    rng = np.random.default_rng(9)
    ctxs, _ = _group(2, oracle)
    try:
        ctxs[1].set_sharding(False)
        for c in (ctx, ctxs[1]):
            for h, w in ((1 << 14, 4), (1 << 16, 1), (5, 7)):
                a = rng.integers(0, P, size=(h, w), dtype=np.uint32)
                assert c.local_rows(h) == (0, h)
                x = _row_major(a, "cuda:%d" % c.device)
                ref = c.import_tensor(x).download(vb.REPR_MONTY_R32)
                m = c.import_tensor_local(x, h)
                assert m.local_rows() == (0, h)
                assert np.array_equal(m.download(vb.REPR_MONTY_R32), ref)
                y = _col_major(_monty(a), "cuda:%d" % c.device, pad=1)
                b = c.borrow_tensor_local(y, h)
                assert b.local_rows() == (0, h)
                for mm in (m, b):
                    assert np.array_equal(_host(mm.local_to_tensor()), _host(mm.to_tensor()))
                    assert np.array_equal(_host(mm.local_to_tensor()), a)
                m.free()
                b.free()
    finally:
        _close(ctxs)


@pytest.fixture(scope="module")
def fib20(built):
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(fib_n(20)), initial_fp=0x1000)
    assert t.main[0].shape[0] == 1 << 20
    return t


def _borrowed_proofs(oracle, t, nranks, merkle_hash=None):
    import valida_b200 as vb

    mats = [_monty(a) for a in t.main + t.preprocessed]
    ctxs, cfgs = _group(nranks, oracle)
    try:
        if merkle_hash is not None:
            for c in ctxs:
                c.set_merkle_hash(merkle_hash)
        tens = [_local_tensors(c, mats, lambda a, d: _col_major(a, d, pad=1)) for c in ctxs]

        def rank(r, c):
            dm = [c.borrow_tensor_local(x, a.shape[0]) for x, a in zip(tens[r], mats)]
            return _prove(cfgs[r], dm)

        return vb.run_ranks(rank, ctxs)
    finally:
        _close(ctxs)


@pytest.mark.parametrize("nranks", [2, 4, 8])
def test_fibonacci_2p20_from_borrowed_local_shards_equals_golden(oracle, fib20, nranks):
    for p in _borrowed_proofs(oracle, fib20, nranks):
        assert_matches_golden(p, "fib_2p20")


def test_poseidon_fibonacci_2p20_from_borrowed_local_shards_equals_golden(oracle, fib20):
    import valida_b200 as vb

    for p in _borrowed_proofs(oracle, fib20, 4, vb.MERKLE_POSEIDON16):
        assert_matches_golden(p, "p16_fib_2p20")


def test_borrow_local_saves_the_local_traces(oracle, fib20):
    """Fibonacci 2^20 over 4 ranks: on every rank the peak of a proof from borrowed shards is lower than from imported shards by
    the rank's local trace bytes."""
    import valida_b200 as vb

    t = fib20
    mats = t.main + t.preprocessed
    ctxs, cfgs = _group(4, oracle)
    try:
        canon = [_local_tensors(c, mats, _row_major) for c in ctxs]
        monty = [_local_tensors(c, [_monty(a) for a in mats], _col_major) for c in ctxs]

        def rank(r, c):
            c.release_cached()
            dm = [c.import_tensor_local(x, a.shape[0]) for x, a in zip(canon[r], mats)]
            c.memory_stats(reset=True)
            p_imp = _prove(cfgs[r], dm)
            peak_imported = c.memory_stats()["peak"]
            for m in dm:
                m.free()
            c.release_cached()
            bm = [c.borrow_tensor_local(x, a.shape[0]) for x, a in zip(monty[r], mats)]
            c.memory_stats(reset=True)
            p_bor = _prove(cfgs[r], bm)
            peak_borrowed = c.memory_stats()["peak"]
            for m in bm:
                m.free()
            c.release_cached()
            local = sum(c.local_rows(a.shape[0])[1] * a.shape[1] * 4 for a in mats)
            return p_imp, p_bor, peak_imported, peak_borrowed, local

        for r, (p_imp, p_bor, peak_imported, peak_borrowed, local) in enumerate(vb.run_ranks(rank, ctxs)):
            assert_matches_golden(p_imp, "fib_2p20")
            assert p_bor == p_imp
            assert local < sum(a.nbytes for a in mats) // 3                 # a rank holds about a quarter of the traces
            assert abs((peak_imported - peak_borrowed) - local) <= 0.01 * local, (r, peak_imported, peak_borrowed, local)
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
    mats = [_monty(a) for a in t.main + t.preprocessed]
    tens = _local_tensors(ctx, mats, lambda a, d: _col_major(a, d, pad=1))
    dm = [ctx.borrow_tensor_local(x, a.shape[0]) for x, a in zip(tens, mats)]
    out[rank] = {"split": dm[2].local_rows() == (rank * (1 << 17) // world, (1 << 17) // world),
                 "rows_only": all(x.shape[0] == ctx.local_rows(a.shape[0])[1] for x, a in zip(tens, mats)),
                 "proof_equal": _prove(cfg, dm) == single}
    for m in dm:
        m.free()
    ctx.close()
    dist.destroy_process_group()


def test_processes_borrow_only_their_rows(built):
    import torch
    import torch.multiprocessing as mp

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs: one process per GPU")
    mgr = mp.Manager()
    out = mgr.dict()
    port = 34500 + (os.getpid() % 2000)
    mp.spawn(_worker, args=(2, port, out), nprocs=2, join=True)
    for rank in range(2):
        assert all(out[rank].values()), (rank, dict(out[rank]))
