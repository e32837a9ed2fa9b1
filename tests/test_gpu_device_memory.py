"""Traces in the caller's GPU memory: import (a strided copy into the library's layout), borrow (proven from in place) and export
(the library's matrices into caller tensors), with torch tensors as the caller's buffers.  Proof bytes equal vgpu_prove on the same
host traces and the oracle's; every import equals upload() of the same words; refusals name the offending word and launch nothing
when they are decided on the host."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from programs import mixed_program, static_data_program

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_large_proof_digests import assert_matches_golden  # noqa: E402

pytestmark = pytest.mark.gpu
P = 2013265921


def _torch():
    import torch

    return torch


def _cuda(a):
    """numpy words -> a row-major torch.int32 CUDA tensor with the same bits."""
    torch = _torch()
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).cuda()


def _host(t):
    return t.cpu().numpy().view(np.uint32)


def _monty(a):
    return ((np.asarray(a, dtype=np.uint64) << np.uint64(32)) % np.uint64(P)).astype(np.uint32)


def _col_major(a, pad=0):
    """A (h, w) column-major CUDA view of `a` (stride(0) == 1, stride(1) == h + pad)."""
    h, w = a.shape
    big = _cuda(np.zeros((w, h + pad), dtype=np.uint32))
    big[:, :h] = _cuda(np.ascontiguousarray(a.T))
    return big[:, :h].t()


PROGRAMS = {
    "fib": lambda vb: vb.run_program(vb.fib_program(((1 << 10) - 17) // 7), initial_fp=0x1000),
    "mixed": lambda vb: vb.run_program(mixed_program(100), initial_fp=0x1000),
    "static_data": lambda vb: vb.run_program(static_data_program()[0], initial_fp=0x1000, static_data=static_data_program()[1]),
}


@pytest.fixture(scope="module")
def cfg(ctx, oracle):
    import valida_b200 as vb

    return vb.StarkConfig(ctx, oracle.rc480)


@pytest.fixture(scope="module")
def proofs(built, oracle, cfg):
    """Per program: (host traces, vgpu_prove bytes) after checking those against the oracle."""
    import valida_b200 as vb

    out = {}
    for name, make in PROGRAMS.items():
        t = make(vb)
        proof = vb.prove_machine(cfg, t)
        assert proof == oracle.prove(t.main, t.preprocessed, debug_checks=False).cbor(), name
        out[name] = (t, proof)
    return out


def _prove(cfg, dm, dp):
    import valida_b200 as vb

    return vb.prove_machine(cfg, None, device_resident=(dm, dp))


@pytest.mark.parametrize("repr_", ["canonical", "monty"])
@pytest.mark.parametrize("name", list(PROGRAMS))
def test_import_tensors_prove_the_host_bytes(ctx, cfg, proofs, name, repr_):
    import valida_b200 as vb

    t, proof = proofs[name]
    conv = (lambda a: a) if repr_ == "canonical" else _monty
    r = vb.REPR_CANONICAL if repr_ == "canonical" else vb.REPR_MONTY_R32
    tens = [_cuda(conv(m)) for m in t.main + t.preprocessed]
    dm = [ctx.import_tensor(x, r) for x in tens[:14]]
    dp = [ctx.import_tensor(x, r) for x in tens[14:]]
    assert _prove(cfg, dm, dp) == proof


LAYOUTS = ["row_major", "col_major_padded", "transposed", "sub_matrix", "every_other"]


def _layout(a, layout):
    torch = _torch()
    h, w = a.shape
    if layout == "row_major":
        return _cuda(a)
    if layout == "col_major_padded":
        return _col_major(a, pad=3)
    if layout == "transposed":
        return _cuda(np.ascontiguousarray(a.T)).t()
    if layout == "sub_matrix":                        # rows and columns of a larger tensor: row_stride > width
        big = torch.full((h + 5, w + 9), -1, dtype=torch.int32, device="cuda")
        big[2:2 + h, 3:3 + w] = _cuda(a)
        return big[2:2 + h, 3:3 + w]
    big = torch.full((2 * h, 2 * w), -1, dtype=torch.int32, device="cuda")   # no unit stride at all
    big[::2, ::2] = _cuda(a)
    return big[::2, ::2]


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("width", [1, 7, 127, 128, 129, 200])
def test_import_layouts_equal_upload(ctx, width, layout):
    """Widths around the 128-column tile and ragged row tiles; the import equals upload of the same words, and exporting it back
    gives the words imported."""
    import valida_b200 as vb

    rng = np.random.default_rng(width * 31 + len(layout))
    for h in [1, 3, 64, 65, 1000, 4097, 1 << 17]:
        if h * width > (1 << 17) * 129 and layout == "every_other":
            continue
        a = rng.integers(0, P, size=(h, width), dtype=np.uint32)
        x = _layout(a, layout)
        assert tuple(x.shape) == (h, width)
        for r in (vb.REPR_CANONICAL, vb.REPR_MONTY_R32):
            got = ctx.import_tensor(x, r)
            ref = ctx.upload(a, r)
            assert np.array_equal(got.download(vb.REPR_MONTY_R32), ref.download(vb.REPR_MONTY_R32)), (h, width, layout, r)
            assert np.array_equal(_host(got.to_tensor(r)), a), (h, width, layout, r)
            got.free()
            ref.free()


def test_import_uint32_tensor_and_empty(ctx):
    import valida_b200 as vb

    torch = _torch()
    a = np.arange(12, dtype=np.uint32).reshape(4, 3)
    x = _cuda(a).view(torch.uint32)
    assert np.array_equal(ctx.import_tensor(x).download(), a)
    e = ctx.import_tensor(torch.empty((0, 5), dtype=torch.int32, device="cuda"))
    assert e.shape == (0, 5)


@pytest.mark.parametrize("pad", [0, 5])
@pytest.mark.parametrize("name", list(PROGRAMS))
def test_borrow_proves_in_place(ctx, cfg, proofs, name, pad):
    """Column-major Montgomery tensors (col_stride = height + pad) prove to the same bytes; the borrow copies nothing and the
    tensors are bit-identical after the proof and after free."""
    t, proof = proofs[name]
    tens = [_col_major(_monty(m), pad) for m in t.main + t.preprocessed]
    before = [x.clone() for x in tens]
    live = ctx.memory_stats()["live"]
    dm = [ctx.borrow_tensor(x) for x in tens[:14]]
    dp = [ctx.borrow_tensor(x) for x in tens[14:]]
    assert ctx.memory_stats()["live"] == live                        # no copy of the borrowed traces
    assert _prove(cfg, dm, dp) == proof
    assert all(_torch().equal(x, y) for x, y in zip(tens, before))
    for m in dm + dp:
        m.free()
    _torch().cuda.synchronize()
    assert all(_torch().equal(x, y) for x, y in zip(tens, before))
    assert ctx.memory_stats()["live"] == live


def test_borrow_the_device_witness_exported_to_tensors(ctx, cfg, proofs):
    """The device witness's traces, exported into column-major tensors and borrowed back, prove to the bytes of the host traces."""
    import valida_b200 as vb

    torch = _torch()
    t, proof = proofs["fib"]
    log = vb.run_program_log(vb.fib_program(((1 << 10) - 17) // 7))
    wm, wp = log.witness_device(ctx)
    tens = []
    for m in wm + wp:
        h, w = m.shape
        tens.append(m.to_tensor(vb.REPR_MONTY_R32, out=torch.empty((w, h), dtype=torch.int32, device="cuda").t()))
    for m in wm + wp:
        m.free()
    dm = [ctx.borrow_tensor(x) for x in tens[:14]]
    dp = [ctx.borrow_tensor(x) for x in tens[14:]]
    assert _prove(cfg, dm, dp) == proof


@pytest.mark.parametrize("bad", [P, 0xFFFFFFFF])
def test_words_not_below_p_are_refused_by_position(ctx, bad):
    import valida_b200 as vb

    a = np.random.default_rng(1).integers(0, P, size=(300, 131), dtype=np.uint32)
    a[217, 129] = bad
    a[250, 3] = bad                                                   # a later row: the first offending word is named
    live = ctx.memory_stats()["live"]
    for x in (_cuda(a), _col_major(a, 2)):
        for r in (vb.REPR_CANONICAL, vb.REPR_MONTY_R32):
            with pytest.raises(vb.VgpuError, match=r"row 217, column 129"):
                ctx.import_tensor(x, r)
    with pytest.raises(vb.VgpuError, match=r"row 217, column 129"):
        ctx.borrow_tensor(_col_major(a, 2))
    assert ctx.memory_stats()["live"] == live                         # no matrix was created
    b = a.copy()
    b[0, 0] = bad
    with pytest.raises(vb.VgpuError, match=r"row 0, column 0"):
        ctx.borrow_tensor(_col_major(b))


def test_host_side_refusals_launch_nothing(ctx):
    import valida_b200 as vb
    from valida_b200.api import _DevMatrix, lib

    torch = _torch()
    host = np.zeros((64, 4), dtype=np.uint32)
    dev = torch.zeros((64, 4), dtype=torch.int32, device="cuda")
    n = ctx.launch_count

    def refused(call, pattern):
        out = C.c_void_p()
        assert call(out) != 0
        assert pattern in lib().vgpu_last_error(ctx._h).decode()
        assert not out.value

    hv = _DevMatrix(host.ctypes.data, 64, 4, 4, 1)
    refused(lambda o: lib().vgpu_dmat_import(ctx._h, C.byref(hv), 0, C.byref(o)), "not device memory")
    refused(lambda o: lib().vgpu_dmat_borrow(ctx._h, host.ctypes.data, 64, 4, 64, C.byref(o)), "not device memory")
    refused(lambda o: lib().vgpu_dmat_borrow(ctx._h, dev.data_ptr(), 64, 4, 63, C.byref(o)), "below the height")
    refused(lambda o: lib().vgpu_dmat_borrow(ctx._h, dev.data_ptr() + 2, 16, 4, 16, C.byref(o)), "4-byte aligned")
    over = _DevMatrix(dev.data_ptr(), 64, 4, 1 << 62, 1)
    refused(lambda o: lib().vgpu_dmat_import(ctx._h, C.byref(over), 0, C.byref(o)), "overflows")
    over = _DevMatrix(dev.data_ptr(), 1 << 40, 1 << 30, 1 << 30, 1)
    refused(lambda o: lib().vgpu_dmat_import(ctx._h, C.byref(over), 0, C.byref(o)), "overflows")
    refused(lambda o: lib().vgpu_dmat_borrow(ctx._h, dev.data_ptr(), 1 << 40, 1 << 30, 1 << 40, C.byref(o)), "overflows")
    past = _DevMatrix(dev.data_ptr(), 64, 4, 4, 1 << 40)             # the last word is not in the allocation
    refused(lambda o: lib().vgpu_dmat_import(ctx._h, C.byref(past), 0, C.byref(o)), "not device memory")
    for bad, exc in ((torch.zeros((4, 4), dtype=torch.int32), ValueError), (dev.float(), TypeError), (dev[0], ValueError), (host, TypeError)):
        with pytest.raises(exc):
            ctx.import_tensor(bad)
        with pytest.raises(exc):
            ctx.borrow_tensor(bad)
    with pytest.raises(ValueError, match="column-major"):
        ctx.borrow_tensor(dev)
    m = ctx.upload(host)
    with pytest.raises(ValueError):
        m.to_tensor(out=torch.zeros((4, 64), dtype=torch.int32, device="cuda"))
    with pytest.raises(ValueError):
        m.to_tensor(out=torch.zeros((64, 4), dtype=torch.int32))
    assert ctx.launch_count == n + 1                                  # the upload's transpose only
    with pytest.raises(vb.VgpuError, match="borrowed"):
        vb.Radix2Dft(ctx).dft_batch(ctx.borrow_tensor(_col_major(host)))


def _stages(ctx, oracle, t):
    """A trace, its committed LDE, its permutation trace and its quotient chunks (bit-reversed rows) for chip 0."""
    import valida_b200 as vb

    ref = oracle.prove(t.main, t.preprocessed, debug_checks=False)
    tr = ref.transcript()
    pcs = vb.TwoAdicFriPcs(ctx)
    main = ctx.upload(t.main[0])
    perm, cs = vb.generate_permutation_trace(ctx, 0, main, None, tr["perm_challenges"])
    _, main_pd = pcs.commit_batches([main])
    _, perm_pd = pcs.commit_batches([perm])
    lde = pcs.get_ldes(main_pd)[0]
    log_degree = t.main[0].shape[0].bit_length() - 1
    q = vb.quotient(ctx, 0, log_degree, None, lde, pcs.get_ldes(perm_pd)[0], cs, tr["perm_challenges"], tr["alpha"])
    assert np.array_equal(q.download(), ref.quotient_chunks(0))
    return {"trace": main, "lde": lde, "perm": perm, "quotient": q}, (main_pd, perm_pd)


def test_export_equals_download(ctx, oracle, proofs):
    import valida_b200 as vb

    torch = _torch()
    mats, _keep = _stages(ctx, oracle, proofs["mixed"][0])
    for name, m in mats.items():
        h, w = m.shape
        for r in (vb.REPR_CANONICAL, vb.REPR_MONTY_R32):
            ref = m.download(r)
            assert np.array_equal(_host(m.to_tensor(r)), ref), (name, r)
            big = torch.full((h + 3, w + 4), -1, dtype=torch.int32, device="cuda")
            m.to_tensor(r, out=big[1:1 + h, 2:2 + w])
            assert np.array_equal(_host(big[1:1 + h, 2:2 + w]), ref), (name, r)
            assert (big[0] == -1).all() and (big[:, :2] == -1).all() and (big[1 + h:] == -1).all() and (big[:, 2 + w:] == -1).all()
            cm = torch.empty((w, h), dtype=torch.uint32, device="cuda").t()
            m.to_tensor(r, out=cm)
            assert np.array_equal(_host(cm.view(torch.int32)), ref), (name, r)


def test_stream_order_through_events(ctx):
    """A tensor written by torch on a side stream is imported with no host synchronisation in between: the context's stream waits
    for the event recorded on that stream, and the imported words are the ones written."""
    import valida_b200 as vb

    torch = _torch()
    h, w = 1 << 16, 33
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        x = torch.zeros((h, w), dtype=torch.int64, device="cuda")
        for _ in range(8):                                            # a few dependent kernels ahead of the final values
            x = (x * 3 + 7) % P
        x = (torch.arange(h * w, device="cuda", dtype=torch.int64).reshape(h, w) * 7919 + x) % P
        y = x.to(torch.int32)
        m = ctx.import_tensor(y)
    expect = _host(y)
    assert np.array_equal(m.download(), expect)
    out = m.to_tensor(vb.REPR_MONTY_R32)                              # torch's current stream waits for the export
    assert np.array_equal(_host(out), _monty(expect))


@pytest.fixture(scope="module")
def fib15(built, oracle, cfg):
    import valida_b200 as vb

    t = vb.run_program(vb.fib_program(((1 << 15) - 17) // 7), initial_fp=0x1000)
    assert t.main[0].shape[0] == 1 << 15 and t.main[2].shape[0] == 1 << 17
    return t, vb.prove_machine(cfg, t)


@pytest.mark.parametrize("nranks", [2, 4])
def test_split_import_rows(oracle, fib15, nranks):
    """Every rank imports its rows of the same tensors (tall traces are split, short ones imported whole): single-GPU bytes."""
    import valida_b200 as vb

    t, single = fib15
    tens = [_cuda(m) for m in t.main + t.preprocessed]
    ctxs = [vb.Context(0) for _ in range(nranks)]
    try:
        vb.comm_init_local(ctxs)
        cfgs = [vb.StarkConfig(c, oracle.rc480) for c in ctxs]

        def rank(r, c):
            mats = [c.import_tensor_rows(x) for x in tens]
            row0, rows = mats[2].local_rows()
            assert rows == (1 << 17) // nranks and row0 == r * rows            # the memory chip is split
            assert mats[13].local_rows() == (0, t.main[13].shape[0])         # a short trace is whole
            return _prove(cfgs[r], mats[:14], mats[14:])

        assert all(p == single for p in vb.run_ranks(rank, ctxs))
    finally:
        for c in ctxs:
            c.close()


def test_full_size_borrow_saves_the_traces(ctx, oracle, cfg):
    """Fibonacci 2^22 from borrowed tensors: the uploaded traces' bytes, which are the recorded oracle proof's, and a peak that is
    lower by the traces' device copy."""
    import valida_b200 as vb

    torch = _torch()
    t = vb.run_program(vb.fib_program(((1 << 22) - 17) // 7), initial_fp=0x1000)
    assert t.main[0].shape[0] == 1 << 22
    mats = t.main + t.preprocessed
    ctx.release_cached()
    dm = [ctx.upload(m) for m in t.main]
    dp = [ctx.upload(m) for m in t.preprocessed]
    try:
        ctx.memory_stats(reset=True)
        proof = vb.prove_machine(cfg, t, device_resident=(dm, dp))
        peak_uploaded = ctx.memory_stats()["peak"]
        assert_matches_golden(proof, "fib_2p22")
    finally:
        for m in dm + dp:
            m.free()
        ctx.release_cached()
    tens = [_col_major(_monty(m)) for m in mats]
    bm = [ctx.borrow_tensor(x) for x in tens]
    try:
        ctx.memory_stats(reset=True)
        assert _prove(cfg, bm[:14], bm[14:]) == proof
        peak_borrowed = ctx.memory_stats()["peak"]
    finally:
        for m in bm:
            m.free()
        ctx.release_cached()
        del tens
        torch.cuda.empty_cache()
    traces = sum(m.nbytes for m in mats)
    assert traces > 2_000_000_000
    assert abs((peak_uploaded - peak_borrowed) - traces) <= 0.01 * traces, (peak_uploaded, peak_borrowed, traces)
    assert oracle.verify(proof, t.preprocessed) == 0
