"""GPU parity: NTT / coset-LDE / Keccak-Merkle commit through the C ABI vs the oracle (bit-exact)."""
import numpy as np
import pytest

P = 2013265921
pytestmark = pytest.mark.gpu


def rand_mat(rng, h, w):
    return rng.integers(0, P, size=(h, w), dtype=np.uint32)


@pytest.mark.parametrize("log_h,w", [(0, 1), (1, 3), (2, 2), (5, 7), (8, 51), (10, 16), (12, 5), (13, 3), (14, 2), (15, 3), (16, 4), (17, 3), (18, 2), (19, 2), (21, 2), (22, 2), (23, 1), (24, 1)])
def test_ntt_forward_inverse_bit_exact(ctx, oracle, log_h, w):
    import valida_b200 as vb

    rng = np.random.default_rng(100 + log_h)
    m = rand_mat(rng, 1 << log_h, w)
    dft = vb.Radix2Dft(ctx)
    d = ctx.upload(m)
    dft.dft_batch(d)
    got = d.download()
    assert np.array_equal(got, oracle.dft(m))
    dft.idft_batch(d)
    assert np.array_equal(d.download(), m)


def test_ntt_monty_repr_and_host_entry(ctx, oracle):
    import ctypes as C
    import valida_b200 as vb
    from valida_b200.api import REPR_MONTY_R32

    rng = np.random.default_rng(7)
    m = rand_mat(rng, 256, 9)
    R = (1 << 32) % P
    monty = (m.astype(np.uint64) * R % P).astype(np.uint32)
    d = ctx.upload(monty, repr=REPR_MONTY_R32)
    vb.Radix2Dft(ctx).dft_batch(d)
    out_monty = d.download(repr=REPR_MONTY_R32)
    rinv = pow(R, P - 2, P)
    assert np.array_equal((out_monty.astype(np.uint64) * rinv % P).astype(np.uint32), oracle.dft(m))
    # host-buffer entry point (the e2e path)
    buf = m.copy()
    ctx.check(vb.lib().vgpu_ntt_batch_host(ctx._h, buf.ctypes.data_as(C.POINTER(C.c_uint32)), 256, 9, 0, 0))
    assert np.array_equal(buf, oracle.dft(m))


@pytest.mark.parametrize("log_h,w,shift", [(0, 2, 31), (1, 1, 31), (3, 4, 31), (9, 14, 31), (12, 3, 31), (13, 5, 31), (15, 2, 7), (16, 2, pow(31, P - 2, P)), (17, 2, 31), (18, 3, 31), (19, 2, 31), (20, 2, 31), (21, 2, 31), (22, 2, 31), (23, 1, 961), (24, 1, 31)])
def test_coset_lde_bit_exact(ctx, oracle, log_h, w, shift):
    import valida_b200 as vb

    rng = np.random.default_rng(200 + log_h)
    m = rand_mat(rng, 1 << log_h, w)
    dft = vb.Radix2Dft(ctx)
    d = ctx.upload(m)
    br = dft.coset_lde_batch(d, 1, shift, bit_reversed=True).download()
    assert np.array_equal(br, oracle.coset_lde(m, 1, shift, bitrev=True))
    nat = dft.coset_lde_batch(d, 1, shift, bit_reversed=False).download()
    assert np.array_equal(nat, oracle.coset_lde(m, 1, shift, bitrev=False))


def test_commit_batches_mixed_heights(ctx, oracle):
    import valida_b200 as vb

    rng = np.random.default_rng(11)
    # the prove_fibonacci (n=25) shape: 14 matrices of heights 256,32,512,128,1,1024,1,1,1,1,1,1,256,1
    heights = [256, 32, 512, 128, 1, 1024, 1, 1, 1, 1, 1, 1, 256, 1]
    widths = [51, 1, 14, 16, 16, 18, 14, 28, 45, 14, 79, 7, 2, 6]
    mats = [rand_mat(rng, h, w) for h, w in zip(heights, widths)]
    pcs = vb.TwoAdicFriPcs(ctx)
    root, pd = pcs.commit_batches(mats)
    exp_root, exp_ldes = oracle.commit_batches(mats, want_ldes=True)
    assert np.array_equal(root, exp_root)
    for lde, exp in zip(pcs.get_ldes(pd), exp_ldes):
        assert np.array_equal(lde.download(), exp)
    # shifted commit (the quotient-chunk commit uses coset_shift = 31^2 per matrix)
    shifts = [31 * 31 % P] * len(mats)
    root2, pd2 = pcs.commit_shifted_batches(mats, shifts)
    assert np.array_equal(root2, oracle.commit_batches(mats, coset_shifts=shifts))
    assert not np.array_equal(root, root2)


def test_commit_wide_rows_multi_block_sponge(ctx, oracle):
    # rows longer than one 136-byte rate block, and exactly at block boundaries (34, 68 words)
    import valida_b200 as vb

    rng = np.random.default_rng(12)
    pcs = vb.TwoAdicFriPcs(ctx)
    for w in [33, 34, 35, 67, 68, 69, 79]:
        mats = [rand_mat(rng, 64, w)]
        root, _ = pcs.commit_batches(mats)
        assert np.array_equal(root, oracle.commit_batches(mats)), w


def test_ntt_linearity_and_roundtrip_large(ctx):
    # size-independent properties at the BASELINE config-2 shape (2^20 x 64): iNTT(NTT(x)) = x, NTT(a+b) = NTT(a)+NTT(b)
    import valida_b200 as vb

    h, w = 1 << 20, 64
    r = np.arange(h, dtype=np.uint64)[:, None]
    c = np.arange(w, dtype=np.uint64)[None, :]
    a = ((r * 64 + c) * 0x9E3779B1 % P).astype(np.uint32)
    b = ((r * 31 + c * 17 + 5) * 0x85EBCA6B % P).astype(np.uint32)
    dft = vb.Radix2Dft(ctx)
    da, db = ctx.upload(a), ctx.upload(b)
    dab = ctx.upload(((a.astype(np.uint64) + b) % P).astype(np.uint32))
    fa = dft.dft_batch(da).download()
    fb = dft.dft_batch(db).download()
    fab = dft.dft_batch(dab).download()
    assert np.array_equal(fab, ((fa.astype(np.uint64) + fb) % P).astype(np.uint32))
    assert np.array_equal(dft.idft_batch(da).download(), a)
    # first output row of a DFT is the column sum
    assert np.array_equal(fa[0], (a.astype(np.uint64).sum(axis=0) % P).astype(np.uint32))


@pytest.mark.parametrize("w", [1, 51, 64])
def test_ntt_config2_full_size_vs_oracle(ctx, oracle, w):
    """BASELINE config 2 at full size (2^20 rows; w = 64 and the w = 1 / w = 51 variants of SURVEY 8(d)): the forward
    transform equals the oracle's on every word, and the inverse returns the input."""
    import valida_b200 as vb

    h = 1 << 20
    r = np.arange(h, dtype=np.uint64)[:, None]
    c = np.arange(w, dtype=np.uint64)[None, :]
    x = ((r * 64 + c) * 0x9E3779B1 % P).astype(np.uint32)
    dft = vb.Radix2Dft(ctx)
    d = ctx.upload(x)
    got = dft.dft_batch(d).download()
    assert np.array_equal(got, oracle.dft(x))
    assert np.array_equal(dft.idft_batch(d).download(), x)


@pytest.mark.parametrize("log_h", [25, 26])
def test_ntt_above_2p24_roundtrip_and_oracle(ctx, oracle, log_h):
    """Natural-order transforms above 2^24 (the split halves exceed the fast 2^12 tiles): forward == oracle, inverse restores."""
    import valida_b200 as vb

    rng = np.random.default_rng(log_h)
    x = rng.integers(0, P, (1 << log_h, 1), dtype=np.uint32)
    dft = vb.Radix2Dft(ctx)
    d = ctx.upload(x)
    dft.dft_batch(d)
    got = d.download()
    if log_h == 25:
        assert np.array_equal(got, oracle.dft(x))
    else:   # two outputs by the defining sum (the oracle would need a minute): X[0] = sum_j x[j], X[n/2] = sum_j (-1)^j x[j]
        col = x[:, 0].astype(np.uint64)
        even, odd = int(col[0::2].sum() % P), int(col[1::2].sum() % P)
        assert int(got[0, 0]) == (even + odd) % P
        assert int(got[1 << (log_h - 1), 0]) == (even - odd) % P
    dft.idft_batch(d)
    assert np.array_equal(d.download(), x)


def test_coset_lde_larger_blowups_natural_order(ctx, oracle):
    import valida_b200 as vb

    rng = np.random.default_rng(77)
    x = rng.integers(0, P, (1 << 9, 3), dtype=np.uint32)
    dft = vb.Radix2Dft(ctx)
    for added_bits in (1, 2, 3, 4):
        got = dft.coset_lde_batch(ctx.upload(x), added_bits, 31).download()
        assert np.array_equal(got, oracle.coset_lde(x, added_bits, 31, False))
    with pytest.raises(vb.VgpuError, match="log_blowup = 1 only"):
        dft.coset_lde_batch(ctx.upload(x), 2, 31, bit_reversed=True)
    with pytest.raises(vb.VgpuError, match="1..4"):
        dft.coset_lde_batch(ctx.upload(x), 5, 31)
