"""PCS openings off the machine's path, byte for byte against the oracle: every width around the column groups of the
barycentric kernel and the parameter-table split of the reduced openings (RO_MAXW = 96), heights below, at and above one
barycentric tile, a base-field opening point, one point shared by several rounds, and leaf rows of many sponge blocks.

The machine's own proofs open at most 79 columns, always at points of the extension field, so none of these run there."""
import ctypes as C

import numpy as np
import pytest

P = 2013265921
GEN = 31                                      # coset shift of every committed LDE
pytestmark = pytest.mark.gpu

WIDTHS = [1, 2, 31, 32, 33, 63, 64, 65, 79, 95, 96, 97, 130, 200]


def ext(rng):
    return [int(v) for v in rng.integers(0, P, 5)]


def off_coset(z, log_lde):
    """z (base field) is not a point of the committed coset GEN * <w_(2^log_lde)>."""
    return pow(z * pow(GEN, P - 2, P) % P, 1 << log_lde, P) != 1


def open_and_compare(ctx, oracle, rounds):
    """rounds: [(matrices, [points of each matrix])].  Commits every round, checks the roots, seeds the challenger with them and
    opens: the bytes must equal the oracle's."""
    import valida_b200 as vb

    pcs = vb.StarkConfig(ctx, oracle.rc480).pcs()
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
    got = pcs.open_multi_batches([(pd, pts) for pd, (_, pts) in zip(pds, rounds)])
    want = oracle.open([mats for mats, _ in rounds], [p for _, pts in rounds for p in pts], obs)
    for pd in pds:
        pd.free()
    assert got == want


@pytest.mark.parametrize("npoints", [1, 2])
@pytest.mark.parametrize("log_h", [9, 10, 14])
def test_open_every_width(ctx, oracle, log_h, npoints):
    """h = 2^9: below one barycentric tile (bary_small_kernel); 2^10: exactly one tile; 2^14: sixteen tiles over several CTAs.
    Widths 31/32/33, 63/64/65 and 95/96/97 sit at the column-group boundaries of bary_kernel (an odd group's surplus column
    shadows the last one); 97, 130 and 200 take several reduced-opening launches, of which only the first subtracts the
    opened values.  All matrices share the first point, the second one is the matrix's own."""
    rng = np.random.default_rng(1000 + 10 * log_h + npoints)
    mats = [rng.integers(0, P, (1 << log_h, w), dtype=np.uint32) for w in WIDTHS]
    z = ext(rng)
    pts = [[z] if npoints == 1 else [z, ext(rng)] for _ in mats]
    open_and_compare(ctx, oracle, [(mats, pts)])


def test_open_base_field_point(ctx, oracle):
    """A point with limbs 1..4 zero takes the other inverse-denominator path (x - z, then the ext5 batch inversion).  In the
    first round it shares a height with an extension-field point, and one matrix is opened at both, so the cache of inverse
    denominators per (height, point) holds both kinds at once."""
    rng = np.random.default_rng(2024)
    zb = [7, 0, 0, 0, 0]
    assert all(off_coset(zb[0], k) for k in (10, 11, 13))
    ze = ext(rng)
    r0 = [rng.integers(0, P, (1 << 10, 7), dtype=np.uint32), rng.integers(0, P, (1 << 10, 40), dtype=np.uint32),
          rng.integers(0, P, (1 << 9, 3), dtype=np.uint32)]
    r1 = [rng.integers(0, P, (1 << 12, 97), dtype=np.uint32), rng.integers(0, P, (1 << 12, 5), dtype=np.uint32)]
    open_and_compare(ctx, oracle, [(r0, [[zb, ze], [ze], [zb]]), (r1, [[zb], [ze, zb]])])


def test_open_shared_point_across_rounds(ctx, oracle):
    """Matrices of one height in three rounds, all opened at one point: each round's reduced openings continue the alpha powers
    where the previous round of that height stopped."""
    rng = np.random.default_rng(77)
    z, z2 = ext(rng), ext(rng)
    rounds = []
    for widths in ([97, 5], [64], [3, 33]):
        mats = [rng.integers(0, P, (1 << 10, w), dtype=np.uint32) for w in widths] + [rng.integers(0, P, (1 << 11, 2), dtype=np.uint32)]
        rounds.append((mats, [[z] for _ in widths] + [[z, z2]]))
    open_and_compare(ctx, oracle, rounds)


def test_commit_and_open_leaf_rows_of_many_sponge_blocks(ctx, oracle):
    """Matrices of one height whose rows together are 205 words: each Merkle leaf is one row of all three, absorbed over seven
    Keccak blocks of 34 words.  A shorter matrix joins the tree at its own level."""
    rng = np.random.default_rng(12)
    mats = [rng.integers(0, P, (1 << 12, w), dtype=np.uint32) for w in (90, 70, 45)] + [rng.integers(0, P, (1 << 10, 3), dtype=np.uint32)]
    z = ext(rng)
    open_and_compare(ctx, oracle, [(mats, [[z]] * 4)])
