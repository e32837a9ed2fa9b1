"""Merkle leaves on each side of every sponge-block boundary, byte for byte against the oracle: a row of w words is absorbed in
w // 34 + 1 Keccak blocks, and rows of one and two blocks take leaf_hash_kernel_blocks<1> / <2> while wider rows take the generic
leaf_hash_kernel.  Roots are compared after every commit, and the opening (opened rows and Merkle paths) after it."""
import numpy as np
import pytest

from test_gpu_open_edges import P, ext, open_and_compare

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("w", [1, 16, 33, 34, 35, 67, 68, 69, 101, 102, 205])
def test_commit_and_open_row_lengths(ctx, oracle, w):
    """The leaf row of w words is split over two matrices of one height (one when w = 1); a shorter 3-column matrix joins the
    tree as an injected one-block group."""
    rng = np.random.default_rng(3000 + w)
    widths = [w] if w == 1 else [w // 2, w - w // 2]
    mats = [rng.integers(0, P, (1 << 9, x), dtype=np.uint32) for x in widths] + [rng.integers(0, P, (1 << 6, 3), dtype=np.uint32)]
    z = ext(rng)
    open_and_compare(ctx, oracle, [(mats, [[z]] * len(mats))])


def test_mixed_heights_injected_two_block_groups(ctx, oracle):
    """Groups injected at every kind of layer: 50 words (two blocks, two matrices) at a layer of 2^16 nodes, hashed before
    compress_layer_kernel; 40 words (two blocks) and 70 words (generic) inside the fused tail; one word near the root."""
    rng = np.random.default_rng(4242)
    shape = [(1 << 16, 5), (1 << 15, 20), (1 << 15, 30), (1 << 12, 40), (1 << 10, 70), (1 << 8, 1)]
    mats = [rng.integers(0, P, s, dtype=np.uint32) for s in shape]
    z = ext(rng)
    open_and_compare(ctx, oracle, [(mats, [[z]] * len(mats))])
