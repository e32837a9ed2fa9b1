"""The Poseidon-16 MMCS (VGPU_MERKLE_POSEIDON16) restated in plain Python from the p3-symmetric definitions — NOT from
tests/c/poseidon_mmcs_oracle.cc — and compared with the oracle, which the GPU tests compare the product with:

  PaddingFreeSponge<Perm16, WIDTH 16, RATE 8, OUT 8>: state zero; the input absorbed 8 elements at a time by OVERWRITING
      state[0..len); a permutation after each chunk, a trailing partial chunk included (ceil(n / 8) permutations); output state[0..8).
  TruncatedPermutation<Perm16, N 2, CHUNK 8, WIDTH 16>: the first 8 elements of permute(left || right).
  FieldMerkleTreeMmcs: leaves hash the concatenated rows of the tallest matrices; a shorter group of matrices joins as
      node = compress(compress(l, r), hash(rows of the group)).

Perm16 is the challenger's permutation (test_pcs_restatement.poseidon).  Also: oracle Poseidon proofs of three programs are
accepted by the oracle verifier and rejected for the right reason when a path digest is flipped, their digests differ from the
Keccak proofs', and the new kernels are in the built library for sm_90a without stack or local memory."""
import os
import re
import shutil
import subprocess

import cbor2
import numpy as np
import pytest

from test_pcs_restatement import poseidon

P = 2013265921
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def sponge(words, rc):
    s = [0] * 16
    for i in range(0, len(words), 8):
        chunk = [int(w) for w in words[i:i + 8]]
        s[:len(chunk)] = chunk
        s = poseidon(s, rc)
    return s[:8]


def compress(left, right, rc):
    return poseidon([int(x) for x in left] + [int(x) for x in right], rc)[:8]


class Tree:
    """FieldMerkleTreeMmcs::commit over matrices given in the caller's order (power-of-two heights)."""

    def __init__(self, mats, rc):
        order = sorted(range(len(mats)), key=lambda i: -mats[i].shape[0])      # stable: equal heights keep the caller's order
        groups = {}
        for i in order:
            groups.setdefault(mats[i].shape[0], []).append(mats[i])
        top = mats[order[0]].shape[0]
        rows = lambda h, r: [w for m in groups[h] for w in m[r]]
        self.layers = [[sponge(rows(top, r), rc) for r in range(top)]]
        while len(self.layers[-1]) > 1:
            prev = self.layers[-1]
            n = len(prev) // 2
            nxt = [compress(prev[2 * i], prev[2 * i + 1], rc) for i in range(n)]
            if n in groups:
                nxt = [compress(nxt[i], sponge(rows(n, i), rc), rc) for i in range(n)]
            self.layers.append(nxt)
        self.root = self.layers[-1][0]

    def path(self, index):
        return [self.layers[i][(index >> i) ^ 1] for i in range(len(self.layers) - 1)]


@pytest.fixture(scope="module")
def mmcs(oracle):
    from poseidon_mmcs import PoseidonOracle

    return PoseidonOracle()


def test_sponge_counts_and_overwrites(oracle):
    """ceil(n / 8) permutations, nothing extra when 8 divides n, and a partial chunk leaves the rest of the rate as it was."""
    rc = oracle.rc480
    w = list(range(1, 10))
    assert sponge(w[:8], rc) == poseidon(list(range(1, 9)) + [0] * 8, rc)[:8]
    s = poseidon(list(range(1, 9)) + [0] * 8, rc)
    s[0] = 9
    assert sponge(w, rc) == poseidon(s, rc)[:8]
    assert sponge([], rc) == [0] * 8


@pytest.mark.parametrize("width", [1, 7, 8, 9, 16, 17, 67])
def test_single_matrix_root_and_openings(mmcs, oracle, width):
    rng = np.random.default_rng(width)
    m = rng.integers(0, P, (4, width), dtype=np.uint32)
    t = Tree([m], oracle.rc480)
    assert mmcs.merkle_root([m]).tolist() == t.root
    for idx in (0, 3):
        rows, path = mmcs.merkle_open([m], idx)
        assert rows[0].tolist() == m[idx].tolist()
        assert path.tolist() == t.path(idx)


def test_mixed_heights_root_and_openings(mmcs, oracle):
    """Heights 2^7 .. 2^0 in one commit, two matrices sharing a height, every width class: groups join at every level."""
    rng = np.random.default_rng(7)
    hw = [(1 << 7, 9), (1 << 5, 67), (1 << 6, 1), (1 << 7, 7), (1 << 4, 8), (1 << 3, 17), (1 << 2, 16), (1 << 1, 7), (1, 9), (1 << 5, 1)]
    mats = [rng.integers(0, P, (h, w), dtype=np.uint32) for h, w in hw]
    t = Tree(mats, oracle.rc480)
    assert mmcs.merkle_root(mats).tolist() == t.root
    assert mmcs.merkle_root(mats).tolist() != oracle.merkle_root(mats).tolist()     # not the Keccak tree
    for idx in (0, 77, 127):
        rows, path = mmcs.merkle_open(mats, idx)
        for m, r in zip(mats, rows):
            assert r.tolist() == m[idx >> (7 - (m.shape[0].bit_length() - 1))].tolist()
        assert path.tolist() == t.path(idx)


# ---- oracle Poseidon proofs -----------------------------------------------------------------------------------------------------
def _programs():
    import programs
    import valida_b200 as vb

    prog, cells = programs.static_data_program()
    return {
        "fib25": lambda: vb.run_program(vb.fib_program(25), initial_fp=0x1000),
        "mixed": lambda: vb.run_program(programs.mixed_program(100), initial_fp=0x1000),
        "static_data": lambda: vb.run_program(prog, initial_fp=0x1000, static_data=cells),
    }


def _flip_word(d, path):
    for k in path[:-1]:
        d = d[k]
    d[path[-1]]["value"] ^= 1      # a felt: {"value": word}


INPUT_PATH = ["opening_proof", "query_openings", 7, 2, "opening_proof", 1, 3]
FRI_PATH = ["opening_proof", "fri_proof", "query_proofs", 0, "commit_phase_openings", 0, "opening_proof", 0, 0]


@pytest.mark.parametrize("name", ["fib25", "mixed", "static_data"])
def test_oracle_poseidon_proofs(built, oracle, mmcs, name):
    t = _programs()[name]()
    proof = mmcs.prove(t.main, t.preprocessed).cbor()
    assert mmcs.verify(proof, t.preprocessed) == 0
    keccak = oracle.prove(t.main, t.preprocessed, debug_checks=False).cbor()
    a, b = cbor2.loads(proof), cbor2.loads(keccak)
    for k in ("main_trace", "perm_trace", "quotient_chunks"):
        assert a["commitments"][k] != b["commitments"][k], k
    assert a["opening_proof"]["fri_proof"]["commit_phase_commits"] != b["opening_proof"]["fri_proof"]["commit_phase_commits"]
    # each verifier refuses the other hash's proof
    assert mmcs.verify(keccak, t.preprocessed) != 0 and oracle.verify(proof, t.preprocessed) != 0
    for path, code in ((INPUT_PATH, -3), (FRI_PATH, -4)):        # oracle/pcs.h verify_multi_batches: -3 input Merkle path, -4 FRI Merkle path
        d = cbor2.loads(proof)
        _flip_word(d, path)
        assert mmcs.verify(cbor2.dumps(d), t.preprocessed) == code, path


LIB = os.path.join(ROOT, "valida_b200", "libvalida_b200.so")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.mark.skipif(not (os.path.exists(LIB) and os.path.exists(CUOBJDUMP)), reason="needs the built library and cuobjdump")
def test_poseidon_kernels_built_for_sm_90a_without_spills():
    out = subprocess.run([CUOBJDUMP, "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    res = {m.group(1): tuple(int(m.group(i)) for i in range(2, 5))
           for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)}
    for name in ("p16_leaf_kernel", "p16_layer_kernel", "p16_tail_kernel", "p16_fri_leaf_kernel", "p16_path_kernel"):
        found = {k: v for k, v in res.items() if name in k}
        assert len(found) == 1, (name, found)
        for k, (reg, stack, local) in found.items():
            assert stack == 0 and local == 0, (k, reg, stack, local)
    elfs = re.findall(r"ELF file\s+\d+:\s+(\S+)", subprocess.run([CUOBJDUMP, "-lelf", LIB], capture_output=True, text=True, check=True).stdout)
    assert any("merkle" in e for e in elfs) and all(e.endswith(".sm_90a.cubin") for e in elfs), elfs
