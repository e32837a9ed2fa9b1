"""Static check of the Keccak round loops in the built library (CPU; cuobjdump ships with the CUDA toolkit).  The Merkle kernels
are bound by the INT ALU pipe, which issues the LOP3s and SHFs of Keccak-f, so a round's count of them sets the hashing rate.  A
round needs 122 LOP3 (theta's column parities 20, theta folded into rho/pi 50, chi 50, iota 2) and 58 SHF (rho 48, theta's
rotations 10); ptxas is known to reassociate theta into 14 more LOP3s when the 3-input xor is not pinned."""
import os
import re
import shutil
import subprocess
from collections import Counter

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "valida_b200", "libvalida_b200.so")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

pytestmark = pytest.mark.skipif(not (os.path.exists(LIB) and os.path.exists(CUOBJDUMP)), reason="needs the built library and cuobjdump")

KERNELS = ("leaf_hash_kernel", "compress_layer_kernel", "fri_leaf_hash_kernel", "tree_tail_kernel")
INSN = re.compile(r"/\*([0-9a-f]+)\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)([^;]*);")


def _functions():
    out = subprocess.run([CUOBJDUMP, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    for body in re.split(r"\n\s*Function : ", out)[1:]:
        name, text = body.split("\n", 1)
        yield name.strip(), [(int(a, 16), op.split(".")[0], args) for a, op, args in INSN.findall(text)]


def _round_loops(insns):
    """Innermost loops (a backward branch and its target) with more than 100 LOP3 + SHF: the Keccak round loops."""
    loops = []
    for addr, op, args in insns:
        m = re.search(r"0x([0-9a-f]+)", args) if op == "BRA" else None
        if m and int(m.group(1), 16) < addr:
            loops.append((int(m.group(1), 16), addr))
    for lo, hi in loops:
        if any(lo <= a and b <= hi and (a, b) != (lo, hi) for a, b in loops):
            continue
        c = Counter(op for addr, op, _ in insns if lo <= addr <= hi)
        if c["LOP3"] + c["SHF"] > 100:
            yield c["LOP3"], c["SHF"]


def test_keccak_round_loops_at_the_instruction_floor():
    found = {k: 0 for k in KERNELS}
    for name, insns in _functions():
        kernel = next((k for k in KERNELS if re.search(r"\d" + k, name)), None)
        if kernel is None:
            continue
        for lop3, shf in _round_loops(insns):
            found[kernel] += 1
            assert lop3 <= 122 and shf <= 58, (name, lop3, shf)
    # every kernel has at least one round loop: leaf (generic and per block count), compress, FRI leaf, tail (thread per node)
    assert all(found.values()), found
