"""Static checks of the device code inside the built library (CPU; cuobjdump ships with the CUDA toolkit): every translation
unit is compiled for sm_90a (H100) and nothing else, the kernels of the hot path are present, and the hot ones keep their state in
registers (no stack frame = no spills)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "valida_b200", "libvalida_b200.so")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

pytestmark = pytest.mark.skipif(not (os.path.exists(LIB) and os.path.exists(CUOBJDUMP)), reason="needs the built library and cuobjdump")


def _run(*args):
    return subprocess.run([CUOBJDUMP, *args, LIB], capture_output=True, text=True, check=True).stdout


def test_every_cubin_is_sm_90a():
    elfs = re.findall(r"ELF file\s+\d+:\s+(\S+)", _run("-lelf"))
    assert len(elfs) >= 10, elfs                                   # one per .cu translation unit
    assert all(e.endswith(".sm_90a.cubin") for e in elfs), elfs
    # no PTX for a JIT to fall back on: the product is sm_90a code, compiled ahead of time
    ptx = subprocess.run([CUOBJDUMP, "-lptx", LIB], capture_output=True, text=True).stdout
    assert "PTX file" not in ptx, ptx


def _resources():
    out = _run("-res-usage")
    res = {}
    for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", out):
        res[m.group(1)] = tuple(int(m.group(i)) for i in range(2, 6))
    return res


def test_hot_kernels_present_and_spill_free():
    res = _resources()
    assert len(res) >= 80, len(res)

    def find(sub):
        return {k: v for k, v in res.items() if sub in k}

    must_exist = ["ntt_pass_kernelILi14E", "ntt_pass_kernelILi8E", "leaf_hash_kernel", "compress_layer_kernel", "fri_leaf_hash_kernel", "tree_tail_kernel",
                  "quotient_kernelILi0E", "quotient_kernelILi13E", "perm_denominators_kernel", "ext_batch_inverse_kernel", "perm_terms_kernel",
                  "bary_kernel", "reduced_opening_kernel", "invden_norm_kernel", "fri_fold_kernel", "pow_grind_kernel", "rm_to_cm_kernel",
                  "cols_to_rows_kernel", "rows_to_cols_kernel", "cpu_rows_kernel", "mem_rows_kernel", "sort_scatter_kernel"]
    for name in must_exist:
        assert find(name), name
    # registers only (REG, STACK, SHARED, LOCAL): no stack frame, no local memory
    for name in ["ntt_pass_kernel", "leaf_hash_kernel", "compress_layer_kernel", "fri_leaf_hash_kernel", "tree_tail_kernel", "reduced_opening_kernel",
                 "bary_kernelILi", "invden_norm_kernel", "fri_fold_kernel", "pow_grind_kernel", "cols_to_rows_kernel", "rows_to_cols_kernel"]:
        for k, (reg, stack, shared, local) in find(name).items():
            assert stack == 0 and local == 0, (k, reg, stack, local)
    # occupancy-relevant ceilings the tuning relied on (512-thread NTT CTAs need <= 64 registers; Keccak kernels <= 80)
    for k, (reg, *_rest) in find("ntt_pass_kernel").items():
        assert reg <= 64, (k, reg)
    for name in ("leaf_hash_kernel", "compress_layer_kernel", "fri_leaf_hash_kernel", "tree_tail_kernel"):
        for k, (reg, *_rest) in find(name).items():
            assert reg <= 80, (k, reg)
    # no kernel anywhere uses local memory
    assert all(v[3] == 0 for v in res.values()), [k for k, v in res.items() if v[3]]
