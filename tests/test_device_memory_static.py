"""The import / export kernels of caller device memory in the built library (CPU; cuobjdump ships with the CUDA toolkit): present,
registers only (no stack frame, no local memory), and loading and storing single 32-bit words, so that a borrowed or imported view
needs 4-byte alignment only, as include/valida_b200.h states."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "valida_b200", "libvalida_b200.so")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

pytestmark = pytest.mark.skipif(not (os.path.exists(LIB) and os.path.exists(CUOBJDUMP)), reason="needs the built library and cuobjdump")

KERNELS = ("import_kernelILb1E", "import_kernelILb0E", "export_kernel")


def _run(*args):
    return subprocess.run([CUOBJDUMP, *args, LIB], capture_output=True, text=True, check=True).stdout


def test_device_io_kernels_use_registers_only():
    res = {m.group(1): tuple(int(m.group(i)) for i in range(2, 6))
           for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", _run("-res-usage"))}
    for k in KERNELS:
        found = {n: v for n, v in res.items() if k in n}
        assert len(found) == 1, (k, found)
        (_, (reg, stack, shared, local)), = found.items()
        assert stack == 0 and local == 0, (k, reg, stack, local)


def test_device_io_kernels_access_caller_memory_by_single_words():
    sass = _run("-sass")
    for k in KERNELS:
        body = re.search(r"Function : \S*%s\S*\n(.*?)(?:\n\s*Function : |\Z)" % k, sass, flags=re.S).group(1)
        global_ops = re.findall(r"\b(LDG|STG)(\.[A-Z0-9_.]+)?", body)
        assert global_ops, k
        wide = [op + mods for op, mods in global_ops if re.search(r"\.(64|128)\b", mods)]
        assert not wide, (k, wide)
