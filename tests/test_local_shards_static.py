"""Row shards in caller device memory, in the built library (CPU): the four entry points are exported and declared in the header and in
both Rust crates, and the exchange kernel that hands a borrowed row shard over to the ranks that extend its columns uses registers
only and loads single 32-bit words, so that the shard needs 4-byte alignment only (cuobjdump ships with the CUDA toolkit)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "valida_b200", "libvalida_b200.so")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
FUNCS = ("vgpu_ctx_local_rows", "vgpu_dmat_import_local", "vgpu_dmat_borrow_local", "vgpu_dmat_export_local")
KERNEL = "rows_to_cols_scalar_kernel"

needs_lib = pytest.mark.skipif(not os.path.exists(LIB), reason="needs the built library")
needs_cuobjdump = pytest.mark.skipif(not (os.path.exists(LIB) and os.path.exists(CUOBJDUMP)), reason="needs the built library and cuobjdump")


def _read(*parts):
    with open(os.path.join(ROOT, *parts)) as f:
        return f.read()


def test_declared_in_the_header_and_both_crates():
    header = _read("include", "valida_b200.h")
    sys_crate = _read("rust", "valida-b200-sys", "src", "lib.rs")
    safe = _read("rust", "valida-b200", "src", "lib.rs")
    for f in FUNCS:
        assert re.search(r"\b%s\(" % f, header), f
        assert re.search(r"pub fn %s\(" % f, sys_crate), f
        assert re.search(r"sys::%s\(" % f, safe), f
    for f in ("fn local_rows(&self, height: u64)", "unsafe fn import_device_local(", "unsafe fn borrow_device_local(",
              "unsafe fn export_device_local("):
        assert f in safe, f


@needs_lib
def test_exported_by_the_library():
    lib = C.CDLL(LIB)
    for f in FUNCS:
        assert hasattr(lib, f), f


def _cuobjdump(*args):
    return subprocess.run([CUOBJDUMP, *args, LIB], capture_output=True, text=True, check=True).stdout


@needs_cuobjdump
def test_scalar_exchange_uses_registers_only():
    res = {m.group(1): tuple(int(m.group(i)) for i in range(2, 6))
           for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", _cuobjdump("-res-usage"))}
    found = {n: v for n, v in res.items() if KERNEL in n}
    assert len(found) == 1, found
    (_, (reg, stack, shared, local)), = found.items()
    assert stack == 0 and local == 0, (reg, stack, local)


@needs_cuobjdump
def test_scalar_exchange_loads_single_words():
    """Its loads read the caller's buffer a 32-bit word at a time; its stores into the symmetric heap may be wide."""
    sass = _cuobjdump("-sass")
    body = re.search(r"Function : \S*%s\S*\n(.*?)(?:\n\s*Function : |\Z)" % KERNEL, sass, flags=re.S).group(1)
    loads = re.findall(r"\bLDG(\.[A-Z0-9_.]+)?", body)
    assert loads
    wide = [mods for mods in loads if re.search(r"\.(64|128)\b", mods)]
    assert not wide, wide
    assert re.search(r"\bSTG\.E\.128\b", body)
