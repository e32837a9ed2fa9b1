"""vgpu_cell_alternatives in the built library, without a GPU: its two kernels (one instance per chip) are sm_90a SASS that keep their
state in registers (no stack frame, no local memory), the CPU instance included, and the call refuses a missing context."""
import ctypes as C
import re

from test_device_code_static import _resources, _run, pytestmark  # noqa: F401


def test_alternative_kernels_present_and_spill_free():
    res = _resources()
    kernels = {k: v for k, v in res.items() if "alt_count_kernel" in k or "alt_write_kernel" in k}
    assert len(kernels) == 28, sorted(kernels)
    assert all(e.endswith(".sm_90a.cubin") for e in re.findall(r"ELF file\s+\d+:\s+(\S+)", _run("-lelf")))
    for k, (reg, stack, shared, local) in kernels.items():
        assert stack == 0 and local == 0, (k, reg, stack, local)


def test_no_context_is_refused():
    import valida_b200 as vb

    n, t, f = C.c_uint64(), C.c_uint64(), C.c_uint64()
    assert vb.lib().vgpu_cell_alternatives(None, vb.lib().vgpu_basic_machine_chip(0), None, None, 0, None, C.byref(n), C.byref(t),
                                           C.byref(f), None) == -1
