"""vgpu_diff_witness in the built library, without a GPU: its two kernels are sm_90a SASS that keep their state in registers (no stack
frame, no local memory), the per-column layout is the chips' columns in order with a name for each, and the call refuses a missing
context."""
import ctypes as C
import re

from test_device_code_static import _resources, _run, pytestmark  # noqa: F401


def test_diff_kernels_present_and_spill_free():
    res = _resources()
    kernels = {k: v for k, v in res.items() if "diff_count_kernel" in k or "diff_write_kernel" in k}
    assert len(kernels) == 2, sorted(kernels)
    assert all(e.endswith(".sm_90a.cubin") for e in re.findall(r"ELF file\s+\d+:\s+(\S+)", _run("-lelf")))
    for k, (reg, stack, shared, local) in kernels.items():
        assert stack == 0 and local == 0, (k, reg, stack, local)


def test_column_layout():
    import valida_b200 as vb

    names = []
    for chip in range(14):
        d = C.cast(vb.lib().vgpu_basic_machine_chip(chip), C.POINTER(C.c_uint32))       # chip_id, width, preprocessed_width
        names += [(chip, vb.TRACE_MAIN, c) for c in range(d[1])]
    names += [(1, vb.TRACE_PREPROCESSED, c) for c in range(7)] + [(12, vb.TRACE_PREPROCESSED, 0)]
    assert vb.witness_column_count() == len(names) == 319
    assert all(vb.column_name(*x) for x in names)
    assert vb.column_name(1, vb.TRACE_PREPROCESSED, 7) is None and vb.column_name(12, vb.TRACE_PREPROCESSED, 1) is None


def test_no_context_is_refused():
    import valida_b200 as vb

    n, t = C.c_uint64(), C.c_uint64()
    assert vb.lib().vgpu_diff_witness(None, None, None, None, 0, None, C.byref(n), C.byref(t), None, None) == -1
