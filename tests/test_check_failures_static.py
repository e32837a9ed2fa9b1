"""Static checks of the kernels of vgpu_check_failures in the built library (CPU; cuobjdump): both passes of every chip and the scan are
sm_90a SASS and keep their state in registers (no stack frame, no local memory)."""
import re

from test_device_code_static import _resources, _run, pytestmark  # noqa: F401


def test_failure_kernels_present_and_spill_free():
    res = _resources()
    counts = {k: v for k, v in res.items() if "fail_count_kernelILi" in k}
    writes = {k: v for k, v in res.items() if "fail_write_kernelILi" in k}
    scans = {k: v for k, v in res.items() if "fail_scan_kernel" in k}
    assert len(counts) == 14 and len(writes) == 14 and len(scans) == 1, (sorted(counts), sorted(writes), sorted(scans))
    assert all(e.endswith(".sm_90a.cubin") for e in re.findall(r"ELF file\s+\d+:\s+(\S+)", _run("-lelf")))
    for k, (reg, stack, shared, local) in {**counts, **writes, **scans}.items():
        assert stack == 0 and local == 0, (k, reg, stack, local)
