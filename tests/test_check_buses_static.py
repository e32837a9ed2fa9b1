"""Static checks of the kernels of vgpu_check_buses in the built library (CPU; cuobjdump): the bucket, count and write sweeps and the
small bucket kernels are sm_90a SASS and keep their state in registers (no stack frame, no local memory)."""
import re

from test_device_code_static import _resources, _run, pytestmark  # noqa: F401

KERNELS = ("bus_bucket_kernel", "bus_count_kernel", "bus_write_kernel", "bus_reduce_kernel", "bus_mark_kernel", "bus_number_kernel")


def test_bus_kernels_present_and_spill_free():
    res = _resources()
    found = {name: [k for k in res if name in k] for name in KERNELS}
    assert all(len(v) == 1 for v in found.values()), found
    assert all(e.endswith(".sm_90a.cubin") for e in re.findall(r"ELF file\s+\d+:\s+(\S+)", _run("-lelf")))
    for name, (k,) in found.items():
        reg, stack, shared, local = res[k]
        assert stack == 0 and local == 0, (k, reg, stack, local)
