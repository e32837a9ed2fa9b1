"""Static checks of the kernels of vgpu_bus_links in the built library (CPU; cuobjdump): the count and write sweeps are sm_90a SASS and
keep their state in registers (no stack frame, no local memory)."""
import re

from test_device_code_static import _resources, _run, pytestmark  # noqa: F401

KERNELS = ("link_count_kernel", "link_write_kernel")


def test_link_kernels_present_and_spill_free():
    res = _resources()
    found = {name: [k for k in res if name in k] for name in KERNELS}
    assert all(len(v) == 1 for v in found.values()), found
    assert all(e.endswith(".sm_90a.cubin") for e in re.findall(r"ELF file\s+\d+:\s+(\S+)", _run("-lelf")))
    for name, (k,) in found.items():
        reg, stack, shared, local = res[k]
        assert stack == 0 and local == 0, (k, reg, stack, local)
