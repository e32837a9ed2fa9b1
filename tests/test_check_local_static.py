"""Static checks of the constraint-check kernels in the built library (CPU; cuobjdump): the run sweep of every chip and the copy kernel of
the boundary windows are present and keep their state in registers (no stack frame)."""
from test_device_code_static import _resources, pytestmark  # noqa: F401


def test_check_kernels_present_and_spill_free():
    res = _resources()
    sweeps = {k: v for k, v in res.items() if "check_kernelILi" in k}
    copies = {k: v for k, v in res.items() if "check_copy_kernel" in k}
    assert len(sweeps) == 14 and len(copies) == 1, (sorted(sweeps), sorted(copies))
    for k, (reg, stack, shared, local) in {**sweeps, **copies}.items():
        assert stack == 0 and local == 0, (k, reg, stack, local)
