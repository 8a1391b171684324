"""The kernels that build 128 x 128 tiles of point pairs on pair_tile.cuh keep their registers and stack frames.

The K build, K* and the likelihood gradient share one staged distance sweep (pair_distances).  Each kernel's register count
sets how many CTAs share an SM, and its stack frame is where its spills go, so a change to the shared sweep that costs
one kernel a register or a spill slot shows up here.  The bounds are the cuobjdump resource table of CUDA 12.9 for sm_90a.
No GPU is needed; the test is skipped when the library is not built or cuobjdump is missing."""
import re

import pytest

from test_kernel_resources import resources  # noqa: F401  (fixture: cuobjdump -res-usage of the built library)

# mangled-name fragment -> (REG, STACK bytes) at most; kernel ids 0..3: SE-ARD, Matern-5/2, Matern-3/2, Exp
BOUNDS = {
    "13kbuild_kernelILi0E": (128, 0),
    "13kbuild_kernelILi1E": (80, 24),
    "13kbuild_kernelILi2E": (80, 16),
    "13kbuild_kernelILi3E": (80, 8),
    "11grad_kernelILi0E": (80, 48),
    "11grad_kernelILi1E": (80, 112),
    "11grad_kernelILi2E": (80, 96),
    "11grad_kernelILi3E": (80, 48),
    "12kstar_kernelE": (124, 0),
}


@pytest.mark.parametrize("kernel", sorted(BOUNDS))
def test_pair_tile_kernel_resources(kernel, resources):  # noqa: F811
    found = {name: res for name, res in resources.items() if re.search(kernel, name)}
    assert len(found) == 1, f"{kernel}: instantiations {sorted(found)}"
    (name, res), = found.items()
    reg, stack = BOUNDS[kernel]
    assert int(res["REG"]) <= reg and int(res["STACK"]) <= stack, f"{name}: {res}, bound REG:{reg} STACK:{stack}"
