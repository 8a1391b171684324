"""The fp64 GEMM core runs on Hopper's native DMMA.16x8x4 (mma.sync m16n8k4), not on DMMA.8x8x4.

On sm_90a the 8x8x4 shape reaches only half the fp64 tensor rate of the m16n8kK shapes (DESIGN.md §4.1), so
every kernel built on the tile GEMM core (gemm.cuh) and the diagonal-block kernel must issue the wide shape.
This reads the SASS of the built library, so a later edit or toolchain cannot bring the 8x8x4 path back
unnoticed.  No GPU is needed; the test is skipped when the library is not built or cuobjdump is missing."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "limbo_b200", "lib", "liblimbo_b200.so")

CORE_KERNELS = ["syrk_kernel", "trsm_panel_kernel", "dchol_update_kernel", "panel_update_kernel", "panel_solve_kernel",
                "trtri_level_kernel", "lauum_kernel", "potf2_inv_kernel"]
SHAPE = "DMMA.16x8x4"


def _cuobjdump():
    for cand in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"), shutil.which("cuobjdump")):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def sass_by_kernel():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    r = subprocess.run([tool, "-sass", LIB], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    # "Function : <mangled name>" starts each kernel's listing
    parts = re.split(r"^\s*Function : (\S+)\s*$", r.stdout, flags=re.M)
    return {parts[i]: parts[i + 1] for i in range(1, len(parts) - 1, 2)}


@pytest.mark.parametrize("kernel", CORE_KERNELS)
def test_core_kernel_issues_wide_dmma(kernel, sass_by_kernel):
    # mangled names carry the identifier with its length prefix, e.g. ...11syrk_kernelIN3lbg3CfgILi64...
    pat = re.compile(rf"{len(kernel)}{kernel}[IE]")
    found = {name: body for name, body in sass_by_kernel.items() if pat.search(name)}
    assert found, f"{kernel} not in the library"
    for name, body in found.items():
        shapes = set(re.findall(r"\bDMMA\.(\w+)", body))
        assert "8x8x4" not in shapes, f"{name} issues DMMA.8x8x4"
        assert shapes == {SHAPE.split(".", 1)[1]}, f"{name}: DMMA shapes {sorted(shapes)}"
