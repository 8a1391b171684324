"""The two-CTA GEMM kernels on the benchmark path run without a stack frame.

`lbg::CfgDual` (gemm.cuh) runs two CTAs per SM.  Each warp holds 64 fp64 accumulators and a stage of
DMMA operands in registers.  A register spill puts local-memory traffic beside the DMMA stream, and a
stack frame in the cuobjdump resource table is what a spill leaves behind.  This test reads that table
from the built library and asserts STACK:0 and LOCAL:0 for every CfgDual instantiation of the kernels
on the benchmark path.  No GPU is needed; the test is skipped when the library is not built or
cuobjdump is missing."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "limbo_b200", "lib", "liblimbo_b200.so")

# kernel -> number of CfgDual instantiations (panel kernels: INV = false and INV = true)
TWO_CTA_KERNELS = {"syrk_kernel": 1, "panel_update_kernel": 2, "panel_solve_kernel": 2, "dchol_update_kernel": 1}
# CfgDual's mangled template arguments start with its tile: BN = 64, WN = 2, BK = 16
DUAL_TILE = "3CfgILi64ELi2ELi16E"


def _cuobjdump():
    for cand in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"), shutil.which("cuobjdump")):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def resources():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    r = subprocess.run([tool, "-res-usage", LIB], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    # " Function <mangled name>:" followed by "  REG:<n> STACK:<n> SHARED:<n> LOCAL:<n> ..."
    found = re.findall(r"^\s*Function (\S+):\s*\n\s*(REG:.*)$", r.stdout, flags=re.M)
    return {name: dict(kv.split(":", 1) for kv in usage.split()) for name, usage in found}


@pytest.mark.parametrize("kernel", sorted(TWO_CTA_KERNELS))
def test_two_cta_kernel_has_no_stack(kernel, resources):
    pat = re.compile(rf"{len(kernel)}{kernel}IN3lbg{DUAL_TILE}")
    found = {name: res for name, res in resources.items() if pat.search(name)}
    assert len(found) == TWO_CTA_KERNELS[kernel], f"{kernel}: CfgDual instantiations {sorted(found)}"
    for name, res in found.items():
        assert int(res["REG"]) <= 255, f"{name}: {res}"
        assert int(res["STACK"]) == 0 and int(res["LOCAL"]) == 0, f"{name} spills: {res}"
