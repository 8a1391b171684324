"""The batched methods of the C++ models (include/limbo_b200/model/gp.hpp, spgp.hpp) against a recording stand-in for the C
library, without a GPU: tests/cpp/binding_calls_test.cpp, built by oracle/ref_shim/Makefile's binding_calls_test against the
reference's headers."""
import os
import subprocess

import pytest

from dropin import ROOT, run_dropin
from oracle import ref


def test_cpp_binding_calls():
    if not ref.available():
        pytest.skip("the reference's sources are not present")
    if os.path.isdir(ref.REF_SRC):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle", "ref_shim"), "CXX=g++", f"REF={ref.REF_ROOT}", "binding_calls_test"],
                       check=True, capture_output=True)
    run_dropin("binding_calls_test", "BINDING CALLS OK", timeout=60)
