"""Runs the compiled drop-in test (tests/cpp/dropin_test.cpp): the reference's own C++ policy templates
(acqui::UCB / EI, model::gp::KernelLFOpt<Rprop>, kernel::*, mean::Data) instantiated over
limbo_b200::model::GP next to limbo::model::GP.  __graft_entry__.build() compiles it into oracle/_ref/ where the reference's
sources are present (oracle/ref.py: REF_SRC); without them the test skips."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "oracle", "_ref", "dropin_test")


@pytest.mark.gpu
def test_reference_policy_templates_over_b200_gp():
    if not os.path.exists(BIN):
        pytest.skip("oracle/_ref/dropin_test not built (needs the reference's sources at build time)")
    env = dict(os.environ, LD_LIBRARY_PATH=os.path.join(ROOT, "limbo_b200", "lib") + ":" + os.environ.get("LD_LIBRARY_PATH", ""))
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=300, env=env)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "DROPIN OK" in r.stdout, r.stdout + r.stderr
