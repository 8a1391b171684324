"""Runs the compiled drop-in test (tests/cpp/dropin_test.cpp): the reference's own C++ policy templates
(acqui::UCB / EI, model::gp::KernelLFOpt<Rprop>, kernel::*, mean::Data) instantiated over
limbo_b200::model::GP next to limbo::model::GP.  __graft_entry__.build() compiles it into oracle/_ref/ where the reference's
sources are present (oracle/ref.py: REF_SRC); without them the test skips."""
import pytest

from dropin import run_dropin


@pytest.mark.gpu
def test_reference_policy_templates_over_b200_gp():
    run_dropin("dropin_test", "DROPIN OK")
