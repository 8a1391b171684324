"""CPU checks of multi-objective BO (experimental/acqui/ehvi.hpp, src/ehvi/ehvi_calculations.cc, experimental/tools/pareto.hpp):
the oracle's ehvi2d restatement and the device's table form against the reference's own code (live where oracle/_ref was built,
and through tests/golden/ehvi), the table form against the reference order on random fronts, the Pareto filter, the Python
host logic, and the new kernels' resource table."""
import glob
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import ehvi as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "ehvi", "*.npz")))
GP_FIXTURES = [p for p in FIXTURES if "X" in np.load(p).files]


def random_front(rng, k, lo=-10.0, hi=0.0):
    """k mutually non-dominated points, in random order."""
    f0 = np.sort(rng.uniform(lo, hi, k))
    f1 = np.sort(rng.uniform(lo, hi, k))[::-1]
    return np.stack([f0, f1], axis=1)[rng.permutation(k)]


def test_fixtures_present():
    assert len(FIXTURES) == 9 and len(GP_FIXTURES) == 7


@pytest.mark.parametrize("path", FIXTURES, ids=os.path.basename)
def test_table_form_equals_reference_fixtures(path):
    """With the C library's exp / erf and the reference's summation order, the table form equals the reference bit for bit."""
    g = np.load(path)
    got, _ = E.ehvi2d_tables(g["front"], g["r"], g["mu"][:, 0], g["s"][:, 0], g["mu"][:, 1], g["s"][:, 1], libm=True)
    assert np.array_equal(got, g["ehvi"])


@pytest.mark.parametrize("path", FIXTURES[:4], ids=os.path.basename)
def test_reference_order_equals_fixtures(path):
    g = np.load(path)
    for q in range(0, len(g["ehvi"]), 37):
        assert E.ehvi2d(g["front"], g["r"], g["mu"][q], g["s"][q]) == g["ehvi"][q]


@pytest.mark.parametrize("path", FIXTURES, ids=os.path.basename)
def test_vectorised_table_form_within_1e13(path):
    """numpy / scipy transcendentals and pairwise row sums: <= 1e-13 relative to the largest value up to k = 512 (the raw k = 2000
    front reaches 2.5e-13: two million cells summed in another order), and within the device tolerance everywhere."""
    g = np.load(path)
    got, scale = E.ehvi2d_tables(g["front"], g["r"], g["mu"][:, 0], g["s"][:, 0], g["mu"][:, 1], g["s"][:, 1])
    err = np.abs(got - g["ehvi"])
    if len(g["front"]) <= 512:
        assert err.max() <= 1e-13 * np.abs(g["ehvi"]).max()
    assert np.all(err <= E.tolerance(g["ehvi"], scale))


@pytest.mark.parametrize("k", [0, 1, 2, 7, 64, 512])
def test_table_form_against_reference_order_random_fronts(k):
    rng = np.random.default_rng(100 + k)
    F = random_front(rng, k)
    M = 6 if k >= 64 else 40
    mu = rng.uniform(-11.0, 1.0, (M, 2))
    s = rng.uniform(0.02, 3.0, (M, 2))
    want = np.array([E.ehvi2d(F, (-11.0, -11.0), mu[q], s[q]) for q in range(M)])
    exact, _ = E.ehvi2d_tables(F, (-11.0, -11.0), mu[:, 0], s[:, 0], mu[:, 1], s[:, 1], libm=True)
    assert np.array_equal(exact, want)
    got, scale = E.ehvi2d_tables(F, (-11.0, -11.0), mu[:, 0], s[:, 0], mu[:, 1], s[:, 1])
    assert np.abs(got - want).max() <= 1e-13 * np.abs(want).max()
    assert np.all(np.abs(got - want) <= E.tolerance(want, scale))


def test_front_order_does_not_matter():
    rng = np.random.default_rng(7)
    F = random_front(rng, 30)
    mu, s = rng.uniform(-11, 1, 2), rng.uniform(0.1, 2, 2)
    assert E.ehvi2d(F, (-11, -11), mu, s) == E.ehvi2d(F[::-1], (-11, -11), mu, s)


@pytest.mark.parametrize("path", FIXTURES, ids=os.path.basename)
def test_driver_equals_fixtures_live(path):
    from oracle import ref_ehvi
    if not ref_ehvi.available():
        pytest.skip("the reference's EHVI is not built and its sources are not present")
    g = np.load(path)
    if "X" in g.files:
        r = ref_ehvi.gp_ehvi(g["X"], g["Y"], g["Xq"], g["r"], float(g["noise"]))
        for key in ("ehvi", "mu", "s", "front"):
            assert np.array_equal(r[key], g[key]), key
    else:
        assert np.array_equal(ref_ehvi.ehvi2d(g["front"], g["r"], g["mu"], g["s"]), g["ehvi"])


@pytest.mark.parametrize("path", GP_FIXTURES, ids=os.path.basename)
def test_fixture_front_is_the_pareto_set_of_the_observations(path):
    """The front the reference built is pareto_set's content, in its order up to runs of exact ties."""
    g = np.load(path)
    idx = E.pareto_set(g["Y"])
    assert np.array_equal(g["Y"][idx], g["front"])


@pytest.mark.parametrize("n,K,dup", [(3000, 2, False), (3000, 3, True), (800, 5, True)])
def test_pareto_set_against_driver_live(n, K, dup):
    from oracle import ref_ehvi
    if not ref_ehvi.available():
        pytest.skip("the reference's EHVI is not built and its sources are not present")
    rng = np.random.default_rng(n + K)
    O = rng.integers(0, 25, (n, K)).astype(np.float64) + (0.0 if dup else rng.random((n, K)) * 1e-3)
    got, want = E.pareto_set(O), ref_ehvi.pareto_set(O)
    assert sorted(got) == sorted(want)
    assert np.array_equal(O[got], O[want])  # same order up to runs of equal points


def test_dominate_flag():
    from limbo_b200 import pareto
    for a, b, f in [((1, 2), (0, 2), 1), ((0, 2), (1, 2), -1), ((1, 0), (0, 1), 0), ((1, 1), (1, 1), 0)]:
        assert pareto.dominate_flag(a, b) == f == E.dominate_flag(a, b)
        assert pareto.dominate(a, b) == (f == 1)


def test_hypervolume_sweep():
    assert E.hypervolume([[1.0, 0.0], [0.0, 1.0]], (-1.0, -1.0)) == 3.0
    assert E.hypervolume([[1.0, 1.0], [0.5, 0.5]], (0.0, 0.0)) == 1.0


def test_params_defaults():
    from limbo_b200.params import get
    assert get(None, "bayes_opt_ehvi", "x_ref") == -11.0 and get(None, "bayes_opt_ehvi", "y_ref") == -11.0


class _Stub:
    """Records what BoMulti feeds a model."""

    def __init__(self, *a, **kw):
        self.args = (a, kw)

    def compute(self, X, Y):
        self.X, self.Y = X, Y


def test_bomulti_refits_one_model_per_objective(monkeypatch):
    from limbo_b200 import bayes_opt, model
    monkeypatch.setattr(model, "GP", _Stub)
    bo = bayes_opt.BoMulti()
    for i in range(5):
        bo.add_new_sample(np.array([i, 2.0 * i]), np.array([float(i), -float(i), 3.0]))
    bo.update_pareto_model()
    first = bo.models()
    assert bo.nb_objs() == 3 and len(first) == 3 and bo.pareto_model() == []
    for j, m in enumerate(first):
        assert m.args[0] == (2, 1) and m.X.shape == (5, 2) and np.array_equal(m.Y[:, 0], np.stack(bo.observations())[:, j])
    bo.update_pareto_model()
    assert all(a is not b for a, b in zip(first, bo.models()))  # from scratch every time


def test_entry_points_exported(lib):
    for name in ("lb_ehvi_argmax", "lb_ehvi_argmax_dev", "lb_pareto_set", "lb_pareto_set_dev"):
        assert hasattr(lib, name)


def test_new_kernels_have_no_stack_frame(lib):
    tool = next((c for c in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"), shutil.which("cuobjdump"))
                 if c and os.path.exists(c)), None)
    if tool is None:
        pytest.skip("cuobjdump not found")
    r = subprocess.run([tool, "-res-usage", os.path.join(ROOT, "limbo_b200", "lib", "liblimbo_b200.so")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    found = dict(re.findall(r"^\s*Function (\S+):\s*\n\s*(REG:.*)$", r.stdout, flags=re.M))
    for kernel in ("ehvi_kernel", "pareto_kernel", "values_argmax_kernel"):
        hits = {n: u for n, u in found.items() if f"{len(kernel)}{kernel}" in n}
        assert len(hits) == 1, (kernel, sorted(hits))
        usage = dict(kv.split(":", 1) for kv in next(iter(hits.values())).split())
        assert int(usage["STACK"]) == 0 and int(usage["LOCAL"]) == 0, (kernel, usage)
