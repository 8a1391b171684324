"""CPU checks of constrained BO (experimental/acqui/eci.hpp, experimental/bayes_opt/cboptimizer.hpp): the oracle's ECI
restatement against the reference's own ECI (live where oracle/_ref was built, and through tests/golden/eci), every branch of
the formula against a SciPy statement of it, the Python ECI functor's scalar path, and CBOptimizer's host logic with stand-in
models (no device needed)."""
import glob
import math
import os

import numpy as np
import pytest
from scipy import stats

from limbo_b200 import acqui, bayes_opt
from oracle import eci as oracle_eci

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "eci")
FIXTURES = sorted(glob.glob(os.path.join(GOLDEN, "*.npz")))


def scipy_eci(mu, s2, mu_c, s2_c, f_max, jitter, obj_empty=False, con_empty=False):
    """eci.hpp:76-130 with scipy's normal distribution."""
    sigma, sigma_c = math.sqrt(s2), math.sqrt(s2_c)
    if sigma < 1e-10 or obj_empty:
        return 0.0
    X = mu - f_max - jitter
    ei = X * stats.norm.cdf(X / sigma) + sigma * stats.norm.pdf(X / sigma)
    pf = 1.0 if (sigma_c < 1e-10 or con_empty) else stats.norm.cdf((mu_c - 1.0) / sigma_c)
    return pf * ei


def _oracle_on(r):
    return oracle_eci.eci(r["mu"], r["sigma2"], r["mu_c"][:, 0], r["sigma2_c"], float(r["f_max"]), float(r["jitter"]), False,
                 r["Yc"].shape[0] == 0)


def test_fixtures_present():
    assert len(FIXTURES) == 4


@pytest.mark.parametrize("path", FIXTURES, ids=os.path.basename)
def test_oracle_eci_equals_reference_live(path):
    """The restatement reproduces the reference's ECI bit for bit on the reference's own mu / sigma^2."""
    from oracle import ref, ref_eci
    if not os.path.isdir(ref.REF_SRC):
        pytest.skip("the reference's sources are not present")
    ref_eci.build()
    g = np.load(path)
    r = ref_eci.eci(int(g["con_kernel"]), g["X"], g["y"], g["Yc"], g["Xq"], float(g["noise"]), float(g["jitter"]))
    r.update(Yc=g["Yc"], jitter=g["jitter"])
    assert np.array_equal(_oracle_on(r), r["eci"])
    for k in ("eci", "mu", "sigma2", "mu_c", "sigma2_c", "f_max"):  # the fixtures are what the reference computes today
        assert np.array_equal(r[k], g[k]), k


@pytest.mark.parametrize("path", FIXTURES, ids=os.path.basename)
def test_oracle_eci_matches_fixtures(path):
    g = dict(np.load(path))
    assert np.array_equal(_oracle_on(g), g["eci"])
    if "jitter" in os.path.basename(path):
        assert np.all(g["eci"] == 0.0)


def test_fixture_f_max_is_the_best_predicted_sample():
    """f_max = max_i mu(x_i) over the objective's samples (eci.hpp:91-99): the mean::Data GP nearly interpolates."""
    for path in FIXTURES:
        g = np.load(path)
        assert abs(float(g["f_max"]) - g["y"].max()) < 0.05 * abs(g["y"].max())


# mu, s2, mu_c, s2_c, f_max, jitter, obj_empty, con_empty
BRANCHES = [
    (0.3, 0.2, 1.4, 0.3, 0.1, 0.0, False, False),     # both models informative
    (0.3, 0.2, 0.2, 0.05, 0.1, 0.0, False, False),    # constraint likely violated
    (0.3, 1e-21, 1.4, 0.3, 0.1, 0.0, False, False),   # sigma < 1e-10: 0 (eci.hpp:86)
    (0.3, 0.2, 1.4, 1e-21, 0.1, 0.0, False, False),   # sigma_c < 1e-10: Pf = 1 (eci.hpp:124)
    (0.3, 0.2, 1.4, 0.3, 0.1, 0.0, True, False),      # no objective samples: 0
    (0.3, 0.2, -3.0, 0.3, 0.1, 0.0, False, True),     # no constraint samples: Pf = 1
    (0.3, 0.2, 1.4, 0.3, 0.1, 0.25, False, False),    # jitter
    (-0.5, 0.04, 1.0, 0.5, 0.1, 0.0, False, False),   # far below f_max, Pf = 1/2
]


@pytest.mark.parametrize("case", BRANCHES)
def test_oracle_eci_branches_against_scipy(oracle_mod, case):
    mu, s2, mu_c, s2_c, f_max, jitter, oe, ce = case
    got = oracle_eci.eci_one(mu, s2, mu_c, s2_c, f_max, jitter, oe, ce)
    want = scipy_eci(*case)
    assert abs(got - want) <= 1e-14 * max(1.0, abs(want)), (got, want)
    if oe or s2 < 1e-20:
        assert got == 0.0
    if ce or s2_c < 1e-20:
        assert got == float(oracle_mod.ei([mu], [s2], f_max, jitter)[0])


class _Model:
    """Host stand-in for the Model concept: query(v) -> (mu, sigma^2) from a function, plus a sample list."""

    def __init__(self, f, samples=(), dim_out=1):
        self.f, self._samples, self._dim_out = f, [np.asarray(s, dtype=np.float64) for s in samples], dim_out
        self.added, self.computed, self.hp_calls = [], None, 0

    def query(self, v):
        return self.f(np.asarray(v, dtype=np.float64))

    def query_batch(self, Xq):
        mus, s2s = zip(*(self.f(x) for x in np.atleast_2d(Xq)))
        return np.stack(mus), np.array(s2s)

    def samples(self):
        return self._samples

    def nb_samples(self):
        return len(self._samples)

    def dim_in(self):
        return 2

    def dim_out(self):
        return self._dim_out

    def compute(self, X, Y):
        self._samples = list(np.asarray(X))
        self.computed = np.asarray(Y).copy()

    def add_sample(self, x, y):
        self._samples.append(np.asarray(x))
        self.added.append(np.asarray(y).copy())

    def optimize_hyperparams(self):
        self.hp_calls += 1


def _obj(x):
    return np.array([x[0] - 0.5 * x[1]]), 0.05 + 0.1 * x[1]


def _con(x):
    return np.array([0.5 + 1.5 * x[0], 7.0]), 0.02 + 0.3 * x[0]


@pytest.mark.parametrize("with_con", [True, False])
def test_python_eci_scalar_path_against_scipy(with_con):
    """acqui.ECI.__call__ follows eci.hpp line by line: f_max over the objective's samples, EI times Pf of the first output."""
    obj = _Model(_obj, samples=[[0.1, 0.2], [0.7, 0.1], [0.4, 0.9]])
    con = _Model(_con, samples=[[0.1, 0.2]], dim_out=2) if with_con else None
    class P:  # noqa: E306
        class acqui_eci:
            jitter = 0.01
    a = acqui.ECI(obj, con, 0, params=P)
    f_max = max(_obj(s)[0][0] for s in obj.samples())
    for v in ([0.3, 0.3], [0.9, 0.05], [0.0, 1.0]):
        mu, s2 = _obj(np.array(v))
        mc, s2c = _con(np.array(v)) if with_con else (np.zeros(2), 1.0)
        want = scipy_eci(mu[0], s2, mc[0], s2c, f_max, 0.01, False, not with_con)
        got = a(v)
        got = got[0] if isinstance(got, tuple) else got
        assert abs(got - want) <= 1e-14 * max(1.0, abs(want))
    assert a._f_max == f_max
    empty = acqui.ECI(_Model(_obj), con, 0, params=P)
    got = empty([0.3, 0.3])
    assert (got[0] if isinstance(got, tuple) else got) == 0.0
    assert empty.argmax_batch(np.zeros((5, 2)), return_values=True)[:2] == (0.0, 0)


# ---- CBOptimizer, host logic -------------------------------------------------------------------------------------------

class _Params:
    class init_randomsampling:
        samples = 3

    class stop_maxiterations:
        iterations = 4

    class bayes_opt_cboptimizer:
        hp_period = 2
        bounded = True


class _FixedPoints:
    """acquiopt stand-in: returns the next of a fixed list of points and records the acquisition objects it was given."""

    def __init__(self, points):
        self.points, self.seen = list(points), []

    def __call__(self, acq, dim, bounded):
        self.seen.append((acq, dim, bounded))
        return np.asarray(self.points.pop(0), dtype=np.float64)


def _sfun(x):
    # objective, then two constraint values; feasible (product > 0) when x0 > 0.5
    return np.array([10.0 * x[1], 1.0 if x[0] > 0.5 else 0.0, 2.0])


def _run(nb_constraints=2, points=None):
    obj, con = _Model(_obj), _Model(_con, dim_out=2)
    pts = points if points is not None else [[0.9, 0.1], [0.2, 0.95], [0.6, 0.3], [0.1, 0.8]]
    aopt = _FixedPoints(pts)
    sfun = _sfun if nb_constraints else (lambda x: _sfun(x)[:1])
    bo = bayes_opt.CBOptimizer(obj, con, params=_Params, acqui=acqui.ECI, acqui_opt=aopt, rng=np.random.default_rng(3))
    bo.optimize(sfun, 2, dim_out=1, nb_constraints=nb_constraints)
    return bo, obj, con, aopt


def test_cboptimizer_splits_every_new_observation():
    """Deviation (a): both models get the parts of the observation just made, not the last one of the initial split."""
    bo, obj, con, aopt = _run()
    obs = bo.observations()
    assert len(obs) == 3 + 4
    assert np.array_equal(obj.computed, np.stack([o[:1] for o in obs[:3]]))
    assert np.array_equal(con.computed, np.stack([o[1:] for o in obs[:3]]))
    for k in range(4):
        assert np.array_equal(obj.added[k], obs[3 + k][:1])
        assert np.array_equal(con.added[k], obs[3 + k][1:])
    assert obj.hp_calls == 2 and con.hp_calls == 2  # hp_period = 2 over 4 iterations, on both models
    for a, dim, bounded in aopt.seen:
        assert isinstance(a, acqui.ECI) and a._constraint_model is con and dim == 2 and bounded


def test_cboptimizer_best_is_feasible_and_paired():
    """Feasibility filter and deviation (b): the best feasible observation and ITS sample."""
    bo, _, _, _ = _run()
    obs, smp = bo.observations(), bo.samples()
    feas = [i for i, o in enumerate(obs) if np.prod(o[1:]) > 0]
    best = max(feas, key=lambda i: obs[i][0])
    assert np.array_equal(bo.best_observation(), obs[best][:1])
    assert np.array_equal(bo.best_sample(), smp[best])
    assert smp[best][0] > 0.5
    # the infeasible point (0.2, 0.95) has the largest objective of all: it must not win
    overall = int(np.argmax([o[0] for o in obs]))
    assert overall != best and obs[overall][1] == 0.0
    # the reference's indexing (cboptimizer.hpp:228) takes the position in the feasible-only list, a different sample here
    assert feas.index(best) != best


def test_cboptimizer_no_feasible_falls_back_to_all():
    bo, _, _, _ = _run(points=[[0.1, 0.1], [0.2, 0.95], [0.3, 0.3], [0.1, 0.8]])
    obs = bo.observations()
    if any(np.prod(o[1:]) > 0 for o in obs):  # the random initial points may be feasible; force the case
        for o in obs:
            o[1] = 0.0
    i = int(np.argmax([o[0] for o in obs]))
    assert np.array_equal(bo.best_observation(), obs[i][:1])
    assert np.array_equal(bo.best_sample(), bo.samples()[i])


def test_cboptimizer_without_constraints():
    """Deviation (c): with nb_constraints == 0 every observation is feasible; no constraint model is used."""
    bo, obj, con, aopt = _run(nb_constraints=0)
    obs = bo.observations()
    assert all(o.size == 1 for o in obs)
    i = int(np.argmax([o[0] for o in obs]))
    assert np.array_equal(bo.best_observation(), obs[i])
    assert np.array_equal(bo.best_sample(), bo.samples()[i])
    assert con.added == [] and con.computed is None and con.hp_calls == 0
    assert all(a._constraint_model is None for a, _, _ in aopt.seen)


def test_cboptimizer_rejects_wrong_observation_size():
    obj, con = _Model(_obj), _Model(_con, dim_out=2)
    bo = bayes_opt.CBOptimizer(obj, con, params=_Params, acqui_opt=_FixedPoints([[0.5, 0.5]] * 4), rng=np.random.default_rng(0))
    with pytest.raises(AssertionError):
        bo.optimize(_sfun, 2, dim_out=1, nb_constraints=1)


def test_params_defaults():
    from limbo_b200.params import get
    assert get(None, "acqui_eci", "jitter") == 0.0
    assert get(None, "bayes_opt_cboptimizer", "hp_period") == -1
    assert get(None, "bayes_opt_cboptimizer", "bounded") is True


def test_eci_entry_points_exported(lib):
    for name in ("lb_eci_argmax", "lb_eci_argmax_dev"):
        assert hasattr(lib, name), name


def test_eci_kernel_has_no_stack_frame(lib):
    """eci_kernel (query.cu) compiles for sm_90a without a stack frame or local memory (cuobjdump's resource table)."""
    import re
    import shutil
    import subprocess
    from limbo_b200 import _lib
    tool = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    tool = tool if os.path.exists(tool) else shutil.which("cuobjdump")
    if tool is None:
        pytest.skip("cuobjdump not found")
    r = subprocess.run([tool, "-res-usage", _lib.LIB_PATH], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    found = re.findall(r"^\s*Function (\S*10eci_kernel\S*):\s*\n\s*(REG:.*)$", r.stdout, flags=re.M)
    assert len(found) == 1, found
    res = dict(kv.split(":", 1) for kv in found[0][1].split())
    assert int(res["STACK"]) == 0 and int(res["LOCAL"]) == 0, res
