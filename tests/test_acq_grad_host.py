"""Candidate gradients without a GPU: the NumPy formulas of oracle/acq_grad.py against central differences of the oracle's own
mu / sigma^2 (the restatement pinned to the reference), the policy logic of bayes_opt.BatchedGradientSearch on a pure-NumPy
acquisition, and the SASS and resources of the new DMMA kernels in the built library."""
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from limbo_b200 import bayes_opt
from oracle import acq_grad as AG

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "limbo_b200", "lib", "liblimbo_b200.so")
H = 1e-5
REL = 1e-6


def _fit(O, kid, N, D, log_sf=0.0, noise=0.01, klam=0, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.random((N, D))
    y = np.sin(3 * X[:, :1]) + X[:, -1:] ** 2
    hp = np.concatenate([np.log(rng.uniform(0.3, 0.8, D)), 0.6 * rng.standard_normal(D * klam), [log_sf]]) if kid == AG.K_SE_ARD \
        else np.array([math.log(0.4), log_sf])
    og = O.OracleGP()
    og.set_data(X, y - y.mean())
    og.set_kernel(kid, hp, noise)
    assert og.fit() <= 0  # 1-based failing pivot otherwise
    return og, X, hp


def _central(og, Xq):
    M, D = Xq.shape
    dmu, ds2 = np.zeros((M, D)), np.zeros((M, D))
    for d in range(D):
        e = np.zeros(D)
        e[d] = H
        mp, sp = og.query(Xq + e)
        mm, sm = og.query(Xq - e)
        dmu[:, d] = (mp[:, 0] - mm[:, 0]) / (2 * H)
        ds2[:, d] = (sp - sm) / (2 * H)
    return dmu, ds2


def _close(an, fd):
    scale = np.maximum(np.abs(an).max(axis=1, keepdims=True), 1e-3)
    assert np.all(np.abs(an - fd) <= REL * scale), np.abs(an - fd).max()


CASES = [(AG.K_SE_ARD, 0), (AG.K_SE_ARD, 2), (AG.K_MATERN52, 0), (AG.K_MATERN32, 0), (AG.K_EXP, 0)]


@pytest.mark.parametrize("kid,klam", CASES)
def test_oracle_gradients_match_central_differences(oracle_mod, kid, klam):
    og, X, hp = _fit(oracle_mod, kid, 40, 3, klam=klam)
    rng = np.random.default_rng(1)
    Xq = rng.random((12, 3))
    mu, s2, dmu, ds2, _ = AG.query_grad(kid, hp, og.noise, X, og.get(1), og.get(2), Xq)
    mu_o, s2_o = og.query(Xq)
    assert np.allclose(mu, mu_o, rtol=0, atol=1e-12) and np.allclose(s2, s2_o, rtol=0, atol=1e-12)
    fd_mu, fd_s2 = _central(og, Xq)
    _close(dmu, fd_mu)
    _close(ds2, fd_s2)
    # UCB and EI through the oracle's own acquisition formulas
    f_max = float(mu_o[:, 0].max()) - 0.05
    for name, fun, args in (("ucb", AG.ucb, (0.7,)), ("ei", AG.ei, (f_max, 0.01))):
        val, grad = fun(mu[:, 0], s2, dmu, ds2, *args)
        ref = oracle_mod.ucb(mu_o[:, 0], s2_o, *args) if name == "ucb" else oracle_mod.ei(mu_o[:, 0], s2_o, *args)
        assert np.allclose(val, ref, rtol=0, atol=1e-12)
        fd = np.zeros_like(grad)
        for d in range(3):
            e = np.zeros(3)
            e[d] = H
            (mp, sp), (mm, sm) = og.query(Xq + e), og.query(Xq - e)
            vp = oracle_mod.ucb(mp[:, 0], sp, *args) if name == "ucb" else oracle_mod.ei(mp[:, 0], sp, *args)
            vm = oracle_mod.ucb(mm[:, 0], sm, *args) if name == "ucb" else oracle_mod.ei(mm[:, 0], sm, *args)
            fd[:, d] = (vp - vm) / (2 * H)
        _close(grad, fd)


@pytest.mark.parametrize("kid", [AG.K_SE_ARD, AG.K_MATERN52])
def test_clamp_and_ei_cutoff(oracle_mod, kid):
    """sigma_f^2 = e^-40 < DBL_EPSILON: the clamp of gp.hpp:623 is active everywhere, grad sigma^2 = 0, and with noise 0 the EI
    cut-off (sigma < 1e-10) makes the EI value and gradient 0 as well"""
    og, X, hp = _fit(oracle_mod, kid, 30, 2, log_sf=-20.0, noise=0.0)
    Xq = np.random.default_rng(2).random((8, 2))
    mu, s2, dmu, ds2, _ = AG.query_grad(kid, hp, 0.0, X, og.get(1), og.get(2), Xq)
    assert np.all(s2 == 0.0) and np.all(ds2 == 0.0)
    fd_mu, fd_s2 = _central(og, Xq)
    assert np.all(fd_s2 == 0.0)
    _close(dmu, fd_mu)
    val, grad = AG.ei(mu[:, 0], s2, dmu, ds2, 0.0)
    assert np.all(val == 0.0) and np.all(grad == 0.0)
    val, grad = AG.ucb(mu[:, 0], s2, dmu, ds2, 0.5)
    assert np.array_equal(grad, dmu)


class _Quadratic:
    """-|x - c|^2 on [0, 1]^D with a known maximum at c; counts the batched gradient calls."""

    def __init__(self, c, with_grad=True):
        self.c = np.asarray(c, dtype=np.float64)
        self.grad_calls = 0
        if not with_grad:
            self.grad_batch = None

    def _f(self, X):
        return -((np.atleast_2d(X) - self.c) ** 2).sum(axis=1)

    def argmax_batch(self, Xq, return_values=False):
        v = self._f(Xq)
        i = int(np.argmax(v))
        return (float(v[i]), i, v) if return_values else (float(v[i]), i)

    def grad_batch(self, Xq):
        self.grad_calls += 1
        return self._f(Xq), -2.0 * (np.atleast_2d(Xq) - self.c)


class _Params:
    class opt_batchedgradient:
        candidates = 200
        starts = 8
        iterations = 40
        alpha = 0.02


def _random_pass_best(acq, seed, dim):
    cand = np.random.default_rng(seed).random((_Params.opt_batchedgradient.candidates, dim))
    _, i = acq.argmax_batch(cand)
    return cand[i]


def test_policy_climbs_and_counts_calls():
    acq = _Quadratic([0.3, 0.8, 0.55])
    x = bayes_opt.BatchedGradientSearch(_Params, np.random.default_rng(5))(acq, 3, True)
    assert acq.grad_calls == _Params.opt_batchedgradient.iterations
    best_random = _random_pass_best(acq, 5, 3)
    assert acq._f(x)[0] >= acq._f(best_random)[0]
    assert np.abs(x - acq.c).max() < 1e-2


def test_policy_stays_in_the_box_and_never_below_the_random_pass():
    acq = _Quadratic([1.4, -0.3])  # the maximum over [0, 1]^2 is the corner (1, 0)
    for seed in range(4):
        x = bayes_opt.BatchedGradientSearch(_Params, np.random.default_rng(seed))(acq, 2, True)
        assert np.all((x >= 0.0) & (x <= 1.0))
        assert acq._f(x)[0] >= acq._f(_random_pass_best(acq, seed, 2))[0]


def test_policy_is_deterministic_under_a_seed():
    acq = _Quadratic([0.2, 0.4, 0.6, 0.8])
    a = bayes_opt.BatchedGradientSearch(_Params, np.random.default_rng(11))(acq, 4, True)
    b = bayes_opt.BatchedGradientSearch(_Params, np.random.default_rng(11))(acq, 4, True)
    assert np.array_equal(a, b)


def test_policy_falls_back_to_the_random_pass_without_gradients():
    acq = _Quadratic([0.5, 0.5], with_grad=False)
    x = bayes_opt.BatchedGradientSearch(_Params, np.random.default_rng(3))(acq, 2, True)
    assert np.array_equal(x, _random_pass_best(acq, 3, 2))


def _cuobjdump():
    for cand in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"), shutil.which("cuobjdump")):
        if cand and os.path.exists(cand):
            return cand
    return None


BWD_KERNELS = ["panel_bwd_update_kernel", "panel_bwd_solve_kernel"]


@pytest.fixture(scope="module")
def cuobjdump_lib():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    return tool


@pytest.mark.parametrize("kernel", BWD_KERNELS)
def test_backward_solve_kernels_issue_wide_dmma_without_stack(kernel, cuobjdump_lib):
    sass = subprocess.run([cuobjdump_lib, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    parts = re.split(r"^\s*Function : (\S+)\s*$", sass, flags=re.M)
    pat = re.compile(rf"{len(kernel)}{kernel}I")
    bodies = [parts[i + 1] for i in range(1, len(parts) - 1, 2) if pat.search(parts[i])]
    assert bodies, f"{kernel} not in the library"
    for body in bodies:
        assert set(re.findall(r"\bDMMA\.(\w+)", body)) == {"16x8x4"}
    res = subprocess.run([cuobjdump_lib, "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    found = [u for name, u in re.findall(r"^\s*Function (\S+):\s*\n\s*(REG:.*)$", res, flags=re.M) if pat.search(name)]
    assert found
    for usage in found:
        kv = dict(x.split(":", 1) for x in usage.split())
        assert int(kv["STACK"]) == 0 and int(kv["LOCAL"]) == 0 and int(kv["REG"]) <= 255, usage


class _NoGradientModel(_Quadratic):
    """an acquisition over a model or mean without candidate gradients: grad_batch exists but raises"""

    def __init__(self, c, exc):
        super().__init__(c)
        self.exc = exc

    def grad_batch(self, Xq):
        raise self.exc("no candidate gradient")


@pytest.mark.parametrize("exc", [AttributeError, NotImplementedError])
def test_policy_falls_back_when_the_model_gives_no_gradient(exc):
    acq = _NoGradientModel([0.5, 0.5], exc)
    x = bayes_opt.BatchedGradientSearch(_Params, np.random.default_rng(4))(acq, 2, True)
    assert np.array_equal(x, _random_pass_best(acq, 4, 2))
