"""Golden vectors produced by the REFERENCE'S OWN code (tests/golden/make_golden.py runs
the reference's src/limbo gp.hpp / kernels / acqui / rprop compiled against the Eigen stand-in).
 * CPU (`not gpu`): the oracle restatement reproduces every fixture;
 * GPU (`gpu`)    : the CUDA path reproduces every fixture through the reference-facing API.
Tolerances: 1e-10 absolute on K, mu, sigma^2, UCB, EI (BASELINE.json); alpha / log-lik / gradient
relative (they scale with cond(K) between any two correct fp64 orderings, SURVEY.md §7)."""
import glob
import os

import numpy as np
import pytest

GOLD = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "*.npz")))
IDS = [os.path.basename(p)[:-4] for p in GOLD]
KNAMES = {0: "SquaredExpARD", 1: "MaternFiveHalves", 2: "MaternThreeHalves", 3: "Exp", 4: "SquaredExpARD"}
# fixture kernel_id 4 = SquaredExpARD with Params::kernel_squared_exp_ard::k() = 2 (Lambda columns); the ABI / oracle id stays 0


def _kid(g):
    kid = int(g["kernel_id"])
    return (0, 2) if kid == 4 else (kid, 0)


def test_fixtures_present():
    assert len(GOLD) >= 10


def _hp_own(g):
    D = int(g["D"])
    kid, klam = _kid(g)
    nh = D + D * klam + 1 if kid == 0 else 2
    hp = np.asarray(g["hp"], dtype=float)  # final h-params the reference reports (incl. noise entry if optimised)
    return hp[:nh], hp


@pytest.mark.parametrize("path", GOLD, ids=IDS)
def test_oracle_reproduces_reference(path, oracle_mod):
    O = oracle_mod
    g = np.load(path)
    X, Y, Xq = g["X"], g["Y"], g["Xq"]
    noise, n0, on, iters = float(g["noise"]), int(g["n0"]), bool(g["optimize_noise"]), int(g["rprop_iters"])
    kid, klam = _kid(g)
    hp_own, hp_full = _hp_own(g)
    og = O.OracleGP()
    if iters > 0:
        hp0 = np.asarray(g["hp_in"], dtype=float)
        nh = X.shape[1] * (1 + klam) + 1 if kid == 0 else 2
        hp0 = hp0 if hp0.size else np.zeros(nh)
        og.set_data(X, Y - Y.mean(axis=0))
        og.set_kernel(kid, hp0, noise)
        og.fit()
        best, ne = og.rprop_lml(hp0, iters)
        assert ne == iters
        assert np.abs(best - hp_full).max() <= 1e-12
    if n0 > 0:
        og.set_data(X[:n0], Y[:n0] - Y[:n0].mean(axis=0))
        og.set_kernel(kid, hp_own, noise)
        og.fit()
        for i in range(n0, X.shape[0]):
            og.append(X[i], Y[: i + 1] - Y[: i + 1].mean(axis=0))
    else:
        og.set_data(X, Y - Y.mean(axis=0))
        og.set_kernel(kid, hp_own, noise)
        og.fit()
    assert np.abs(og.get(0) - g["K"]).max() <= 1e-15
    assert np.abs(og.get(1) - g["L"]).max() <= 1e-12
    assert np.abs(og.get(2) - g["alpha"]).max() <= 1e-11 * np.abs(g["alpha"]).max()
    mu, s2 = og.query(Xq)
    mu = mu + Y.mean(axis=0)
    assert np.abs(mu - g["mu"]).max() <= 1e-12 and np.abs(s2 - g["sigma2"]).max() <= 1e-13
    assert abs(og.log_lik() - float(g["loglik"])) <= 1e-12 * abs(float(g["loglik"]))
    gr = og.grad(optimize_noise=on)
    assert np.abs(gr - g["grad"]).max() <= 1e-10 * max(1.0, np.abs(g["grad"]).max())
    assert np.abs(O.ucb(mu[:, 0], s2, 0.5) - g["ucb"]).max() <= 1e-12
    mtr, _ = og.query(X)
    f_max = float((mtr[:, 0] + Y.mean(axis=0)[0]).max())
    assert np.abs(O.ei(mu[:, 0], s2, f_max, 0.0) - g["ei"]).max() <= 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize("path", GOLD, ids=IDS)
def test_cuda_path_reproduces_reference(path):
    from limbo_b200 import acqui, kernel, mean, model, opt
    g = np.load(path)
    X, Y, Xq = g["X"], g["Y"], g["Xq"]
    noise, n0, on, iters = float(g["noise"]), int(g["n0"]), bool(g["optimize_noise"]), int(g["rprop_iters"])
    kid, klam = _kid(g)
    hp_own, hp_full = _hp_own(g)

    class Prm:
        class kernel:
            pass

        class kernel_squared_exp_ard:
            k = klam
            sigma_sq = 1.0

        class opt_rprop:
            iterations = max(iters, 1)
            eps_stop = 0.0
    Prm.kernel.noise = noise
    Prm.kernel.optimize_noise = on
    D, P = X.shape[1], Y.shape[1]
    gp = model.GP(D, P, params=Prm, kernel=getattr(kernel, KNAMES[kid]), mean=mean.Data,
                  hp_opt=model.KernelLFOpt(Prm, opt.Rprop(Prm)))
    hp_in = np.asarray(g["hp_in"], dtype=float)
    if iters > 0:
        if hp_in.size:
            gp.kernel_function().set_h_params(hp_in)
        gp.compute(list(X), list(Y))
        gp.optimize_hyperparams()
        assert np.abs(gp.kernel_function().h_params() - hp_full).max() <= 1e-9
    else:
        gp.kernel_function().set_h_params(hp_full)
        if n0 > 0:
            gp.compute(list(X[:n0]), list(Y[:n0]))
            for i in range(n0, X.shape[0]):
                gp.add_sample(X[i], Y[i])
        else:
            gp.compute(list(X), list(Y))
    assert np.abs(gp.kernel_matrix() - g["K"]).max() <= 1e-10
    assert np.abs(gp.matrixL() - g["L"]).max() <= 1e-10
    assert np.abs(gp.alpha() - g["alpha"]).max() <= 1e-10 * np.abs(g["alpha"]).max()
    mu, s2 = gp.query_batch(Xq)
    assert np.abs(mu - g["mu"]).max() <= 1e-10 and np.abs(s2 - g["sigma2"]).max() <= 1e-10
    ll = gp.compute_log_lik()
    assert abs(ll - float(g["loglik"])) <= 1e-11 * abs(float(g["loglik"]))
    gr = gp.compute_kernel_grad_log_lik()
    assert np.abs(gr - g["grad"]).max() <= 1e-9 * max(1.0, np.abs(g["grad"]).max())
    _, _, ucb = acqui.UCB(gp, params=Prm).argmax_batch(Xq, return_values=True)
    assert np.abs(ucb - g["ucb"]).max() <= 1e-10
    best, idx, ei = acqui.EI(gp, params=Prm).argmax_batch(Xq, return_values=True)
    assert np.abs(ei - g["ei"]).max() <= 1e-10
    assert abs(best - g["ei"].max()) <= 1e-10
