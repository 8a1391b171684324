"""Pins the oracle restatement against the reference ITSELF: the reference's own headers compiled against the Eigen/Boost
stand-in (oracle/ref_shim -> oracle/_ref) were run on these seeded inputs and their outputs stored under
tests/golden/oracle_ref/ (tests/golden/make_golden_oracle_ref.py regenerates them)."""
import os

import numpy as np
import pytest

from limbo_b200 import synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_ref")
KIDS = [0, 1, 2, 3]
SHAPES = [(5, 1, 1), (33, 3, 2), (120, 6, 1)]
NOISE = 0.015


def restatement_inputs(kid, N, D, P):
    rng = np.random.default_rng(100 * kid + N)
    nh = D + 1 if kid == 0 else 2
    hp = rng.uniform(-0.7, 0.7, nh)
    X = synth.points(77 + N, N, D)
    y = synth.targets(X)
    Y = np.stack([y * (p + 1) - 0.3 * p for p in range(P)], axis=1)
    Xq = synth.points(78, 25, D)
    return {"hp": hp, "X": X, "Y": Y, "Xq": Xq}


def sampled_lower(N, n=300):
    """Row / column indices of the stored K and L entries: the whole lower triangle up to n entries, else a seeded sample."""
    i, j = np.tril_indices(N)
    if i.size > n:
        keep = np.sort(np.random.default_rng(N).choice(i.size, n, replace=False))
        i, j = i[keep], j[keep]
    return i, j


def restatement_name(kid, N, D, P):
    return f"restatement_k{kid}_n{N}_d{D}_p{P}.npz"


def rprop_inputs():
    X = synth.points(5, 50, 2)
    return X, synth.targets(X)


def incremental_inputs():
    X = synth.points(6, 40, 2)
    return X, synth.targets(X)[:, None]


@pytest.mark.parametrize("kid", KIDS)
@pytest.mark.parametrize("N,D,P", SHAPES)
def test_restatement_equals_reference(oracle_mod, kid, N, D, P):
    O = oracle_mod
    inp = restatement_inputs(kid, N, D, P)
    X, Y, Xq, hp = inp["X"], inp["Y"], inp["Xq"], inp["hp"]
    r = np.load(os.path.join(GOLDEN, restatement_name(kid, N, D, P)))
    og = O.OracleGP()
    og.set_data(X, Y - Y.mean(axis=0))
    og.set_kernel(kid, hp, NOISE)
    assert og.fit() == -1
    i, j = sampled_lower(N)
    assert np.abs(og.get(0)[i, j] - r["K"]).max() <= 1e-15
    assert np.abs(og.get(1)[i, j] - r["L"]).max() <= 1e-12
    assert np.abs(og.get(2) - r["alpha"]).max() <= 1e-11 * np.abs(r["alpha"]).max()
    mu, s2 = og.query(Xq)
    assert np.abs(mu + Y.mean(axis=0) - r["mu"]).max() <= 1e-12
    assert np.abs(s2 - r["sigma2"]).max() <= 1e-13
    assert abs(og.log_lik() - float(r["loglik"])) <= 1e-12 * abs(float(r["loglik"]))
    assert np.abs(og.grad() - r["grad"]).max() <= 1e-10 * max(1.0, np.abs(r["grad"]).max())


def test_rprop_trajectory_equals_reference(oracle_mod):
    """KernelLFOpt<Rprop> in the reference vs the restated Rprop on the restated objective."""
    O = oracle_mod
    X, y = rprop_inputs()
    r = np.load(os.path.join(GOLDEN, "rprop10_se_ard_n50_d2.npz"))
    og = O.OracleGP()
    og.set_data(X, (y - y.mean())[:, None])
    og.set_kernel(0, np.zeros(3), 0.01)
    og.fit()
    best, ne = og.rprop_lml(np.zeros(3), 10)
    assert ne == 10 and np.abs(best - r["hp"]).max() <= 1e-12


def test_incremental_equals_reference(oracle_mod):
    O = oracle_mod
    X, y = incremental_inputs()
    r = np.load(os.path.join(GOLDEN, "incremental_matern52_n40_d2.npz"))
    og = O.OracleGP()
    og.set_data(X[:25], y[:25] - y[:25].mean())
    og.set_kernel(1, np.zeros(2), 0.01)
    og.fit()
    for i in range(25, 40):
        og.append(X[i], y[: i + 1] - y[: i + 1].mean())
    assert np.abs(og.get(1) - r["L"]).max() <= 1e-12
    assert np.abs(og.get(2) - r["alpha"]).max() <= 1e-11 * np.abs(r["alpha"]).max()
