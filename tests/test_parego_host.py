"""ParEGO without a GPU: the scalarisation against the reference's own GPParego (oracle/_ref/libref_parego.so, built where the
reference's sources are present), the oracle model against tests/golden/parego, the weight bookkeeping of model.GPParego, the
q > 1 proposal rules of bayes_opt.Parego, the new entry points and their argument errors, and the new kernels' resources."""
import ctypes as C
import glob
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from limbo_b200 import _lib, bayes_opt, kernel
from limbo_b200.model import gp_parego as G
from oracle import oracle as O, parego as OP, ref_parego

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "parego", "*.npz")))
LIB = os.path.join(ROOT, "limbo_b200", "lib", "liblimbo_b200.so")


def _objectives(rng, N, K, negative):
    F = rng.normal(size=(N, K)) if negative else rng.random((N, K))
    F[3] = F[4]  # a repeated observation
    return F


@pytest.mark.parametrize("K", [2, 3])
@pytest.mark.parametrize("rho", [0.0, 0.05])
@pytest.mark.parametrize("negative", [False, True])
def test_scalarisation_matches_the_reference_bit_for_bit(K, rho, negative):
    if not ref_parego.available():
        pytest.skip("needs the reference's sources or a built oracle/_ref/libref_parego.so")
    rng = np.random.default_rng(K * 7 + int(rho * 100) + negative)
    X, F, W = rng.random((40, 2)), _objectives(rng, 40, K, negative), rng.random((1, K))
    scal, _, _ = ref_parego.parego(X, F, W, X[:1], rho=rho)
    assert np.array_equal(scal, OP.scalarise(OP.normalise(W[0]), F, rho))
    assert np.array_equal(scal, G.scalarise(G.normalise(W[0]), F, rho))


def test_add_sample_sequence_rescalarises_with_the_last_draw():
    if not ref_parego.available():
        pytest.skip("needs the reference's sources or a built oracle/_ref/libref_parego.so")
    rng = np.random.default_rng(5)
    X, F, W = rng.random((30, 3)), rng.normal(size=(30, 2)), rng.random((6, 2))
    scal, _, _ = ref_parego.parego(X, F, W, X[:1], n0=25)
    assert np.array_equal(scal, OP.scalarise(OP.normalise(W[-1]), F, 0.05))


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_oracle_matches_the_golden_files(path):
    g = np.load(path)
    X, F, draws, n0, rho = g["X"], g["F"], g["draws"], int(g["n0"]), float(g["rho"])
    D = X.shape[1]
    op = OP.OracleParego(O.K_MATERN52, kernel.MaternFiveHalves(None, D).params(), 0.01, rho)
    op.compute(X[:n0], F[:n0], draws[:1])
    for i in range(n0, X.shape[0]):
        op.add_sample(X[i], F[i], draws[1 + i - n0: 2 + i - n0])
    assert np.array_equal(op.Y[:, 0], g["scal"])
    mu, s2 = op.query(g["Xq"])
    assert np.abs(mu[:, 0] - g["mu"]).max() < 1e-12 and np.abs(s2 - g["sigma2"]).max() < 1e-12
    assert np.abs(op.ucb(g["Xq"], 0.5)[:, 0] - g["ucb"]).max() < 1e-12
    assert np.abs(op.ei(g["Xq"])[:, 0] - g["ei"]).max() < 1e-12


def _host_only_parego(q, seed):
    m = G.GPParego.__new__(G.GPParego)
    m._q, m._rng, m._params = q, np.random.default_rng(seed), None
    m._raw, m._lambda, m._draws = np.zeros((0, 0)), np.zeros((q, 0)), 0
    return m


def test_one_draw_per_column_per_update_from_the_models_generator():
    q, K = 3, 2
    m = _host_only_parego(q, 11)
    m._raw = np.random.default_rng(0).normal(size=(10, K))
    Y = m._scalarised(None)
    expect = np.random.default_rng(11)
    draws = [expect.random(K) for _ in range(q)]
    assert m.lambda_draws() == q and Y.shape == (10, q)
    for r in range(q):
        assert np.array_equal(m.lambdas()[r], G.normalise(draws[r]))
        assert np.array_equal(Y[:, r], OP.scalarise(OP.normalise(draws[r]), m._raw, 0.05))
    m._raw = np.vstack([m._raw, [[1.0, -2.0]]])  # add_sample's step: every row rescalarised with fresh draws
    Y2 = m._scalarised(None)
    assert m.lambda_draws() == 2 * q and Y2.shape == (11, q)
    assert np.array_equal(Y2[:, 0], OP.scalarise(OP.normalise(expect.random(K)), m._raw, 0.05))
    pinned = np.array([[1.0, 3.0], [2.0, 2.0], [5.0, 1.0]])
    Y3 = m._scalarised(pinned)
    assert np.array_equal(m.lambdas(), np.stack([G.normalise(p) for p in pinned])) and m.lambda_draws() == 3 * q
    assert np.array_equal(Y3[:, 2], OP.scalarise(OP.normalise(pinned[2]), m._raw, 0.05))


def test_distinct_rows_drops_repeated_proposals_in_order():
    X = np.array([[0.1, 0.2], [0.3, 0.4], [0.1, 0.2], [0.5, 0.6], [0.3, 0.4]])
    assert np.array_equal(bayes_opt.distinct_rows(X), X[[0, 1, 3]])


class _FakeModel:
    def __init__(self):
        self.added = []

    def compute(self, X, F):
        self.computed = len(X)

    def add_sample(self, x, f):
        self.added.append(np.array(x))

    def optimize_hyperparams(self):
        pass


class _FakePolicy:
    """proposes q = 3 points per call, the second equal to the first"""

    def __init__(self):
        self.calls = 0

    def propose_batch(self, acqui, dim, bounded=True):
        self.calls += 1
        x = np.full(dim, 0.01 * self.calls)
        return np.stack([x, x, x + 0.5])


def test_q_batch_loop_counts_each_evaluated_point_and_drops_duplicates():
    class P:
        class stop_maxiterations:
            iterations = 5

        class init_randomsampling:
            samples = 2

    bo = bayes_opt.Parego.__new__(bayes_opt.Parego)
    bayes_opt.BOptimizer.__init__(bo, _FakeModel(), P, lambda m, it, params=None: None, _FakePolicy(), np.random.default_rng(0))
    bo._q = 3
    evals = []
    bo.optimize(lambda x: (evals.append(x), np.array([x.sum(), -x.sum()]))[1], 2)
    # 2 initial samples, then 2 distinct points per proposal: 2 + 2 + 1 (the fifth iteration ends the loop mid-batch)
    assert len(evals) == 7 and bo._current_iteration == 5 and bo._acqui_opt.calls == 3
    assert len(bo.model().added) == 5


def test_gradient_policy_refuses_q_batches():
    with pytest.raises(NotImplementedError):
        bayes_opt.BatchedGradientSearch().propose_batch(None, 2)


def test_new_symbols_are_declared_and_exported():
    lib = _lib.load()
    for name in ("lb_acq_argmax_cols", "lb_acq_argmax_cols_dev", "lb_acq_cmaes_cols"):
        assert hasattr(lib, name) and name in _lib.DECLARED_SYMBOLS


def test_argument_errors_are_raised_before_any_device_work():
    lib = _lib.load()
    v = np.zeros(8)
    i = np.zeros(8, dtype=np.int64)
    # NULL handle, NULL outputs, M <= 0: LB_ERR_ARG before the handle is touched
    assert lib.lb_acq_argmax_cols(None, 0, 1, v.ctypes.data, 4, v.ctypes.data, None, v.ctypes.data, None, v.ctypes.data, i.ctypes.data) == -1
    assert lib.lb_acq_argmax_cols_dev(None, 0, 1, v.ctypes.data, 0, v.ctypes.data, None, v.ctypes.data, None, v.ctypes.data,
                                      i.ctypes.data) == -1
    opts = _lib.CmaesOpts(0, 0.1, 10, 1e-6, 1, 1)
    cols = np.zeros(2, dtype=np.int32)
    assert lib.lb_acq_cmaes_cols(None, 0, 1, v.ctypes.data, v.ctypes.data, C.byref(opts), 2, v.ctypes.data, cols.ctypes.data,
                                 v.ctypes.data, v.ctypes.data, i.ctypes.data) == -1


def test_new_kernels_have_no_stack_frame():
    tool = next((c for c in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"), shutil.which("cuobjdump"))
                 if c and os.path.exists(c)), None)
    if tool is None:
        pytest.skip("cuobjdump not found")
    r = subprocess.run([tool, "-res-usage", LIB], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    found = dict(re.findall(r"^\s*Function (\S+):\s*\n\s*(REG:.*)$", r.stdout, flags=re.M))
    for k in ("acq_cols_kernel", "argmax_final_kernel"):
        hits = {n: u for n, u in found.items() if f"{len(k)}{k}" in n}
        assert len(hits) == 1, (k, sorted(hits))
        usage = dict(kv.split(":", 1) for kv in next(iter(hits.values())).split())
        assert int(usage["STACK"]) == 0 and int(usage["LOCAL"]) == 0 and int(usage["REG"]) <= 64, (k, usage)
