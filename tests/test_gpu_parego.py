"""ParEGO on the device: lb_acq_argmax_cols / _dev and lb_acq_cmaes_cols (limbo_b200/csrc/query.cu: acq_cols_kernel) against
the oracle (oracle/parego.py over oracle.OracleGP), against lb_acq_argmax and one-output handles, model.GPParego's incremental
add_sample against a full compute with the same weights, the device values against tests/golden/parego, and bayes_opt.Parego on
MOP2 against an oracle replay of the same weights and candidate sets."""
import ctypes as C
import functools
import glob
import os

import numpy as np
import pytest

from limbo_b200 import acqui, bayes_opt, kernel, mean, model, synth
from oracle import ehvi as OE, oracle as O, parego as OP

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "parego", "*.npz")))
TOL = 1e-10  # the bound of the UCB / EI parity tests (tests/test_gpu_parity.py)


class _ColumnMean(mean.Data):
    """an input-dependent mean: mean::Data plus 0.1 (r + 1) x_0 in column r, so that mean_at_q is an M x q array"""

    def batch(self, xs, gp):
        base = super().batch(xs, gp)
        return base + 0.1 * np.asarray(xs)[:, :1] * np.arange(1, base.shape[1] + 1)[None, :]

    def __call__(self, v, gp):
        return self.batch(np.atleast_2d(v), gp)[0]

    def is_constant(self) -> bool:
        return False


def _problem(N, D=6, K=2, seed=3):
    X = synth.points(seed + N, N, D)
    F = OE.zdt2(X) if K == 2 else np.concatenate([OE.zdt2(X), -OE.zdt2(X)[:, :1]], axis=1)
    return X, F


@functools.lru_cache(maxsize=None)
def _fitted(N, q, column_mean):
    """(GPParego, its oracle (OracleGP on the same scalarised columns), candidates) with pinned weights"""
    X, F = _problem(N)
    draws = np.random.default_rng(N + q).random((q, 2))
    gp = model.GPParego(6, q, kernel=kernel.MaternFiveHalves, mean=_ColumnMean if column_mean else mean.Data)
    gp.compute(X, F, lambdas=draws)
    og = O.OracleGP()
    og.set_data(X, gp.obs_mean())
    og.set_kernel(O.K_MATERN52, gp.kernel_function().params(), gp.kernel_function().noise())
    og.fit()
    Xq = synth.points(7 + N, 1000, 6)
    return gp, og, Xq


def _oracle_values(gp, og, Xq, acq):
    mu, s2 = og.query(Xq)
    mu = mu + gp.mean_function().batch(Xq, gp)
    if acq == "ei":
        ms, _ = og.query(gp._sample_matrix())
        f_max = (ms + gp.mean_function().batch(gp._sample_matrix(), gp)).max(axis=0)
        return np.stack([O.ei(mu[:, r], s2, f_max[r], 0.0) for r in range(mu.shape[1])], axis=1)
    alpha = acqui.GP_UCB(gp, 10)._alpha() if acq == "gp_ucb" else 0.5
    return np.stack([O.ucb(mu[:, r], s2, alpha) for r in range(mu.shape[1])], axis=1)


def _acq(name, gp):
    return {"ucb": lambda: acqui.UCB(gp), "gp_ucb": lambda: acqui.GP_UCB(gp, 10), "ei": lambda: acqui.EI(gp)}[name]()


@pytest.mark.parametrize("N", [60, 300, 2048])
@pytest.mark.parametrize("q", [1, 3, 16])
@pytest.mark.parametrize("acq", ["ucb", "gp_ucb", "ei"])
@pytest.mark.parametrize("column_mean", [False, True], ids=["const_mean", "array_mean"])
def test_argmax_cols_matches_oracle(N, q, acq, column_mean):
    gp, og, Xq = _fitted(N, q, column_mean)
    best, idx, vals = _acq(acq, gp).argmax_cols(Xq, return_values=True)
    want = _oracle_values(gp, og, Xq, acq)
    assert vals.shape == (len(Xq), q)
    assert np.abs(vals - want).max() <= TOL * max(1.0, np.abs(want).max())
    for r in range(q):
        assert vals[idx[r], r] == best[r] and best[r] == vals[:, r].max() and idx[r] == int(np.argmax(vals[:, r]))


@pytest.mark.parametrize("M", [100, 1000])
@pytest.mark.parametrize("acq", ["ucb", "ei"])
@pytest.mark.parametrize("column_mean", [False, True], ids=["const_mean", "array_mean"])
def test_one_column_equals_acq_argmax_bit_for_bit(M, acq, column_mean):
    gp, _, Xq = _fitted(300, 1, column_mean)
    a = _acq(acq, gp)
    best, idx, vals = a.argmax_cols(Xq[:M], return_values=True)
    b1, i1, v1 = a.argmax_batch(Xq[:M], return_values=True)
    assert np.array_equal(vals[:, 0], v1) and best[0] == b1 and idx[0] == i1


@pytest.mark.parametrize("M", [100, 1000])
def test_each_column_equals_a_one_output_handle(M):
    """sigma^2 bit for bit; mu (hence the values) within the bound, and the test prints whether it is bit for bit"""
    q = 3
    gp, _, Xq = _fitted(300, q, False)
    vals = acqui.UCB(gp).argmax_cols(Xq[:M], return_values=True)[2]
    _, s2 = gp.query_batch(Xq[:M])
    same = []
    for r in range(q):
        one = model.GP(6, 1, kernel=kernel.MaternFiveHalves, mean=mean.Data)
        one.compute(gp._sample_matrix(), gp.observations_matrix()[:, r:r + 1])
        _, _, v1 = acqui.UCB(one).argmax_batch(Xq[:M], return_values=True)
        mu1, s21 = one.query_batch(Xq[:M])
        assert np.array_equal(s2, s21)
        assert np.abs(vals[:, r] - v1).max() <= TOL
        same.append(bool(np.array_equal(vals[:, r], v1)))
    print("columns bit-identical to one-output handles:", same)


def test_dev_equals_host():
    import torch
    from limbo_b200 import _lib
    gp, _, Xq = _fitted(300, 3, True)
    a = acqui.EI(gp)
    params = np.ascontiguousarray(a._col_params(), dtype=np.float64)
    best, idx, vals = gp.acq_argmax_cols(_lib.ACQ_EI, params, Xq, return_values=True)
    dev = torch.device("cuda", 0)
    dX = torch.from_numpy(Xq).to(dev)
    dMean = torch.from_numpy(np.ascontiguousarray(gp.mean_function().batch(Xq, gp))).to(dev)
    dVals = torch.empty((len(Xq), 3), dtype=torch.float64, device=dev)
    dBest = torch.empty(3, dtype=torch.float64, device=dev)
    dIdx = torch.empty(3, dtype=torch.int64, device=dev)
    zero = np.zeros(3)
    torch.cuda.synchronize()
    _lib.check(gp._lib.lb_acq_argmax_cols_dev(gp._h, _lib.ACQ_EI, 3, params.ctypes.data, len(Xq), dX.data_ptr(), dMean.data_ptr(),
                                              zero.ctypes.data, dVals.data_ptr(), dBest.data_ptr(), dIdx.data_ptr()), "dev")
    gp._lib.lb_sync(gp._h)
    assert np.array_equal(dVals.cpu().numpy(), vals) and np.array_equal(dBest.cpu().numpy(), best)
    assert np.array_equal(dIdx.cpu().numpy(), idx)


def test_argument_errors():
    from limbo_b200 import _lib
    gp, _, Xq = _fitted(60, 3, False)
    p = np.zeros(6)
    b, i = np.zeros(3), np.zeros(3, dtype=np.int64)
    call = gp._lib.lb_acq_argmax_cols
    assert call(gp._h, 0, 2, p.ctypes.data, 10, Xq.ctypes.data, None, b.ctypes.data, None, b.ctypes.data, i.ctypes.data) == -1  # q != P
    assert call(gp._h, 7, 3, p.ctypes.data, 10, Xq.ctypes.data, None, b.ctypes.data, None, b.ctypes.data, i.ctypes.data) == -5
    S = np.random.default_rng(0).random((4, 6))
    opts = _lib.CmaesOpts(0, 0.1, 5, 1e-6, 1, 1)
    for cols in ([0, 1, 1, 1], [0, 1, 2, 3]):  # column 2 without an instance; a column outside [0, q)
        c = np.array(cols, dtype=np.int32)
        bx = np.zeros((3, 6))
        n = C.c_int64()
        assert gp._lib.lb_acq_cmaes_cols(gp._h, 0, 3, p.ctypes.data, b.ctypes.data, C.byref(opts), 4, S.ctypes.data, c.ctypes.data,
                                         bx.ctypes.data, b.ctypes.data, C.addressof(n)) == -1
    with pytest.raises(NotImplementedError):
        model.GPParego(6, 2, precision="tf32")


def test_incremental_add_sample_matches_full_compute():
    X, F = _problem(301)
    draws = np.random.default_rng(1).random((2, 3, 2))
    inc = model.GPParego(6, 3, kernel=kernel.MaternFiveHalves)
    inc.compute(X[:300], F[:300], lambdas=draws[0])
    n0 = inc.append_count()
    inc.add_sample(X[300], F[300], lambdas=draws[1])
    assert inc.append_count() == n0 + 1 and inc.lambda_draws() == 6
    assert np.array_equal(inc.raw_observations(), F)
    full = model.GPParego(6, 3, kernel=kernel.MaternFiveHalves)
    full.compute(X, F, lambdas=draws[1])
    assert np.array_equal(inc.observations_matrix(), full.observations_matrix())
    Xq = synth.points(99, 500, 6)
    for a, b in ((inc.matrixL(), full.matrixL()), (inc.alpha(), full.alpha())):
        assert np.abs(a - b).max() <= 1e-10
    (m1, s1), (m2, s2) = inc.query_batch(Xq), full.query_batch(Xq)
    assert np.abs(m1 - m2).max() <= 1e-10 and np.abs(s1 - s2).max() <= 1e-10


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_device_values_match_golden(path):
    g = np.load(path)
    X, F, draws, n0, rho = g["X"], g["F"], g["draws"], int(g["n0"]), float(g["rho"])

    class P:
        class model_gp_parego:
            pass
    P.model_gp_parego.rho = rho
    gp = model.GPParego(X.shape[1], 1, params=P, kernel=kernel.MaternFiveHalves)
    gp.compute(X[:n0], F[:n0], lambdas=draws[:1])
    for i in range(n0, X.shape[0]):
        gp.add_sample(X[i], F[i], lambdas=draws[1 + i - n0: 2 + i - n0])
    assert np.array_equal(gp.observations_matrix()[:, 0], g["scal"])
    mu, s2 = gp.query_batch(g["Xq"])
    assert np.abs(mu[:, 0] - g["mu"]).max() <= TOL and np.abs(s2 - g["sigma2"]).max() <= TOL
    assert np.abs(acqui.UCB(gp).argmax_cols(g["Xq"], return_values=True)[2][:, 0] - g["ucb"]).max() <= TOL
    assert np.abs(acqui.EI(gp).argmax_cols(g["Xq"], return_values=True)[2][:, 0] - g["ei"]).max() <= TOL


def _trace(lib, R, lam, D):
    n = lib.lb_debug_cmaes_trace(None, 0)
    buf = np.empty(n)
    lib.lb_debug_cmaes_trace(buf.ctypes.data, n)
    M = R * lam
    return buf[n - M * D - M:n - M].reshape(M, D), buf[n - M:]


@pytest.mark.parametrize("acq", ["ucb", "ei"])
def test_cmaes_cols_scores_deterministic_and_q1(acq):
    from oracle import cmaes as OC
    gp, _, _ = _fitted(300, 3, False)
    a = _acq(acq, gp)
    R, D = 6, 6
    lam = OC.default_lambda(D)
    starts = np.random.default_rng(2).random((R, D))
    cols = [0, 1, 2, 2, 1, 0]
    gp._lib.lb_debug_cmaes_capture(1)
    bx, bv, n = a.cmaes_cols(starts, cols, generations=6, tolx=1e-9, seed=5)
    cand, vals = _trace(gp._lib, R, lam, D)
    gp._lib.lb_debug_cmaes_capture(0)
    full = a.argmax_cols(cand, return_values=True)[2]
    inst = np.repeat(np.asarray(cols), lam)
    assert np.array_equal(vals, full[np.arange(len(cand)), inst])
    assert n == 6 * R * lam and bx.shape == (3, D)
    for r in range(3):
        assert abs(a.argmax_cols(bx[r][None], return_values=True)[2][0, r] - bv[r]) <= 1e-12 * max(1.0, abs(bv[r]))
    again = a.cmaes_cols(starts, cols, generations=6, tolx=1e-9, seed=5)
    assert np.array_equal(again[0], bx) and np.array_equal(again[1], bv)
    g1, _, _ = _fitted(300, 1, False)
    a1 = _acq(acq, g1)
    x1, v1, n1 = a1.cmaes_cols(starts, [0] * R, generations=6, tolx=1e-9, seed=5)
    x0, v0, n0 = a1.cmaes_batch(starts, generations=6, tolx=1e-9, seed=5)
    assert np.array_equal(x1[0], x0) and v1[0] == v0 and n1 == n0


class _Recording(bayes_opt.BatchedRandomSearch):
    """BatchedRandomSearch that keeps every candidate set it scores"""

    def __init__(self, params, rng):
        super().__init__(params, rng)
        self.sets = []

    def __call__(self, acq, dim, bounded=True):
        m = int(bayes_opt._get(self._params, "opt_batchedrandom", "candidates"))
        cand = self._rng.random((m, dim))
        self.sets.append(cand)
        return cand[acq.argmax_batch(cand)[1]].copy()

    def propose_batch(self, acq, dim, bounded=True):
        cand = self._rng.random((int(bayes_opt._get(self._params, "opt_batchedrandom", "candidates")), dim))
        self.sets.append(cand)
        return cand[np.asarray(acq.argmax_cols(cand)[1])].copy()


def _mop2(x):
    return OE.mop2(np.asarray(x)[None, :])[0]


@pytest.mark.parametrize("q", [1, 4])
def test_parego_loop_matches_oracle_replay(q):
    class P:
        class stop_maxiterations:
            iterations = 8

        class init_randomsampling:
            samples = 10

        class opt_batchedrandom:
            candidates = 2000

        class kernel:
            noise = 1e-4

    rng = np.random.default_rng(21)
    bo = bayes_opt.Parego(P, q=q, acqui=acqui.UCB, acqui_opt=_Recording(P, rng), rng=rng)
    bo.model()._rng = np.random.default_rng(42)  # the weights on their own generator, replayed below
    bo.optimize(_mop2, 2)
    X = np.stack(bo.samples())
    replay = np.random.default_rng(42)
    op = OP.OracleParego(O.K_MATERN52, kernel.MaternFiveHalves(None, 2).params(), 1e-4)
    op.compute(X[:10], OE.mop2(X[:10]), [replay.random(2) for _ in range(q)])
    n, margins = 10, []
    for cand in bo._acqui_opt.sets:
        v = op.ucb(cand, 0.5)
        order = np.argsort(-v, axis=0)
        margins += [v[order[0, r], r] - v[order[1, r], r] for r in range(q)]
        picks = bayes_opt.distinct_rows(cand[order[0]])
        for x in picks:
            if n == X.shape[0]:
                break
            assert np.array_equal(X[n], x), (n, X[n], x)
            op.add_sample(x, _mop2(x), [replay.random(2) for _ in range(q)])
            n += 1
    assert n == X.shape[0] == 18
    assert min(margins) > 1e-8, min(margins)  # every pick is decided by far more than the parity bound


def test_cpp_parego_dropin():
    """tests/cpp/parego_dropin_test.cpp: the GPParego specialisation against the reference's GPParego under the same weights,
    Parego's loop over it with BatchedRandom on MOP2, and GP::acq_argmax_cols"""
    from dropin import run_dropin
    run_dropin("parego_dropin_test", "PAREGO DROPIN OK")
