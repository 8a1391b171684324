"""Constrained BO on the device: lb_eci_argmax (the objective's and the constraint's queries on their own streams, the fused
eci_kernel epilogue) against the reference's own ECI (tests/golden/eci), against the oracle on both query paths, against EI
where it must degenerate to it, and through the Python and C++ callers."""
import ctypes as C
import glob
import os
import subprocess
import threading

import numpy as np
import pytest

from oracle import eci as oracle_eci

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "eci", "*.npz")))
LB_ERR_ARG = -1


def _params(noise=0.01, jitter=0.0, constant=0.25):
    class P:
        class kernel:
            pass

        class mean_constant:
            pass

        class acqui_eci:
            pass
    P.kernel.noise = noise
    P.mean_constant.constant = constant
    P.acqui_eci.jitter = jitter
    return P


def _models(P, X, y, Xc, Yc, obj_kernel="SquaredExpARD", obj_mean="Data", con_kernel="Exp", **kw):
    from limbo_b200 import kernel, mean, model
    D = X.shape[1]
    gp = model.GP(D, 1, params=P, kernel=getattr(kernel, obj_kernel), mean=getattr(mean, obj_mean), **kw.get("obj", {}))
    gp.compute(X, np.asarray(y).reshape(-1, 1))
    con = model.GP(D, 2, params=P, kernel=getattr(kernel, con_kernel), mean=mean.Constant, **kw.get("con", {}))
    if len(Yc):
        con.compute(Xc, Yc)
    return gp, con


@pytest.mark.parametrize("path", GOLDEN, ids=os.path.basename)
def test_eci_matches_reference_fixtures(path):
    from limbo_b200 import acqui
    g = np.load(path)
    nc = g["Yc"].shape[0]
    P = _params(float(g["noise"]), float(g["jitter"]))
    gp, con = _models(P, g["X"], g["y"], g["X"][:nc], g["Yc"], con_kernel={1: "MaternFiveHalves", 3: "Exp"}[int(g["con_kernel"])])
    a = acqui.ECI(gp, con, 0, params=P)
    best, idx, vals = a.argmax_batch(g["Xq"], return_values=True)
    assert abs(a._f_max - float(g["f_max"])) <= 1e-10
    assert np.abs(vals - g["eci"]).max() <= 1e-10
    assert idx == int(np.argmax(g["eci"])) and best == vals[idx]
    if float(g["jitter"]) > 0:  # every value is 0: the lowest index wins
        assert np.all(vals == 0.0) and idx == 0


def _oracle_side(O, kid, X, obs, mean_add, Xq, noise=0.01):
    og = O.OracleGP()
    og.set_data(X, obs - mean_add)
    og.set_kernel(kid, np.zeros(X.shape[1] + 1 if kid == O.K_SE_ARD else 2), noise)
    assert og.fit() == -1
    mu, s2 = og.query(Xq)
    mu_x, _ = og.query(X)
    return mu + mean_add, s2, mu_x + mean_add


@pytest.mark.parametrize("M", [100, 3000])  # slab path, panel path
@pytest.mark.parametrize("obj_kernel", ["SquaredExpARD", "MaternFiveHalves"])
@pytest.mark.parametrize("obj_mean", ["Data", "Constant"])
def test_eci_matches_oracle(oracle_mod, M, obj_kernel, obj_mean):
    from limbo_b200 import acqui, synth
    O = oracle_mod
    D, N, Nc = 4, 300, 180
    X = synth.points(31, N, D)
    y = synth.targets(X)
    Yc = np.stack([0.3 + 1.5 * X[:Nc, 0] + 0.2 * np.sin(7 * X[:Nc, 2]), 1.0 + X[:Nc, 1]], axis=1)
    Xq = synth.points(32, M, D)
    P = _params()
    gp, con = _models(P, X, y, X[:Nc], Yc, obj_kernel=obj_kernel, obj_mean=obj_mean)
    best, idx, vals = acqui.ECI(gp, con, 0, params=P).argmax_batch(Xq, return_values=True)
    kid = {"SquaredExpARD": O.K_SE_ARD, "MaternFiveHalves": O.K_MATERN52}[obj_kernel]
    m_obj = y.mean() if obj_mean == "Data" else 0.25
    mu, s2, mu_x = _oracle_side(O, kid, X, y[:, None], m_obj, Xq)
    mu_c, s2_c, _ = _oracle_side(O, O.K_EXP, X[:Nc], Yc, 0.25, Xq)
    want = oracle_eci.eci(mu[:, 0], s2, mu_c[:, 0], s2_c, mu_x[:, 0].max(), 0.0)
    assert np.abs(vals - want).max() <= 1e-10
    assert idx == int(np.argmax(want)) and best == vals[idx] and best > 0
    with np.errstate(invalid="ignore", divide="ignore"):
        pf = want / O.ei(mu[:, 0], s2, mu_x[:, 0].max(), 0.0)
    assert np.nanmax(pf) - np.nanmin(pf) > 0.5  # the constraint model matters here


def test_eci_degenerates_to_ei_bit_for_bit():
    """con = NULL, and a constraint handle without samples: Pf = 1, values and argmax equal lb_acq_argmax(LB_ACQ_EI)."""
    from limbo_b200 import _lib, kernel, mean, model, synth
    D = 3
    X = synth.points(41, 200, D)
    y = synth.targets(X)
    P = _params()
    gp, _ = _models(P, X, y, X[:0], np.zeros((0, 2)))
    empty = model.GP(D, 2, params=P, kernel=kernel.Exp, mean=mean.Constant)
    for M in (100, 3000):
        Xq = synth.points(42 + M, M, D)
        ei = gp.acq_argmax_batch(_lib.ACQ_EI, [1.7, 0.01], Xq, return_values=True)
        for con in (None, empty):
            got = gp.eci_argmax_batch(con, 1.7, 0.01, Xq, return_values=True)
            assert got[:2] == ei[:2] and np.array_equal(got[2], ei[2])


def test_eci_empty_objective_scores_zero():
    from limbo_b200 import kernel, mean, model, synth
    P = _params()
    gp = model.GP(2, 1, params=P, kernel=kernel.SquaredExpARD, mean=mean.Constant)
    X = synth.points(5, 50, 2)
    _, con = _models(P, X, X[:, 0], X, np.stack([X[:, 0] * 2, X[:, 1]], axis=1))
    best, idx, vals = gp.eci_argmax_batch(con, 0.0, 0.0, synth.points(6, 700, 2), return_values=True)
    assert best == 0.0 and idx == 0 and np.all(vals == 0.0)


def _fitted_pair(D=3, N=260, Nc=200, M=2000, **kw):
    from limbo_b200 import synth
    X = synth.points(51, N, D)
    y = synth.targets(X)
    Yc = np.stack([0.2 + 1.6 * X[:Nc, 0], 2.0 - X[:Nc, 1]], axis=1)
    P = _params()
    gp, con = _models(P, X, y, X[:Nc], Yc, **kw)
    return gp, con, synth.points(52, M, D), P


def test_eci_dev_equals_host():
    import torch
    from limbo_b200 import _lib
    lib = _lib.load()
    gp, con, Xq, _ = _fitted_pair()
    M = Xq.shape[0]
    mean_obj = np.ascontiguousarray(gp.mean_function().batch(Xq, gp)[:, 0])
    ref = gp.eci_argmax_batch(con, 2.1, 0.0, Xq, return_values=True)
    dXq = torch.from_numpy(Xq).cuda()
    dmean = torch.from_numpy(mean_obj).cuda()
    dacq = torch.empty(M, dtype=torch.float64, device="cuda")
    dbest = torch.empty(1, dtype=torch.float64, device="cuda")
    didx = torch.empty(1, dtype=torch.int64, device="cuda")
    ep = np.array([2.1, 0.0])
    rc = lib.lb_eci_argmax_dev(gp._h, con._h, ep.ctypes.data, M, dXq.data_ptr(), dmean.data_ptr(), 0.0, None, 0.25,
                               dacq.data_ptr(), dbest.data_ptr(), didx.data_ptr())
    assert rc == 0
    assert lib.lb_sync(gp._h) == 0
    assert float(dbest.item()) == ref[0] and int(didx.item()) == ref[1]
    assert np.array_equal(dacq.cpu().numpy(), ref[2])


def test_eci_argument_errors():
    from limbo_b200 import _lib
    lib = _lib.load()
    gp, con, Xq, _ = _fitted_pair(M=300)
    ep = np.array([0.0, 0.0])
    best, idx = C.c_double(), C.c_int64()
    args = lambda o, c, M, bv, bi: lib.lb_eci_argmax(o, c, ep.ctypes.data, M, Xq.ctypes.data, None, 0.0, None, 0.0, None, bv, bi)  # noqa: E731
    assert args(gp._h, gp._h, 300, C.addressof(best), C.addressof(idx)) == LB_ERR_ARG
    assert args(gp._h, con._h, 0, C.addressof(best), C.addressof(idx)) == LB_ERR_ARG
    assert args(gp._h, con._h, -5, C.addressof(best), C.addressof(idx)) == LB_ERR_ARG
    assert args(gp._h, con._h, 300, None, C.addressof(idx)) == LB_ERR_ARG
    assert args(gp._h, con._h, 300, C.addressof(best), None) == LB_ERR_ARG
    assert args(gp._h, con._h, 300, C.addressof(best), C.addressof(idx)) == 0


def test_eci_reduced_precision_composition():
    """FP16X3 objective, TF32 constraint: ECI is the formula applied to those handles' own lb_query outputs."""
    from limbo_b200 import acqui
    gp, con, Xq, P = _fitted_pair(D=4, N=512, Nc=400, M=1500, obj={"precision": "fp16x3"}, con={"precision": "tf32"})
    a = acqui.ECI(gp, con, 0, params=P)
    best, idx, vals = a.argmax_batch(Xq, return_values=True)
    mu, s2 = gp.query_batch(Xq)
    mu_c, s2_c = con.query_batch(Xq)
    want = oracle_eci.eci(mu[:, 0], s2, mu_c[:, 0], s2_c, a._f_max, 0.0)
    assert np.abs(vals - want).max() <= 1e-12
    assert best == vals[idx] and vals[idx] == vals.max()


def test_eci_threads_with_swapped_pairs():
    """Two threads score (g1, g2) and (g2, g1) 20 times each while a third queries g2: scoped_lock keeps them deadlock-free and
    the join events keep every result equal to the serial one."""
    gp1, gp2, Xq, _ = _fitted_pair(M=3000)
    r12 = gp1.eci_argmax_batch(gp2, 2.0, 0.0, Xq, return_values=True)
    r21 = gp2.eci_argmax_batch(gp1, 0.5, 0.0, Xq, return_values=True)
    q2 = gp2.query_batch(Xq)
    errors = []

    def run(fn):
        try:
            fn()
        except Exception as e:  # reported below
            errors.append(repr(e))

    def a():
        for _ in range(20):
            r = gp1.eci_argmax_batch(gp2, 2.0, 0.0, Xq, return_values=True)
            if r[:2] != r12[:2] or not np.array_equal(r[2], r12[2]):
                errors.append("g1,g2 differs")

    def b():
        for _ in range(20):
            r = gp2.eci_argmax_batch(gp1, 0.5, 0.0, Xq, return_values=True)
            if r[:2] != r21[:2] or not np.array_equal(r[2], r21[2]):
                errors.append("g2,g1 differs")

    def c():
        for _ in range(20):
            m, s = gp2.query_batch(Xq)
            if not (np.array_equal(m, q2[0]) and np.array_equal(s, q2[1])):
                errors.append("lb_query on g2 differs")

    th = [threading.Thread(target=run, args=(f,), daemon=True) for f in (a, b, c)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=600)
    assert not any(t.is_alive() for t in th), "a thread did not finish"
    assert not errors, errors


def test_eci_sharded_equals_unsharded():
    from limbo_b200 import acqui, dist
    gp, con, Xq, P = _fitted_pair(M=3000)
    a = acqui.ECI(gp, con, 0, params=P)
    want = a.argmax_batch(Xq)
    for world in (1, 2, 3):
        recs = [dist.sharded_acq_argmax(a, Xq, r, world) for r in range(world)]
        got = dist.reduce_records(np.array([v for v, _ in recs]), np.array([i for _, i in recs]))
        assert got == want, (world, got, want)
        for r in range(world):  # chunk by chunk: every shard's record is its own range's argmax
            lo, hi = dist.shard_range(len(Xq), r, world)
            v, i = a.argmax_batch(Xq[lo:hi])
            assert recs[r] == (v, i + lo)


def test_cboptimizer_converges_to_constrained_optimum():
    """max -|x - (0.25, 0.75)|^2 subject to x0 + x1 >= 1.2: the optimum is the projection (0.35, 0.85) onto the boundary."""
    from limbo_b200 import bayes_opt, kernel, mean, model

    class P:
        class kernel:
            noise = 1e-6

        class kernel_maternfivehalves:
            sigma_sq = 1.0
            l = 0.3

        class init_randomsampling:
            samples = 10

        class stop_maxiterations:
            iterations = 30

        class opt_batchedrandom:
            candidates = 20000
            refinements = 2
            shrink = 0.1
    sol = np.array([0.25, 0.75])
    target = np.array([0.35, 0.85])

    def f(x):
        return np.array([-float(((x - sol) ** 2).sum()), 1.0 if x[0] + x[1] >= 1.2 else 0.0])
    gp = model.GP(2, 1, params=P, kernel=kernel.MaternFiveHalves, mean=mean.Data)
    con = model.GP(2, 1, params=P, kernel=kernel.MaternFiveHalves, mean=mean.Constant)
    bo = bayes_opt.CBOptimizer(gp, con, params=P, rng=np.random.default_rng(0))
    bo.optimize(f, 2, dim_out=1, nb_constraints=1)
    assert len(bo.samples()) == 40 and gp.nb_samples() == 40 and con.nb_samples() == 40
    x = bo.best_sample()
    print("best sample", x, "distance^2", ((x - target) ** 2).sum())
    assert x[0] + x[1] >= 1.2
    # 2e-3, not the 1e-3 of the unconstrained loop: this seed ends at (0.342, 0.884), 1.25e-3 away (H100, deterministic).  The
    # constraint GP smooths the 0/1 step over its length scale (0.3), so Pf is about 1/2 on both sides of the boundary and the
    # loop spends samples on the infeasible side instead of refining along it.
    assert ((x - target) ** 2).sum() < 2e-3


def test_cpp_eci_dropin():
    binary = os.path.join(ROOT, "oracle", "_ref", "eci_dropin_test")
    if not os.path.exists(binary):
        pytest.skip("oracle/_ref/eci_dropin_test not built (needs the reference's sources at build time)")
    r = subprocess.run([binary], capture_output=True, text=True, timeout=600)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "ECI DROPIN OK" in r.stdout, r.stdout + r.stderr
