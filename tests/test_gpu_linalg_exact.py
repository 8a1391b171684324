"""The fp64 factorisation, inverse, solves, likelihood gradient and query on matrices with an exactly known answer
(tests/linalg_exact.py), at every tile-schedule shape: T = 1 .. 13 covers every tail of the quad schedule (nc2 = 1,
nca < 4, ncb == 0, every T mod 4) and of the recursive trtri (short last problem), T = 15 .. 17 and 31 .. 33 the
ragged 16-tile super-blocks of the panel query, N mod 128 in {0, 1, 127} the edge tiles.  Every bar is a first-order
rounding-error bound; each case prints its observed / bound ratio."""
import math
import threading

import numpy as np
import pytest

import linalg_exact as E

pytestmark = pytest.mark.gpu

EXACT = E.exact_shapes()
RATIOS = {}


def _ratio(name, obs, bound):
    r = float(np.max(np.asarray(obs) / np.asarray(bound)))
    RATIOS[name] = max(RATIOS.get(name, 0.0), r)
    return r


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nlargest observed / bound:", {k: f"{v:.2e}" for k, v in sorted(RATIOS.items())})


@pytest.fixture(scope="module")
def handle(lib):
    h = E.Handle(lib)
    yield h
    h.close()


def _check_factor(h, case, tag=""):
    """L, alpha, K^-1 and log det of an exact case already factored on h (alpha refitted with case.Y)."""
    N = case.N
    L = h.get(1)
    assert np.all(np.triu(L, 1) == 0.0), f"{tag} upper part of L not zero: {E.worst_tile(np.triu(L, 1))}"
    eL = np.linalg.norm(L - case.L0)
    bL = E.bound_L(case)
    alpha = h.get(2)
    ea = np.linalg.norm(alpha - case.A0, axis=0)
    ba = E.bound_alpha(case)
    Ki = h.get(3)
    assert np.array_equal(Ki, Ki.T), f"{tag} K^-1 not exactly symmetric: {E.worst_tile(Ki - Ki.T)}"
    eK = np.linalg.norm(Ki - case.ref()["kinv"])
    bK = E.bound_kinv(case)
    print(f"{tag} N={N} T={case.T} P={case.P} kappa={case.ref()['kappa']:.2f} ratio L={eL / bL:.2e} "
          f"alpha={np.max(ea / ba):.2e} Kinv={eK / bK:.2e}")
    assert eL <= bL, f"{tag} L: ||err||_F {eL:.3e} > {bL:.3e}; {E.worst_tile(L - case.L0)}"
    assert np.all(ea <= ba), f"{tag} alpha: {ea} > {ba}; {E.worst_tile(alpha - case.A0)}"
    assert eK <= bK, f"{tag} K^-1: ||err||_F {eK:.3e} > {bK:.3e}; {E.worst_tile(Ki - case.ref()['kinv'])}"
    _ratio("L", eL, bL)
    _ratio("alpha", ea, ba)
    _ratio("Kinv", eK, bK)
    return L, alpha, Ki


def test_lambda_gradient_shapes_are_covered():
    """The Lambda entries of the likelihood gradient (dk_build over 1024 column slices of wdot) are checked against the
    reference at N > 1024 (a second pass of the slice loop) on at least two shapes, and with k = 4 (LB_MAX_LAMBDA)."""
    lam = [(N, E.exact_objective(i, N)[2]) for i, (N, _, _) in enumerate(EXACT) if E.exact_objective(i, N)[2] > 0]
    checked = [(N, k) for N, k in lam if N <= 2200 or N == 4223]
    assert sum(N > 1024 for N, _ in checked) >= 2, checked
    assert any(k == 4 for _, k in checked), checked
    assert {k for _, k in lam} == {1, 2, 4}, lam


@pytest.mark.parametrize("N,P,seed", EXACT, ids=[f"N{n}_P{p}" for n, p, _ in EXACT])
def test_exact_factor_solve_inverse_logdet_grad(handle, N, P, seed):
    h = handle
    case = E.ExactCase(N, P, seed)
    assert case.ref()["kappa"] < 16.0
    rng = np.random.default_rng(seed + 1)
    i = EXACT.index((N, P, seed))
    kid, D, klam, optimize_noise = E.exact_objective(i, N)  # SE-ARD with k Lambda columns: lb_launch_grad_lambda
    X = rng.uniform(0.0, 1.0, size=(N, D))
    p = E.exact_objective_params(kid, D, klam, rng)
    noise = 0.01
    h.set_data(X, case.Y)
    h.set_kernel(kid, p, noise)
    assert h.factor(case.K) == 0
    h.refit_alpha(case.Y)
    _check_factor(h, case, f"[{E.KERNEL_NAMES[kid]}]")

    # gradient: 0.5 sum_ij (alpha alpha^T - K^-1)_ij dk_ij / dtheta, alpha = A0 and K^-1 from LAPACK
    g = h.grad(optimize_noise)
    if N <= 2200 or N == 4223:
        gr, absum, fro = E.grad_reference(kid, p, X, case.A0, case.ref()["kinv"], noise, optimize_noise)
        bg = E.bound_grad(case, kid, p, X, absum, fro, E.bound_alpha(case), E.bound_kinv(case))
        eg = np.abs(g - gr)
        print(f"  grad {E.KERNEL_NAMES[kid]} D={D} k={klam} noise={optimize_noise} ratio={np.max(eg / bg):.2e}")
        assert np.all(eg <= bg), (g, gr, bg)
        _ratio("grad", eg, bg)
        if klam:
            _ratio("grad_lambda", eg[D:D * (1 + klam)], bg[D:D * (1 + klam)])

    # log det: with alpha = 0, loglik = -0.5 log det K - 0.5 N log(2 pi)
    h.refit_alpha(np.zeros((N, P)))
    ld = -2.0 * h.log_lik() - N * math.log(2.0 * math.pi)
    bl = E.bound_logdet(case)
    assert abs(ld - case.logdet) <= bl, (ld, case.logdet, bl)
    _ratio("logdet", abs(ld - case.logdet), bl)


# ---- query on a loaded factor ----------------------------------------------------------------------------------------
POOL = 2049
PATHS = [("point", 1, False), ("slab", 7, False), ("slab", 72, False), ("slab", 73, False), ("slab", 255, False),
         ("multi_launch", 100, True), ("panel", 256, False), ("panel", 640, False), ("panel", 1000, False), ("panel", 2049, False)]


def _query_check(h, qc, kid, p, noise, Xq, paths, tag):
    L, mu, s2, V, Ks = qc.reference(kid, p, noise, Xq)
    c = float(L[0, 0])
    h.set_data(qc.X, np.zeros((qc.N, qc.P)))
    h.set_kernel(kid, p, noise)
    h.load_factor(L, qc.alpha)
    xmax = 1.0
    bm = E.bound_mu(kid, p, Ks, qc.alpha, xmax, qc.D)
    bs = E.bound_s2(kid, p, V, c, qc.norm_E(), xmax, qc.D, noise)
    for name, M, unfused in paths:
        m, s = h.query(Xq[:M], unfused=unfused)
        em, es = np.abs(m - mu[:M]), np.abs(s - s2[:M])
        rm, rs = float(np.max(em / bm[:M])), float(np.max(es / bs[:M]))
        print(f"{tag} {name} M={M} ratio mu={rm:.2e} s2={rs:.2e}")
        assert rm <= 1.0, f"{tag} {name} M={M} mu: {E.worst_tile(em / bm[:M])}"
        assert rs <= 1.0, f"{tag} {name} M={M} sigma2: worst candidate {int(np.argmax(es / bs[:M]))}, ratio {rs:.3e}"
        _ratio("mu", rm, 1.0)
        _ratio("sigma2", rs, 1.0)


@pytest.mark.parametrize("kid", E.KERNELS, ids=[E.KERNEL_NAMES[k] for k in E.KERNELS])
@pytest.mark.parametrize("T", E.QUERY_T)
def test_query_paths_on_loaded_factor(handle, lib, T, kid):
    N = 100 if T == 1 else (128 * T - 1 if T % 2 else 128 * T)
    qc = E.QueryCase(N, 3, 2, 7000 + 10 * T + kid)
    assert qc.norm_E() <= 0.25
    p = E.kernel_params(kid, 3, qc.rng)
    Xq = qc.rng.uniform(0.0, 1.0, size=(POOL, 3))
    _query_check(h=handle, qc=qc, kid=kid, p=p, noise=0.01, Xq=Xq, paths=PATHS, tag=f"[T={T} {E.KERNEL_NAMES[kid]}]")


@pytest.mark.parametrize("T", (1, 2, 15))
def test_query_slab_widths_8_and_9(handle, lib, T):
    """A batch of just over 8 n8-tiles per SM, below the panel threshold: the slab kernel's compile-time widths 8 and 9."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    M = 8 * (sms * 8 + sms // 2) - 3
    N = 100 if T == 1 else 128 * T - 1
    kid = (0, 1, 3)[(1, 2, 15).index(T)]
    qc = E.QueryCase(N, 3, 1, 7500 + T)
    p = E.kernel_params(kid, 3, qc.rng)
    Xq = qc.rng.uniform(0.0, 1.0, size=(M, 3))
    lib.lb_debug_set_query_panel_min(1 << 40)
    try:
        _query_check(handle, qc, kid, p, 0.01, Xq, [("slab89", M, False)], f"[T={T} {E.KERNEL_NAMES[kid]}]")
    finally:
        lib.lb_debug_set_query_panel_min(0)


@pytest.mark.parametrize("T", (2, 17))
@pytest.mark.parametrize("what", ("D20", "P5"))
def test_query_multi_launch_from_shape(handle, T, what):
    """D = 20 (more than the fused kernels' 16 staged dimensions) or P = 5 (more than their 4 outputs): multi-launch path."""
    N = 128 * T - 1
    if what == "D20":
        qc = E.QueryCase(N, 20, 1, 7700 + T)
        kid, p = 0, np.concatenate([qc.rng.uniform(0.3, 0.8, 20), [0.1]])
    else:
        qc = E.QueryCase(N, 3, 5, 7800 + T)
        kid = 2
        p = E.kernel_params(kid, 3, qc.rng)
    Xq = qc.rng.uniform(0.0, 1.0, size=(300, qc.D))
    _query_check(handle, qc, kid, p, 0.01, Xq, [("point", 1, False), ("batch", 100, False), ("panel", 300, False)],
                 f"[T={T} {what}]")


# ---- repeatability, races, grouping, pivots --------------------------------------------------------------------------
def test_factor_repeatable_across_calls_and_handles(lib):
    case = E.ExactCase(128 * 9 - 1, 2, 77)
    X = np.random.default_rng(78).uniform(0.0, 1.0, size=(case.N, 2))
    h1, h2 = E.Handle(lib), E.Handle(lib)
    try:
        a = E.factor_outputs(h1, case, X)
        b = E.factor_outputs(h1, case, X)
        c = E.factor_outputs(h2, case, X)
    finally:
        h1.close()
        h2.close()
    for k in a:
        assert np.array_equal(a[k], b[k]), f"{k} differs between two factorisations on one handle: {E.worst_tile(a[k] - b[k])}"
        assert np.array_equal(a[k], c[k]), f"{k} differs between two handles: {E.worst_tile(a[k] - c[k])}"


def test_concurrent_factorisations_match_sequential(lib):
    cases = [E.ExactCase(128 * 13 + 1, 1, 81), E.ExactCase(128 * 24 - 1, 3, 82)]
    Xs = [np.random.default_rng(90 + i).uniform(0.0, 1.0, size=(c.N, 2)) for i, c in enumerate(cases)]
    hs = [E.Handle(lib), E.Handle(lib)]
    try:
        seq = [E.factor_outputs(hs[i], cases[i], Xs[i]) for i in range(2)]
        par, errs = [None, None], []

        def work(i):
            try:
                for _ in range(3):
                    par[i] = E.factor_outputs(hs[i], cases[i], Xs[i])
                    for k in seq[i]:
                        assert np.array_equal(par[i][k], seq[i][k]), f"handle {i} {k}: {E.worst_tile(par[i][k] - seq[i][k])}"
            except Exception as e:  # noqa: BLE001 - reported below
                errs.append(e)

        ts = [threading.Thread(target=work, args=(i,)) for i in range(2)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        assert not errs, errs
    finally:
        for h in hs:
            h.close()


@pytest.mark.parametrize("N,P,seed", [(2048, 1, 21), (4097, 2, 22)], ids=["T16", "T33"])
def test_panel_grouping_bit_identical(handle, lib, N, P, seed):
    """The panel query walks its candidate column tiles in four stream groups when a launch of all of them is under one
    round of the machine, otherwise on one stream.  Nested prefixes of one candidate set on either side of that rule give
    bit-identical mu and sigma^2 for the shared candidates: the grouping does not change any tile's arithmetic, and a
    candidate's value does not depend on the batch it is in."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    slots = 2 * sms  # CfgDual: two CTAs per SM
    per_ct = 2 * 16  # CTAs per 128-candidate column tile in one launch: two 64-wide tiles x a 16-row-tile super-block

    def groups(M):
        ct = -(-M // 128)
        return 4 if ct >= 4 and ct * per_ct < slots else 1

    m4 = (slots - 1) // per_ct * 128  # the largest batch that takes four groups
    m1 = m4 + 1                       # the smallest batch above it, on one stream
    mid = (4 * 128 + m4) // 2 - 3     # a ragged batch with four uneven groups
    sizes = (m1, m4, mid)
    assert [groups(M) for M in sizes] == [1, 4, 4], (sms, sizes)
    assert min(sizes) >= 256  # all on the panel path

    qc = E.QueryCase(N, 3, P, seed)
    p = E.kernel_params(1, 3, qc.rng)
    Xq = qc.rng.uniform(0.0, 1.0, size=(m1, 3))
    L, _, _, _, _ = qc.reference(1, p, 0.01, Xq)
    handle.set_data(qc.X, np.zeros((N, P)))
    handle.set_kernel(1, p, 0.01)
    handle.load_factor(L, qc.alpha)
    handle.query(Xq[:m1])  # builds the cached diagonal-block inverses, so every query below launches the same fixed kernels
    T = -(-N // 128)
    nsb = -(-T // 16)  # super-blocks
    out, fixed = {}, set()
    for M in sizes:
        n0 = lib.lb_launch_count(handle.h)
        out[M] = handle.query(Xq[:M])
        # one update and one solve launch per super-block and group; the rest of the query launches the same for every M
        fixed.add(lib.lb_launch_count(handle.h) - n0 - 2 * nsb * groups(M))
    assert len(fixed) == 1, f"the launch count does not follow the grouping rule: {fixed}"
    for M in sizes[1:]:
        for k, (a, b) in enumerate(zip(out[M], out[m1])):
            assert np.array_equal(a, b[:M]), f"M={M} {('mu', 'sigma2')[k]}: {E.worst_tile(a - b[:M])}"


PIVOT_T = (1, 3, 5, 9)


@pytest.mark.parametrize("T", PIVOT_T)
def test_pivot_reporting_matches_dpotrf(handle, T):
    import scipy.linalg as sl
    N = 128 * T - 1 if T > 1 else 100
    case = E.ExactCase(N, 1, 900 + T)
    X = np.random.default_rng(901 + T).uniform(0.0, 1.0, size=(N, 2))
    h = handle
    h.set_data(X, case.Y)
    h.set_kernel(1, np.array([-0.5, 0.0]), 0.01)
    ps = sorted({p for p in (0, 31, 32, 127, 128, 255, 256, 511, 512, N - 1) if p < N})
    for p in ps:
        Kb = case.with_bad_pivot(p)
        _, info_lapack = sl.lapack.dpotrf(Kb, lower=1)
        assert info_lapack == p + 1
        info = h.factor(Kb)
        assert info == p + 1, f"T={T} pivot {p}: info {info}, dpotrf {info_lapack}"
    # the same handle factors a positive-definite matrix correctly afterwards
    assert h.factor(case.K) == 0
    h.refit_alpha(case.Y)
    _check_factor(h, case, f"[after pivots T={T}]")
