"""The objectives the hyper-parameter optimisers climb, against bounded references (tests/linalg_exact.py):
  - LOO-CV value and gradient (loo.cu: dk_build, loo_zeta on 128 x 128 DMMA tiles over a T x T grid, the 1024-thread
    reductions) and K^-1 obs_mean (kinv_obs over 32 slices of N) on exact factors at every tile-schedule shape;
  - the batched log-likelihood and gradient (lml_batch.cu) on a table of shapes that covers its sweeps and layouts;
  - a factor grown by lb_append answers bit for bit like the same factor loaded into a fresh handle (no stale cache).
Every bar is a first-order rounding-error bound; the module prints the largest observed / bound ratio per quantity."""
import functools
import math

import numpy as np
import pytest

import linalg_exact as E

pytestmark = pytest.mark.gpu

EXACT = E.exact_shapes()
RATIOS = {}


def _ratio(name, obs, bound):
    r = float(np.max(np.asarray(obs, dtype=np.float64) / np.asarray(bound, dtype=np.float64)))
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


# ---- LOO-CV and K^-1 obs_mean on exact factors -----------------------------------------------------------------------
def _loo_reference_checked(N):
    """The host reference of the LOO gradient costs N^3 per hyper-parameter: where the likelihood-gradient test computes its
    reference (tests/test_gpu_linalg_exact.py)."""
    return N <= 2200 or N == 4223


def test_loo_shapes_are_covered():
    """LOO cases with N > 1024 (a second pass of the 1024-thread row loops) and N a multiple of 128, P >= 3, Lambda columns
    and D = 20 on SE-ARD, the noise entry on and off; the gradient reference runs on some N > 1024."""
    objs = [(N, P) + E.exact_objective(i, N) for i, (N, P, _) in enumerate(EXACT)]
    assert any(N > 1024 and _loo_reference_checked(N) for N, *_ in objs)
    assert any(N % 128 == 0 and N > 128 for N, *_ in objs)
    assert {P for _, P, *_ in objs} >= {1, 3, 5}
    assert {k for _, _, kid, _, k, _ in objs if kid == 0} == set(E.EXACT_KLAM)
    assert any(D == 20 for _, _, _, D, _, _ in objs)
    assert {on for *_, on in objs} == {False, True}
    assert {kid for _, _, kid, *_ in objs} == set(E.KERNELS)


@pytest.mark.parametrize("N,P,seed", EXACT, ids=[f"N{n}_P{p}" for n, p, _ in EXACT])
def test_loo_and_kinv_obs_on_exact_factor(handle, N, P, seed):
    h = handle
    case = E.ExactCase(N, P, seed)
    assert case.ref()["kappa"] < 16.0
    i = EXACT.index((N, P, seed))
    kid, D, klam, on = E.exact_objective(i, N)
    rng = np.random.default_rng(seed + 2)
    X = rng.uniform(0.0, 1.0, size=(N, D))
    p = E.exact_objective_params(kid, D, klam, rng)
    noise = 0.01
    h.set_data(X, case.Y)
    h.set_kernel(kid, p, noise)
    assert h.factor(case.K) == 0
    h.refit_alpha(case.Y)
    tag = f"[N={N} T={case.T} P={P} {E.KERNEL_NAMES[kid]} D={D} k={klam} noise={on}]"
    ba, bk = E.bound_alpha(case), E.bound_kinv(case)
    kinv = case.ref()["kinv"]

    # K^-1 obs_mean: exactly A0 in exact arithmetic
    ko = h.kinv_obs()
    eko, bko = np.linalg.norm(ko - case.A0, axis=0), E.bound_kinv_obs(case, bk)
    assert np.all(eko <= bko), f"{tag} K^-1 obs_mean: {eko} > {bko}; {E.worst_tile(ko - case.A0)}"
    _ratio("kinv_obs", eko, bko)

    # LOO value (O(N)) at every shape
    v = h.loo_cv()
    vr = E.loo_value(case.A0, kinv)
    ev_, bv = abs(v - vr), E.bound_loo(case, ba, bk)
    assert ev_ <= bv, f"{tag} LOO value {v!r} vs {vr!r}: |err| {ev_:.3e} > {bv:.3e}"
    _ratio("loo", ev_, bv)

    g = h.loo_grad(on)
    assert g.size == p.size + int(on) and np.all(np.isfinite(g)), (tag, g)
    msg = f"{tag} ratio kinv_obs={np.max(eko / bko):.2e} loo={ev_ / bv:.2e}"
    if _loo_reference_checked(N):
        _, gr = E.loo_reference(kid, p, X, case.A0, kinv, noise, on)
        bg = E.bound_loo_grad(case, kid, p, X, noise, on, ba, bk)
        eg = np.abs(g - gr)
        msg += f" loo_grad={np.max(eg / bg):.2e}"
        assert np.all(eg <= bg), f"{tag} LOO gradient: entries {np.flatnonzero(eg > bg)}; {g} vs {gr}, bound {bg}"
        _ratio("loo_grad", eg, bg)
        if klam:
            _ratio("loo_grad_lambda", eg[D:D * (1 + klam)], bg[D:D * (1 + klam)])
    print(msg)


# ---- lb_lml_grad_batch on a shape table ------------------------------------------------------------------------------
# lml_batch.cu's layout rule, restated: the vector's matrix has leading dimension ld = N | 1, and the workspace of
#   ws_doubles = ld N + De N + 2 P N + N   (matrix, staged coordinates De = D + k, obs_mean / alpha and the forward solution,
#                                           one vector)
# lives in shared memory when N <= 128 and ws_doubles * 8 <= 200 KiB, otherwise in a global workspace (one CTA per SM).
# SE-ARD's ell / Lambda entries, D (1 + k) of them, are reduced GCH = 8 per sweep.
GCH = 8
SMEM_MAX_N, SMEM_BYTES_MAX = 128, 200 * 1024
MAX_THREADS_PER_SM, NT = 2048, 256


def ws_doubles(N, De, P):
    return (N | 1) * N + De * N + 2 * P * N + N


def in_smem(N, De, P):
    return N <= SMEM_MAX_N and 8 * ws_doubles(N, De, P) <= SMEM_BYTES_MAX


def resident_bounds(N, De, P, sms):
    """(at most, at least) resident CTAs: the global layout runs one per SM; in shared memory at most 2048 / 256 per SM."""
    return (sms * MAX_THREADS_PER_SM // NT, sms) if in_smem(N, De, P) else (sms, sms)


# (kernel id, N, D, k, P, R, optimize_noise); R = "above": 7 more vectors than the most CTAs that can be resident
BATCH = [
    (1, 1, 2, 0, 1, 3, True), (0, 1, 3, 0, 2, "above", False), (3, 2, 1, 0, 1, "above", True),
    (0, 31, 7, 0, 1, 5, True), (0, 32, 8, 0, 2, 4, False), (0, 33, 9, 0, 1, 3, True), (0, 32, 4, 3, 2, 3, True),
    (0, 31, 8, 1, 4, 2, False), (0, 33, 17, 0, 1, 2, True), (2, 33, 3, 0, 3, 7, False),
    (0, 127, 60, 4, 4, 2, True), (0, 127, 60, 4, 5, 2, False), (0, 128, 60, 4, 3, 2, False), (0, 128, 60, 4, 4, 2, True),
    (1, 128, 64, 0, 4, "above", True), (3, 127, 3, 0, 1, 9, False), (0, 129, 3, 2, 2, 3, True), (2, 129, 5, 0, 1, 4, True),
    (0, 199, 16, 0, 2, 2, False), (1, 200, 3, 0, 1, 3, True), (0, 200, 2, 1, 1, 2, True), (3, 200, 4, 0, 2, "above", False),
]


def _rows(sms):
    out = []
    for kid, N, D, k, P, R, on in BATCH:
        De = D + k if kid == 0 else D
        if R == "above":
            R = resident_bounds(N, De, P, sms)[0] + 7
        out.append((kid, N, D, k, P, R, on))
    return out


def test_lml_batch_table_covers_the_kernel(lib):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows = _rows(sms)
    assert {N for _, N, *_ in rows} >= {1, 2, 31, 32, 33, 127, 128, 129, 199, 200}
    nent = {D * (1 + k) for kid, _, D, k, *_ in rows if kid == 0}
    assert nent >= {7, 8, 9, 16, 17}, nent                          # a second GCH sweep from 9 entries on
    assert any(kid == 0 and D + k == 64 and k == 4 for kid, _, D, k, *_ in rows)   # De = 64: 38 sweeps of Lambda entries
    assert {P for kid, _, D, k, P, *_ in rows if kid == 0} >= {2, 4}
    lay = {(N, in_smem(N, (D + k) if kid == 0 else D, P)) for kid, N, D, k, P, *_ in rows}
    assert {(127, True), (127, False), (128, True), (128, False)} <= lay, lay   # the global workspace at N <= 128
    below = any(R < resident_bounds(N, (D + k) if kid == 0 else D, P, sms)[1] for kid, N, D, k, P, R, _ in rows)
    above = any(R > resident_bounds(N, (D + k) if kid == 0 else D, P, sms)[0] for kid, N, D, k, P, R, _ in rows)
    assert below and above


@functools.lru_cache(maxsize=None)
def _batch_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("row", range(len(BATCH)))
def test_lml_batch_rows_against_reference(handle, row):
    kid, N, D, k, P, R, on = _rows(_batch_sms())[row]
    rng = np.random.default_rng(5000 + row)
    X = rng.uniform(0.0, 1.0, size=(N, D))
    Y = rng.normal(size=(N, P))
    H = np.stack([E.grad_params(kid, D, k, rng) for _ in range(R)])
    noise = np.array([0.01 + N * math.exp(2 * h[-1]) / 8000.0 for h in H])  # kappa_2(K) <= 1e4, asserted below
    h = handle
    h.set_data(X, Y)
    lik, grad, info = h.lml_grad_batch(kid, H, noise, on)
    tag = f"[row {row}: {E.KERNEL_NAMES[kid]} N={N} D={D} k={k} P={P} R={R} noise={on} smem={in_smem(N, D + k, P)}]"
    assert np.all(info == 0), f"{tag} info {info[info != 0]}"
    assert np.all(np.isfinite(lik)) and np.all(np.isfinite(grad)), tag
    # the reference for every row of small batches, a spread of rows of large ones (the host cost is per row)
    check = range(R) if R <= 16 else sorted(set(np.linspace(0, R - 1, 12).astype(int)))
    worst = [0.0, 0.0]
    for r in check:
        c = E.LmlCase(kid, H[r], noise[r], X, Y, on)
        assert c.kappa <= 1e4, (tag, r, c.kappa)
        bl, bg = c.bound()
        el, eg = abs(lik[r] - c.lik), np.abs(grad[r] - c.grad)
        assert el <= 2 * bl, f"{tag} row {r} likelihood {lik[r]!r} vs {c.lik!r}: |err| {el:.3e} > 2 x {bl:.3e}"
        bad = np.flatnonzero(eg > 2 * bg)
        assert bad.size == 0, f"{tag} row {r} gradient entries {bad}: {grad[r][bad]} vs {c.grad[bad]}, bound 2 x {bg[bad]}"
        worst = [max(worst[0], _ratio("lml_batch_lik", el, 2 * bl)), max(worst[1], _ratio("lml_batch_grad", eg, 2 * bg))]
    print(f"{tag} ratio lik={worst[0]:.2e} grad={worst[1]:.2e}")


# ---- appended factors answer like fresh ones --------------------------------------------------------------------------
def _appended_reference(qc, kid, p, noise, Xn):
    """The host extension of L = c (I + E) by the rows of the points Xn (l = L^-1 k, d^2 = k(x, x) + noise + 1e-8 - |l|^2),
    with c such that |L^-1 k|^2 <= sf^2 / 16 for each of them against the first N points."""
    import scipy.linalg as sl
    sf2 = math.exp(2 * p[-1])
    A = np.eye(qc.N) + qc.E
    V1 = sl.solve_triangular(A, E.kernel_matrix(kid, p, qc.X, Xn), lower=True)
    c = math.sqrt(16.0 * float((V1 * V1).sum(0).max()) / sf2)
    L = c * A
    Xall = qc.X
    rows = []
    for x in Xn:
        n = L.shape[0]
        kv = E.kernel_matrix(kid, p, Xall, x[None, :])[:, 0]
        l = sl.solve_triangular(L, kv, lower=True)
        d2 = sf2 + noise + E.JITTER - float(l @ l)
        rows.append((l, d2, kv))
        L = np.block([[L, np.zeros((n, 1))], [l[None, :], np.array([[math.sqrt(d2)]])]])
        Xall = np.vstack([Xall, x[None, :]])
    return c, L, rows


def _row_bound(kid, p, l, kv, Lprev, c, normE, noise, D):
    """|l^ - l| (2-norm) and |d^ - d| of one appended row, one evaluation: the solve's forward error through kappa_2 of the
    factor it runs on and the kernel evaluation (bound_s2's dv), then d^2 = knn - |l|^2 (2 ||l|| ||dl|| + gamma_{n+2} |l|^2 +
    4u knn) and the square root."""
    n = l.size
    s = np.linalg.svd(Lprev, compute_uv=False)
    kap = float(s[0] / s[-1])
    ev = E.kernel_eval_err(kid, p, 1.0, D)
    dl = kap * kap * E.gamma(n) * float(np.linalg.norm(l)) + ev * math.sqrt(n) / float(s[-1])
    knn = math.exp(2 * p[-1]) + noise + E.JITTER
    d2 = knn - float(l @ l)
    dd2 = 2.0 * float(np.linalg.norm(l)) * dl + E.gamma(n + 2) * float(l @ l) + 4.0 * E.U * knn
    return dl, dd2 / (2.0 * math.sqrt(d2)) + E.U * math.sqrt(d2)


def _outputs(h, Xq, on):
    """Everything derived from the factor: panel, slab and one-point queries, candidate gradients, likelihood gradient, LOO
    value and gradient, K^-1 obs_mean."""
    out = {}
    out["panel"] = h.query(Xq[:300])
    out["slab"] = h.query(Xq[:100])
    out["point"] = h.query(Xq[:1])
    out["query_grad"] = h.query_grad(Xq[:50])
    out["grad"] = h.grad(on)
    out["loo"] = h.loo_cv()
    out["loo_grad"] = h.loo_grad(on)
    out["kinv_obs"] = h.kinv_obs()
    return out


APPEND_T = (1, 2, 16, 17)


@pytest.mark.parametrize("T", APPEND_T)
def test_appended_factor_answers_like_fresh(lib, T):
    N0 = 128 * T - 1
    assert (N0 + 1) % 128 == 0 and N0 + 2 > 128 * T  # the first append fills the last tile, the second grows the capacity
    kid = E.KERNELS[APPEND_T.index(T)]
    D, P, noise, on = 3, 2, 0.01, bool(T % 2)
    qc = E.QueryCase(N0, D, P, 9100 + T)
    p = E.kernel_params(kid, D, qc.rng)
    Xn = np.vstack([qc.rng.uniform(0.0, 0.1, size=(1, D)), qc.rng.uniform(0.9, 1.0, size=(1, D))])
    Yall = qc.rng.normal(size=(N0 + 2, P))
    Xq = qc.rng.uniform(0.0, 1.0, size=(300, D))
    c, Lext, rows = _appended_reference(qc, kid, p, noise, Xn)
    sf2 = math.exp(2 * p[-1])
    for _, d2, _ in rows:  # on the host, before any device call: both new pivots are well away from zero
        assert d2 >= sf2 / 4, (d2, sf2)

    hs = [E.Handle(lib), E.Handle(lib, precision=3)]
    fresh = []
    try:
        for h in hs:
            h.set_data(qc.X, Yall[:N0])
            h.set_kernel(kid, p, noise)
            h.load_factor(Lext[:N0, :N0], qc.alpha)
            h.query(Xq)  # build every cache: the panel query's inverse levels (or the reduced-precision copy), K^-1, L^-1
            if h is hs[0]:
                h.query(Xq[:100])
                h.grad(on)
                h.loo_grad(on)
        h = hs[0]
        Lprev = Lext[:N0, :N0]
        for j in range(2):
            n = N0 + j
            hs[0].append(Xn[j], Yall[:n + 1])
            hs[1].append(Xn[j], Yall[:n + 1])
            L = h.get(1)
            l, d2, kv = rows[j]
            dl, dd = _row_bound(kid, p, l, kv, Lext[:n, :n], c, qc.norm_E(), noise, D)
            el, ed = float(np.linalg.norm(L[n, :n] - l)), abs(L[n, n] - math.sqrt(d2))
            assert el <= 2 * dl, f"T={T} append {j}: new row ||err|| {el:.3e} > 2 x {dl:.3e}"
            assert ed <= 2 * dd, f"T={T} append {j}: new pivot |err| {ed:.3e} > 2 x {dd:.3e}"
            assert np.array_equal(L[:n, :n], Lprev), f"T={T} append {j}: the old factor changed"
            Lprev = L
            _ratio("append_row", el, 2 * dl)
            _ratio("append_pivot", ed, 2 * dd)
            # alpha against the host solve on the host extension: the solve's backward error, and the new rows' errors
            # entering K = L L^T by 2 ||dL|| ||L||, through ||K^-1||_2
            import scipy.linalg as sl
            Lr = Lext[:n + 1, :n + 1]
            ar = sl.cho_solve((Lr, True), Yall[:n + 1])
            s = np.linalg.svd(Lr, compute_uv=False)
            absL = np.abs(Lr)
            dK = 2.0 * E.gamma(3 * (n + 1) + 1) * float(np.linalg.norm(absL @ absL.T, 2)) + 2.0 * 2.0 * (dl + dd) * float(s[0])
            ba = dK / float(s[-1]) ** 2 * np.linalg.norm(ar, axis=0)
            ea = np.linalg.norm(h.get(2) - ar, axis=0)
            assert np.all(ea <= ba), f"T={T} append {j}: alpha ||err|| {ea} > {ba}"
            _ratio("append_alpha", ea, ba)
        Ldev, adev = h.get(1), h.get(2)
        Xall = np.vstack([qc.X, Xn])
        for prec, ha in ((0, hs[0]), (3, hs[1])):
            hf = E.Handle(lib, precision=prec)
            fresh.append(hf)
            hf.set_data(Xall, Yall)
            hf.set_kernel(kid, p, noise)
            hf.load_factor(Ldev, adev)
            assert np.array_equal(ha.get(1), Ldev) and np.array_equal(ha.get(2), adev)
            if prec == 0:
                a_out, f_out = _outputs(ha, Xq, on), _outputs(hf, Xq, on)
            else:
                a_out, f_out = {"reduced": ha.query(Xq)}, {"reduced": hf.query(Xq)}
            for name in a_out:
                a, f = a_out[name], f_out[name]
                for x, y in zip(a if isinstance(a, tuple) else (a,), f if isinstance(f, tuple) else (f,)):
                    assert np.array_equal(np.asarray(x), np.asarray(y)), \
                        f"T={T} precision {prec} {name}: appended and fresh handles differ; {E.worst_tile(np.asarray(x) - np.asarray(y))}"
        print(f"T={T} {E.KERNEL_NAMES[kid]}: N {N0} -> {N0 + 2}, appended == fresh for every output")
    finally:
        for x in hs + fresh:
            x.close()
