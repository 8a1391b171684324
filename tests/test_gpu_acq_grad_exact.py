"""Candidate gradients on the device (lb_query_grad / lb_acq_grad) on loaded factors of known conditioning
(tests/linalg_exact.py: QueryCase.grad_reference, grad_bounds, bound_acq): every 16-tile super-block shape of the backward
walk W = L^-T V, staged widths across the 16-coordinate passes of the gradient kernel, several outputs, the stream grouping
of the backward walk, the _dev entry points, the candidate-chunk boundary of the fp64 panel path, and Matern kernels at
subnormal squared distances.  Every bar is a first-order rounding-error bound; the largest observed / bound ratio per
quantity is printed at the end."""
import math

import numpy as np
import pytest

import linalg_exact as E
from oracle import acq_grad as AG

pytestmark = pytest.mark.gpu

RATIOS = {}
POOL = 2049
SIZES = (1, 127, 256, 640, 2049)
NOISE = 0.01


def _ratio(name, r):
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


def _load(h, qc, kid, p, L):
    h.set_data(qc.X, np.zeros((qc.N, qc.P)))
    h.set_kernel(kid, p, NOISE)
    h.load_factor(L, qc.alpha)


def _assert_within(name, got, ref, bound, tag):
    err = np.abs(got - ref)
    r = float(np.max(err / bound))
    assert r <= 1.0, f"{tag} {name}: ratio {r:.3e}; {E.worst_tile(err / bound)}"
    return _ratio(name, r)


def _check_acq(h, Xq, mu, s2, dmu, ds2, tag):
    """UCB and EI values and gradients from lb_acq_grad against oracle/acq_grad's epilogue on the device's own mu (output
    0), sigma^2, grad mu and grad sigma^2."""
    mu0 = mu[:, 0]
    f_max = float(np.median(mu0))
    for acq_id, params in ((0, [0.6]), (1, [f_max, 0.01])):
        v, g = h.acq_grad(acq_id, params, Xq)
        rv, rg = AG.ucb(mu0, s2, dmu, ds2, params[0]) if acq_id == 0 else AG.ei(mu0, s2, dmu, ds2, *params)
        bv, bg = E.bound_acq(acq_id, params, mu0, s2, dmu, ds2)
        name = ("ucb", "ei")[acq_id]
        _assert_within(name, v, rv, bv, tag)
        _assert_within(name + "_grad", g, rg, bg, tag)


def _check_grad(h, qc, kid, p, Xq, sizes, tag, acq=True):
    """lb_query_grad on the prefixes `sizes` of Xq against the reference within twice the one-evaluation bounds."""
    r = qc.grad_reference(kid, p, NOISE, Xq)
    b = E.grad_bounds(kid, p, qc.X, Xq, qc.alpha, NOISE, qc.norm_E(), r)
    _load(h, qc, kid, p, r["L"])
    out = {}
    for M in sizes:
        got = h.query_grad(Xq[:M])
        ratios = [_assert_within(name, g, r[name][:M], 2.0 * b[name][:M], f"{tag} M={M}")
                  for name, g in zip(("mu", "s2", "dmu", "ds2"), got)]
        assert all(np.all(np.isfinite(g)) for g in got)
        print(f"{tag} M={M} ratio mu={ratios[0]:.2e} s2={ratios[1]:.2e} dmu={ratios[2]:.2e} ds2={ratios[3]:.2e}")
        if acq:
            _check_acq(h, Xq[:M], *got, f"{tag} M={M}")
        out[M] = got
    return r, out


# ---- every super-block shape of the backward walk ----------------------------------------------------------------------
@pytest.mark.parametrize("kid", E.KERNELS, ids=[E.KERNEL_NAMES[k] for k in E.KERNELS])
@pytest.mark.parametrize("T", E.QUERY_T)
def test_grad_every_super_block_shape(handle, T, kid):
    N = 100 if T == 1 else (128 * T - 1 if T % 2 else 128 * T)
    qc = E.QueryCase(N, 3, 2, 9000 + 10 * T + kid)
    assert qc.norm_E() <= 0.25
    p = E.kernel_params(kid, 3, qc.rng)
    Xq = qc.rng.uniform(0.0, 1.0, size=(POOL, 3))
    _check_grad(handle, qc, kid, p, Xq, SIZES, f"[T={T} {E.KERNEL_NAMES[kid]}]")


# ---- staged widths: the gradient kernel's 16-coordinate passes ----------------------------------------------------------
WIDTHS = ([(1, D, 0) for D in (1, 15, 16, 17, 32, 33, 64)] + [(3, D, 0) for D in (1, 15, 16, 17, 32, 33, 64)]
          + [(0, 15, 1), (0, 15, 2), (0, 16, 1), (0, 60, 4), (0, 64, 0)])


@pytest.mark.parametrize("kid,D,klam", WIDTHS, ids=[f"{E.KERNEL_NAMES[k]}_D{d}_k{m}" for k, d, m in WIDTHS])
@pytest.mark.parametrize("T", (2, 17))
def test_grad_staged_widths(handle, T, kid, D, klam):
    """De = D + klam staged coordinates in {1, 15, 16, 17, 32, 33, 64}: one pass, a full pass, a ragged last pass of 1 or 15,
    four full passes; SE-ARD's Lambda columns push De across 16 and the map back through J mixes them into every x_r."""
    qc = E.QueryCase(128 * T - 1, D, 1, 9500 + 100 * T + 10 * D + klam + kid)
    p = E.grad_params(kid, D, klam, qc.rng)
    Xq = qc.rng.uniform(0.0, 1.0, size=(300, D))
    _check_grad(handle, qc, kid, p, Xq, (300,), f"[T={T} {E.KERNEL_NAMES[kid]} D={D} klam={klam}]")


# ---- several outputs ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", (2, 17))
def test_grad_five_outputs(handle, T):
    """P = 5: grad mu and EI follow output 0 (the bounds are of output 0's gradient and EI on mu[:, 0]; the other outputs'
    gradients are far outside them), and mu equals lb_query's bit for bit."""
    qc = E.QueryCase(128 * T - 1, 3, 5, 9800 + T)
    kid = 1
    p = E.kernel_params(kid, 3, qc.rng)
    Xq = qc.rng.uniform(0.0, 1.0, size=(300, 3))
    r, out = _check_grad(handle, qc, kid, p, Xq, (256, 300), f"[T={T} P=5]")
    for M, (mu, s2, dmu, _) in out.items():
        mq, sq = handle.query(Xq[:M])
        assert np.array_equal(mu, mq) and np.array_equal(s2, sq)
    b = E.grad_bounds(kid, p, qc.X, Xq, qc.alpha, NOISE, qc.norm_E(), r)
    dmu = out[300][2]
    for o in range(1, 5):  # the gradient of another output would be detected
        other = np.stack([(r["c"] * q).T @ qc.alpha[:, o] for q in r["Q"]], axis=1)
        assert np.max(np.abs(other - dmu) / (2.0 * b["dmu"])) > 1.0


# ---- grouping and batch independence of the backward walk ----------------------------------------------------------------
@pytest.mark.parametrize("N,P,seed", [(2048, 1, 31), (4097, 2, 32)], ids=["T16", "T33"])
def test_grad_panel_grouping_bit_identical(handle, lib, N, P, seed):
    """The forward and the backward walk take their candidate column tiles in four stream groups when a launch of all of
    them is under one round of the machine, otherwise on one stream (lb_query_panel_groups).  Nested prefixes on either
    side of that rule give bit-identical mu, sigma^2, grad mu and grad sigma^2; each super-block and group costs two
    forward and two backward launches."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    slots = 2 * sms  # CfgDual: two CTAs per SM
    per_ct = 2 * 16  # CTAs per 128-candidate column tile in one launch: two 64-wide tiles x a 16-row-tile super-block

    def groups(M):
        ct = -(-M // 128)
        return 4 if ct >= 4 and ct * per_ct < slots else 1

    m4 = (slots - 1) // per_ct * 128
    m1 = m4 + 1
    mid = (4 * 128 + m4) // 2 - 3
    sizes = (m1, m4, mid)
    assert [groups(M) for M in sizes] == [1, 4, 4], (sms, sizes)
    assert min(sizes) >= 256

    qc = E.QueryCase(N, 3, P, seed)
    kid = 2
    p = E.kernel_params(kid, 3, qc.rng)
    Xq = qc.rng.uniform(0.0, 1.0, size=(m1, 3))
    r, out = _check_grad(handle, qc, kid, p, Xq, (m1,), f"[grouping N={N}]", acq=False)
    T = -(-N // 128)
    nsb = -(-T // 16)
    fixed = set()
    for M in sizes:
        n0 = lib.lb_launch_count(handle.h)
        out[M] = handle.query_grad(Xq[:M])
        fixed.add(lib.lb_launch_count(handle.h) - n0 - 4 * nsb * groups(M))
    assert len(fixed) == 1, f"the launch count does not follow the grouping rule: {fixed}"
    for M in sizes[1:]:
        for k, (a, b) in enumerate(zip(out[M], out[m1])):
            assert np.array_equal(a, b[:M]), f"M={M} {('mu', 'sigma2', 'dmu', 'ds2')[k]}: {E.worst_tile(a - b[:M])}"


# ---- the _dev entry points -----------------------------------------------------------------------------------------------
def test_dev_variants_equal_host_variants(handle, lib):
    import torch
    qc = E.QueryCase(128 * 17 - 1, 4, 3, 9900)
    kid = 0
    p = E.grad_params(kid, 4, 1, qc.rng)
    Xq = qc.rng.uniform(0.0, 1.0, size=(700, 4))
    r = qc.grad_reference(kid, p, NOISE, Xq)
    _load(handle, qc, kid, p, r["L"])
    h = handle
    M, D, P = Xq.shape[0], 4, 3
    mean = qc.rng.normal(size=M)
    mgrad = qc.rng.normal(size=(M, D))
    host = h.query_grad(Xq)
    dev = torch.device("cuda:0")
    tX = torch.from_numpy(Xq).to(dev)
    tmu, ts2 = torch.empty((M, P), dtype=torch.float64, device=dev), torch.empty(M, dtype=torch.float64, device=dev)
    tdmu, tds2 = (torch.empty((M, D), dtype=torch.float64, device=dev) for _ in range(2))
    torch.cuda.synchronize()
    check = h._lib.check
    check(lib.lb_query_grad_dev(h.h, M, tX.data_ptr(), tmu.data_ptr(), ts2.data_ptr(), tdmu.data_ptr(), tds2.data_ptr()), "lb_query_grad_dev")
    torch.cuda.synchronize()
    for name, a, b in zip(("mu", "s2", "dmu", "ds2"), host, (tmu, ts2, tdmu, tds2)):
        assert np.array_equal(a, b.cpu().numpy()), name
    tmean, tmg = torch.from_numpy(mean).to(dev), torch.from_numpy(mgrad).to(dev)
    for acq_id, params in ((0, [0.6]), (1, [float(np.median(host[0][:, 0])), 0.01])):
        for with_mean in (False, True):
            v, g = h.acq_grad(acq_id, params, Xq, mean=mean if with_mean else None, mean_const=0.25,
                              mean_grad=mgrad if with_mean else None)
            ap = np.array(list(params) + [0.0] * (2 - len(params)))
            tv, tg = torch.empty(M, dtype=torch.float64, device=dev), torch.empty((M, D), dtype=torch.float64, device=dev)
            torch.cuda.synchronize()
            check(lib.lb_acq_grad_dev(h.h, acq_id, ap.ctypes.data, M, tX.data_ptr(), tmean.data_ptr() if with_mean else None, 0.25,
                                   tmg.data_ptr() if with_mean else None, tv.data_ptr(), tg.data_ptr()), "lb_acq_grad_dev")
            torch.cuda.synchronize()
            assert np.array_equal(v, tv.cpu().numpy()) and np.array_equal(g, tg.cpu().numpy()), (acq_id, with_mean)


# ---- the candidate-chunk boundary of the fp64 panel path -------------------------------------------------------------------
def test_candidate_chunk_boundary(lib):
    """A fitted N = 16384, D = 6 handle and a batch two candidates chunks long (the chunk: V = Np x Mc doubles within 6 GiB,
    as in abi.cu): every output of lb_query, lb_acq_argmax, lb_query_grad and lb_acq_grad (with per-candidate means and
    mean gradients) equals separate calls on the leading chunk and on the rest, bit for bit."""
    N, D = 16384, 6
    Np = -(-N // 128) * 128
    Mc = max(128, (6 << 30) // (8 * Np) // 128 * 128)
    M = Mc + 300
    assert -(-M // 128) * 128 > Mc and Mc == 49152, Mc  # the batch spans two chunks
    rng = np.random.default_rng(9950)
    X = rng.uniform(0.0, 1.0, size=(N, D))
    Y = np.sin(3.0 * X[:, :1]) + X[:, 1:2] ** 2
    Xq = rng.uniform(0.0, 1.0, size=(M, D))
    mean = rng.normal(size=M)
    mgrad = rng.normal(size=(M, D))
    h = E.Handle(lib)
    try:
        h.set_data(X, Y)
        h.set_kernel(0, np.concatenate([np.full(D, math.log(0.5)), [0.0]]), NOISE)
        h.fit()
        parts = (slice(0, Mc), slice(Mc, M))

        def both(f):
            whole = f(slice(0, M))
            split = [f(s) for s in parts]
            return whole, split

        whole, split = both(lambda s: h.query(Xq[s]))
        for k in range(2):
            assert np.array_equal(whole[k], np.concatenate([sp[k] for sp in split])), ("lb_query", k)
        whole, split = both(lambda s: h.query_grad(Xq[s]))
        for k in range(4):
            assert np.array_equal(whole[k], np.concatenate([sp[k] for sp in split])), ("lb_query_grad", k)
        f_max = float(np.quantile(whole[0][:, 0], 0.9))
        for acq_id, params in ((0, [0.6]), (1, [f_max, 0.01])):
            whole, split = both(lambda s: h.acq_argmax(acq_id, params, Xq[s], mean=mean[s]))
            vals = np.concatenate([sp[0] for sp in split])
            assert np.array_equal(whole[0], vals), ("lb_acq_argmax values", acq_id)
            assert whole[2] == int(np.argmax(vals)) and whole[1] == vals[whole[2]], ("lb_acq_argmax best", acq_id)
            whole, split = both(lambda s: h.acq_grad(acq_id, params, Xq[s], mean=mean[s], mean_grad=mgrad[s]))
            for k in range(2):
                assert np.array_equal(whole[k], np.concatenate([sp[k] for sp in split])), ("lb_acq_grad", acq_id, k)
    finally:
        h.close()


# ---- Matern kernels at subnormal squared distances -------------------------------------------------------------------------
@pytest.mark.parametrize("kid", (1, 2), ids=("matern52", "matern32"))
def test_subnormal_squared_distances(lib, oracle_mod, kid):
    """Training points at 0 and 1e-160 e_i, candidates at 0, 1e-170 e_1 and 1e-155 (1, ..., 1): squared distances below
    DBL_MIN.  The fit, the query on the one-point, slab and panel paths, the gradients and the reduced-precision path's
    mean are finite and agree with the oracle as everywhere else."""
    O = oracle_mod
    D = 3
    rng = np.random.default_rng(9960 + kid)
    X = np.vstack([np.zeros((1, D)), 1e-160 * np.eye(D), rng.uniform(0.0, 1.0, size=(296, D))])
    Y = np.sin(3.0 * X[:, :1]) + X[:, 1:2]
    Y = Y - Y.mean()
    special = np.vstack([np.zeros((1, D)), 1e-170 * np.eye(D)[:1], np.full((1, D), 1e-155)])
    Xq = np.vstack([special, X[:2], rng.uniform(0.0, 1.0, size=(295, D))])
    hp = np.array([math.log(0.4), 0.0])
    og = O.OracleGP()
    og.set_data(X, Y)
    og.set_kernel(kid, hp, NOISE)
    og.fit()
    mu_o, s2_o = og.query(Xq)
    _, _, dmu_o, ds2_o, mag = AG.query_grad(kid, hp, og.noise, X, og.get(1), og.get(2), Xq)
    h = E.Handle(lib)
    tf = E.Handle(lib, precision=1)
    try:
        for hh in (h, tf):
            hh.set_data(X, Y)
            hh.set_kernel(kid, hp, NOISE)
            hh.fit()
        assert np.all(np.isfinite(h.get(1))) and np.all(np.isfinite(h.get(2)))
        for name, M in (("point", 1), ("point", 2), ("point", 3), ("slab", 7), ("panel", Xq.shape[0])):
            Xm = Xq[M - 1:M] if name == "point" else Xq[:M]
            mu, s2 = h.query(Xm)
            ref_mu, ref_s2 = (mu_o[M - 1:M], s2_o[M - 1:M]) if name == "point" else (mu_o[:M], s2_o[:M])
            assert np.all(np.isfinite(mu)) and np.all(np.isfinite(s2)), (name, M, mu, s2)
            assert np.allclose(mu, ref_mu, rtol=0, atol=1e-10) and np.allclose(s2, ref_s2, rtol=0, atol=1e-10), (name, M)
        mu, s2, dmu, ds2 = h.query_grad(Xq)
        assert all(np.all(np.isfinite(a)) for a in (mu, s2, dmu, ds2))
        assert np.allclose(mu, mu_o, rtol=0, atol=1e-10) and np.allclose(s2, s2_o, rtol=0, atol=1e-10)
        for a, b in ((dmu, dmu_o), (ds2, ds2_o)):
            assert np.all(np.abs(a - b) <= 1e-9 * mag + 1e-15), np.abs(a - b).max()
        mu32, s232 = tf.query(Xq)
        assert np.all(np.isfinite(mu32)) and np.all(np.isfinite(s232))
        assert np.abs(mu32 - mu_o).max() <= 1e-9
    finally:
        h.close()
        tf.close()
