"""Lease balance of the handles' device buffers: a round of calls over every model and acquisition, then its handles
dropped, returns every pool lease it took (lb_debug_pool_live), including on the argument-error paths of the call-scoped
temporaries."""
import ctypes as C
import gc

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LB_ERR_ARG = -1


class _SparseParams:
    class model_sparse_gp:
        max_points = 150


def _gp_round(lib):
    import torch
    from limbo_b200 import kernel, model, pareto

    rng = np.random.default_rng(7)
    D = 3
    X = rng.random((120, D))
    Y = np.stack([np.sin(3 * X[:, 0]) + X[:, 1], np.cos(2 * X[:, 1]) - X[:, 2]], axis=1)
    Xq = rng.random((300, D))

    gp = model.GP(D, 1, kernel=kernel.MaternFiveHalves)
    gp.compute(list(X), list(Y[:, :1]))
    gp.query_batch(Xq[:40])  # slab path
    lib.lb_debug_set_query_panel_min(16)
    try:
        gp.query_batch(Xq)  # panel path
    finally:
        lib.lb_debug_set_query_panel_min(0)
    gp.query(Xq[0])  # one-point path
    gp.acq_argmax_batch(0, [0.5], Xq, return_values=True)  # UCB
    gp.acq_argmax_batch(1, [0.0, float(Y[:, 0].max())], Xq, return_values=True)  # EI
    con = model.GP(D, 1)
    con.compute(list(X), list(Y[:, 1:]))
    gp.eci_argmax_batch(con, float(Y[:, 0].max()), 0.0, Xq, return_values=True)
    gp.ehvi_argmax_batch(con, [-3.0, -3.0], np.array([[1.0, 0.5], [0.5, 1.0]]), Xq, return_values=True)
    gp.query_grad_batch(Xq[:50])
    gp.acq_grad_batch(1, [0.0, float(Y[:, 0].max())], Xq[:50])
    gp.eci_grad_batch(con, float(Y[:, 0].max()), 0.0, Xq[:50])
    gp.ehvi_grad_batch(con, [-3.0, -3.0], np.array([[1.0, 0.5], [0.5, 1.0]]), Xq[:50])
    k = gp.kernel_function()
    gp.lml_grad_batch(np.tile(k.h_params(), (5, 1)) + rng.uniform(-0.5, 0.5, (5, k.h_params_size())))
    dXq = torch.from_numpy(Xq[:50]).cuda()
    dMu, dS2, dDmu, dDs2, dAcq, dGrad = (torch.zeros(n, dtype=torch.float64, device="cuda") for n in (50, 50, 50 * D, 50 * D, 50, 50 * D))
    ep = np.array([float(Y[:, 0].max()), 0.0])
    torch.cuda.synchronize()
    assert lib.lb_query_grad_dev(gp._h, 50, dXq.data_ptr(), dMu.data_ptr(), dS2.data_ptr(), dDmu.data_ptr(), dDs2.data_ptr()) == 0
    assert lib.lb_eci_grad_dev(gp._h, con._h, ep.ctypes.data, 50, dXq.data_ptr(), None, 0.0, None, None, 0.0, None, dAcq.data_ptr(),
                               dGrad.data_ptr()) == 0
    torch.cuda.synchronize()
    del dXq, dMu, dS2, dDmu, dDs2, dAcq, dGrad
    gp.kernel_matrix(); gp.matrixL(); gp.inv_kernel()
    gp.compute_kernel_grad_log_loo_cv()
    gp.compute_mean_grad_log_lik()  # lb_kinv_obs_mean
    cp = gp.copy()
    cp.recompute()
    cp.query_batch(Xq[:10])
    for i in range(10):  # 120 -> 130 samples: lb_append grows the padded size past 128
        gp.add_sample(rng.random(D), np.array([0.1 * i]))
    gp.query_batch(Xq[:10])
    del cp, con

    tf = model.GP(D, 1, precision="tf32")
    tf.compute(list(X), list(Y[:, :1]))
    tf.query_batch(Xq)
    del tf

    h = pareto._handle(0)
    P = np.ascontiguousarray(rng.random((200, 2)))
    pareto.pareto_set_indices(P)
    dP = torch.from_numpy(P).cuda()
    dIdx = torch.zeros(200, dtype=torch.int64, device="cuda")
    nf = C.c_int64(-1)
    torch.cuda.synchronize()
    assert lib.lb_pareto_set_dev(h, 200, 2, dP.data_ptr(), dIdx.data_ptr(), C.addressof(nf)) == 0

    sg = model.SparsifiedGP(D, 1, params=_SparseParams)
    Xs = rng.random((400, D))
    sg.sparsify(Xs)
    dXs = torch.from_numpy(Xs).cuda()
    dk = torch.zeros(400, dtype=torch.int64, device="cuda")
    dr = torch.zeros(400, dtype=torch.int64, device="cuda")
    ds = torch.zeros(400, dtype=torch.float64, device="cuda")
    nk = C.c_int64(-1)
    torch.cuda.synchronize()
    assert lib.lb_sparsify_dev(sg._h, 400, D, dXs.data_ptr(), 150, dk.data_ptr(), C.addressof(nk), dr.data_ptr(), ds.data_ptr()) == 0
    assert nk.value == 150
    torch.cuda.synchronize()
    del sg, dP, dIdx, dXs, dk, dr, ds

    sp = model.SPGP(rng=np.random.default_rng(0))
    xs = rng.random((100, 1)) * 6.0
    sp.compute(xs, np.cos(xs))
    sp.query_batch(xs[:20])
    sp.acq_argmax_batch(0, [0.5], xs[:50], return_values=True)
    del sp, gp


def _live(lib):
    gc.collect()
    return lib.lb_debug_pool_live()


def test_round_returns_every_lease():
    from limbo_b200 import _lib
    lib = _lib.load()
    _gp_round(lib)  # warm-up: lazily created globals (the Pareto handle) keep their buffers
    live = _live(lib)
    _gp_round(lib)
    assert _live(lib) == live


def test_argument_errors_return_their_temporaries():
    from limbo_b200 import _lib, pareto
    lib = _lib.load()
    h = pareto._handle(0)
    rng = np.random.default_rng(3)
    objs = np.ascontiguousarray(rng.random((64, 2)))
    objs[17, 1] = np.nan
    idx = np.zeros(64, dtype=np.int64)
    nf = C.c_int64(-1)
    live = _live(lib)
    assert lib.lb_pareto_set(h, 64, 2, objs.ctypes.data, idx.ctypes.data, C.addressof(nf)) == LB_ERR_ARG
    assert _live(lib) == live
    X = np.ascontiguousarray(rng.random((500, 3)))
    X[123, 2] = np.inf
    kept = np.zeros(500, dtype=np.int64)
    nk = C.c_int64(-1)
    assert lib.lb_sparsify(h, 500, 3, X.ctypes.data, 100, kept.ctypes.data, C.addressof(nk), None, None) == LB_ERR_ARG
    assert _live(lib) == live
