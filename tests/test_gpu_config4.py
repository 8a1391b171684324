"""Reduced-precision candidate scoring pinned AT CONFIG-4 SIZE (BASELINE.json configs[3]: N=16384, D=12, SquaredExpARD,
>= 10^5 EI candidates) against the fp64 DMMA path of the same handle type - which is itself pinned to the oracle /
reference at 1e-10 (tests/test_gpu_parity.py, tests/test_golden.py) and, at this size, by the residual / batch==single
properties of tests/test_gpu_fullsize.py.

Stated tolerances (model/gp.hpp:618-624 computes sigma^2 = k(v,v) - |L^-1 k*|^2 in fp64; here the GEMM operands carry an
11-bit significand, fp32 accumulation):
    |d mu|                <= 1e-9           (the mean never leaves fp64)
  one-plane modes (tf32, fp16), measured on an H100 at this size (cond(K) ~ 1.6e6):
    |d sigma^2|           <= 5e-3 k(v,v)    absolute, every candidate (max 4.2e-3; mean -1.5e-3: the modelled rounding bias
                                            under-corrects at this conditioning)
    |d sigma^2| / sigma^2 <= 0.35 max, <= 0.15 median: sigma^2 sits at its floor (0.010 .. 0.043, the noise is 0.01), so the
                                            absolute error IS a 12 % median relative error - these modes rank candidates, they do
                                            not report calibrated variances
    EI regret             <= 2 %: EI_fp64(argmax EI_reduced) >= 0.98 max EI_fp64 (measured 0: same candidate)
  split-operand mode (fp16x3: hi + 2^-11 lo planes, three products, fp64 combination):
    |d sigma^2|           <= 2e-4 absolute (measured 8.8e-5, mean -4.6e-5), <= 1e-2 relative to sigma^2 (measured 5e-3);
                          EI regret <= 1e-4.  The floor is the fp32 accumulation of the tensor core over K = 16384 terms of a
                          heavily cancelling sum (partial sums ~10^2 x the result at cond(K) ~ 1.6e6); at N <= 4096 the same
                          mode is at <= 2e-5 (tests/test_gpu_tf32.py).  Exact variances: LB_PREC_FP64.
The measured table is printed as one JSON line (pytest -s shows it); records/h100_config4_parity.json is that line from an H100 run."""
import json

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def test_reduced_precision_at_config4_size():
    import torch
    from limbo_b200 import acqui, kernel, mean, model, synth
    if torch.cuda.mem_get_info()[0] < 40e9:
        pytest.skip("needs ~40 GB of device memory")
    N, D, M = 16384, 12, 131072
    X = synth.points(1234, N, D)
    y = synth.targets(X)
    Xq = synth.points(4321, M, D)
    kw = dict(kernel=kernel.SquaredExpARD, mean=mean.Data)
    g64 = model.GP(D, 1, **kw)
    g64.compute(X, y[:, None])
    mu64, s64 = g64.query_batch(Xq)
    ei64 = acqui.EI(g64)
    best64, i64, v64 = ei64.argmax_batch(Xq, return_values=True)
    table = {"config": f"N={N}, D={D}, SquaredExpARD (ell=1, sigma_f=1, noise=0.01), M={M} candidates", "sigma2_fp64": {
        "min": float(s64.min()), "median": float(np.median(s64)), "max": float(s64.max())}, "ei_fp64_max": float(best64), "modes": {}}
    del g64
    for prec in ("tf32", "fp16", "fp16x3"):
        g = model.GP(D, 1, precision=prec, **kw)
        g.compute(X, y[:, None])
        mu, s2 = g.query_batch(Xq)
        best, idx, v = acqui.EI(g).argmax_batch(Xq, return_values=True)
        d = np.abs(s2 - s64)
        rel = d / s64
        regret = float((best64 - v64[idx]) / best64) if best64 > 0 else 0.0
        row = {"max_abs_dmu": float(np.abs(mu - mu64).max()), "max_abs_dsigma2": float(d.max()), "mean_dsigma2": float((s2 - s64).mean()),
               "rel_dsigma2": {"median": float(np.median(rel)), "p90": float(np.percentile(rel, 90)), "p99": float(np.percentile(rel, 99)),
                               "p999": float(np.percentile(rel, 99.9)), "max": float(rel.max())},
               "ei_argmax_same_index": bool(idx == i64), "ei_regret_rel": regret, "max_abs_dei": float(np.abs(v - v64).max()),
               "ei_rank_of_choice_under_fp64": int((v64 > v64[idx]).sum())}
        table["modes"][prec] = row
        del g
    print(json.dumps(table))
    for prec, row in table["modes"].items():
        assert row["max_abs_dmu"] <= 1e-9, (prec, row)
        if prec == "fp16x3":
            assert row["max_abs_dsigma2"] <= 2e-4 and row["rel_dsigma2"]["max"] <= 1e-2 and row["ei_regret_rel"] <= 1e-4, (prec, row)
            continue
        assert row["max_abs_dsigma2"] <= 5e-3, (prec, row)
        assert row["rel_dsigma2"]["max"] <= 0.35 and row["rel_dsigma2"]["median"] <= 0.15, (prec, row)
        assert row["ei_regret_rel"] <= 0.02, (prec, row)
