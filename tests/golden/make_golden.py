"""Generates tests/golden/*.npz by running the REFERENCE'S OWN code
(oracle/_ref/libref_gp.so = the reference's src/limbo headers compiled against the
Eigen/Boost stand-in, see oracle/ref_shim/) on seeded inputs.  Run where __graft_entry__.build()
has built that library:   python tests/golden/make_golden.py
The fixtures pin the kernel formulas, noise placement, mean::Data, clamp, +noise, log-lik,
gradient, UCB / EI (with the reference's f_max loop) and the incremental Cholesky path."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from limbo_b200 import synth  # noqa: E402
from oracle import ref  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))

CASES = [
    # name, kernel_id, N, D, P, M, noise, hp (None = defaults), n0 (incremental start), optimize_noise, rprop_iters
    ("se_ard_n3_d1", 0, 3, 1, 1, 7, 0.01, None, 0, False, 0),
    ("se_ard_n8_d2", 0, 8, 2, 1, 16, 0.01, [0.2, -0.3, 0.1], 0, False, 0),
    ("se_ard_n40_d4_p2", 0, 40, 4, 2, 32, 0.01, [0.1, -0.2, 0.3, 0.0, 0.2], 0, False, 0),
    ("se_ard_n100_d6", 0, 100, 6, 1, 64, 0.01, None, 0, False, 0),
    ("se_ard_n150_d6_noiseopt", 0, 150, 6, 1, 32, 0.02, [0, 0, 0, 0, 0, 0, 0, float(np.log(np.sqrt(0.02)))], 0, True, 0),
    ("matern52_n50_d1", 1, 50, 1, 1, 40, 0.01, None, 0, False, 0),
    ("matern52_n200_d6", 1, 200, 6, 1, 64, 0.01, [-0.5, 0.3], 0, False, 0),
    ("matern32_n60_d3", 2, 60, 3, 1, 20, 0.01, [0.2, -0.1], 0, False, 0),
    ("exp_n60_d3", 3, 60, 3, 1, 20, 0.01, [0.3, 0.1], 0, False, 0),
    ("matern52_incremental_n100_d1", 1, 100, 1, 1, 30, 0.01, None, 60, False, 0),
    ("se_ard_incremental_cross128_d3", 0, 140, 3, 1, 30, 0.01, None, 120, False, 0),
    ("se_ard_rprop8_n60_d2", 0, 60, 2, 1, 10, 0.01, None, 0, False, 8),
    # kernel_id 4 = SquaredExpARD with Params::kernel_squared_exp_ard::k() = 2 (Lambda columns): hp = [ell (D), A(:,0), A(:,1), sigma_f]
    ("se_ard_lambda2_n90_d3", 4, 90, 3, 1, 24, 0.01, [-0.3, -0.5, -0.2, 0.5, -0.4, 0.3, 0.1, 0.7, -0.6, 0.2], 0, False, 0),
    ("se_ard_lambda2_incremental_n140_d2_p2", 4, 140, 2, 2, 16, 0.02, [-0.4, -0.1, 0.6, -0.3, -0.2, 0.5, 0.1], 126, False, 0),
    ("se_ard_lambda2_rprop5_n50_d2", 4, 50, 2, 1, 8, 0.01, None, 0, False, 5),
]

ONLY = sys.argv[1:]  # optional: regenerate only the named fixtures
for name, kid, N, D, P, M, noise, hp, n0, on, iters in CASES:
    if ONLY and name not in ONLY:
        continue
    X = synth.points(1234, N, D)
    y = synth.targets(X)
    Y = np.stack([y * (p + 1) + 0.1 * p for p in range(P)], axis=1)
    Xq = synth.points(1235, M, D)
    r = ref.run(kid, X, Y, noise, hp=hp, Xq=Xq, n0=n0, rprop_iters=iters, optimize_noise=on)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), kernel_id=kid, N=N, D=D, P=P, M=M, noise=noise,
                        hp_in=np.array([] if hp is None else hp, dtype=float), n0=n0, optimize_noise=on, rprop_iters=iters,
                        X=X, Y=Y, Xq=Xq, K=r["K"], L=r["L"], alpha=r["alpha"], mu=r["mu"], sigma2=r["sigma2"], loglik=r["loglik"],
                        grad=r["grad"], ucb=r["ucb"], ei=r["ei"], hp=r["hp"])
    print(name, "ok", r["loglik"])
