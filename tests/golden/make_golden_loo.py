"""Generates tests/golden/loo/*.npz from the REFERENCE'S OWN code (oracle/_ref/libref_gp.so, see make_golden.py):
 * loo_*       : GP::compute_log_loo_cv / compute_kernel_grad_log_loo_cv            (gp.hpp:339-399)
 * meangrad_*  : GP::compute_log_lik / compute_mean_grad_log_lik with mean::FunctionARD<mean::Constant>  (gp.hpp:313-330)
Run where oracle/_ref/libref_gp.so is built:   python tests/golden/make_golden_loo.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from limbo_b200 import synth  # noqa: E402
from oracle import ref  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "loo")
os.makedirs(OUT, exist_ok=True)

LOO_CASES = [
    # name, kernel_id, N, D, P, noise, hp, optimize_noise
    ("loo_se_ard_n8_d2", 0, 8, 2, 1, 0.01, [0.2, -0.3, 0.1], False),
    ("loo_se_ard_n60_d3_p2", 0, 60, 3, 2, 0.01, [-0.4, -0.2, 0.1, 0.2], False),
    ("loo_se_ard_n150_d6_noiseopt", 0, 150, 6, 1, 0.02, [-0.5, -0.3, -0.6, -0.2, -0.4, -0.1, 0.1, float(np.log(np.sqrt(0.02)))], True),
    ("loo_matern52_n130_d2", 1, 130, 2, 1, 0.01, [-0.5, 0.3], False),
    ("loo_matern32_n70_d3_noiseopt", 2, 70, 3, 1, 0.05, [0.2, -0.1, float(np.log(np.sqrt(0.05)))], True),
    ("loo_exp_n70_d3", 3, 70, 3, 1, 0.01, [-0.3, 0.1], False),
    ("loo_se_ard_n260_d4", 0, 260, 4, 1, 0.01, [-0.7, -0.5, -0.6, -0.8, 0.0], False),
    ("loo_se_ard_lambda2_n80_d2", 4, 80, 2, 1, 0.01, [-0.4, -0.1, 0.6, -0.3, -0.2, 0.5, 0.1], False),  # kernel_id 4: k = 2
]
ONLY = sys.argv[1:]
for name, kid, N, D, P, noise, hp, on in LOO_CASES:
    if ONLY and name not in ONLY:
        continue
    X = synth.points(4321, N, D)
    y = synth.targets(X)
    Y = np.stack([y * (p + 1) + 0.1 * p for p in range(P)], axis=1)
    v, g = ref.loo(kid, X, Y, noise, hp=hp, optimize_noise=on)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), kernel_id=kid, N=N, D=D, P=P, noise=noise, hp_in=np.array(hp, dtype=float),
                        optimize_noise=on, X=X, Y=Y, loo=v, loo_grad=g)
    print(name, v, g)

MEAN_CASES = [
    # name, kernel_id, N, D, P, noise, kernel hp, mean hp [tr row-major P x (P+1), constant]
    ("meangrad_se_ard_n50_d2_p1", 0, 50, 2, 1, 0.01, [-0.3, -0.2, 0.1], [0.8, 0.3, 0.5]),
    ("meangrad_matern52_n140_d3_p2", 1, 140, 3, 2, 0.01, [-0.4, 0.2], [1.1, 0.2, -0.1, -0.3, 0.9, 0.4, 0.7]),
]
for name, kid, N, D, P, noise, hp, mh in MEAN_CASES:
    if ONLY and name not in ONLY:
        continue
    X = synth.points(4322, N, D)
    y = synth.targets(X)
    Y = np.stack([y * (p + 1) + 0.1 * p for p in range(P)], axis=1)
    ll, g, mu0 = ref.mean_grad(kid, X, Y, mh, noise, hp=hp)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), kernel_id=kid, N=N, D=D, P=P, noise=noise, hp_in=np.array(hp, dtype=float),
                        mean_hp=np.array(mh, dtype=float), X=X, Y=Y, loglik=ll, mean_grad=g, mu_at_x0=mu0)
    print(name, ll, g)
