"""Generates tests/golden/lml_batch/*.npz from the REFERENCE'S OWN code (oracle/_ref/libref_gp.so, see make_golden.py): for several
kernel states of one data set, GP::compute_log_lik and GP::compute_kernel_grad_log_lik (gp.hpp:267-311) as
KernelLFOptimization evaluates them (kernel_lf_opt.hpp:77-92) - the rows lb_lml_grad_batch evaluates at once.
Each case holds R = 4 h-param vectors (kernel.h_params() layout, noise entry last when optimised) with long and short length
scales.  Run where oracle/_ref/libref_gp.so is built:   python tests/golden/make_golden_lml_batch.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from limbo_b200 import synth  # noqa: E402
from oracle import ref  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lml_batch")
os.makedirs(OUT, exist_ok=True)

CASES = [
    # name, kernel_id (4 = SE-ARD with k = 2 Lambda columns), N, D, P, noise, optimize_noise
    ("se_ard_n3_d1", 0, 3, 1, 1, 0.01, False),
    ("se_ard_n8_d2", 0, 8, 2, 1, 0.01, False),
    ("matern52_n60_d3", 1, 60, 3, 1, 0.01, False),
    ("se_ard_n60_d3_p2", 0, 60, 3, 2, 0.01, False),
    ("se_ard_lambda2_n60_d2", 4, 60, 2, 1, 0.01, False),
    ("matern32_n127_d2_noiseopt", 2, 127, 2, 1, 0.02, True),
    ("exp_n128_d3", 3, 128, 3, 1, 0.01, False),
    ("se_ard_n129_d4_noiseopt", 0, 129, 4, 1, 0.01, True),
    ("matern52_n129_d3_p2", 1, 129, 3, 2, 0.01, False),
    ("se_ard_lambda2_n190_d2", 4, 190, 2, 1, 0.01, False),  # the reference driver has no Lambda + noise parameter set
    ("matern52_n256_d2", 1, 256, 2, 1, 0.01, False),
    ("exp_n257_d3_noiseopt", 3, 257, 3, 1, 0.05, True),
    ("se_ard_n513_d2", 0, 513, 2, 1, 0.01, False),
]
R = 4
ONLY = sys.argv[1:]
for name, kid, N, D, P, noise, on in CASES:
    if ONLY and name not in ONLY:
        continue
    X = synth.points(777 + N, N, D)
    y = synth.targets(X)
    Y = np.stack([y * (p + 1) + 0.1 * p for p in range(P)], axis=1)
    nk = D + 1 if kid == 0 else (3 * D + 1 if kid == 4 else 2)
    rng = np.random.default_rng(N + 10 * kid)
    H = np.zeros((R, nk + (1 if on else 0)))
    for r in range(R):
        scale = [-1.5, -0.6, 0.0, 0.8][r]  # short to long length scales
        if kid in (0, 4):
            H[r, :D] = scale + rng.uniform(-0.2, 0.2, D)
            if kid == 4:
                H[r, D:3 * D] = rng.uniform(-0.5, 0.5, 2 * D)
        else:
            H[r, 0] = scale
        H[r, nk - 1] = rng.uniform(-0.3, 0.3)  # log sigma_f
        if on:
            H[r, nk] = float(np.log(np.sqrt(noise))) + rng.uniform(-0.5, 0.5)
    lik, grad = np.empty(R), np.empty_like(H)
    for r in range(R):
        out = ref.run(kid, X, Y, noise, hp=H[r], optimize_noise=on)
        lik[r], grad[r] = out["loglik"], out["grad"]
    np.savez_compressed(os.path.join(OUT, name + ".npz"), kernel_id=kid, N=N, D=D, P=P, noise=noise, optimize_noise=on, X=X, Y=Y,
                        H=H, lik=lik, grad=grad)
    print(name, lik)
