"""Generates tests/golden/oracle_ref/*.npz: the REFERENCE'S OWN outputs (oracle/_ref/libref_gp.so, see
oracle/ref_shim/) on the seeded inputs of tests/test_oracle_vs_ref.py, so that the restatement in oracle/ stays pinned
to the reference on machines without its sources.  Needs a built oracle/_ref/libref_gp.so:
    python tests/golden/make_golden_oracle_ref.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ref  # noqa: E402
import test_oracle_vs_ref as T  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "oracle_ref")
os.makedirs(OUT, exist_ok=True)

for kid in T.KIDS:
    for N, D, P in T.SHAPES:
        inp = T.restatement_inputs(kid, N, D, P)
        r = ref.run(kid, inp["X"], inp["Y"], T.NOISE, hp=inp["hp"], Xq=inp["Xq"])
        i, j = T.sampled_lower(N)  # K and L at a fixed sample of lower-triangle positions (keeps every file small)
        np.savez_compressed(os.path.join(OUT, T.restatement_name(kid, N, D, P)), K=r["K"][i, j], L=r["L"][i, j],
                            **{k: np.asarray(r[k]) for k in ("alpha", "mu", "sigma2", "loglik", "grad")})
X, y = T.rprop_inputs()
np.savez_compressed(os.path.join(OUT, "rprop10_se_ard_n50_d2"), hp=ref.run(0, X, y, 0.01, rprop_iters=10)["hp"])
X, y = T.incremental_inputs()
r = ref.run(1, X, y, 0.01, n0=25)
np.savez_compressed(os.path.join(OUT, "incremental_matern52_n40_d2"), L=r["L"], alpha=r["alpha"])
print("wrote", OUT)
