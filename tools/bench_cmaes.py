"""Batched CMA-ES acquisition search on the device (lb_acq_cmaes) against the same algorithm driven from the host (oracle/cmaes.py's
update, one acqui.UCB.argmax_batch per generation, candidates and values crossing PCIe every generation) and against
BatchedRandomSearch at equal evaluations.  The host-driven time is mostly the oracle's per-instance NumPy update (a Python loop
over the R instances every generation), not the copies: it measures what a host loop written that way costs, not the PCIe
round trips alone.  UCB on a Matern-5/2 GP of Hartmann6 (D = 6), N in {256, 2048, 16384}, R = 32 instances
started from the best distinct points of a 10000-point random pass.  Also sweeps sigma0 and the generation budget of the
device search at N = 2048, the measurement behind bayes_opt.defaults_bo.opt_batchedcmaes.  Prints one JSON object (DESIGN.md
§4.15) with the card's name and power limit.

    python tools/bench_cmaes.py [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from limbo_b200 import acqui, bayes_opt, kernel, mean, model, synth  # noqa: E402
from oracle import cmaes as OC  # noqa: E402

D, R, RANDOM_PASS, REPEATS = 6, 32, 10000, 5


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def params():
    class P:
        class kernel:
            noise = 1e-6

        class acqui_ucb:
            alpha = 0.5
    return P


def fitted(N):
    X = synth.points(17, N, D)
    gp = model.GP(D, 1, params=params(), kernel=kernel.MaternFiveHalves, mean=mean.Data)
    gp.compute(X, synth.hartmann6(X)[:, None])
    return gp


def timed(f):
    """median wall time (ms) over REPEATS calls (each ends in a device synchronise) after one warm-up, and the last result"""
    out = f()
    ts = []
    for _ in range(REPEATS):
        t0 = time.perf_counter()
        out = f()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "D": D, "R": R, "random_pass": RANDOM_PASS, "runs": [], "sweep": []}
    for N in (256, 2048, 16384):
        acq = acqui.UCB(fitted(N), params=params())
        cand = np.random.default_rng(N).random((RANDOM_PASS, D))
        best0, _, vals = acq.argmax_batch(cand, return_values=True)
        starts = bayes_opt._best_distinct(cand, vals, R)
        kw = dict(generations=50, tolx=1e-6, seed=3)
        t_dev, (bx, bv, n) = timed(lambda: acq.cmaes_batch(starts, **kw))
        score = lambda X: acq.argmax_batch(X, return_values=True)[2]  # noqa: E731
        t_host, (hx, hv, hn) = timed(lambda: OC.run(score, starts, kw["generations"], tolx=kw["tolx"], seed=kw["seed"]))

        class PR:
            class opt_batchedrandom:
                candidates = (RANDOM_PASS + n) // 3
                refinements = 2
                shrink = 0.1
        t_rand, xr = timed(lambda: bayes_opt.BatchedRandomSearch(PR, np.random.default_rng(0))(acq, D))
        row = {"N": N, "evaluations": RANDOM_PASS + n, "random_pass_best": best0,
               "device": {"ms": t_dev, "best": max(bv, best0), "evals": n},
               "host_driven": {"ms": t_host, "best": max(hv, best0), "evals": hn},
               "random_search": {"ms": t_rand, "best": float(score(xr[None])[0]), "evals": 3 * PR.opt_batchedrandom.candidates}}
        print(json.dumps(row), flush=True)
        res["runs"].append(row)
        if N == 2048:
            for sigma0 in (0.1, 0.3, 0.5):
                for gens in (25, 50, 100):
                    bests = [max(acq.cmaes_batch(starts, sigma0=sigma0, generations=gens, tolx=1e-6, seed=s)[1], best0) for s in range(5)]
                    t, _ = timed(lambda: acq.cmaes_batch(starts, sigma0=sigma0, generations=gens, tolx=1e-6, seed=0))
                    res["sweep"].append({"sigma0": sigma0, "generations": gens, "ms": t, "best_mean": float(np.mean(bests)),
                                         "best_min": float(np.min(bests))})
                    print(json.dumps(res["sweep"][-1]), flush=True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
