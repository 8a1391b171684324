"""The batched device CMA-ES over ECI (lb_eci_cmaes) and over the pseudo-input sparse GP (lb_spgp_acq_cmaes), each against the same
algorithm driven from the host (oracle/cmaes.py's update, one argmax_batch per generation) and against BatchedRandomSearch at
equal evaluations, as tools/bench_cmaes.py measures UCB over a GP.  D = 6, R = 32 instances started from the best distinct points
of a 10000-point random pass, 50 generations.
  * ECI: a Matern-5/2 objective GP of Hartmann6 and a constraint GP that rules out part of the box, N in {256, 2048, 16384}.
    Every generation scores both models.
  * SPGP: UCB and EI over an SPGP of Hartmann6 with N = 16384 samples and M = 1638 pseudo-inputs (the default 10 %), computed at
    its starting vector.  Every generation predicts in QCHUNK-candidate chunks.
Prints one JSON object (DESIGN.md §4.15) with the card's name and power limit.

    python tools/bench_cmaes_eci_spgp.py [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_cmaes import D, R, RANDOM_PASS, card, timed  # noqa: E402
from limbo_b200 import acqui, bayes_opt, kernel, mean, model, synth  # noqa: E402
from oracle import cmaes as OC  # noqa: E402

GENERATIONS = 50


def params():
    class P:
        class kernel:
            noise = 1e-6

        class acqui_ucb:
            alpha = 0.5

        class acqui_ei:
            jitter = 0.0

        class acqui_eci:
            jitter = 0.0
    return P


def constraint(X):
    return 1.0 + np.cos(4.0 * X[:, 0] + X[:, -1])


def eci(N):
    X = synth.points(17, N, D)
    obj = model.GP(D, 1, params=params(), kernel=kernel.MaternFiveHalves, mean=mean.Data)
    obj.compute(X, synth.hartmann6(X)[:, None])
    con = model.GP(D, 1, params=params(), kernel=kernel.MaternFiveHalves, mean=mean.Constant)
    con.compute(X, constraint(X)[:, None])
    return acqui.ECI(obj, con, params=params())


def spgp(N):
    X = synth.points(17, N, D)
    s = model.SPGP(D, 1, params=params(), mean=mean.Data, hp_opt=lambda f, init, bounded: init, rng=np.random.default_rng(0))
    s.compute(X, synth.hartmann6(X)[:, None])
    return s


def arm(name, N, acq, extra=None):
    cand = np.random.default_rng(N).random((RANDOM_PASS, D))
    best0, _, vals = acq.argmax_batch(cand, return_values=True)
    starts = bayes_opt._best_distinct(cand, vals, R)
    kw = dict(generations=GENERATIONS, tolx=1e-6, seed=3)
    t_dev, (bx, bv, n) = timed(lambda: acq.cmaes_batch(starts, **kw))
    score = lambda X: acq.argmax_batch(X, return_values=True)[2]  # noqa: E731
    t_host, (hx, hv, hn) = timed(lambda: OC.run(score, starts, kw["generations"], tolx=kw["tolx"], seed=kw["seed"]))

    class PR:
        class opt_batchedrandom:
            candidates = (RANDOM_PASS + n) // 3
            refinements = 2
            shrink = 0.1
    t_rand, xr = timed(lambda: bayes_opt.BatchedRandomSearch(PR, np.random.default_rng(0))(acq, D))
    t_pass, _ = timed(lambda: acq.argmax_batch(np.tile(starts, (OC.default_lambda(D), 1))))  # one generation's R lambda candidates
    row = {"acquisition": name, "N": N, **(extra or {}), "evaluations": RANDOM_PASS + n, "random_pass_best": best0,
           "one_generation_argmax_ms": t_pass,
           "device": {"ms": t_dev, "best": max(bv, best0), "evals": n},
           "host_driven": {"ms": t_host, "best": max(hv, best0), "evals": hn},
           "random_search": {"ms": t_rand, "best": float(score(xr[None])[0]), "evals": 3 * PR.opt_batchedrandom.candidates}}
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "D": D, "R": R, "random_pass": RANDOM_PASS, "generations": GENERATIONS, "runs": []}
    for N in (256, 2048, 16384):
        res["runs"].append(arm("eci", N, eci(N)))
    s = spgp(16384)
    for name, acq in (("spgp_ucb", acqui.UCB(s, params=params())), ("spgp_ei", acqui.EI(s, params=params()))):
        res["runs"].append(arm(name, 16384, acq, {"M": s.nb_pseudo_samples()}))
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
