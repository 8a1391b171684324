"""ParEGO on the device (DESIGN.md §4.16), Matern-5/2 GPs over ZDT2 (D = 6, K = 2), noise 1e-6:
  (a) one model update at N in {2048, 16384}: model.GPParego.add_sample (the factor grown by one row, alpha re-solved against the
      rescalarised observations) against a full refit with the same weights (compute, as the reference's add_sample does);
  (b) q in {1, 4, 16} proposals from 20 000 candidates at N = 2048: one acqui.UCB.argmax_cols on a q-column GPParego against q
      one-output GPs, each fitted to one column and queried (q fits + q queries);
  (c) a 50-generation acqui.UCB.cmaes_cols with 32 instances (8 per column, q = 4) at N = 2048.
Times are medians of wall time around calls that end in a device synchronise, after one warm-up.  Prints one JSON object with
the card's name and power limit, read in the same run, and writes it to --out (records/h100_parego.json by default).

    python tools/bench_parego.py [--out FILE]
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

from limbo_b200 import acqui, kernel, mean, model, synth  # noqa: E402
from oracle import ehvi as OE  # noqa: E402

D, REPEATS = 6, 5


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


class P:
    class kernel:
        noise = 1e-6


def timed(f, repeats=REPEATS):
    out = f()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = f()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), out


def parego(N, q, seed=5):
    X = synth.points(seed, N + 1, D)
    F = OE.zdt2(X)
    draws = np.random.default_rng(seed).random((q, 2))
    gp = model.GPParego(D, q, params=P, kernel=kernel.MaternFiveHalves)
    gp.compute(X[:N], F[:N], lambdas=draws)
    return gp, X, F, draws


def update(N):
    """one add_sample on a freshly fitted N-sample model against a full compute of the N + 1 samples"""
    def incremental():
        gp, X, F, draws = parego(N, 1)
        gp._lib.lb_sync(gp._h)
        t0 = time.perf_counter()
        gp.add_sample(X[N], F[N], lambdas=draws)
        gp._lib.lb_sync(gp._h)
        assert gp.append_count() == 1
        return (time.perf_counter() - t0) * 1e3

    incremental()
    t_inc = float(np.median([incremental() for _ in range(REPEATS)]))
    _, X, F, draws = parego(N, 1)
    full = model.GPParego(D, 1, params=P, kernel=kernel.MaternFiveHalves)
    t_full, _ = timed(lambda: (full.compute(X, F, lambdas=draws), full._lib.lb_sync(full._h)))
    return {"N": N, "append_ms": t_inc, "refit_ms": t_full}


def proposals(q, N=2048, M=20000):
    gp, X, F, draws = parego(N, q)
    cand = np.random.default_rng(1).random((M, D))
    t_cols, _ = timed(lambda: acqui.UCB(gp).argmax_cols(cand))
    Y = gp.observations_matrix()

    def separate():
        out = []
        for r in range(q):
            one = model.GP(D, 1, params=P, kernel=kernel.MaternFiveHalves, mean=mean.Data)
            one.compute(X[:N], Y[:, r:r + 1])
            out.append(acqui.UCB(one).argmax_batch(cand))
        return out

    t_sep, _ = timed(separate, repeats=3)
    return {"q": q, "N": N, "candidates": M, "argmax_cols_ms": t_cols, "q_fits_and_queries_ms": t_sep}


def cmaes(N=2048, q=4, R=32, generations=50):
    gp, _, _, _ = parego(N, q)
    starts = np.random.default_rng(2).random((R, D))
    cols = [i % q for i in range(R)]
    t, (_, _, n) = timed(lambda: acqui.UCB(gp).cmaes_cols(starts, cols, sigma0=0.1, generations=generations, tolx=1e-12, seed=3))
    return {"N": N, "q": q, "instances": R, "generations": generations, "evaluations": int(n), "ms": t}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "records", "h100_parego.json"))
    a = ap.parse_args()
    res = {"card": card(), "update": [], "proposals": [], "cmaes_cols": None}
    for N in (2048, 16384):
        res["update"].append(update(N))
        print(json.dumps(res["update"][-1]), flush=True)
    for q in (1, 4, 16):
        res["proposals"].append(proposals(q))
        print(json.dumps(res["proposals"][-1]), flush=True)
    res["cmaes_cols"] = cmaes()
    res["card_after"] = card()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
