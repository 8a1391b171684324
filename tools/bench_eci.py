"""Constrained BO on one GPU: what one ECI step costs next to bench.py's UCB step, on bench.py's workload.

Headline leg (N = 16384, D = 6): an SE-ARD / mean::Data objective GP on Hartmann6 and an Exp / mean::Constant constraint GP on a
synthetic 0/1 feasibility column (x0 + x1 >= 0.9) over the same samples.  Per step, each part timed with CUDA events on the
objective's stream (every call below returns after its device work, the constraint stream is joined in first):
    fit_obj, fit_con   GP.compute on each model
    f_max              max_i mu(x_i): one N-point query of the objective (what EI pays too)
    eci                acqui.ECI.argmax_batch over 20 000 candidates: both queries (own streams) + the fused epilogue
    two_queries        the same two queries back to back on the host (obj then con), for comparison with `eci`
    ucb_step           bench.py's step: fit + UCB over 10^4 candidates + argmax (alternated with the ECI step)
Small-N leg (N = 1024, 2000 candidates): eci.hpp's one-point contract (two one-point queries per candidate, the Python
acqui.ECI.__call__) against one batched call.

Prints one JSON line with the card's name, power limit and max SM clock read in the same run.
    python tools/bench_eci.py [--steps 3]"""
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


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": out[0], "power_limit_w": float(out[1]), "sm_clock_max_mhz": float(out[2])}
    except Exception as e:  # the timing below is still valid; the line says what is missing
        return {"gpu": None, "card_query_error": repr(e)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--n", type=int, default=16384)
    ap.add_argument("--candidates", type=int, default=20000)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_eci needs a CUDA device"
    import __graft_entry__  # noqa: F401  (puts the repository on sys.path)
    from limbo_b200 import acqui, kernel, mean, model, synth

    info = card()
    D = 6
    s_obj, s_con = torch.cuda.Stream(), torch.cuda.Stream()

    def timed(fn):
        """ms of fn() between CUDA events on the objective's stream (constraint stream joined before the end event)."""
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s_obj)
        r = fn()
        s_obj.wait_stream(s_con)
        e1.record(s_obj)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), r

    def models(n, params=None):
        X = synth.points(1234, n, D)
        y = synth.targets(X)
        c = (X[:, 0] + X[:, 1] >= 0.9).astype(np.float64)
        gp = model.GP(D, 1, params=params, kernel=kernel.SquaredExpARD, mean=mean.Data)
        con = model.GP(D, 1, params=params, kernel=kernel.Exp, mean=mean.Constant)
        gp.set_stream(s_obj.cuda_stream)
        con.set_stream(s_con.cuda_stream)
        return X, y, c, gp, con

    # ---- headline leg ----
    N, M = args.n, args.candidates
    X, y, c, gp, con = models(N)
    Xq = synth.points(1235, M, D)
    Xq_ucb = Xq[:10000]
    eci = acqui.ECI(gp, con, 0)
    parts = {k: [] for k in ("fit_obj", "fit_con", "f_max", "eci", "query_obj", "query_con", "two_queries", "eci_step", "ucb_step")}
    best = None

    def eci_step():
        nonlocal best
        t = {}
        t["fit_obj"], _ = timed(lambda: gp.compute(X, y[:, None]))
        t["fit_con"], _ = timed(lambda: con.compute(X, c[:, None]))
        eci._nb_samples = -1
        t["f_max"], _ = timed(lambda: eci._update_f_max(acqui.first_elem))
        t["eci"], best = timed(lambda: eci.argmax_batch(Xq))
        t["query_obj"], _ = timed(lambda: gp.query_batch(Xq))
        t["query_con"], _ = timed(lambda: con.query_batch(Xq))
        t["two_queries"] = t["query_obj"] + t["query_con"]
        t["eci_step"] = t["fit_obj"] + t["fit_con"] + t["f_max"] + t["eci"]
        return t

    def ucb_step():
        return timed(lambda: (gp.compute(X, y[:, None]), acqui.UCB(gp).argmax_batch(Xq_ucb)))[0]

    ucb_step()  # warm-up of every shape
    eci_step()
    for _ in range(args.steps):  # alternated in one process
        parts["ucb_step"].append(ucb_step())
        for k, v in eci_step().items():
            parts[k].append(v)
    med = {k: float(np.median(v)) for k, v in parts.items()}
    rng = {k: [float(min(v)), float(max(v))] for k, v in parts.items()}

    # ---- small-N leg: one point at a time (eci.hpp's contract) against one batched call ----
    n_s, m_s = 1024, 2000
    Xs, ys, cs, gps, cons = models(n_s)
    gps.compute(Xs, ys[:, None])
    cons.compute(Xs, cs[:, None])
    Xqs = synth.points(1236, m_s, D)
    a = acqui.ECI(gps, cons, 0)
    a(Xqs[0])  # f_max and warm-up
    a.argmax_batch(Xqs)
    t0 = time.perf_counter()
    vals = np.array([a(x)[0] for x in Xqs])  # (value, no gradient), optimizer.hpp:66-69
    one_ms = (time.perf_counter() - t0) * 1e3
    t_b = []
    for _ in range(5):
        t0 = time.perf_counter()
        b_best, b_idx, b_vals = a.argmax_batch(Xqs, return_values=True)
        t_b.append((time.perf_counter() - t0) * 1e3)
    batched_ms = float(np.median(t_b))

    out = dict(info)
    out.update({
        "tool": "bench_eci", "workload": f"N={N}, D={D}, SE-ARD objective (Hartmann6) + Exp constraint (0/1 column), {M} ECI candidates",
        "steps": args.steps, "ms_median": {k: round(v, 3) for k, v in med.items()}, "ms_range": {k: [round(x, 3) for x in v] for k, v in rng.items()},
        "eci_over_two_queries": round(med["eci"] / med["two_queries"], 3),
        "f_max_share_of_eci_step": round(med["f_max"] / med["eci_step"], 3),
        "eci_step_over_ucb_step": round(med["eci_step"] / med["ucb_step"], 3),
        "eci_best": [float(best[0]), int(best[1])],
        "small_n": {"N": n_s, "candidates": m_s, "one_point_ms": round(one_ms, 2), "batched_ms": round(batched_ms, 3),
                    "speedup": round(one_ms / batched_ms, 1), "same_argmax": int(np.argmax(vals)) == int(b_idx),
                    "max_abs_diff": float(np.abs(vals - b_vals).max())},
    })
    print(json.dumps(out))


if __name__ == "__main__":
    main()
