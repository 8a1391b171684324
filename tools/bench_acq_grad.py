"""Candidate gradients on one GPU: what lb_acq_grad costs next to lb_acq_argmax, and what the gradient acquisition optimiser buys.

For N = 16384 training points (SE-ARD, mean::Data, Hartmann6-style targets from synth), D = 6 and D = 12:
  argmax_ms[M] / grad_ms[M]   lb_acq_argmax (UCB) and lb_acq_grad (UCB) over M = 256, 1024, 4096 candidates; host clock around the
                              call, which returns after a stream synchronise; median of --steps after a warm-up call
  ratio[M]                    grad_ms / argmax_ms
  bwd_ms[M], bwd_tflops[M]    the backward solve W = L^-T V (panel_bwd_update_kernel + panel_bwd_solve_kernel), device time summed
                              from torch.profiler (CUDA activity) in a separate pass; M N^2 flops
  fwd_ms[M], fwd_tflops[M]    the forward panel solve (panel_update_kernel + panel_solve_kernel) in the same pass, same flop count
  gradpass_ms[M]              query_grad_kernel in the same pass
  policy                      BatchedRandomSearch (its defaults) and BatchedGradientSearch (its defaults) with the same seed, on UCB
                              and EI: whole-policy wall time and the acquisition value of the returned point, median of three runs,
                              the two policies alternated

Prints one JSON line with the card's name, power limit and max SM clock read in the same run.
    python tools/bench_acq_grad.py [--steps 5] [--out FILE]"""
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

MS = (256, 1024, 4096)


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": out[0], "power_limit_w": float(out[1]), "sm_clock_max_mhz": float(out[2])}
    except Exception as e:
        return {"gpu": None, "card_query_error": repr(e)}


def timed(fn, steps):
    fn()
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def profile_kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    tot = {"bwd": 0.0, "fwd": 0.0, "gradpass": 0.0}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        ms = e.device_time / 1e3 if hasattr(e, "device_time") else e.cuda_time / 1e3
        if "panel_bwd_" in e.name:
            tot["bwd"] += ms
        elif "panel_update_kernel" in e.name or "panel_solve_kernel" in e.name:
            tot["fwd"] += ms
        elif "query_grad_kernel" in e.name:
            tot["gradpass"] += ms
    return tot


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--n", type=int, default=16384)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_acq_grad needs a CUDA device"
    from limbo_b200 import acqui, bayes_opt, kernel, mean, model, synth

    res = {"bench": "acq_grad", "n": args.n, **card()}
    for D in (6, 12):
        rng = np.random.default_rng(D)
        X = rng.random((args.n, D))
        gp = model.GP(D, 1, kernel=kernel.SquaredExpARD, mean=mean.Data)
        gp.compute(X, synth.targets(X)[:, None])
        r = {}
        for M in MS:
            Xq = rng.random((M, D))
            a = timed(lambda: gp.acq_argmax_batch(0, [0.5], Xq), args.steps)
            g = timed(lambda: gp.acq_grad_batch(0, [0.5], Xq), args.steps)
            k = profile_kernels(lambda: gp.acq_grad_batch(0, [0.5], Xq))
            fl = float(M) * args.n ** 2
            r[str(M)] = {"argmax_ms": a, "grad_ms": g, "ratio": g / a, "bwd_ms": k["bwd"], "bwd_tflops": fl / (k["bwd"] * 1e9),
                         "fwd_ms": k["fwd"], "fwd_tflops": fl / (k["fwd"] * 1e9), "gradpass_ms": k["gradpass"]}
        pol = {}
        for name in ("UCB", "EI"):
            acq = getattr(acqui, name)(gp, 0)
            runs = {"random": [], "gradient": []}
            for rep in range(3):
                for label, cls in (("random", bayes_opt.BatchedRandomSearch), ("gradient", bayes_opt.BatchedGradientSearch)):
                    opt = cls(None, np.random.default_rng(100 + rep))
                    t0 = time.perf_counter()
                    x = opt(acq, D, True)
                    t = (time.perf_counter() - t0) * 1e3
                    v = float(acq.grad_batch(np.atleast_2d(x))[0][0])
                    runs[label].append((t, v))
            pol[name] = {lab: {"wall_ms": float(np.median([t for t, _ in rr])), "value": float(np.median([v for _, v in rr]))}
                         for lab, rr in runs.items()}
        res[f"D{D}"] = {"calls": r, "policy": pol}
        del gp
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
