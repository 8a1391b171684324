"""Small-N hyper-parameter fits on one GPU: lb_lml_grad_batch against the evaluations it replaces.

For N = 50, 100, 200, 400, 800, 1024 training points (synth targets), D = 6, SE-ARD and Matern-5/2, mean::Data:
  batch_dev_ms[R]   one lb_lml_grad_batch call of R vectors (likelihood and gradient): CUDA events on the handle's stream around
                    the call (upload of the R vectors, the launch, the read-back); median of --steps after a warm-up call
  batch_host_ms[R]  the same call on a host clock (it returns after a stream synchronise)
  seq_ms[R]         the same R evaluations through _KernelLFOptimization(gp)(x, True) (GP copy, lb_set_kernel, lb_fit, lb_log_lik,
                    lb_kernel_grad_log_lik), host clock ending in a synchronise; median of --steps
  max_rel_lik[R], max_rel_grad[R]   largest deviation of the batched results from the sequential ones (grad: over max(1, |g|inf))
  fit_seq_s, fit_batch_s   a whole KernelLFOpt (10 restarts x 300 Rprop iterations) with ParallelRepeater(Rprop) and with
                    BatchedParallelRepeater, same seed; fit_dh = largest h-param difference of the two results
for R = 1, 10, 32, 132.  The library must accept every N measured (LB_LML_BATCH_MAX_N at least the largest).

Prints one JSON line with the card's name, power limit and max SM clock read in the same run.
    python tools/bench_lml_batch.py [--steps 5] [--ns 50,100,200] [--no-fit] [--out FILE]"""
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

NS = (50, 100, 200, 400, 800, 1024)
RS = (1, 10, 32, 132)


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": out[0], "power_limit_w": float(out[1]), "sm_clock_max_mhz": float(out[2])}
    except Exception as e:
        return {"gpu": None, "card_query_error": repr(e)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--ns", default=",".join(map(str, NS)))
    ap.add_argument("--no-fit", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from limbo_b200 import _lib, kernel, mean, model, opt, synth
    assert torch.cuda.is_available(), "bench_lml_batch needs a GPU"
    st = torch.cuda.Stream()
    rec = {"tool": "bench_lml_batch", "D": 6, "max_n_lib": _lib.LML_BATCH_MAX_N, **card(), "rows": []}
    for n in [int(s) for s in a.ns.split(",")]:
        for kname, kcls in (("se_ard", kernel.SquaredExpARD), ("matern52", kernel.MaternFiveHalves)):
            X = synth.points(1, n, 6)
            y = synth.targets(X)[:, None]
            gp = model.GP(6, 1, kernel=kcls, mean=mean.Data)
            gp.compute(X, y)
            gp.set_stream(st.cuda_stream)
            f = model.hp_opt._KernelLFOptimization(gp)
            row = {"N": n, "kernel": kname}
            rng = np.random.default_rng(n)
            for R in RS:
                H = np.tile(gp.kernel_function().h_params(), (R, 1)) + rng.uniform(-0.5, 0.5, (R, gp.kernel_function().h_params_size()))
                gp.lml_grad_batch(H)  # warm-up
                dev, host = [], []
                for _ in range(a.steps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(st)
                    t0 = time.perf_counter()
                    lik, grad, _ = gp.lml_grad_batch(H)
                    host.append((time.perf_counter() - t0) * 1e3)
                    e1.record(st)
                    e1.synchronize()
                    dev.append(e0.elapsed_time(e1))
                f(H[0], True)  # warm-up
                seq = []
                for _ in range(a.steps):
                    t0 = time.perf_counter()
                    outs = [f(H[r], True) for r in range(R)]
                    torch.cuda.synchronize()
                    seq.append((time.perf_counter() - t0) * 1e3)
                sl = np.array([o[0] for o in outs])
                sg = np.stack([o[1] for o in outs])
                row[f"batch_dev_ms[{R}]"] = float(np.median(dev))
                row[f"batch_host_ms[{R}]"] = float(np.median(host))
                row[f"seq_ms[{R}]"] = float(np.median(seq))
                row[f"max_rel_lik[{R}]"] = float(np.max(np.abs(lik - sl) / np.maximum(1.0, np.abs(sl))))
                row[f"max_rel_grad[{R}]"] = float(max(np.abs(grad[r] - sg[r]).max() / max(1.0, np.abs(sg[r]).max()) for r in range(R)))
            if not a.no_fit:
                res = []
                for batched in (False, True):
                    g2 = model.GP(6, 1, kernel=kcls, mean=mean.Data)
                    g2.compute(X, y)
                    rep = opt.BatchedParallelRepeater(None, rng=np.random.default_rng(0)) if batched else \
                        opt.ParallelRepeater(None, opt.Rprop(None), rng=np.random.default_rng(0))
                    t0 = time.perf_counter()
                    model.KernelLFOpt(None, rep)(g2)
                    torch.cuda.synchronize()
                    res.append((time.perf_counter() - t0, g2.kernel_function().h_params(), g2.get_log_lik()))
                row["fit_seq_s"], row["fit_batch_s"] = res[0][0], res[1][0]
                row["fit_dh"] = float(np.abs(res[0][1] - res[1][1]).max())
                row["fit_lik"] = [res[0][2], res[1][2]]
            rec["rows"].append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
