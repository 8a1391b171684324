"""Timing of the SPGP candidate gradients (lb_spgp_acq_grad, limbo_b200/csrc/spgp.cu) next to the acquisition argmax over the
same model (lb_spgp_acq_argmax).

  python tools/bench_spgp_grad.py [--out DIR] [--N 16384] [--M 1638] [--D 6] [--mq 32,20000] [--reps 7]

For each batch size Mq: ms per synchronising call of lb_spgp_acq_argmax and of lb_spgp_acq_grad (UCB), the median of --reps
calls after warm-up; then, in a separate profiled run of each call, a per-kernel breakdown from torch.profiler with the achieved
TFLOP/s of the four triangular products (L^-1 K*, Lm^-1 ., Lm^-T ., L^-T ., each Mp^2 nqp flops per chunk from the shapes).  Last,
one bayes_opt.BatchedGradientSearch step and one BatchedRandomSearch step over acqui.UCB on the model, with their times and the
acquisition value each reaches.  Prints one JSON line (also DIR/bench_spgp_grad.json) with the card name and power limit read in
the same run."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

QCHUNK = 8192


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def tri_flops(M, Mq):
    """flops of the triangular products per call: per chunk of nqp (padded) candidates, an upper or lower Mp x Mp factor
    against Mp x nqp streams about Mp^2 nqp multiply-adds (half the full 2 Mp^2 nqp)"""
    Mp = -(-M // 128) * 128
    total = 0.0
    for q0 in range(0, Mq, QCHUNK):
        nqp = -(-min(QCHUNK, Mq - q0) // 128) * 128
        total += float(Mp) * Mp * nqp
    return total  # per product


def profile_call(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    classes = {}
    for ev in prof.key_averages():
        cls = "other"
        for key in ("spgp_gemm", "spgp_query_grad", "spgp_resid", "spgp_kmat", "spgp_stage", "spgp_coldot", "spgp_pred", "acq_kernel",
                    "argmax_final", "Memcpy"):
            if key in ev.key:
                cls = key
                break
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        classes[cls] = classes.get(cls, 0.0) + t / 1e3  # ms
    return classes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--N", type=int, default=16384)
    ap.add_argument("--M", type=int, default=1638)
    ap.add_argument("--D", type=int, default=6)
    ap.add_argument("--mq", default="32,20000")
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    import torch  # noqa: F401  (CUDA context for the profiler)
    from limbo_b200 import _lib, acqui, bayes_opt, model, synth
    from oracle import spgp as O

    lib = _lib.load()
    rec = {"card": card(), "N": args.N, "M": args.M, "D": args.D, "calls": []}
    N, M, D = args.N, args.M, args.D
    X = synth.points(7, N, D)
    y = synth.targets(X)
    y = y - y.mean()
    w = O.init_w(X, y, M, np.random.default_rng(0).permutation(N)) + np.random.default_rng(1).normal(0, 0.05, (M + 1) * D + 2)
    h = C.c_void_p()
    assert lib.lb_spgp_create(C.byref(h), 0) == 0
    assert lib.lb_spgp_set_data(h, N, D, X.ctypes.data, y.ctypes.data) == 0
    assert lib.lb_spgp_compute(h, M, w.size, w.ctypes.data, 1e-6) == 0
    params = np.array([0.5, 0.0])
    best, idx = C.c_double(), C.c_int64()
    for Mq in (int(v) for v in args.mq.split(",")):
        Xq = np.ascontiguousarray(synth.points(8, Mq, D))
        vals, grads = np.empty(Mq), np.empty((Mq, D))

        def argmax():
            assert lib.lb_spgp_acq_argmax(h, 0, params.ctypes.data, Mq, Xq.ctypes.data, 1, None, 0.0, vals.ctypes.data,
                                          C.addressof(best), C.addressof(idx)) == 0

        def grad():
            assert lib.lb_spgp_acq_grad(h, 0, params.ctypes.data, Mq, Xq.ctypes.data, 1, None, 0.0, None, vals.ctypes.data,
                                        grads.ctypes.data) == 0
        times = {}
        for name, fn in (("argmax", argmax), ("grad", grad)):
            for _ in range(3):
                fn()
            ts = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                fn()
                ts.append(time.perf_counter() - t0)
            times[name] = 1e3 * float(np.median(ts))
        prof = {name: profile_call(fn) for name, fn in (("argmax", argmax), ("grad", grad))}
        f1 = tri_flops(M, Mq)
        gemm_ms = prof["grad"].get("spgp_gemm", float("nan"))
        entry = {"Mq": Mq, "acq_argmax_ms": times["argmax"], "acq_grad_ms": times["grad"], "grad_over_argmax": times["grad"] / times["argmax"],
                 "kernels_argmax_ms": prof["argmax"], "kernels_grad_ms": prof["grad"],
                 "tri_products_tflops": 4.0 * f1 / (gemm_ms * 1e-3) / 1e12 if gemm_ms == gemm_ms else None}
        rec["calls"].append(entry)
        print(json.dumps(entry), file=sys.stderr)
    lib.lb_spgp_destroy(h)

    # one search step of each policy over acqui.UCB on an SPGP at the same (N, M, D) and w
    class P:
        class acqui_ucb:
            alpha = 0.5

        class opt_batchedgradient:
            candidates = 20000
            starts = 32
            iterations = 30
            alpha = 0.01

        class opt_batchedrandom:
            candidates = 20000
            refinements = 2
            shrink = 0.1
    m = model.SPGP(params=P, rng=np.random.default_rng(0))
    m._set(X, (y + 1.0)[:, None])
    m._m = M
    m.compute_at(w)
    m._optimized = True
    acq = acqui.UCB(m, 0, params=P)
    steps = {}
    for name, pol in (("BatchedGradientSearch", bayes_opt.BatchedGradientSearch), ("BatchedRandomSearch", bayes_opt.BatchedRandomSearch)):
        pol(P, np.random.default_rng(1))(acq, D, True)  # warm-up
        t0 = time.perf_counter()
        x = pol(P, np.random.default_rng(2))(acq, D, True)
        dt = time.perf_counter() - t0
        steps[name] = {"ms": 1e3 * dt, "value": float(acq.grad_batch(x[None, :])[0][0])}
    rec["search_step"] = steps
    rec["card_after"] = card()
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_spgp_grad.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
