"""Timing of the pseudo-input sparse GP on the device (lb_spgp_*, limbo_b200/csrc/spgp.cu).

  python tools/bench_spgp.py [--out DIR] [--sizes 16384:1638,65536:6553] [--D 6] [--reps 3]

For each (N, M): one likelihood + gradient evaluation, the value alone, one _compute + a 10^4-candidate prediction, and a
per-kernel-class breakdown of one gradient evaluation from torch.profiler, with achieved TFLOP/s of the DMMA products from flop
counts derived from the shapes.  Then one whole SPGP.compute (Rprop at the default 300 iterations) at the first size, and the
reference's own SPGP (the Eigen stand-in build, one CPU core; evaluation + _compute) at N = 1024 and 2048 where it is built.  Prints
one JSON line (also written to DIR/bench_spgp.json) with the card name and power limit read in the same run."""
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


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


class Raw:
    """lb_spgp handle over the raw ABI (the calls timed here)."""

    def __init__(self):
        import ctypes as C
        from limbo_b200 import _lib
        self.C, self.lib, self.h = C, _lib.load(), C.c_void_p()
        assert self.lib.lb_spgp_create(C.byref(self.h), 0) == 0

    def __del__(self):
        self.lib.lb_spgp_destroy(self.h)

    def set_data(self, X, y):
        X, y = np.ascontiguousarray(X, dtype=np.float64), np.ascontiguousarray(y, dtype=np.float64)
        return self.lib.lb_spgp_set_data(self.h, X.shape[0], X.shape[1], X.ctypes.data, y.ctypes.data)

    def lik(self, M, w, grad=True, jitter=1e-6):
        f = self.C.c_double()
        g = np.empty(w.size) if grad else None
        rc = self.lib.lb_spgp_lik(self.h, M, w.size, w.ctypes.data, jitter, self.C.addressof(f), g.ctypes.data if grad else None)
        return rc, f.value, g

    def compute(self, M, w, jitter=1e-6):
        return self.lib.lb_spgp_compute(self.h, M, w.size, w.ctypes.data, jitter)

    def query(self, Xq):
        Xq = np.ascontiguousarray(Xq, dtype=np.float64)
        mu, s2 = np.empty(len(Xq)), np.empty(len(Xq))
        return self.lib.lb_spgp_query(self.h, len(Xq), Xq.ctypes.data, 1, mu.ctypes.data, s2.ctypes.data), mu, s2


def gemm_flops(N, M):
    # DMMA products of one gradient evaluation: five triangular M x M by M x N products (V, Lm^-1 V~, Lm^-T ., L^-T ., L^-T V~)
    # at M^2 N each, two full M x N x M products (the SYRK of A and TT) at 2 M^2 N each, and Z, Z^T Z at about 2/3 M^3 each
    return 9.0 * M * M * N + 4.0 / 3.0 * M ** 3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--sizes", default="16384:1638,65536:6553")
    ap.add_argument("--D", type=int, default=6)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-compute", action="store_true", help="skip the whole SPGP.compute")
    args = ap.parse_args()
    import torch
    from limbo_b200 import model, synth
    from oracle import spgp as O

    rec = {"card": card(), "sizes": []}
    D = args.D
    for spec in args.sizes.split(","):
        N, M = (int(v) for v in spec.split(":"))
        X = synth.points(7, N, D)
        y = synth.targets(X)
        y = y - y.mean()
        w = O.init_w(X, y, M, np.random.default_rng(0).permutation(N)) + np.random.default_rng(1).normal(0, 0.05, (M + 1) * D + 2)
        s = Raw()
        assert s.set_data(X, y) == 0
        assert s.lik(M, w)[0] == 0  # warm-up: allocations, module load
        t_grad, t_val = [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            rc, f, g = s.lik(M, w)
            t_grad.append(time.perf_counter() - t0)
            assert rc == 0 and np.isfinite(f) and np.all(np.isfinite(g))
            t0 = time.perf_counter()
            s.lik(M, w, grad=False)
            t_val.append(time.perf_counter() - t0)
        Xq = synth.points(8, 10000, D)
        assert s.compute(M, w) == 0
        s.query(Xq)
        t_pred = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            assert s.compute(M, w) == 0
            rc, mu, s2 = s.query(Xq)
            t_pred.append(time.perf_counter() - t0)
        # per-kernel-class breakdown of one gradient evaluation
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            s.lik(M, w)
            torch.cuda.synchronize()
        classes = {}
        for ev in prof.key_averages():
            name = ev.key
            cls = "other"
            for key in ("spgp_gemm", "spgp_split_reduce", "spgp_pass", "spgp_kmat", "spgp_ep", "spgp_coldot", "spgp_rowdot", "potf2",
                        "trsm_panel", "syrk_kernel", "trtri", "lauum", "symmetrize"):
                if key in name:
                    cls = key
                    break
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            classes[cls] = classes.get(cls, 0.0) + t / 1e3  # ms
        gf = gemm_flops(N, M)
        size = {"N": N, "M": M, "D": D, "lik_grad_ms": 1e3 * float(np.median(t_grad)), "lik_value_ms": 1e3 * float(np.median(t_val)),
                "compute_plus_predict_1e4_ms": 1e3 * float(np.median(t_pred)), "kernel_class_ms": classes,
                "gemm_tflops": gf / (classes.get("spgp_gemm", float("nan")) * 1e-3) / 1e12 if classes.get("spgp_gemm") else None}
        rec["sizes"].append(size)
        print(json.dumps(size), file=sys.stderr)
        del s
    if not args.no_compute:
        N, M = (int(v) for v in args.sizes.split(",")[0].split(":"))
        X = synth.points(9, N, D)
        y = synth.targets(X)
        m = model.SPGP(rng=np.random.default_rng(0))
        t0 = time.perf_counter()
        m.compute(X, y[:, None])
        rec["spgp_compute_rprop300_s"] = {"N": N, "M": M, "D": D, "seconds": time.perf_counter() - t0}
    # the reference's own _likelihood(w, true) (oracle/_ref/libref_spgp.so: the Eigen stand-in, one core), where it was built
    from oracle import ref_spgp
    if os.path.exists(ref_spgp.LIB_PATH):
        rec["reference_stand_in_lik_grad_s"] = {}
        for N in (1024, 2048):
            M = O.n_pseudo(N)
            X = synth.points(7, N, D)
            y = synth.targets(X)
            w = O.init_w(X, y - y.mean(), M, np.random.default_rng(0).permutation(N)) + np.random.default_rng(1).normal(0, 0.05, (M + 1) * D + 2)
            t0 = time.perf_counter()
            ref_spgp.run(X, y, M, w, X[:1])  # one _likelihood(w, true) + one _compute(false) + a one-point _predict
            rec["reference_stand_in_lik_grad_s"][f"N={N},M={M}"] = time.perf_counter() - t0
    rec["card_after"] = card()
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_spgp.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
