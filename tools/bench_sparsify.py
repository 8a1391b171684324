"""Device-event times of the sparsified model (model::SparsifiedGP, limbo_b200/csrc/sparsify.cu).

    python tools/bench_sparsify.py --out DIR          (on the GPU) N = 65536, D = 6 synth points -> 16384: k-NN init, greedy loop
                                                      (total and per removal), the following fit; the steady-state
                                                      SparsifiedGP.add_sample at max_points = 16384 next to GP.add_sample.
                                                      Writes DIR/bench_sparsify.json and DIR/sparsify_kept.npz.
    python tools/bench_sparsify.py --check DIR        (CPU) the saved kept set and removal order against oracle/sparsify.py.
    python tools/bench_sparsify.py --ref              (CPU) the reference's own _sparsify (oracle/_ref/libref_sparse.so) at
                                                      N = 1024 and 2048, extrapolated to N = 65536 -> 16384 with the sum-of-n^2 law.
"""
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

N, D, MAXP = 65536, 6, 16384


def _card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip()


def gpu(out: str) -> None:
    import torch
    from limbo_b200 import _lib, model, synth
    lib = _lib.load()
    X = np.ascontiguousarray(synth.points(4242, N, D))
    y = synth.targets(X)[:, None]
    gp = model.GP(D, 1)
    lib.lb_debug_sparsify_timing(1)
    kept = np.empty(N, dtype=np.int64)
    removed = np.empty(N, dtype=np.int64)
    score = np.empty(N)
    nk = C.c_int64()
    ms = np.zeros(2)
    runs = []
    for rep in range(3):  # the first call also loads the module
        t0 = time.perf_counter()
        _lib.check(lib.lb_sparsify(gp._h, N, D, X.ctypes.data, MAXP, kept.ctypes.data, C.addressof(nk), removed.ctypes.data,
                                   score.ctypes.data), "lb_sparsify")
        wall = time.perf_counter() - t0
        lib.lb_debug_sparsify_last_ms(ms.ctypes.data)
        runs.append({"init_ms": ms[0], "loop_ms": ms[1], "call_wall_ms": wall * 1e3})
    lib.lb_debug_sparsify_timing(0)
    nrem = N - nk.value
    np.savez_compressed(os.path.join(out, "sparsify_kept.npz"), seed=4242, kept=kept[:nk.value], removed=removed[:nrem],
                        removed_score=score[:nrem])
    # the following fit on the kept rows (device events around lb_fit)
    kx, ky = X[kept[:nk.value]], y[kept[:nk.value]]
    fit = model.GP(D, 1)
    fit_ms = []
    for rep in range(3):
        fit.compute(kx, ky, False)
        fit._push_data()
        fit._push_kernel()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        _lib.check(lib.lb_fit(fit._h), "lb_fit")
        b.record()
        torch.cuda.synchronize()
        fit_ms.append(a.elapsed_time(b))
    # steady state of add_sample at max_points: SparsifiedGP re-sparsifies max_points + 1 samples and refits; GP appends
    class P:
        class model_sparse_gp:
            max_points = MAXP
    extra = synth.points(4343, 8, D)
    sgp = model.SparsifiedGP(D, 1, params=P)
    sgp.compute(kx, ky)
    pgp = model.GP(D, 1)
    pgp.compute(kx, ky)
    s_ms, g_ms = [], []
    for i in range(4):
        for m, acc in ((sgp, s_ms), (pgp, g_ms)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            m.add_sample(extra[i], [float(synth.targets(extra[i:i + 1])[0])])
            torch.cuda.synchronize()
            acc.append((time.perf_counter() - t0) * 1e3)
    res = {
        "card": _card(),
        "N": N, "D": D, "max_points": MAXP, "removals": int(nrem),
        "sparsify_runs": runs,
        "init_ms_median": float(np.median([r["init_ms"] for r in runs[1:]])),
        "loop_ms_median": float(np.median([r["loop_ms"] for r in runs[1:]])),
        "loop_us_per_removal": float(np.median([r["loop_ms"] for r in runs[1:]]) * 1e3 / max(nrem, 1)),
        "fit_ms": fit_ms,
        "sparsified_add_sample_ms": s_ms, "gp_add_sample_ms": g_ms,
        "sgp_nb_samples": sgp.nb_samples(), "gp_nb_samples": pgp.nb_samples(),
    }
    with open(os.path.join(out, "bench_sparsify.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res))


def check(out: str) -> None:
    from limbo_b200 import synth
    from oracle import sparsify as O
    g = np.load(os.path.join(out, "sparsify_kept.npz"))
    X = np.ascontiguousarray(synth.points(int(g["seed"]), N, D))
    t0 = time.perf_counter()
    kept, removed, score = O.sparsify(X, MAXP)
    print(json.dumps({"kept_equal": bool(np.array_equal(kept, g["kept"])), "order_equal": bool(np.array_equal(removed, g["removed"])),
                      "scores_bit_equal": bool(np.array_equal(score.view(np.uint64), g["removed_score"].view(np.uint64))),
                      "oracle_s": time.perf_counter() - t0}))


def ref() -> None:
    from limbo_b200 import synth
    from oracle import ref_sparse
    lib = ref_sparse.load()
    lib.ref_sparsify_only.argtypes = [C.c_long, C.c_int, C.c_void_p, C.c_long]
    lib.ref_sparsify_only.restype = C.c_long
    out = {}
    for n in (1024, 2048):
        X = np.ascontiguousarray(synth.points(4242, n, D))
        t0 = time.perf_counter()
        lib.ref_sparsify_only(n, D, X.ctypes.data, n // 4)
        out[n] = time.perf_counter() - t0
    # the removal loop costs ~ sum of n^2 over the remaining sizes n (one N x N scan of sorted rows and matrix moves per removal)
    def law(n0):
        m = np.arange(n0 // 4 + 1, n0 + 1, dtype=np.float64)
        return float((m ** 2).sum())
    c = out[2048] / law(2048)
    print(json.dumps({"ref_s": out, "ratio_2048_over_1024": out[2048] / out[1024], "law_ratio": law(2048) / law(1024),
                      "extrapolated_65536_to_16384_s": c * law(N), "note": "extrapolation, not a measurement"}))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--check")
    ap.add_argument("--ref", action="store_true")
    a = ap.parse_args()
    if a.check:
        check(a.check)
    elif a.ref:
        ref()
    else:
        if not a.out:
            ap.error("--out DIR, --check DIR or --ref")
        os.makedirs(a.out, exist_ok=True)
        gpu(a.out)
