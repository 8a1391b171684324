"""CPU-side checks of the batched hyper-parameter fit: opt.BatchedRprop / opt.BatchedParallelRepeater run every lane exactly as
opt.Rprop / opt.ParallelRepeater run that start (the same points evaluated in the same order, the same returned vector, bit for
bit) over NumPy objectives, and the batched likelihood kernel has no stack frame.  No GPU is needed."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from limbo_b200 import opt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "limbo_b200", "lib", "liblimbo_b200.so")


def _params(iterations, eps_stop=0.0, repeats=10, epsilon=1e-2):
    class Prm:
        class opt_rprop:
            pass

        class opt_parallelrepeater:
            pass
    Prm.opt_rprop.iterations, Prm.opt_rprop.eps_stop = iterations, eps_stop
    Prm.opt_parallelrepeater.repeats, Prm.opt_parallelrepeater.epsilon = repeats, epsilon
    return Prm


class Recorder:
    """f(x, grad) that logs every point it is asked for; the batched optimisers see it without a batch method."""

    def __init__(self, fn):
        self.fn, self.log = fn, []

    def __call__(self, x, compute_grad):
        self.log.append(np.array(x, copy=True))
        v, g = self.fn(np.asarray(x))
        return (v, g) if compute_grad else (v, None)


class BatchRecorder:
    """The same objective with a batch method, logging the rows of every call."""

    def __init__(self, fn):
        self.fn, self.calls = fn, []

    def batch(self, X, compute_grad):
        self.calls.append(np.array(X, copy=True))
        vals, grads = zip(*(self.fn(x) for x in X))
        return np.array(vals), (np.stack(grads) if compute_grad else None)


def _quadratic_with_holes(x):
    """A concave quadratic that is NaN on a band of its first coordinate (an objective the optimiser must step through)."""
    c = np.linspace(0.3, -0.2, x.size)
    v = -float(np.sum((x - c) ** 2))
    g = -2.0 * (x - c)
    if 0.05 < x[0] < 0.12:
        return float("nan"), np.full(x.size, np.nan)
    return v, g


def _oracle_objective(kernel_id, n, d, hp_size):
    O = pytest.importorskip("oracle.oracle")
    rng = np.random.default_rng(11)
    X = rng.random((n, d))
    y = np.sin(3 * X).sum(axis=1)[:, None]
    og = O.OracleGP()
    og.set_data(X, y - y.mean())
    og.set_kernel(kernel_id, np.zeros(hp_size), 0.01)
    og.fit()
    return lambda x: og.lml_eval(x, True)


def _objectives():
    yield "quadratic", _quadratic_with_holes, 3
    yield "oracle_se_ard", _oracle_objective(0, 30, 2, 3), 3
    yield "oracle_matern52", _oracle_objective(1, 25, 3, 2), 2


@pytest.mark.parametrize("bounded", [False, True])
@pytest.mark.parametrize("eps_stop", [0.0, 0.5])
def test_batched_rprop_lanes_replay_rprop(bounded, eps_stop):
    for name, fn, n in _objectives():
        P = _params(25, eps_stop)
        starts = np.random.default_rng(5).random((4, n)) * 0.4 - 0.1
        got = opt.BatchedRprop(P)(BatchRecorder(fn), starts, bounded)
        rows = Recorder(fn)
        got_rows = opt.BatchedRprop(P)(rows, starts, bounded)  # no batch method: row-by-row evaluation
        assert np.array_equal(got_rows, got, equal_nan=True)
        seqs = _split_lanes(rows.log, starts, fn, P, bounded)
        for r in range(4):
            rec = Recorder(fn)
            want = opt.Rprop(P)(rec, starts[r], bounded)
            assert np.array_equal(got[r], want, equal_nan=True), (name, r)
            assert len(seqs[r]) == len(rec.log), (name, r)
            for a, b in zip(seqs[r], rec.log):
                assert np.array_equal(a, b, equal_nan=True), (name, r)


def _split_lanes(log, starts, fn, P, bounded):
    """The row-by-row log of a BatchedRprop run, split into lanes: each iteration evaluates the running lanes in lane order,
    and a lane stops when Rprop would (replayed here from each lane's own Rprop run)."""
    lengths = []
    for r in range(starts.shape[0]):
        rec = Recorder(fn)
        opt.Rprop(P)(rec, starts[r], bounded)
        lengths.append(len(rec.log))
    seqs = [[] for _ in lengths]
    pos = 0
    for it in range(max(lengths)):
        for r, ln in enumerate(lengths):
            if it < ln:
                seqs[r].append(log[pos])
                pos += 1
    assert pos == len(log)
    return seqs


def test_eps_stop_stops_lanes_early():
    P = _params(300, eps_stop=0.6)
    starts = np.random.default_rng(2).random((3, 3))
    batch = BatchRecorder(lambda x: (-float(np.sum((x - 0.3) ** 2)), -2.0 * (x - 0.3)))
    opt.BatchedRprop(P)(batch, starts, False)
    sizes = [X.shape[0] for X in batch.calls]
    assert sizes[0] == 3 and len(sizes) < 300  # every lane came close enough to the maximum and left
    assert sizes == sorted(sizes, reverse=True)


@pytest.mark.parametrize("bounded", [False, True])
def test_batched_parallel_repeater_matches_parallel_repeater(bounded):
    for name, fn, n in _objectives():
        P = _params(20, repeats=6, epsilon=0.3)
        init = np.full(n, 0.1)
        want = opt.ParallelRepeater(P, opt.Rprop(P), rng=np.random.default_rng(123))(Recorder(fn), init, bounded)
        got = opt.BatchedParallelRepeater(P, rng=np.random.default_rng(123))(BatchRecorder(fn), init, bounded)
        got_rows = opt.BatchedParallelRepeater(P, rng=np.random.default_rng(123))(Recorder(fn), init, bounded)
        assert np.array_equal(got, want, equal_nan=True), name
        assert np.array_equal(got_rows, want, equal_nan=True), name


def test_batched_parallel_repeater_keeps_init_when_nothing_is_finite():
    P = _params(5, repeats=3)
    nan = lambda x: (float("nan"), np.full(x.size, np.nan))  # noqa: E731
    init = np.array([0.2, -0.4])
    got = opt.BatchedParallelRepeater(P, rng=np.random.default_rng(0))(BatchRecorder(nan), init, False)
    want = opt.ParallelRepeater(P, opt.Rprop(P), rng=np.random.default_rng(0))(Recorder(nan), init, False)
    assert np.array_equal(got, want) and np.array_equal(got, init)


def test_lml_batch_kernel_has_no_stack():
    tool = None
    for cand in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"), shutil.which("cuobjdump")):
        if cand and os.path.exists(cand):
            tool = cand
            break
    if tool is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    r = subprocess.run([tool, "-res-usage", LIB], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    found = re.findall(r"^\s*Function (\S*lml_batch_kernel\S*):\s*\n\s*(REG:.*)$", r.stdout, flags=re.M)
    assert len(found) == 4, found  # one instantiation per kernel functor
    for name, usage in found:
        res = dict(kv.split(":", 1) for kv in usage.split())
        assert int(res["STACK"]) == 0 and int(res["LOCAL"]) == 0, f"{name}: {res}"


GOLDEN = sorted(__import__("glob").glob(os.path.join(ROOT, "tests", "golden", "lml_batch", "*.npz")))


def test_lml_batch_fixtures_present():
    assert len(GOLDEN) >= 13


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_oracle_matches_lml_batch_fixtures(path):
    """The oracle's restatement reproduces the reference's own likelihood and gradient at every row of every fixture (the
    tolerances of test_golden.py)."""
    O = pytest.importorskip("oracle.oracle")
    g = np.load(path)
    on = bool(g["optimize_noise"])
    H = g["H"]
    nk = H.shape[1] - (1 if on else 0)
    og = O.OracleGP()
    og.set_data(g["X"], g["Y"] - g["Y"].mean(axis=0))
    for r in range(H.shape[0]):
        noise = float(np.exp(2.0 * H[r, nk])) if on else float(g["noise"])  # kernel.hpp:116-123
        og.set_kernel(int(g["kernel_id"]) % 4, H[r, :nk], noise)  # fixture id 4 = SE-ARD with k = 2
        og.fit()
        v, gr = og.log_lik(), og.grad(on)
        assert abs(v - g["lik"][r]) <= 1e-11 * max(1.0, abs(g["lik"][r])), (r, v, g["lik"][r])
        assert np.abs(gr - g["grad"][r]).max() <= 1e-9 * max(1.0, np.abs(g["grad"][r]).max()), r
