"""The SPGP candidate gradients without a GPU: oracle/spgp_grad.py against central differences of the reference's own _predict
(oracle/ref_spgp.py, where it was built) and of oracle/spgp.py's State.predict, its UCB / EI gradients, and the new entry points
and kernels of the built library (exported, no stack frame)."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import acq_grad as AG
from oracle import spgp as O
from oracle import spgp_grad as SG

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "limbo_b200", "lib", "liblimbo_b200.so")
JITTER = 1e-6
H = 1e-6
REL = 1e-6

SHAPES = [(1, 1, 40), (10, 3, 120), (129, 6, 300), (10, 6, 200), (129, 1, 260)]


def _case(M, D, N, seed=0):
    rng = np.random.default_rng(seed + 17 * M + D)
    X = rng.random((N, D))
    y = np.sin(3.0 * X).sum(axis=1) + 0.05 * rng.normal(size=N)
    y = y - y.mean()
    w = O.init_w(X, y, M, rng.permutation(N))
    w[:M * D] += rng.normal(0.0, 0.02, M * D)
    w[M * D:(M + 1) * D] = np.log(rng.uniform(2.0, 8.0, D))
    w[(M + 1) * D] = np.log(0.8)
    w[(M + 1) * D + 1] = np.log(0.05)
    Xq = np.vstack([rng.random((12, D)), rng.random((3, D)) * 3.0 - 1.0])  # some candidates outside the data's box
    return X, y, w, Xq


def _central(predict, Xq):
    Mq, D = Xq.shape
    dmu, ds2 = np.zeros((Mq, D)), np.zeros((Mq, D))
    for d in range(D):
        e = np.zeros(D)
        e[d] = H
        mp, sp = predict(Xq + e)
        mm, sm = predict(Xq - e)
        dmu[:, d] = (mp - mm) / (2 * H)
        ds2[:, d] = (sp - sm) / (2 * H)
    return dmu, ds2


def _close(an, fd):
    scale = np.maximum(np.abs(an).max(axis=1, keepdims=True), 1e-3)
    assert np.all(np.abs(an - fd) <= REL * scale), np.abs(an - fd).max()


@pytest.mark.parametrize("optimized", [0, 1])
@pytest.mark.parametrize("M,D,N", SHAPES)
def test_oracle_matches_central_differences_of_its_prediction(M, D, N, optimized):
    X, y, w, Xq = _case(M, D, N)
    st = O.State(w, X, y, M, JITTER)
    mu, s2, dmu, ds2, mag = SG.query_grad(st, Xq, bool(optimized))
    mu_p, s2_p = st.predict(Xq, bool(optimized))
    assert np.allclose(mu, mu_p, rtol=0, atol=1e-12) and np.allclose(s2, s2_p, rtol=0, atol=1e-12)
    assert np.all(np.abs(dmu) <= mag) and np.all(np.abs(ds2) <= mag)
    fd_mu, fd_s2 = _central(lambda Z: st.predict(Z, bool(optimized)), Xq)
    _close(dmu, fd_mu)
    _close(ds2, fd_s2)
    f_max = float(mu.max()) - 0.05
    for name, fun, args in (("ucb", AG.ucb, (0.7,)), ("ei", AG.ei, (f_max, 0.01))):
        _, grad = fun(mu, s2, dmu, ds2, *args)
        fd = np.zeros_like(grad)
        for d in range(D):
            e = np.zeros(D)
            e[d] = H
            (mp, sp), (mm, sm) = st.predict(Xq + e, bool(optimized)), st.predict(Xq - e, bool(optimized))
            fd[:, d] = (fun(mp, sp, dmu, ds2, *args)[0] - fun(mm, sm, dmu, ds2, *args)[0]) / (2 * H)
        _close(grad, fd)


@pytest.mark.parametrize("M,D,N", SHAPES)
def test_oracle_matches_central_differences_of_the_reference(M, D, N):
    from oracle import ref_spgp
    if not ref_spgp.available():
        pytest.skip("the reference's SPGP is not built and its sources are not present")
    X, y, w, Xq = _case(M, D, N)
    st = O.State(w, X, y, M, JITTER)
    _, _, dmu, ds2, _ = SG.query_grad(st, Xq)

    def ref_predict(Z):
        r = ref_spgp.run(X, y, M, w, Z)
        return r["mu"], r["s2"]
    fd_mu, fd_s2 = _central(ref_predict, Xq)
    _close(dmu, fd_mu)
    _close(ds2, fd_s2)


def test_optimized_flag_moves_sigma2_only():
    X, y, w, Xq = _case(10, 3, 120)
    st = O.State(w, X, y, 10, JITTER)
    a = SG.query_grad(st, Xq, False)
    b = SG.query_grad(st, Xq, True)
    assert np.array_equal(a[0], b[0]) and np.allclose(b[1] - a[1], st.sig, rtol=0, atol=1e-15)
    assert all(np.array_equal(p, q) for p, q in zip(a[2:], b[2:]))


def test_entry_points_exported():
    from limbo_b200 import _lib
    lib = _lib.load()
    for name in ("lb_spgp_query_grad", "lb_spgp_acq_grad"):
        assert hasattr(lib, name) and name in _lib.DECLARED_SYMBOLS


def test_new_kernels_have_no_stack_frame():
    tool = next((c for c in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"), shutil.which("cuobjdump"))
                 if c and os.path.exists(c)), None)
    if tool is None:
        pytest.skip("cuobjdump not found")
    r = subprocess.run([tool, "-res-usage", LIB], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    found = dict(re.findall(r"^\s*Function (\S+):\s*\n\s*(REG:.*)$", r.stdout, flags=re.M))
    for kernel in ("spgp_query_grad_kernel", "spgp_resid_kernel"):
        hits = {n: u for n, u in found.items() if f"{len(kernel)}{kernel}" in n}
        assert len(hits) == 1, (kernel, sorted(hits))
        usage = dict(kv.split(":", 1) for kv in next(iter(hits.values())).split())
        assert int(usage["STACK"]) == 0 and int(usage["LOCAL"]) == 0 and int(usage["REG"]) <= 255, (kernel, usage)
