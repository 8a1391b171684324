"""The SPGP oracle (oracle/spgp.py) without a GPU: its gradient against central differences of its own value, the kept
integer-division quirk of the value, the parameter layout and initialisation, M's rounding, the regrouped gradient the device
computes (limbo_b200/csrc/spgp.cu) restated in NumPy, and the new kernels' resource table (no stack frame)."""
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import spgp as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "limbo_b200", "lib", "liblimbo_b200.so")
JITTER = 1e-6


def _case(seed, N, D, M=None):
    rng = np.random.default_rng(seed)
    X = rng.random((N, D))
    y = np.sin(3.0 * X).sum(axis=1)
    y = y - y.mean()
    M = O.n_pseudo(N) if M is None else M
    w = O.init_w(X, y, M, rng.permutation(N)) + rng.normal(0.0, 0.05, (M + 1) * D + 2)
    return X, y, M, w


@pytest.mark.parametrize("seed,N,D,M", [(0, 60, 3, 6), (1, 40, 2, 4), (2, 12, 1, 2)])
def test_oracle_gradient_matches_central_differences(seed, N, D, M):
    assert (N - M) % 2 == 0  # with odd N - M the value lacks 1/2 log sig, the gradient does not
    X, y, M, w = _case(seed, N, D, M)
    _, g = O.likelihood(w, X, y, M, JITTER)
    h = 1e-6
    fd = np.array([(O.likelihood(w + h * e, X, y, M, JITTER, grad=False)[0] - O.likelihood(w - h * e, X, y, M, JITTER, grad=False)[0])
                   / (2 * h) for e in np.eye(w.size)])
    assert np.abs(fd - g).max() <= 1e-6 * np.abs(g).max()


def test_odd_n_minus_m_lacks_half_log_sig():
    X, y, M, w = _case(3, 41, 2)
    assert (41 - M) % 2 == 1
    f, _ = O.likelihood(w, X, y, M, JITTER, grad=False)
    ff, _ = O.likelihood(w, X, y, M, JITTER, grad=False, fix_integer_division=True)
    sig = O.unpack(w, M, 2)[3]
    assert abs((f - ff) - 0.5 * math.log(sig)) <= 1e-12 * abs(f)
    Xe, ye, Me, we = _case(3, 40, 2)
    assert O.likelihood(we, Xe, ye, Me, JITTER, grad=False)[0] == O.likelihood(we, Xe, ye, Me, JITTER, grad=False,
                                                                              fix_integer_division=True)[0]


def test_w_layout_and_row_major_initialisation():
    rng = np.random.default_rng(4)
    X = rng.random((9, 3))
    y = rng.random(9)
    perm = rng.permutation(9)
    M = 2
    w = O.init_w(X, y, M, perm)
    assert w.size == O.n_params(M, 3) == 11
    # the first M*D entries are the chosen samples one after another (row-major) ...
    assert np.array_equal(w[:6], np.concatenate([X[perm[0]], X[perm[1]]]))
    xb, b, c, sig = O.unpack(w, M, 3)
    # ... read back column-major: xb(j, i) = w[i*M + j], so for D > 1 the pseudo-inputs mix coordinates of different samples
    for i in range(3):
        for j in range(M):
            assert xb[j, i] == w[i * M + j]
    assert not np.array_equal(xb[0], X[perm[0]])
    assert np.allclose(b, ((X.max(0) - X.min(0)) / 2.0) ** -2)
    assert c == pytest.approx(np.mean(y ** 2)) and sig == pytest.approx(np.mean(y ** 2) / 4)


@pytest.mark.parametrize("N,M", [(1, 1), (5, 1), (9, 1), (10, 1), (19, 1), (20, 2), (100, 10), (16384, 1638), (65536, 6553)])
def test_m_rounding(N, M):
    assert O.n_pseudo(N) == M


def test_regrouped_gradient_equals_oracle():
    """The device's regrouping of the D-loop (spgp.cu header) in NumPy, against the oracle's loop."""
    X, y, M, w = _case(0, 60, 3, 6)
    f, g = O.likelihood(w, X, y, M, JITTER)
    N, D = X.shape
    xb, b, c, sig = O.unpack(w, M, D)
    dl = JITTER
    bs = np.sqrt(b)
    xbt, xt = xb * bs, X * bs
    Q = c * np.exp(-0.5 * ((xbt[:, None, :] - xbt[None, :, :]) ** 2).sum(-1)) + dl * np.eye(M)
    K = c * np.exp(-0.5 * ((xbt[:, None, :] - xt[None, :, :]) ** 2).sum(-1))
    Li = np.linalg.inv(np.linalg.cholesky(Q))
    V = Li @ K
    ep = 1 + (c - (V ** 2).sum(0)) / sig
    Kt, Vt, yt = K / np.sqrt(ep), V / np.sqrt(ep), y / np.sqrt(ep)
    Lmi = np.linalg.inv(np.linalg.cholesky(sig * np.eye(M) + Vt @ Vt.T))
    invLmV = Lmi @ Vt
    bet = invLmV @ yt
    B1 = Li.T @ (Lmi.T @ invLmV)
    u = Lmi.T @ bet
    b1 = Li.T @ u
    invLV = Li.T @ Vt
    invQ = Li.T @ Li
    Z = Lmi @ Li
    invA = Z.T @ Z
    mu = u @ Vt
    r = yt - mu
    big = yt * (bet @ invLmV) / sig - (invLmV ** 2).sum(0) / 2 - (yt ** 2 + mu ** 2) / (2 * sig) + 0.5
    TT = invLV @ (invLV * big).T
    G = Kt * (B1 - np.outer(b1, r) / sig - (2 / sig) * invLV * big)
    H = Q * (invQ - sig * invA - (2 / sig) * TT - np.outer(b1, b1))
    dfxb = (G @ xt - xbt * G.sum(1)[:, None]) + (xbt * H.sum(1)[:, None] - H @ xbt)
    dfb = np.array([(G * xt[:, i][None, :] * (xbt[:, i][:, None] - xt[:, i][None, :])).sum() for i in range(D)])
    dfxb = dfxb * bs
    dfb = (dfb / bs + (dfxb * xbt).sum(0) / b) * bs / 2
    epc = (c / ep - (Vt ** 2).sum(0) - dl * (invLV ** 2).sum(0)) / sig
    dfc = ((M + dl * (np.trace(invQ) - sig * np.trace(invA)) - sig * (invA * Q).sum()) / 2 - mu @ r / sig
           + (b1 @ Q @ b1 - dl * b1 @ b1) / 2 + epc @ big)
    dfsig = (big / ep).sum()
    g2 = -np.concatenate([dfxb.T.reshape(-1), dfb, [dfc, dfsig]])
    assert np.abs(g2 - g).max() <= 1e-12 * np.abs(g).max()


def test_new_kernels_have_no_stack_frame():
    tool = next((c for c in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"), shutil.which("cuobjdump"))
                 if c and os.path.exists(c)), None)
    if tool is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    out = subprocess.run([tool, "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"^\s*Function (\S*spgp_\S*):\s*\n\s*(REG:.*)$", out, flags=re.M)
    names = {re.search(r"\d(spgp_[a-z_]+?_kernel)", n).group(1) for n, _ in found}
    assert {"spgp_gemm_kernel", "spgp_pass_kernel", "spgp_kmat_kernel", "spgp_ep_kernel", "spgp_coldot_kernel", "spgp_nvec_kernel",
            "spgp_final_kernel", "spgp_dfxb_kernel"} <= names, names
    for name, usage in found:
        res = dict(kv.split(":", 1) for kv in usage.split())
        assert int(res["STACK"]) == 0 and int(res["LOCAL"]) == 0, f"{name}: {res}"


GOLDEN = sorted(__import__("glob").glob(os.path.join(ROOT, "tests", "golden", "spgp", "*.npz")))


def test_golden_cases_present():
    names = {os.path.basename(p)[:-4] for p in GOLDEN}
    assert {"cos1d_n100", "n40_d2", "n41_d2_odd", "n5_d2_m1", "n300_d3", "hartmann6_n2000"} <= names


def _against_reference(g, fo, go, st, mo, so):
    assert abs(fo - g["f"]) <= 1e-12 * abs(g["f"])
    assert np.abs(go - g["grad"]).max() <= 1e-10 * np.abs(g["grad"]).max()
    assert np.abs(st.L - g["L"]).max() <= 1e-10 and np.abs(st.Lm - g["Lm"]).max() <= 1e-10
    assert np.abs(st.bet - g["bet"]).max() <= 1e-9 * max(1.0, np.abs(g["bet"]).max())
    c = st.c
    assert np.abs(mo + g["y"].mean() - g["mu"]).max() <= 1e-10 * c
    assert np.abs(so - g["s2"]).max() <= 1e-10 * c


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_oracle_equals_reference_fixtures(path):
    """The restatement against the reference's own SPGP (tests/golden/spgp, made by oracle/ref_shim/spgp_driver.cpp)."""
    g = np.load(path)
    X, y, M, w, jit = g["X"], g["y"], int(g["M"]), g["w"], float(g["jitter"])
    yz = y - y.mean()
    fo, go = O.likelihood(w, X, yz, M, jit)
    st = O.State(w, X, yz, M, jit)
    mo, so = st.predict(g["Xq"])
    _against_reference(g, fo, go, st, mo, so)


@pytest.mark.parametrize("seed,N,D", [(11, 60, 3), (12, 57, 2), (13, 400, 4), (14, 30, 1)])
def test_oracle_equals_reference_driver(seed, N, D):
    """The same comparison on fresh cases, where the reference driver is built (oracle/_ref/libref_spgp.so)."""
    from oracle import ref_spgp
    if not ref_spgp.available():
        pytest.skip("the reference's SPGP is not built and its sources are not present; the fixtures cover it")
    rng = np.random.default_rng(seed)
    X = rng.random((N, D))
    y = np.cos(4.0 * X).sum(axis=1)
    M = O.n_pseudo(N)
    w = O.init_w(X, y - y.mean(), M, rng.permutation(N)) + rng.normal(0.0, 0.05, (M + 1) * D + 2)
    Xq = rng.random((100, D))
    r = dict(ref_spgp.run(X, y, M, w, Xq), y=y)
    fo, go = O.likelihood(w, X, y - y.mean(), M, JITTER)
    st = O.State(w, X, y - y.mean(), M, JITTER)
    mo, so = st.predict(Xq)
    _against_reference(r, fo, go, st, mo, so)
