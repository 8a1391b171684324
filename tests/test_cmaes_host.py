"""CPU checks of the batched CMA-ES (DESIGN.md §4.15): the strategy constants, the box transform and its inverse, the NumPy
restatement (oracle/cmaes.py) converging on standard test functions, and the library's exports."""
import math

import numpy as np
import pytest

from oracle import cmaes as OC


@pytest.mark.parametrize("D", range(1, 65))
def test_constants(D):
    k = OC.constants(D)
    assert k.lam == 4 + int(math.floor(3 * math.log(D))) and k.mu == k.lam // 2
    assert abs(k.w[:k.mu].sum() - 1.0) < 1e-15 and np.all(k.w[:k.mu] > 0) and np.all(np.diff(k.w) <= 0)
    assert k.c1 + k.cmu <= 1.0 and 0 < k.cs < 1 and 0 < k.cc <= 1 and k.ds > 1
    # the negative weights keep C positive definite: sum |w-| <= alpha_posdef (and the two other bounds)
    sneg = np.abs(k.w[k.mu:]).sum()
    assert sneg <= min(k.alpha_mu_neg, k.alpha_mueff_neg, k.alpha_posdef_neg) * (1 + 1e-15)
    assert k.c1 + k.cmu * k.w.sum() <= 1.0 + 1e-15 or k.cmu * sneg <= 1.0 - k.c1 - k.cmu + 1e-15
    assert abs(k.chi - math.sqrt(D) * (1 - 1 / (4 * D) + 1 / (21 * D * D))) == 0.0
    k256 = OC.constants(D, 256)
    assert k256.lam == 256 and abs(k256.w[:128].sum() - 1.0) < 1e-14


def test_transform_identity_seams_range_and_inverse():
    lb, ub = 0.0, 1.0
    al, au = 0.05, 0.1
    inner = np.linspace(lb + al, ub - au, 101)
    assert np.array_equal(OC.transform(inner), inner)
    x = np.linspace(-7.3, 8.1, 200001)
    y = OC.transform(x)
    assert y.min() >= lb and y.max() <= ub and y.min() < 1e-9 and y.max() > 1 - 1e-9
    assert OC.transform(np.array([lb - al, ub + au])).tolist() == [lb, ub]
    # C1 at the four seams lb - al, lb + al, ub - au, ub + au: matching one-sided difference quotients
    h = 1e-7
    for s in (lb - al, lb + al, ub - au, ub + au):
        left = (OC.transform(np.array([s])) - OC.transform(np.array([s - h])))[0] / h
        right = (OC.transform(np.array([s + h])) - OC.transform(np.array([s])))[0] / h
        assert abs(left - right) < 1e-5, s
    # periodic: one period further gives the same phenotype
    r = 2 * (ub - lb + al + au)
    assert np.allclose(OC.transform(x + r), y, atol=1e-12)
    u = np.linspace(0, 1, 1001)
    assert np.allclose(OC.transform(OC.inverse(u)), u, atol=1e-15)
    assert np.array_equal(OC.inverse(inner), inner)


def test_normals_are_the_documented_stream():
    from limbo_b200 import synth
    z = OC.normals(5, 2, 3, 4, 6)
    c = ((2 * 3 + 1) * 4 + 2) * 6 + 5
    u = synth.uniform(5, 2, 2 * c)
    assert z[1, 2, 5] == math.sqrt(-2 * math.log(1 - u[0])) * math.cos(2 * math.pi * u[1])
    assert abs(z.mean()) < 0.5


def _problems(D, rng):
    c = 0.3 + 0.4 * rng.random(D)
    scale = 10.0 ** (3 * np.arange(D) / max(D - 1, 1))
    cf = c.copy()
    cf[0] = 1.3

    def rosen(X):
        Y = 4 * X - 1  # maximum at x = 0.5
        return -(100 * (Y[:, 1:] - Y[:, :-1] ** 2) ** 2 + (1 - Y[:, :-1]) ** 2).sum(1)
    return [("sphere", lambda X: -((X - c) ** 2).sum(1), c), ("ellipsoid", lambda X: -(scale * (X - c) ** 2).sum(1), c),
            ("rosenbrock", rosen, np.full(D, 0.5)), ("face", lambda X: -((X - cf) ** 2).sum(1), np.r_[1.0, c[1:]])]


@pytest.mark.parametrize("D", [2, 6])
def test_oracle_converges(D):
    rng = np.random.default_rng(D)
    for name, f, xo in _problems(D, rng):
        bx, bv, n = OC.run(f, np.full((1, D), 0.6), 3000, tolx=1e-13, seed=7)
        assert np.abs(bx - xo).max() < 1e-8, (name, bx, xo)
        assert np.all((bx >= 0) & (bx <= 1))


def test_oracle_unbounded_and_several_instances():
    c = np.array([2.0, -3.0, 0.5])
    bx, bv, n = OC.run(lambda X: -((X - c) ** 2).sum(1), np.zeros((3, 3)), 2000, tolx=1e-13, seed=1, bounded=False)
    assert np.abs(bx - c).max() < 1e-8 and n % (3 * OC.default_lambda(3)) == 0


def test_library_exports_cmaes(lib):
    from limbo_b200 import _lib
    for name in ("lb_acq_cmaes", "lb_ehvi_cmaes"):
        assert hasattr(lib, name) and name in _lib.DECLARED_SYMBOLS
    assert _lib.CmaesOpts.sigma0.offset == 8 and _lib.CmaesOpts.seed.offset == 32


def test_cpp_header_compiles_against_the_reference(tmp_path):
    """include/limbo_b200/opt/batched_cmaes.hpp with the batch-aware UCB / EI and the acqui::Ehvi specialisation, over the
    reference's headers and the Eigen stand-in (oracle/ref_shim): one translation unit that instantiates BatchedCmaes over each."""
    import os
    import subprocess
    from oracle import ref
    if not os.path.isdir(ref.REF_SRC):
        pytest.skip("the reference's sources are not present")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-w", "-I", os.path.join(root, "oracle", "ref_shim"), "-I", ref.REF_ROOT,
                        "-I", os.path.join(root, "include"), os.path.join(root, "tests", "cpp", "cmaes_dropin_test.cpp")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
