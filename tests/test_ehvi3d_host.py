"""Three-objective EHVI without a GPU: oracle/ehvi3d.py against the reference's own ehvi3d_sliceupdate, ehvi3d_5term, ehvi3d_8term
and hvol3d (oracle/ref_ehvi3d.py, where the reference's sources were present at build time), the fixtures under
tests/golden/ehvi3d against the oracle, the z_ref default, the exported entry points and the new kernels' resources."""
import glob
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import ehvi as E2
from oracle import ehvi3d as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "ehvi3d", "*.npz")))


@pytest.fixture(scope="module")
def ref():
    from oracle import ref_ehvi3d as R
    if not R.available():
        pytest.skip("the reference's EHVI is not built and its sources are not present")
    return R


def _sphere(rng, k):
    v = np.abs(rng.normal(size=(k, 3)))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _fronts():
    """(tag, front) over k = 0, 1, 8, 32, with tied coordinates and duplicated points"""
    rng = np.random.default_rng(7)
    for k in (0, 1, 8, 32):
        yield f"k{k}", _sphere(rng, k)
    yield "tied", np.round(_sphere(rng, 20) * 4) / 4
    F = _sphere(rng, 10)
    yield "duplicates", np.concatenate([F, F[:3], F[:1]])


def _cands(seed, M=6):
    rng = np.random.default_rng(seed)
    return rng.uniform(-0.1, 1.2, (M, 3)), rng.uniform(0.02, 0.6, (M, 3))


R0 = np.array([-0.1, -0.2, -0.15])


@pytest.mark.parametrize("tag,front", list(_fronts()), ids=[t for t, _ in _fronts()])
def test_oracle_equals_reference_bit_for_bit(ref, tag, front):
    mu, s = _cands(len(front))
    want = ref.ehvi3d_sliceupdate(front, R0, mu, s)
    got = np.array([E.ehvi3d(front, R0, mu[q], s[q]) for q in range(len(mu))])
    assert np.array_equal(got, want), (tag, got - want)
    tab, scale = E.ehvi3d_tables(front, R0, mu, s)
    assert np.all(np.abs(tab - want) <= E2.tolerance(want, scale)), tag
    assert np.all(np.abs(E.ehvi3d_tables(front, R0, mu, s, libm=True)[0] - want) <= E2.tolerance(want, scale)), tag


@pytest.mark.parametrize("tag,front", [(t, f) for t, f in _fronts() if t in ("k1", "k8", "k32", "tied", "duplicates")],
                         ids=["k1", "k8", "k32", "tied", "duplicates"])
def test_independent_schemes_agree(ref, tag, front):
    """ehvi3d_5term and ehvi3d_8term (ehvi_calculations.cc) against the slice-update scheme, to 1e-13 relative"""
    mu, s = _cands(100 + len(front))
    want = ref.ehvi3d_sliceupdate(front, R0, mu, s)
    tab = E.ehvi3d_tables(front, R0, mu, s)[0]
    for name in ("ehvi3d_5term", "ehvi3d_8term"):
        other = getattr(ref, name)(front, R0, mu, s)
        assert np.all(np.abs(other - want) <= 1e-13 * np.abs(want).max()), (tag, name)
        assert np.all(np.abs(other - tab) <= 1e-13 * np.abs(want).max()), (tag, name)


@pytest.mark.parametrize("tag,front", [(t, f) for t, f in _fronts() if t != "k0"], ids=[t for t, _ in _fronts() if t != "k0"])
def test_tie_order_does_not_change_the_tested_fronts(ref, tag, front):
    """The reference sorts with std::sort, which is not stable, and the oracle and the device sort stably by input index: with
    tied coordinates the reference's Pstruct could depend on the order of the ties.  On every tested front, five permutations of
    the input leave the reference's values and the oracle's unchanged, bit for bit."""
    mu, s = _cands(200 + len(front))
    want = ref.ehvi3d_sliceupdate(front, R0, mu, s)
    rng = np.random.default_rng(len(front))
    for _ in range(5):
        P = front[rng.permutation(len(front))]
        assert np.array_equal(ref.ehvi3d_sliceupdate(P, R0, mu, s), want), tag
        assert np.array_equal(np.array([E.ehvi3d(P, R0, mu[q], s[q]) for q in range(len(mu))]), want), tag


def test_gp_fixtures_reproduce_from_the_reference(ref):
    """The GP fixtures are what the reference's three GPs and ehvi3d_sliceupdate give for their inputs (rerun here)."""
    for name in ("dtlz2_n60_d3", "on_samples", "duplicated_obs", "prior"):
        g = np.load(os.path.join(ROOT, "tests", "golden", "ehvi3d", name + ".npz"))
        out = ref.gp_ehvi3d(g["X"], g["Y"], g["Xq"], g["r"], float(g["noise"]))
        for k in ("ehvi", "mu", "s", "front"):
            assert np.array_equal(out[k], g[k]), (name, k)


def test_small_s_approaches_the_hypervolume_gain(ref):
    """With s = 1e-9 on every axis and mu off the front's coordinates, EHVI is the hypervolume the point mu adds."""
    rng = np.random.default_rng(9)
    F = _sphere(rng, 12)
    for mu in (np.array([0.7, 0.65, 0.6]), np.array([0.2, 0.3, 1.05]), np.array([1.1, 0.05, 0.1])):
        gain = ref.hv3d(np.vstack([F, mu]), R0) - ref.hv3d(F, R0)
        v = E.ehvi3d(F, R0, mu, np.full(3, 1e-9))
        assert gain > 0 and abs(v - gain) <= 1e-7 * gain, (mu, v, gain)
        assert abs(E.hypervolume3d(np.vstack([F, mu]), R0) - E.hypervolume3d(F, R0) - gain) <= 1e-12


def test_hypervolume3d_against_reference(ref):
    rng = np.random.default_rng(10)
    for k in (1, 5, 40):
        F = _sphere(rng, k)
        assert abs(E.hypervolume3d(F, R0) - ref.hv3d(F, R0)) <= 1e-14 * ref.hv3d(F, R0)


def test_fixtures_present():
    names = {os.path.basename(p) for p in FIXTURES}
    assert {"raw_k64.npz", "raw_k256.npz", "one_point.npz", "duplicates.npz", "tied.npz", "tiny_s.npz", "dtlz2_n60_d3.npz",
            "dtlz2_n300_d6.npz", "on_samples.npz", "duplicated_obs.npz", "prior.npz"} <= names


@pytest.mark.parametrize("path", FIXTURES, ids=os.path.basename)
def test_fixtures_reproduce_from_oracle(path):
    g = np.load(path)
    want, scale = E.ehvi3d_tables(g["front"], g["r"], g["mu"], g["s"])
    assert np.all(np.abs(want - g["ehvi"]) <= E2.tolerance(g["ehvi"], scale)), os.path.basename(path)
    if len(g["front"]) <= 16:
        exact = np.array([E.ehvi3d(g["front"], g["r"], g["mu"][q], g["s"][q]) for q in range(len(g["mu"]))])
        assert np.array_equal(exact, g["ehvi"])


def test_params_defaults():
    from limbo_b200.params import get
    assert get(None, "bayes_opt_ehvi", "z_ref") == -11.0


def test_entry_points_exported():
    from limbo_b200 import _lib
    lib = _lib.load()
    for name in ("lb_ehvi3d_argmax", "lb_ehvi3d_argmax_dev"):
        assert hasattr(lib, name) and name in _lib.DECLARED_SYMBOLS


def test_new_kernels_have_no_stack_frame():
    tool = next((c for c in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"), shutil.which("cuobjdump"))
                 if c and os.path.exists(c)), None)
    if tool is None:
        pytest.skip("cuobjdump not found")
    r = subprocess.run([tool, "-res-usage", os.path.join(ROOT, "limbo_b200", "lib", "liblimbo_b200.so")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    found = dict(re.findall(r"^\s*Function (\S+):\s*\n\s*(REG:.*)$", r.stdout, flags=re.M))
    for kernel in ("ehvi3d_dom_kernel", "ehvi3d_slice_kernel", "ehvi3d_chunk_kernel", "ehvi3d_cells_kernel", "ehvi3d_sum_kernel"):
        hits = {n: u for n, u in found.items() if f"{len(kernel)}{kernel}" in n}
        assert len(hits) == 1, (kernel, sorted(hits))
        usage = dict(kv.split(":", 1) for kv in next(iter(hits.values())).split())
        assert int(usage["STACK"]) == 0 and int(usage["LOCAL"]) == 0, (kernel, usage)
