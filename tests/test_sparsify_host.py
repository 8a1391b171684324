"""CPU checks of the sparsified model (model/sparsified_gp.hpp): the NumPy restatement (oracle/sparsify.py) against the reference's
own _sparsify, through tests/golden/sparsify and, where oracle/_ref was built, live on fresh random and lattice sets; the parameter
default; the C++ drop-in header against the Eigen stand-in; and the resource table of the new kernels (no device needed)."""
import glob
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from limbo_b200 import params
from oracle import sparsify as oracle_sparsify

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "sparsify")
FIXTURES = sorted(glob.glob(os.path.join(GOLDEN, "*.npz")))
LIB = os.path.join(ROOT, "limbo_b200", "lib", "liblimbo_b200.so")


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def test_fixtures_present():
    assert len(FIXTURES) == 7


@pytest.mark.parametrize("path", FIXTURES, ids=os.path.basename)
def test_oracle_matches_fixtures(path):
    """kept set, removal order and densities, bit for bit"""
    g = np.load(path)
    kept, removed, score = oracle_sparsify.sparsify(g["X"], int(g["max_points"]))
    assert np.array_equal(kept, g["kept"])
    assert np.array_equal(removed, g["removed"])
    assert np.array_equal(score.view(np.uint64), g["removed_score"].view(np.uint64))
    assert len(kept) == min(len(g["X"]), int(g["max_points"]))


def test_lattice_fixture_pins_the_tie_rule():
    """on the lattice most removals are decided among exactly equal densities: the lowest index wins"""
    g = np.load(os.path.join(GOLDEN, "lattice16x16_max64.npz"))
    s = g["removed_score"]
    assert len(np.unique(s)) < len(s) // 4


def _ref_or_skip():
    from oracle import ref, ref_sparse
    if not os.path.isdir(ref.REF_SRC):
        pytest.skip("the reference's sources are not present")
    ref_sparse.build()
    return ref_sparse


@pytest.mark.parametrize("path", FIXTURES, ids=os.path.basename)
def test_fixtures_are_what_the_reference_computes(path):
    ref_sparse = _ref_or_skip()
    g = np.load(path)
    assert _same(ref_sparse.sparsify(g["X"], int(g["max_points"])), (g["kept"], g["removed"], g["removed_score"]))


@pytest.mark.parametrize("seed,N,D,max_points", [(1, 120, 1, 40), (2, 200, 2, 60), (3, 150, 5, 30), (4, 90, 12, 12), (5, 300, 3, 299)])
def test_oracle_equals_reference_random(seed, N, D, max_points):
    ref_sparse = _ref_or_skip()
    X = np.random.default_rng(seed).normal(size=(N, D))
    assert _same(oracle_sparsify.sparsify(X, max_points), ref_sparse.sparsify(X, max_points))


@pytest.mark.parametrize("shape,max_points", [((10, 10), 30), ((5, 5, 5), 20), ((40,), 7)])
def test_oracle_equals_reference_lattice(shape, max_points):
    ref_sparse = _ref_or_skip()
    X = np.stack(np.meshgrid(*[np.arange(float(n)) for n in shape], indexing="ij"), -1).reshape(-1, len(shape))
    assert _same(oracle_sparsify.sparsify(X, max_points), ref_sparse.sparsify(X, max_points))


def test_params_default():
    assert params.defaults.model_sparse_gp.max_points == 200  # sparsified_gp.hpp:56-60
    assert params.get(None, "model_sparse_gp", "max_points") == 200

    class P:
        class model_sparse_gp:
            max_points = 33

    assert params.get(P, "model_sparse_gp", "max_points") == 33


def test_multigp_takes_the_inner_model_class():
    import inspect
    from limbo_b200 import model
    assert inspect.signature(model.MultiGP).parameters["gp_class"].default is model.GP
    assert issubclass(model.SparsifiedGP, model.GP)


def test_dropin_header_compiles():
    """limbo_b200::model::SparsifiedGP with the reference's defaults, and model::MultiGP over it, against the Eigen stand-in"""
    from oracle import ref
    if not os.path.isdir(ref.REF_SRC):
        pytest.skip("the reference's sources are not present")
    src = r"""
#include <limbo/kernel/matern_five_halves.hpp>
#include <limbo/kernel/squared_exp_ard.hpp>
#include <limbo/mean/constant.hpp>
#include <limbo/mean/data.hpp>
#include <limbo/model/gp.hpp>
#include <limbo/model/multi_gp.hpp>
#include <limbo_b200/model/sparsified_gp.hpp>
struct Params {
    struct kernel : public limbo::defaults::kernel {};
    struct kernel_maternfivehalves : public limbo::defaults::kernel_maternfivehalves {};
    struct kernel_squared_exp_ard : public limbo::defaults::kernel_squared_exp_ard {};
    struct mean_constant : public limbo::defaults::mean_constant {};
    struct model_sparse_gp { BO_PARAM(int, max_points, 50); };
};
template class limbo_b200::model::SparsifiedGP<Params>;
template class limbo::model::MultiGP<Params, limbo_b200::model::SparsifiedGP, limbo::kernel::SquaredExpARD<Params>,
    limbo::mean::Constant<Params>>;
static_assert(std::is_base_of<limbo_b200::model::GP<Params, limbo::kernel::MaternFiveHalves<Params>, limbo::mean::Data<Params>,
    limbo::model::gp::NoLFOpt<Params>>, limbo_b200::model::SparsifiedGP<Params>>::value, "defaults");
"""
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-w", "-x", "c++", "-I", os.path.join(ROOT, "oracle", "ref_shim"), "-I",
                        ref.REF_ROOT, "-I", os.path.join(ROOT, "include"), "-"], input=src, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]


def test_sparsify_kernels_have_no_stack():
    tool = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    if not os.path.exists(tool):
        tool = shutil.which("cuobjdump")
    if not tool:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    r = subprocess.run([tool, "-res-usage", LIB], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    found = re.findall(r"^\s*Function (\S+):\s*\n\s*(REG:.*)$", r.stdout, flags=re.M)
    res = {name: dict(kv.split(":", 1) for kv in usage.split()) for name, usage in found}
    mine = {n: v for n, v in res.items() if re.search(r"sparsify_(soa|knn_init|greedy|compact)_kernel", n)}
    assert len(mine) == 4, sorted(mine)
    for name, v in mine.items():
        assert int(v["STACK"]) == 0 and int(v["LOCAL"]) == 0, f"{name}: {v}"
