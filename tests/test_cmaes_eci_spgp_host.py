"""CPU checks of the device CMA-ES over ECI and over SPGP (lb_eci_cmaes, lb_spgp_acq_cmaes and the SPGP _dev scorers): the C
declarations are plain C with the documented prototypes, the library exports them, and the C++ drop-ins compile against the
reference's headers with BatchedCmaes instantiated over the batch-aware ECI and over UCB / EI on model::SPGP."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("lb_eci_cmaes", "lb_spgp_query_dev", "lb_spgp_acq_argmax_dev", "lb_spgp_acq_cmaes")


def test_declarations_are_plain_c(tmp_path):
    """Each new entry point is assigned to a pointer of its documented type, so a changed prototype fails to compile as C."""
    src = tmp_path / "t.c"
    src.write_text('#include "limbo_b200.h"\n'
                   "int (*eci)(const lb_gp*, const lb_gp*, const double*, double, double, const lb_cmaes_opts*, int64_t, const double*,"
                   " double*, double*, int64_t*) = lb_eci_cmaes;\n"
                   "int (*qdev)(const lb_spgp*, int64_t, const double*, int, double*, double*) = lb_spgp_query_dev;\n"
                   "int (*adev)(const lb_spgp*, int, const double*, int64_t, const double*, int, const double*, double, double*, double*,"
                   " int64_t*) = lb_spgp_acq_argmax_dev;\n"
                   "int (*scm)(const lb_spgp*, int, const double*, int, double, const lb_cmaes_opts*, int64_t, const double*, double*,"
                   " double*, int64_t*) = lb_spgp_acq_cmaes;\n"
                   "int main(void) { return LB_OK; }\n")
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_library_exports_the_new_entry_points(lib):
    from limbo_b200 import _lib
    for name in NEW:
        assert hasattr(lib, name) and name in _lib.DECLARED_SYMBOLS


def test_cpp_headers_compile_against_the_reference():
    """tests/cpp/cmaes_eci_spgp_dropin_test.cpp over the reference's headers and the Eigen stand-in of oracle/ref_shim/spgp_eigen:
    BatchedCmaes over limbo_b200::acqui::ECI and over UCB / EI on limbo_b200::model::SPGP, whose device search is selected through
    detail::has_device_cmaes."""
    from oracle import ref
    if not os.path.isdir(ref.REF_SRC):
        pytest.skip("the reference's sources are not present")
    shim = os.path.join(ROOT, "oracle", "ref_shim")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-w", "-I", os.path.join(shim, "spgp_eigen"), "-I", shim, "-I", ref.REF_ROOT,
                        "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "cmaes_eci_spgp_dropin_test.cpp")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]


def test_device_search_is_selected_on_the_model_type(tmp_path):
    """has_device_cmaes is true for SPGP with an input-free mean and false with one that depends on the input, and the batch-aware
    ECI's device search is compiled in for a pair of device GPs with input-free means only."""
    from oracle import ref
    if not os.path.isdir(ref.REF_SRC):
        pytest.skip("the reference's sources are not present")
    src = tmp_path / "t.cpp"
    src.write_text("""#include <Eigen/Core>
#include <limbo/kernel/exp.hpp>
#include <limbo/kernel/squared_exp_ard.hpp>
#include <limbo/mean/constant.hpp>
#include <limbo/mean/data.hpp>
#include <limbo/model/gp.hpp>
#include <limbo/opt/rprop.hpp>
#include <limbo_b200/model/gp.hpp>
#include <limbo_b200/model/spgp.hpp>
#include <limbo_b200/opt/batched_cmaes.hpp>
using namespace limbo;
struct Params {
    struct kernel : public defaults::kernel {};
    struct kernel_squared_exp_ard : public defaults::kernel_squared_exp_ard {};
    struct kernel_exp : public defaults::kernel_exp {};
    struct model_spgp : public defaults::model_spgp {};
    struct opt_rprop : public defaults::opt_rprop {};
    struct mean_constant { BO_PARAM(double, constant, 0.5); };
};
struct XMean { // a mean that depends on the input
    XMean(int = 1) {}
    template <typename GP> Eigen::VectorXd operator()(const Eigen::VectorXd& v, const GP&) const { return v.head(1); }
};
using K = kernel::SquaredExpARD<Params>;
using S1 = limbo_b200::model::SPGP<Params, K, mean::Data<Params>, opt::Rprop<Params>>;
using S2 = limbo_b200::model::SPGP<Params, K, XMean, opt::Rprop<Params>>;
using G1 = limbo_b200::model::GP<Params, K, mean::Data<Params>, model::gp::NoLFOpt<Params>>;
using G2 = limbo_b200::model::GP<Params, kernel::Exp<Params>, mean::Constant<Params>, model::gp::NoLFOpt<Params>>;
using G3 = limbo_b200::model::GP<Params, K, XMean, model::gp::NoLFOpt<Params>>;
using R1 = model::GP<Params, K, mean::Data<Params>>;
static_assert(limbo_b200::acqui::detail::has_device_cmaes<S1>::value, "SPGP, input-free mean");
static_assert(!limbo_b200::acqui::detail::has_device_cmaes<S2>::value, "SPGP, input-dependent mean");
template <typename A> struct Probe : A { static constexpr bool value = A::has_cmaes; };
static_assert(Probe<limbo_b200::acqui::ECI<Params, G1, G2>>::value, "ECI over two device GPs");
static_assert(!Probe<limbo_b200::acqui::ECI<Params, G3, G2>>::value, "ECI, input-dependent objective mean");
static_assert(!Probe<limbo_b200::acqui::ECI<Params, G1, G3>>::value, "ECI, input-dependent constraint mean");
static_assert(!Probe<limbo_b200::acqui::ECI<Params, R1, G2>>::value, "ECI over the reference's GP");
int main() { return 0; }
""")
    shim = os.path.join(ROOT, "oracle", "ref_shim")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-w", "-I", os.path.join(shim, "spgp_eigen"), "-I", shim, "-I", ref.REF_ROOT,
                        "-I", os.path.join(ROOT, "include"), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
