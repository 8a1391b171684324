// oracle/ref_shim/eci_driver.cpp — TEST INFRASTRUCTURE ONLY.
//
// Runs the REFERENCE'S OWN experimental::acqui::ECI (experimental/acqui/eci.hpp) over two of the reference's model::GP, with
// the dense linear algebra supplied by the stand-in in ./Eigen.  Used to pin the ECI restatement (oracle/eci.py,
// tests/test_eci_host.py) and to generate tests/golden/eci/*.npz (tests/golden/make_golden_eci.py).
// No reference source is copied: this file only instantiates its templates.
#include <algorithm>
#include <limits>
#include <limbo/acqui/ucb.hpp>
#include <limbo/experimental/acqui/eci.hpp>
#include <limbo/kernel/exp.hpp>
#include <limbo/kernel/matern_five_halves.hpp>
#include <limbo/kernel/squared_exp_ard.hpp>
#include <limbo/mean/constant.hpp>
#include <limbo/mean/data.hpp>
#include <limbo/model/gp.hpp>

using namespace limbo;

struct Params {
    struct kernel {
        BO_DYN_PARAM(double, noise);
        BO_PARAM(bool, optimize_noise, false);
    };
    struct kernel_squared_exp_ard : public defaults::kernel_squared_exp_ard {};
    struct kernel_maternfivehalves : public defaults::kernel_maternfivehalves {};
    struct kernel_exp : public defaults::kernel_exp {};
    struct mean_constant {
        BO_PARAM(double, constant, 0.25);
    };
    struct acqui_eci { // run-time jitter (Params::acqui_eci::jitter)
        BO_DYN_PARAM(double, jitter);
    };
};
BO_DECLARE_DYN_PARAM(double, Params::kernel, noise);
BO_DECLARE_DYN_PARAM(double, Params::acqui_eci, jitter);

// bayes_opt/bo_base.hpp:99-105 (FirstElem) restated: bo_base.hpp itself needs Boost.Parameter/Fusion
struct FirstElem {
    double operator()(const Eigen::VectorXd& x) const { return x(0); }
};

namespace {

std::vector<Eigen::VectorXd> rows_of(const double* a, long n, int d)
{
    std::vector<Eigen::VectorXd> v;
    for (long i = 0; i < n; ++i) {
        Eigen::VectorXd x((Eigen::Index)d);
        for (int k = 0; k < d; ++k) x(k) = a[i * d + k];
        v.push_back(x);
    }
    return v;
}

// The reference's experimental::acqui::ECI (eci.hpp:76-130) over an objective GP (SE-ARD, mean::Data, N samples, P = 1) and a
// constraint GP (Exp or Matern-5/2, mean::Constant, P = 2) fitted on the first Nc samples (Nc = 0: a constraint model without
// samples), default hyper-parameters, one candidate at a time.  Returns ECI, both models' mu and sigma^2, and f_max.
template <typename ConKernel>
int run_eci(long N, int D, const double* X, const double* Y, long Nc, const double* Yc, double noise, double jitter, long M,
    const double* Xq, double* eci, double* mu, double* s2, double* mu_c, double* s2_c, double* f_max)
{
    using P = Params;
    P::kernel::set_noise(noise);
    P::acqui_eci::set_jitter(jitter);
    using GPo_t = model::GP<P, kernel::SquaredExpARD<P>, mean::Data<P>>;
    using GPc_t = model::GP<P, ConKernel, mean::Constant<P>>;
    auto samples = rows_of(X, N, D);
    GPo_t gp(D, 1);
    gp.compute(samples, rows_of(Y, N, 1));
    GPc_t gpc(D, 2);
    if (Nc > 0) gpc.compute(std::vector<Eigen::VectorXd>(samples.begin(), samples.begin() + Nc), rows_of(Yc, Nc, 2));
    experimental::acqui::ECI<P, GPo_t, GPc_t> acq(gp, gpc);
    FirstElem afun;
    *f_max = -std::numeric_limits<double>::max(); // eci.hpp:91-99
    for (const auto& x : samples) *f_max = std::max(*f_max, afun(gp.mu(x)));
    for (long q = 0; q < M; ++q) {
        Eigen::VectorXd v((Eigen::Index)D);
        for (int k = 0; k < D; ++k) v(k) = Xq[q * D + k];
        Eigen::VectorXd m;
        double s;
        std::tie(m, s) = gp.query(v);
        mu[q] = m(0);
        s2[q] = s;
        std::tie(m, s) = gpc.query(v);
        mu_c[2 * q] = m(0);
        mu_c[2 * q + 1] = m(1);
        s2_c[q] = s;
        eci[q] = opt::fun(acq(v, afun, false));
    }
    return 0;
}

} // namespace

extern "C" {

// con_kernel_id: 1 MaternFiveHalves, 3 Exp.  Y: N objective observations; Yc: Nc x 2 row-major constraint observations of the
// first Nc samples.  mu_c is M x 2 row-major.
int ref_gp_eci(int con_kernel_id, long N, int D, const double* X, const double* Y, long Nc, const double* Yc, double noise, double jitter,
    long M, const double* Xq, double* eci, double* mu, double* s2, double* mu_c, double* s2_c, double* f_max)
{
    if (con_kernel_id == 1)
        return run_eci<kernel::MaternFiveHalves<Params>>(N, D, X, Y, Nc, Yc, noise, jitter, M, Xq, eci, mu, s2, mu_c, s2_c, f_max);
    if (con_kernel_id == 3) return run_eci<kernel::Exp<Params>>(N, D, X, Y, Nc, Yc, noise, jitter, M, Xq, eci, mu, s2, mu_c, s2_c, f_max);
    return 1;
}
}
