// oracle/ref_shim/parego_driver.cpp — TEST INFRASTRUCTURE ONLY.
//
// Runs the REFERENCE'S OWN experimental::model::GPParego (experimental/model/gp_parego.hpp) over its model::GP (Matern-5/2,
// mean::Data, default hyper-parameters), with the dense linear algebra supplied by the stand-in in ./Eigen and the weight
// vectors replayed through ./parego_shim (tools::random_vector).  Used to pin the scalarisation of limbo_b200.model.GPParego and
// oracle/parego.py (tests/test_parego_host.py) and to generate tests/golden/parego/*.npz (tests/golden/make_golden_parego.py).
// No reference source is copied: this file only instantiates its templates.
#include <limbo/tools/random_generator.hpp> // first: the replaying tools::random_vector of ./parego_shim
#include <limbo/kernel/matern_five_halves.hpp>
#include <limbo/mean/data.hpp>
#include <limbo/model/gp.hpp> // with tools.hpp: the macros and tools::make_vector gp_parego.hpp uses without including them
#include <limbo/experimental/model/gp_parego.hpp>

using namespace limbo;

struct Params {
    struct kernel {
        BO_DYN_PARAM(double, noise);
        BO_PARAM(bool, optimize_noise, false);
    };
    struct kernel_maternfivehalves : public defaults::kernel_maternfivehalves {};
    struct model_gp_parego {
        BO_DYN_PARAM(double, rho);
    };
};
BO_DECLARE_DYN_PARAM(double, Params::kernel, noise);
BO_DECLARE_DYN_PARAM(double, Params::model_gp_parego, rho);

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
} // namespace

extern "C" {

// GPParego over the first N0 of the N samples (X: N x D, F: N x K row-major) with compute(), then add_sample() for each of the
// others; draws holds the K raw weights of each of the 1 + N - N0 calls.  Returns the final scalarised observations (N), and mu
// and sigma^2 at the M query points.
int ref_parego(long N, long N0, int D, int K, const double* X, const double* F, const double* draws, double rho, double noise, long M,
    const double* Xq, double* scal, double* mu, double* s2)
{
    using P = Params;
    P::kernel::set_noise(noise);
    P::model_gp_parego::set_rho(rho);
    using GP_t = experimental::model::GPParego<P, model::GP<P, kernel::MaternFiveHalves<P>, mean::Data<P>>>;
    limbo_parego_replay(draws, (size_t)K * (size_t)(1 + N - N0));
    auto xs = rows_of(X, N, D);
    auto fs = rows_of(F, N, K);
    GP_t gp(D, K);
    gp.compute(std::vector<Eigen::VectorXd>(xs.begin(), xs.begin() + N0), std::vector<Eigen::VectorXd>(fs.begin(), fs.begin() + N0));
    for (long i = N0; i < N; ++i) gp.add_sample(xs[(size_t)i], fs[(size_t)i]);
    const auto obs = gp.observations();
    for (long i = 0; i < N; ++i) scal[i] = obs[(size_t)i](0);
    for (long q = 0; q < M; ++q) {
        Eigen::VectorXd v((Eigen::Index)D);
        for (int k = 0; k < D; ++k) v(k) = Xq[q * D + k];
        Eigen::VectorXd m;
        double s;
        std::tie(m, s) = gp.query(v);
        mu[q] = m(0);
        s2[q] = s;
    }
    return 0;
}
}
