// tests/cpp/spgp_dropin_test.cpp — the reference's experimental::model::SPGP next to limbo_b200::model::SPGP, built by
// oracle/ref_shim/spgp.mk against the Eigen stand-in of oracle/ref_shim/spgp_eigen and run by tests/test_gpu_spgp.py.
// At a fixed w both models' _likelihood(w, true) and _compute(false) + predict must agree (value <= 1e-10 relative, gradient
// <= 1e-7 |g|inf, mu and sigma^2 <= 1e-9 c); then limbo_b200's public compute + query runs with the reference's Rprop.
// Prints "SPGP DROPIN OK" on success.
#include <Eigen/Core>
#include <cmath>
#include <cstdio>
#include <vector>

namespace nlopt {
enum algorithm { LD_LBFGS = 11 };
}
namespace limbo {
namespace opt {
template <typename Params, nlopt::algorithm Algorithm>
struct NLOptGrad;
}
} // namespace limbo

#include <limbo/experimental/model/spgp.hpp>
#include <limbo/kernel/squared_exp_ard.hpp>
#include <limbo/mean/data.hpp>
#include <limbo/opt/rprop.hpp>

#include <limbo_b200/model/spgp.hpp>

using namespace limbo;

struct Params {
    struct kernel : public defaults::kernel {};
    struct kernel_squared_exp_ard : public defaults::kernel_squared_exp_ard {};
    struct model_spgp : public defaults::model_spgp {};
    struct opt_rprop : public defaults::opt_rprop {
        BO_PARAM(int, iterations, 30);
    };
};
using Kern = kernel::SquaredExpARD<Params>;
using Mean = mean::Data<Params>;
using Ref = model::SPGP<Params, Kern, Mean, opt::Rprop<Params>>;
using Ours = limbo_b200::model::SPGP<Params, Kern, Mean, opt::Rprop<Params>>;

struct RefX : Ref {
    void init(const Eigen::MatrixXd& X, const Eigen::MatrixXd& Y) { this->_init(X, Y); }
    opt::eval_t lik(const Eigen::VectorXd& w) const { return this->_likelihood(w, true); }
    void compute_at(const Eigen::VectorXd& w)
    {
        typename Ref::HyperParams hp(w, this->_m, this->_dim_in);
        this->_pseudo_samples = hp.xb;
        this->_b = hp.b.transpose();
        this->_c = hp.c;
        this->_sig = hp.sig;
        this->_optimized = true;
        this->_compute(false);
    }
    size_t m() const { return this->_m; }
};

struct OursX : Ours {
    void init(const std::vector<Eigen::VectorXd>& s, const std::vector<Eigen::VectorXd>& o) { this->_init(s, o); }
    opt::eval_t lik(const Eigen::VectorXd& w) const { return this->_likelihood(w, true); }
    void compute_at(const Eigen::VectorXd& w)
    {
        this->_optimized = true;
        this->_compute_at(w);
    }
};

int main()
{
    const int N = 300, D = 3;
    std::vector<Eigen::VectorXd> s, o;
    Eigen::MatrixXd X(N, D), Y(N, 1);
    unsigned st = 12345u;
    auto uni = [&]() { st = st * 1664525u + 1013904223u; return (double)(st >> 8) / (double)(1u << 24); };
    for (int i = 0; i < N; ++i) {
        Eigen::VectorXd x(D);
        double y = 0.0;
        for (int d = 0; d < D; ++d) { x(d) = uni(); X(i, d) = x(d); y += std::sin(3.0 * x(d)); }
        s.push_back(x);
        o.push_back(Eigen::VectorXd::Constant(1, y));
        Y(i, 0) = y;
    }
    RefX ref;
    ref.init(X, Y);
    OursX ours;
    ours.init(s, o);
    const size_t M = ref.m();
    // the reference's starting layout for the permutation i -> 7 i mod N, moved off the samples
    Eigen::VectorXd w((M + 1) * D + 2);
    for (size_t i = 0; i < M; ++i)
        for (int d = 0; d < D; ++d) w(i * D + d) = X((7 * i) % N, d) + 0.01 * std::cos((double)(i * D + d));
    for (int d = 0; d < D; ++d) w(M * D + d) = 2.0 + 0.1 * d;
    w((M + 1) * D) = std::log(0.8);
    w((M + 1) * D + 1) = std::log(0.05);
    auto a = ref.lik(w), b = ours.lik(w);
    const Eigen::VectorXd ga = std::get<1>(a).get(), gb = std::get<1>(b).get();
    double gmax = 0.0, gerr = 0.0;
    for (int i = 0; i < (int)ga.size(); ++i) { gmax = std::max(gmax, std::fabs(ga(i))); gerr = std::max(gerr, std::fabs(ga(i) - gb(i))); }
    const double ferr = std::fabs(std::get<0>(a) - std::get<0>(b)) / std::fabs(std::get<0>(a));
    ref.compute_at(w);
    ours.compute_at(w);
    const double c = 0.8;
    Eigen::MatrixXd xq(200, D);
    for (int i = 0; i < 200; ++i) for (int d = 0; d < D; ++d) xq(i, d) = uni();
    auto pa = ref.predict(xq);
    auto pb = ours.predict(xq);
    double merr = 0.0, serr = 0.0;
    for (int i = 0; i < 200; ++i) {
        merr = std::max(merr, std::fabs(pa.first(i, 0) - pb.first(i, 0)));
        serr = std::max(serr, std::fabs(pa.second(i, 0) - pb.second(i, 0)));
    }
    std::printf("M = %zu: |df|/|f| = %.2e, |dg|/|g|inf = %.2e, |dmu|/c = %.2e, |ds2|/c = %.2e\n", M, ferr, gerr / gmax, merr / c, serr / c);
    bool ok = ferr <= 1e-10 && gerr <= 1e-7 * gmax && merr <= 1e-9 * c && serr <= 1e-9 * c;
    // the public path: compute (reference initialisation + Rprop over the device likelihood), then query
    Ours model;
    model.compute(s, o);
    double rmse = 0.0, var = 0.0, ym = 0.0;
    for (int i = 0; i < N; ++i) ym += Y(i, 0) / N;
    for (int i = 0; i < N; ++i) {
        auto q = model.query(s[(size_t)i]);
        rmse += std::pow(std::get<0>(q)(0) - Y(i, 0), 2) / N;
        var += std::pow(Y(i, 0) - ym, 2) / N;
    }
    std::printf("compute: %d pseudo-inputs, rmse %.3e, std(y) %.3e\n", model.nb_pseudo_samples(), std::sqrt(rmse), std::sqrt(var));
    ok = ok && model.nb_pseudo_samples() == (int)M && std::sqrt(rmse) < std::sqrt(var);
    if (ok) std::printf("SPGP DROPIN OK\n");
    return ok ? 0 : 1;
}
