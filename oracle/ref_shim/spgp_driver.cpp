// oracle/ref_shim/spgp_driver.cpp — TEST INFRASTRUCTURE ONLY.
//
// Runs the REFERENCE'S OWN experimental::model::SPGP (experimental/model/spgp.hpp) with the dense linear algebra supplied by
// the stand-in in ./spgp_eigen: its _likelihood(w, true) (:446-580), and _compute(false) + _predict (:389-407, 582-610) at a
// fixed w.  Used to pin the restatement (oracle/spgp.py, tests/test_spgp_host.py) and to generate tests/golden/spgp/*.npz
// (tests/golden/make_golden_spgp.py).  No reference source is copied: this file only instantiates its templates.
#include <Eigen/Core> // first: the stand-in extended for spgp.hpp (spgp_eigen/Eigen/Core)
#include <algorithm>
#include <cstring>
#include <vector>

// the default optimiser template argument of SPGP names NLopt, which is not built here (no USE_NLOPT)
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

using namespace limbo;

struct Params {
    struct kernel : public defaults::kernel {};
    struct kernel_squared_exp_ard : public defaults::kernel_squared_exp_ard {};
    struct model_spgp : public defaults::model_spgp {};
    struct opt_rprop : public defaults::opt_rprop {};
};

using Model = model::SPGP<Params, kernel::SquaredExpARD<Params>, mean::Data<Params>, opt::Rprop<Params>>;

namespace {

// exposes the protected members of the reference's SPGP
struct Exposed : public Model {
    void init(const Eigen::MatrixXd& X, const Eigen::MatrixXd& Y, size_t m)
    {
        this->_init(X, Y);
        this->_m = m; // _init sets _m = max(samples_percent * N / 100, min_m); the caller's M is the same by default
    }
    double lik(const Eigen::VectorXd& w, double* grad) const
    {
        opt::eval_t r = this->_likelihood(w, true);
        const Eigen::VectorXd g = std::get<1>(r).get();
        std::copy(g.data(), g.data() + g.size(), grad);
        return std::get<0>(r);
    }
    // _compute(false) at HyperParams(w), as _optimize_hyperparams leaves the members (:436-443)
    void compute_at(const Eigen::VectorXd& w)
    {
        typename Model::HyperParams hp(w, this->_m, this->_dim_in);
        this->_pseudo_samples = hp.xb;
        this->_b = hp.b.transpose();
        this->_c = hp.c;
        this->_sig = hp.sig;
        this->_optimized = true;
        this->_compute(false);
    }
    std::pair<Eigen::MatrixXd, Eigen::MatrixXd> predict(const Eigen::MatrixXd& xt) const { return this->_predict(xt, true, true); }
    const Eigen::MatrixXd& L() const { return this->_matrixL; }
    const Eigen::MatrixXd& Lm() const { return this->_Lm; }
    const Eigen::MatrixXd& bet() const { return this->_bet; }
};

Eigen::MatrixXd rows(const double* p, long n, int d)
{
    Eigen::MatrixXd m(n, d);
    for (long i = 0; i < n; ++i)
        for (int j = 0; j < d; ++j) m(i, j) = p[i * d + j];
    return m;
}

} // namespace

extern "C" {

// X: N x D row-major, y: N observations (the model subtracts mean::Data itself), w: (M+1) D + 2, Xq: nq x D row-major.
// Out (each may be NULL): f = _likelihood value, grad ((M+1) D + 2), mu (nq, mean(v) included), s2 (nq), L and Lm (M x M
// column-major), bet (M).
int ref_spgp(long N, int D, const double* X, const double* y, long M, const double* w, long nq, const double* Xq, double* f, double* grad,
    double* mu, double* s2, double* L, double* Lm, double* bet)
{
    Exposed m;
    Eigen::MatrixXd Y(N, 1);
    for (long i = 0; i < N; ++i) Y(i, 0) = y[i];
    m.init(rows(X, N, D), Y, (size_t)M);
    const long nw = (M + 1) * D + 2;
    Eigen::VectorXd wv(nw);
    for (long i = 0; i < nw; ++i) wv(i) = w[i];
    std::vector<double> g((size_t)nw);
    const double fv = m.lik(wv, g.data());
    if (f) *f = fv;
    if (grad) std::copy(g.begin(), g.end(), grad);
    m.compute_at(wv);
    if (L) std::memcpy(L, m.L().data(), sizeof(double) * M * M);
    if (Lm) std::memcpy(Lm, m.Lm().data(), sizeof(double) * M * M);
    if (bet) std::memcpy(bet, m.bet().data(), sizeof(double) * M);
    if (nq > 0) {
        auto r = m.predict(rows(Xq, nq, D));
        for (long i = 0; i < nq; ++i) {
            if (mu) mu[i] = r.first(i, 0);
            if (s2) s2[i] = r.second(i, 0);
        }
    }
    return 0;
}

} // extern "C"
