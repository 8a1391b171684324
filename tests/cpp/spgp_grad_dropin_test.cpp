// tests/cpp/spgp_grad_dropin_test.cpp — the batch-aware acquisitions over limbo_b200::model::SPGP, next to the reference's
// experimental::model::SPGP at the same w; built by oracle/ref_shim/Makefile's spgp_grad_dropin_test against the Eigen stand-in
// of oracle/ref_shim/spgp_eigen and run by tests/test_gpu_spgp_grad.py:
//   (1) limbo_b200::acqui::UCB / EI operator()(v, afun, true) (one lb_spgp_acq_grad) agrees with central differences of
//       operator()(v, afun, false) to 1e-6 relative;
//   (2) BatchedRandom's BatchRequest is answered with one device argmax (lb_spgp_acq_argmax: the launches of one SPGP::acq_argmax
//       plus the functor's own one-point query), and every filed value equals the reference SPGP's one-point UCB / EI to 1e-10;
//   (3) limbo_b200::opt::BatchedGradient takes grad_steps() > 0 gradient steps and returns a point no worse than its random pass.
// Needs a GPU to run; prints "SPGP GRAD DROPIN OK".
#include <Eigen/Core>
#include <cmath>
#include <cstdio>
#include <vector>
#include "dropin_common.hpp"

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
#include <limbo_b200/opt/batched_gradient.hpp>

using namespace limbo;

struct Params {
    struct kernel : public defaults::kernel {};
    struct kernel_squared_exp_ard : public defaults::kernel_squared_exp_ard {};
    struct model_spgp : public defaults::model_spgp {};
    struct opt_rprop : public defaults::opt_rprop {};
    struct acqui_ucb {
        BO_PARAM(double, alpha, 0.5);
    };
    struct acqui_ei {
        BO_PARAM(double, jitter, 0.01);
    };
    struct opt_batchedgradient {
        BO_PARAM(int, candidates, 500);
        BO_PARAM(int, starts, 8);
        BO_PARAM(int, iterations, 25);
        BO_PARAM(double, alpha, 0.01);
    };
};
using Kern = kernel::SquaredExpARD<Params>;
using Mean = mean::Data<Params>;
using Ref = model::SPGP<Params, Kern, Mean, opt::Rprop<Params>>;
using Ours = limbo_b200::model::SPGP<Params, Kern, Mean, opt::Rprop<Params>>;

struct RefX : Ref {
    void init(const Eigen::MatrixXd& X, const Eigen::MatrixXd& Y) { this->_init(X, Y); }
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

// the acquisitions are instantiated over Ours itself (their gradient path is selected on the model type), OursX only reaches the
// protected set-up and the launch counter
struct OursX : Ours {
    void init(const std::vector<Eigen::VectorXd>& s, const std::vector<Eigen::VectorXd>& o) { this->_init(s, o); }
    void compute_at(const Eigen::VectorXd& w)
    {
        this->_optimized = true;
        this->_compute_at(w);
    }
    long long launches() const { return lb_spgp_launch_count(this->_h); }
};

static double uni(unsigned& st)
{
    st = st * 1664525u + 1013904223u;
    return (double)(st >> 8) / (double)(1u << 24);
}

template <typename Acq>
static int check_point_gradient(const OursX& model, const char* name, unsigned& st)
{
    Acq acq(model, 0);
    FirstElem afun;
    int bad = 0;
    double worst = 0;
    const int D = model.dim_in();
    for (int t = 0; t < 6; ++t) {
        Eigen::VectorXd v(D);
        for (int d = 0; d < D; ++d) v(d) = 0.05 + 0.9 * uni(st);
        auto fg = acq(v, afun, true);
        const Eigen::VectorXd g = opt::grad(fg);
        double scale = 1e-3;
        for (int d = 0; d < D; ++d) scale = std::max(scale, std::fabs(g(d)));
        const double h = 1e-5;
        for (int d = 0; d < D; ++d) {
            Eigen::VectorXd a = v, b = v;
            a(d) += h;
            b(d) -= h;
            const double fd = (opt::fun(acq(a, afun, false)) - opt::fun(acq(b, afun, false))) / (2 * h);
            worst = std::max(worst, std::fabs(fd - g(d)) / scale);
            if (std::fabs(fd - g(d)) > 1e-6 * scale) ++bad;
        }
    }
    std::printf("%s over SPGP: operator()(v, afun, true) vs central differences, max rel %.3e: %s\n", name, worst, bad ? "FAILED" : "ok");
    return bad ? 1 : 0;
}

// BatchedRandom's request through the functor: one device argmax, values against the reference's one-point acquisition
template <typename Acq, typename RefValue>
static int check_batch(const OursX& model, const char* name, const std::vector<Eigen::VectorXd>& cands, const RefValue& ref_value)
{
    Acq acq(model, 0);
    FirstElem afun;
    acq(cands[0], afun, false); // EI refreshes f_max here, outside the counted call
    std::vector<double> direct;
    long long l0 = model.launches();
    model.query(cands[0]);
    const long long per_query = model.launches() - l0;
    l0 = model.launches();
    model.acq_argmax(0, 0.0, 0.0, cands, &direct);
    const long long per_argmax = model.launches() - l0;
    std::vector<double> values;
    limbo_b200::opt::BatchRequest req;
    req.candidates = &cands;
    req.values = &values;
    limbo_b200::opt::current_batch() = &req;
    l0 = model.launches();
    acq(cands[0], afun, false);
    const long long used = model.launches() - l0;
    limbo_b200::opt::current_batch() = nullptr;
    double worst = 0.0;
    long best_i = 0;
    for (size_t i = 0; i < cands.size(); ++i) {
        const double r = ref_value(cands[i]);
        worst = std::max(worst, std::fabs(values[i] - r) / std::max(1.0, std::fabs(r)));
        if (values[i] > values[(size_t)best_i]) best_i = (long)i;
    }
    const bool ok = req.answered && req.gradients && used == per_argmax + per_query && values.size() == cands.size() && worst <= 1e-10
        && req.best_index == best_i && req.best_value == values[(size_t)best_i];
    std::printf("%s BatchRequest over SPGP: answered %d, %lld launches (argmax %lld + query %lld), max rel vs reference %.3e: %s\n", name,
        (int)req.answered, used, per_argmax, per_query, worst, ok ? "ok" : "FAILED");
    return ok ? 0 : 1;
}

template <typename Acq>
static int check_batched_gradient(const OursX& model, const char* name)
{
    Acq acq(model, 0);
    FirstElem afun;
    double random_best = -INFINITY;
    long grad_calls = 0;
    auto f = [&](const Eigen::VectorXd& x, bool g) {
        if (g) ++grad_calls;
        limbo_b200::opt::BatchRequest* req = limbo_b200::opt::current_batch();
        auto r = acq(x, afun, g);
        if (req && req->answered) random_best = std::max(random_best, req->best_value);
        return r;
    };
    limbo_b200::opt::BatchedGradient<Params> bg;
    const Eigen::VectorXd x = bg(f, Eigen::VectorXd::Zero(model.dim_in()), true);
    const double vx = opt::eval(f, x);
    bool inside = true;
    for (int d = 0; d < (int)x.size(); ++d) inside = inside && x(d) >= 0.0 && x(d) <= 1.0;
    const bool ok = bg.grad_steps() > 0 && grad_calls == 0 && inside && vx >= random_best - 1e-12;
    std::printf("BatchedGradient over limbo_b200::acqui::%s<SPGP>: %d gradient steps, value %.6f vs random pass %.6f: %s\n", name,
        bg.grad_steps(), vx, random_best, ok ? "ok" : "FAILED");
    return ok ? 0 : 1;
}

int main()
{
    const int N = 300, D = 3;
    std::vector<Eigen::VectorXd> s, o;
    Eigen::MatrixXd X(N, D), Y(N, 1);
    unsigned st = 777u;
    for (int i = 0; i < N; ++i) {
        Eigen::VectorXd x(D);
        double y = 0.0;
        for (int d = 0; d < D; ++d) { x(d) = uni(st); X(i, d) = x(d); y += std::sin(3.0 * x(d)); }
        s.push_back(x);
        o.push_back(Eigen::VectorXd::Constant(1, y));
        Y(i, 0) = y;
    }
    RefX ref;
    ref.init(X, Y);
    OursX ours;
    ours.init(s, o);
    const size_t M = ref.m();
    Eigen::VectorXd w((M + 1) * D + 2);
    for (size_t i = 0; i < M; ++i)
        for (int d = 0; d < D; ++d) w(i * D + d) = X((7 * i) % N, d) + 0.01 * std::cos((double)(i * D + d));
    for (int d = 0; d < D; ++d) w(M * D + d) = 2.0 + 0.1 * d;
    w((M + 1) * D) = std::log(0.8);
    w((M + 1) * D + 1) = std::log(0.05);
    ref.compute_at(w);
    ours.compute_at(w);

    int fails = 0;
    fails += check_point_gradient<limbo_b200::acqui::UCB<Params, Ours>>(ours, "UCB", st);
    fails += check_point_gradient<limbo_b200::acqui::EI<Params, Ours>>(ours, "EI", st);

    std::vector<Eigen::VectorXd> cands;
    for (int i = 0; i < 1000; ++i) {
        Eigen::VectorXd v(D);
        for (int d = 0; d < D; ++d) v(d) = uni(st);
        cands.push_back(v);
    }
    auto ref_mu_s2 = [&](const Eigen::VectorXd& v) { // the reference's one-point query (spgp.hpp:193-197)
        Eigen::MatrixXd xt(1, D);
        for (int d = 0; d < D; ++d) xt(0, d) = v(d);
        auto p = ref.predict(xt);
        return std::make_pair(p.first(0, 0), p.second(0, 0));
    };
    fails += check_batch<limbo_b200::acqui::UCB<Params, Ours>>(ours, "UCB", cands, [&](const Eigen::VectorXd& v) {
        auto q = ref_mu_s2(v);
        return q.first + Params::acqui_ucb::alpha() * std::sqrt(q.second);
    });
    double f_max = -INFINITY; // ei.hpp:100-108 over the reference's own posterior mean
    for (const auto& x : s) f_max = std::max(f_max, ref_mu_s2(x).first);
    fails += check_batch<limbo_b200::acqui::EI<Params, Ours>>(ours, "EI", cands, [&](const Eigen::VectorXd& v) { // ei.hpp:85-116
        auto q = ref_mu_s2(v);
        const double sigma = std::sqrt(q.second);
        if (sigma < 1e-10) return 0.0;
        const double Xv = q.first - f_max - Params::acqui_ei::jitter();
        const double Z = Xv / sigma;
        const double phi = std::exp(-0.5 * std::pow(Z, 2.0)) / std::sqrt(2.0 * M_PI);
        const double Phi = 0.5 * std::erfc(-Z / std::sqrt(2));
        return Xv * Phi + sigma * phi;
    });
    fails += check_batched_gradient<limbo_b200::acqui::UCB<Params, Ours>>(ours, "UCB");
    fails += check_batched_gradient<limbo_b200::acqui::EI<Params, Ours>>(ours, "EI");
    if (fails == 0) std::printf("SPGP GRAD DROPIN OK\n");
    return fails ? 1 : 0;
}
