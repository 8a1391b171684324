// tests/cpp/acq_grad_dropin_test.cpp — candidate gradients through the C++ drop-ins, compiled against the reference's own headers:
//   (1) limbo_b200::acqui::UCB / EI operator()(v, afun, true) (one lb_acq_grad) agrees with central differences of
//       operator()(v, afun, false) to 1e-6 relative, and bit for bit with GP::acq_grad over a batch that holds the same point;
//   (2) the reference's unmodified opt::GradientAscent and opt::Adam drive limbo_b200::acqui::UCB as the acquisition optimiser of
//       the inner loop of bayes_opt::BOptimizer::optimize (boptimizer.hpp:139-170; BOptimizer itself needs Boost.Parameter);
//   (3) limbo_b200::opt::BatchedGradient over the batch-aware UCB takes `iterations` gradient steps, one lb_acq_grad each, and
//       returns a point no worse than its random pass;
//   (4) over the reference's acqui::UCB it never calls f with gradient = true and returns the best point of its random pass.
// Needs a GPU to run; prints "ACQ GRAD DROPIN OK".  (Eigen is the stand-in from oracle/ref_shim.)
#include <cmath>
#include <cstdio>
#include <vector>

#include <Eigen/Core>
#include "dropin_common.hpp"

#include <limbo/acqui/ucb.hpp>
#include <limbo/kernel/matern_five_halves.hpp>
#include <limbo/mean/data.hpp>
#include <limbo/model/gp.hpp>
#include <limbo/opt/adam.hpp>
#include <limbo/opt/gradient_ascent.hpp>

#include <limbo_b200/model/gp.hpp>
#include <limbo_b200/opt/batched_gradient.hpp>

using namespace limbo;

struct Params {
    struct kernel : public defaults::kernel {};
    struct kernel_maternfivehalves : public defaults::kernel_maternfivehalves {};
    struct acqui_ucb : public defaults::acqui_ucb {};
    struct acqui_ei {
        BO_PARAM(double, jitter, 0.0);
    };
    struct opt_gradient_ascent : public defaults::opt_gradient_ascent {
        BO_PARAM(int, iterations, 40);
        BO_PARAM(double, alpha, 0.01);
    };
    struct opt_adam : public defaults::opt_adam {
        BO_PARAM(int, iterations, 40);
        BO_PARAM(double, alpha, 0.01);
    };
    struct opt_batchedgradient {
        BO_PARAM(int, candidates, 500);
        BO_PARAM(int, starts, 8);
        BO_PARAM(int, iterations, 25);
        BO_PARAM(double, alpha, 0.01);
    };
};

using GP_t = limbo_b200::model::GP<Params, kernel::MaternFiveHalves<Params>, mean::Data<Params>, model::gp::NoLFOpt<Params>>;

static Eigen::VectorXd target(const Eigen::VectorXd& x)
{
    Eigen::VectorXd y((Eigen::Index)1);
    y(0) = std::sin(5.0 * x(0)) * std::cos(3.0 * x(1)) + 0.3 * x(0);
    return y;
}

static void fit(GP_t& gp, int N, unsigned long long& seed)
{
    std::vector<Eigen::VectorXd> S, O;
    for (int i = 0; i < N; ++i) {
        Eigen::VectorXd x((Eigen::Index)2);
        x(0) = u01(seed);
        x(1) = u01(seed);
        S.push_back(x);
        O.push_back(target(x));
    }
    gp.compute(S, O);
}

template <typename Acq>
static int check_point_gradient(const GP_t& gp, const char* name, int acq_id, double p0, double p1, unsigned long long& seed)
{
    Acq acq(gp, 0);
    FirstElem afun;
    int bad = 0;
    double worst = 0;
    for (int t = 0; t < 6; ++t) {
        Eigen::VectorXd v((Eigen::Index)2);
        v(0) = 0.05 + 0.9 * u01(seed);
        v(1) = 0.05 + 0.9 * u01(seed);
        auto fg = acq(v, afun, true);
        const Eigen::VectorXd g = opt::grad(fg);
        const double h = 1e-5;
        double scale = std::max(std::max(std::fabs(g(0)), std::fabs(g(1))), 1e-3);
        for (int d = 0; d < 2; ++d) {
            Eigen::VectorXd a = v, b = v;
            a(d) += h;
            b(d) -= h;
            const double fd = (opt::fun(acq(a, afun, false)) - opt::fun(acq(b, afun, false))) / (2 * h);
            worst = std::max(worst, std::fabs(fd - g(d)) / scale);
            if (std::fabs(fd - g(d)) > 1e-6 * scale) ++bad;
        }
        // the same point inside a batch: bit for bit
        std::vector<Eigen::VectorXd> batch;
        for (int k = 0; k < 5; ++k) {
            Eigen::VectorXd w((Eigen::Index)2);
            w(0) = u01(seed);
            w(1) = u01(seed);
            batch.push_back(k == 3 ? v : w);
        }
        Eigen::VectorXd vals;
        Eigen::MatrixXd grads;
        gp.acq_grad(acq_id, acq_id == LB_ACQ_EI ? p0 : Params::acqui_ucb::alpha(), p1, batch, vals, grads);
        if (!(vals(3) == opt::fun(fg) && grads(3, 0) == g(0) && grads(3, 1) == g(1))) ++bad;
    }
    std::printf("%s: operator()(v, afun, true) vs central differences, max rel %.3e; batch bit-identical: %s\n", name, worst,
        bad ? "no" : "yes");
    return bad ? 1 : 0;
}

// the inner loop of BOptimizer::optimize with a reference optimiser as acquiopt
template <typename Opt>
static int run_loop(const char* name, unsigned long long& seed)
{
    GP_t gp(2, 1);
    fit(gp, 20, seed);
    Opt acqui_optimizer;
    FirstElem afun;
    int bad = 0;
    for (int it = 0; it < 5; ++it) {
        limbo_b200::acqui::UCB<Params, GP_t> acqui(gp, it);
        auto f = [&](const Eigen::VectorXd& x, bool g) { return acqui(x, afun, g); };
        Eigen::VectorXd start((Eigen::Index)2);
        start(0) = u01(seed);
        start(1) = u01(seed);
        const Eigen::VectorXd nx = acqui_optimizer(f, start, true);
        const double v0 = opt::eval(f, start), v1 = opt::eval(f, nx);
        if (!(std::isfinite(v1) && nx(0) >= 0 && nx(0) <= 1 && nx(1) >= 0 && nx(1) <= 1 && v1 >= v0 - 1e-12)) ++bad;
        gp.add_sample(nx, target(nx));
    }
    std::printf("%s drives limbo_b200::acqui::UCB in the BO loop: %s\n", name, bad ? "FAILED" : "ok");
    return bad ? 1 : 0;
}

int main()
{
    unsigned long long seed = 2024;
    GP_t gp(2, 1);
    fit(gp, 60, seed);
    int fails = 0;
    fails += check_point_gradient<limbo_b200::acqui::UCB<Params, GP_t>>(gp, "UCB", LB_ACQ_UCB, 0.0, 0.0, seed);
    { // EI's f_max: max_i mu(x_i), as the functor computes it (ei.hpp:100-108)
        Eigen::MatrixXd mus;
        Eigen::VectorXd s2;
        gp.query_batch(gp.samples(), mus, s2);
        double f_max = -1e300;
        for (long i = 0; i < (long)mus.rows(); ++i) f_max = std::max(f_max, mus(i, 0));
        fails += check_point_gradient<limbo_b200::acqui::EI<Params, GP_t>>(gp, "EI", LB_ACQ_EI, f_max, 0.0, seed);
    }
    fails += run_loop<opt::GradientAscent<Params>>("opt::GradientAscent", seed);
    fails += run_loop<opt::Adam<Params>>("opt::Adam", seed);

    { // BatchedGradient over the batch-aware UCB
        limbo_b200::acqui::UCB<Params, GP_t> acqui(gp, 0);
        FirstElem afun;
        long grad_calls = 0;
        std::vector<std::pair<Eigen::VectorXd, double>> seen;
        auto f = [&](const Eigen::VectorXd& x, bool g) {
            if (g) ++grad_calls;
            return acqui(x, afun, g);
        };
        limbo_b200::opt::BatchedGradient<Params> bg;
        Eigen::VectorXd init = Eigen::VectorXd::Zero(2);
        const Eigen::VectorXd x = bg(f, init, true);
        const bool ok = bg.grad_steps() == Params::opt_batchedgradient::iterations() && grad_calls == 0 && x(0) >= 0 && x(0) <= 1
            && x(1) >= 0 && x(1) <= 1;
        std::printf("BatchedGradient over limbo_b200::acqui::UCB: %d gradient steps (one lb_acq_grad each), value %.6f: %s\n",
            bg.grad_steps(), opt::eval(f, x), ok ? "ok" : "FAILED");
        fails += ok ? 0 : 1;
    }
    { // BatchedGradient over the reference's acqui::UCB: no gradient request, the random pass's best point
        acqui::UCB<Params, GP_t> acqui(gp, 0);
        FirstElem afun;
        long grad_calls = 0;
        double best = -1e300;
        Eigen::VectorXd best_x;
        auto f = [&](const Eigen::VectorXd& x, bool g) {
            if (g) ++grad_calls;
            auto r = acqui(x, afun, false);
            if (opt::fun(r) > best) { best = opt::fun(r); best_x = x; }
            return r;
        };
        limbo_b200::opt::BatchedGradient<Params> bg;
        Eigen::VectorXd init = Eigen::VectorXd::Zero(2);
        const Eigen::VectorXd x = bg(f, init, true);
        const bool ok = grad_calls == 0 && bg.grad_steps() == 0 && x(0) == best_x(0) && x(1) == best_x(1);
        std::printf("BatchedGradient over the reference's acqui::UCB: %ld gradient calls, random-pass best returned: %s\n", grad_calls,
            ok ? "ok" : "FAILED");
        fails += ok ? 0 : 1;
    }
    if (fails == 0) std::printf("ACQ GRAD DROPIN OK\n");
    return fails ? 1 : 0;
}
