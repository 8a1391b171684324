// tests/cpp/pair_grad_dropin_test.cpp — gradients of the two-model acquisitions through the C++ drop-ins, compiled against the
// reference's own headers:
//   (1) limbo_b200::acqui::ECI operator()(v, afun, true) (one lb_eci_grad) agrees with central differences of operator()(v, afun,
//       false) to 1e-6 relative, and bit for bit with GP::eci_grad over a batch that holds the same point;
//   (2) the reference's unmodified opt::Adam drives limbo_b200::acqui::ECI in experimental::bayes_opt::CBOptimizer's inner loop
//       (cboptimizer.hpp:171-176: acqui(x, afun, g) handed to the acquisition optimiser);
//   (3) limbo_b200::opt::BatchedGradient in that loop takes grad_steps() > 0 (one lb_eci_grad each) and returns a point no worse
//       than its random pass;
//   (4) limbo_b200::opt::BatchedGradient in experimental::bayes_opt::Ehvi's inner loop (ehvi.hpp:134-137: opt::no_grad(acqui(x)),
//       never a gradient flag) over the acqui::Ehvi specialisation takes grad_steps() > 0 (one lb_ehvi_grad each), and the
//       specialisation's GradRequest answer agrees with central differences of its own values.
// CBOptimizer and Ehvi themselves need Boost.Parameter (bayes_opt/bo_base.hpp), which the stand-in does not provide, so their
// inner loops are restated here with the reference's own lambdas.  Needs a GPU to run; prints "PAIR GRAD DROPIN OK".
#include <cmath>
#include <cstdio>
#include <deque>
#include <vector>

#include <Eigen/Core>

#include "dropin_common.hpp"

#include <limbo/kernel/exp.hpp>
#include <limbo/kernel/matern_five_halves.hpp>
#include <limbo/kernel/squared_exp_ard.hpp>
#include <limbo/mean/constant.hpp>
#include <limbo/mean/data.hpp>
#include <limbo/model/gp.hpp>
#include <limbo/opt/adam.hpp>

#include <limbo_b200/acqui/ehvi.hpp>
#include <limbo_b200/model/gp.hpp>
#include <limbo_b200/opt/batched_gradient.hpp>

using namespace limbo;

struct Params {
    struct kernel : public defaults::kernel {};
    struct kernel_squared_exp_ard : public defaults::kernel_squared_exp_ard {};
    struct kernel_exp : public defaults::kernel_exp {};
    struct kernel_maternfivehalves : public defaults::kernel_maternfivehalves {};
    struct acqui_eci {
        BO_PARAM(double, jitter, 0.0);
    };
    struct mean_constant {
        BO_PARAM(double, constant, 0.5);
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

using ObjGP = limbo_b200::model::GP<Params, kernel::SquaredExpARD<Params>, mean::Data<Params>, model::gp::NoLFOpt<Params>>;
using ConGP = limbo_b200::model::GP<Params, kernel::Exp<Params>, mean::Constant<Params>, model::gp::NoLFOpt<Params>>;
using MoGP = limbo_b200::model::GP<Params, kernel::MaternFiveHalves<Params>, mean::Data<Params>, model::gp::NoLFOpt<Params>>;
using ECI_t = limbo_b200::acqui::ECI<Params, ObjGP, ConGP>;

static Eigen::VectorXd point(unsigned long long& seed, double lo = 0.0, double hi = 1.0)
{
    Eigen::VectorXd x((Eigen::Index)2);
    x(0) = lo + (hi - lo) * u01(seed);
    x(1) = lo + (hi - lo) * u01(seed);
    return x;
}

static Eigen::VectorXd objective(const Eigen::VectorXd& x)
{
    return Eigen::VectorXd::Constant(1, std::sin(5.0 * x(0)) * std::cos(3.0 * x(1)) + 0.3 * x(0));
}
static Eigen::VectorXd constraint(const Eigen::VectorXd& x) { return Eigen::VectorXd::Constant(1, 1.0 + std::cos(4.0 * x(0) + x(1))); }
static Eigen::VectorXd objective2(const Eigen::VectorXd& x) { return Eigen::VectorXd::Constant(1, std::cos(3.0 * x(0)) - 0.5 * x(1)); }

static void fit_pair(ObjGP& o, ConGP& c, int N, unsigned long long& seed)
{
    std::vector<Eigen::VectorXd> S, Yo, Yc;
    for (int i = 0; i < N; ++i) {
        S.push_back(point(seed));
        Yo.push_back(objective(S.back()));
        Yc.push_back(constraint(S.back()));
    }
    o.compute(S, Yo);
    c.compute(S, Yc);
}

static int check_eci_point_gradient(const ObjGP& o, const ConGP& c, unsigned long long& seed)
{
    ECI_t acq(o, c, 0);
    FirstElem afun;
    int bad = 0, live = 0;
    double worst = 0;
    for (int t = 0; t < 16; ++t) {
        const Eigen::VectorXd v = point(seed, 0.05, 0.95);
        auto fg = acq(v, afun, true);
        const Eigen::VectorXd g = opt::grad(fg);
        const double h = 1e-5, scale = std::max(std::max(std::fabs(g(0)), std::fabs(g(1))), 1e-3);
        if (std::max(std::fabs(g(0)), std::fabs(g(1))) > 1e-3) ++live;
        for (int d = 0; d < 2; ++d) {
            Eigen::VectorXd a = v, b = v;
            a(d) += h;
            b(d) -= h;
            const double fd = (opt::fun(acq(a, afun, false)) - opt::fun(acq(b, afun, false))) / (2 * h);
            worst = std::max(worst, std::fabs(fd - g(d)) / scale);
            if (std::fabs(fd - g(d)) > 1e-6 * scale) ++bad;
        }
        std::vector<Eigen::VectorXd> batch;
        for (int k = 0; k < 5; ++k) batch.push_back(k == 2 ? v : point(seed));
        Eigen::MatrixXd mus;
        Eigen::VectorXd s2, vals;
        Eigen::MatrixXd grads;
        o.query_batch(o.samples(), mus, s2);
        double f_max = -1e300;
        for (long i = 0; i < (long)mus.rows(); ++i) f_max = std::max(f_max, mus(i, 0));
        o.eci_grad(c, f_max, Params::acqui_eci::jitter(), batch, vals, grads);
        if (!(vals(2) == opt::fun(fg) && grads(2, 0) == g(0) && grads(2, 1) == g(1))) ++bad;
    }
    std::printf("ECI: operator()(v, afun, true) vs central differences at %d points with |grad| > 1e-3, max rel %.3e; batch "
                "bit-identical: %s\n", live, worst, bad ? "no" : "yes");
    return (bad || live < 3) ? 1 : 0;
}

// CBOptimizer's inner loop (cboptimizer.hpp:171-176) with acquiopt Opt for `iters` iterations; returns the failures
template <bool Batched, typename Opt>
static int cb_loop(const char* name, Opt& acqui_optimizer, unsigned long long& seed, int* steps)
{
    ObjGP o(2, 1);
    ConGP c(2, 1);
    fit_pair(o, c, 20, seed);
    FirstElem afun;
    int bad = 0;
    for (int it = 0; it < 5; ++it) {
        ECI_t acqui(o, c, it);
        long grad_calls = 0;
        auto acqui_optimization = [&](const Eigen::VectorXd& x, bool g) {
            if (g) ++grad_calls;
            return acqui(x, afun, g);
        };
        const Eigen::VectorXd start = point(seed);
        const Eigen::VectorXd nx = acqui_optimizer(acqui_optimization, start, true);
        const double v0 = opt::fun(acqui(start, afun, false)), v1 = opt::fun(acqui(nx, afun, false));
        if (!(std::isfinite(v1) && nx(0) >= 0 && nx(0) <= 1 && nx(1) >= 0 && nx(1) <= 1 && v1 >= v0 - 1e-12)) ++bad;
        if constexpr (Batched) { // gradient steps through GradRequest, never a gradient flag
            *steps += acqui_optimizer.grad_steps();
            if (acqui_optimizer.grad_steps() <= 0 || grad_calls != 0) ++bad;
        }
        else if (grad_calls == 0)
            ++bad; // opt::Adam asks for gradients
        o.add_sample(nx, objective(nx));
        c.add_sample(nx, constraint(nx));
    }
    std::printf("%s drives limbo_b200::acqui::ECI in CBOptimizer's inner loop: %s\n", name, bad ? "FAILED" : "ok");
    return bad;
}

static int ehvi_loop(unsigned long long& seed)
{
    std::vector<Eigen::VectorXd> S;
    std::vector<Eigen::VectorXd> Y0, Y1;
    for (int i = 0; i < 12; ++i) { // few samples: wide posteriors, so that most candidates may still improve the front
        S.push_back(point(seed));
        Y0.push_back(objective(S.back()));
        Y1.push_back(objective2(S.back()));
    }
    std::vector<MoGP> models;
    models.emplace_back(2, 1);
    models.emplace_back(2, 1);
    models[0].compute(S, Y0);
    models[1].compute(S, Y1);
    std::vector<individual> store;
    for (size_t i = 0; i < S.size(); ++i) { // the data's non-dominated points (maximisation)
        bool dominated = false;
        for (size_t j = 0; j < S.size() && !dominated; ++j)
            dominated = (Y0[j](0) >= Y0[i](0) && Y1[j](0) >= Y1[i](0)) && (Y0[j](0) > Y0[i](0) || Y1[j](0) > Y1[i](0));
        if (!dominated) {
            individual p;
            p.f[0] = Y0[i](0);
            p.f[1] = Y1[i](0);
            p.f[2] = 0;
            store.push_back(p);
        }
    }
    std::deque<individual*> pop;
    for (auto& p : store) pop.push_back(&p);
    Eigen::VectorXd r(3);
    r << -1.5, -1.5, 0.0;
    acqui::Ehvi<Params, MoGP> acqui(models, pop, r);
    // Ehvi's inner loop (ehvi.hpp:134-137)
    limbo_b200::opt::BatchedGradient<Params> inner_opt;
    long grad_calls = 0;
    auto acqui_optimization = [&](const Eigen::VectorXd& x, bool g) {
        if (g) ++grad_calls;
        return opt::no_grad(acqui(x));
    };
    const Eigen::VectorXd x = inner_opt(acqui_optimization, point(seed), true);
    int bad = 0;
    const bool ok = inner_opt.grad_steps() == Params::opt_batchedgradient::iterations() && grad_calls == 0 && x(0) >= 0 && x(0) <= 1
        && x(1) >= 0 && x(1) <= 1 && std::isfinite(acqui(x));
    // the GradRequest answer against central differences of the specialisation's own values
    std::vector<Eigen::VectorXd> pts;
    for (int k = 0; k < 12; ++k) { // around the returned point, where EHVI is not 0 (a candidate the front dominates scores 0)
        Eigen::VectorXd p = x + (point(seed) - Eigen::VectorXd::Constant(2, 0.5)) * 0.2;
        for (int d = 0; d < 2; ++d) p(d) = std::min(0.95, std::max(0.05, p(d)));
        pts.push_back(p);
    }
    limbo_b200::opt::GradRequest greq;
    greq.points = &pts;
    limbo_b200::opt::current_grad_batch() = &greq;
    acqui(pts[0]);
    limbo_b200::opt::current_grad_batch() = nullptr;
    double worst = 0;
    int live = 0; // points where EHVI has a gradient
    if (!greq.answered) ++bad;
    else
        for (size_t k = 0; k < pts.size(); ++k) {
            const double gmax = std::max(std::fabs(greq.grads((Eigen::Index)k, 0)), std::fabs(greq.grads((Eigen::Index)k, 1)));
            const double scale = std::max(gmax, 1e-3);
            if (gmax > 1e-3) ++live;
            // one point scores on the small-batch path, the request on the panel path: equal to 1e-12
            if (std::fabs(greq.values((Eigen::Index)k) - acqui(pts[k])) > 1e-12 * std::max(1.0, std::fabs(acqui(pts[k])))) ++bad;
            for (int d = 0; d < 2; ++d) {
                Eigen::VectorXd a = pts[k], b = pts[k];
                a(d) += 1e-6;
                b(d) -= 1e-6;
                const double fd = (acqui(a) - acqui(b)) / 2e-6, e = std::fabs(fd - greq.grads((Eigen::Index)k, d)) / scale;
                worst = std::max(worst, e);
                if (e > 1e-6) ++bad;
            }
        }
    if (!ok || live < 6) ++bad;
    std::printf("Ehvi (k = %zu): GradRequest vs central differences at %d points with |grad| > 1e-3, max rel %.3e; BatchedGradient in Ehvi's inner loop: %d gradient "
                "steps, ehvi(x) = %.6e: %s\n",
        pop.size(), live, worst, inner_opt.grad_steps(), acqui(x), bad ? "FAILED" : "ok");
    return bad;
}

int main()
{
    unsigned long long seed = 2025;
    int fails = 0;
    {
        ObjGP o(2, 1);
        ConGP c(2, 1);
        fit_pair(o, c, 8, seed); // few samples: ECI and its gradient are far from 0 between them
        fails += check_eci_point_gradient(o, c, seed);
    }
    {
        opt::Adam<Params> adam;
        fails += cb_loop<false>("opt::Adam", adam, seed, nullptr);
    }
    {
        limbo_b200::opt::BatchedGradient<Params> bg;
        int steps = 0;
        fails += cb_loop<true>("limbo_b200::opt::BatchedGradient", bg, seed, &steps);
        std::printf("BatchedGradient in CBOptimizer's inner loop: %d gradient steps over 5 iterations (one lb_eci_grad each)\n", steps);
    }
    fails += ehvi_loop(seed);
    if (fails == 0) std::printf("PAIR GRAD DROPIN OK\n");
    return fails ? 1 : 0;
}
