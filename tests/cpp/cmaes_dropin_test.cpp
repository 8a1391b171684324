// tests/cpp/cmaes_dropin_test.cpp — the batched CMA-ES through the C++ drop-ins, compiled against the reference's own headers:
//   (1) limbo_b200::opt::BatchedCmaes over the batch-aware limbo_b200::acqui::UCB and EI answers its CmaesRequest with one
//       lb_acq_cmaes (n_evals > 0) and returns a point in the box no worse than the best of its random pass;
//   (2) over the reference's acqui::UCB it runs the random pass one point at a time, requests no search and returns the best
//       point of that pass;
//   (3) over the acqui::Ehvi specialisation with three device models on a three-objective DTLZ2 it answers the request with one
//       lb_ehvi_cmaes and returns a point whose EHVI is no worse than the best of the random pass.
// Needs a GPU to run; prints "CMAES DROPIN OK".  (Eigen is the stand-in from oracle/ref_shim.)
#include <cmath>
#include <cstdio>
#include <deque>
#include <vector>

#include <Eigen/Core>
#include "dropin_common.hpp"

#include <limbo/acqui/ucb.hpp>
#include <limbo/experimental/tools/pareto.hpp>
#include <limbo/kernel/matern_five_halves.hpp>
#include <limbo/mean/data.hpp>
#include <limbo/model/gp.hpp>

#include <limbo_b200/acqui/ehvi.hpp>
#include <limbo_b200/model/gp.hpp>
#include <limbo_b200/opt/batched_cmaes.hpp>

using namespace limbo;

struct Params {
    struct kernel : public defaults::kernel {};
    struct kernel_maternfivehalves : public defaults::kernel_maternfivehalves {};
    struct acqui_ucb : public defaults::acqui_ucb {};
    struct acqui_ei {
        BO_PARAM(double, jitter, 0.0);
    };
    struct opt_batchedcmaes : public limbo_b200::defaults::opt_batchedcmaes {
        BO_PARAM(int, candidates, 500);
        BO_PARAM(int, starts, 8);
        BO_PARAM(int, generations, 30);
    };
};

using GP_t = limbo_b200::model::GP<Params, kernel::MaternFiveHalves<Params>, mean::Data<Params>, model::gp::NoLFOpt<Params>>;

static Eigen::VectorXd dtlz2(const Eigen::VectorXd& x) // three objectives, negated so that they are maximised
{
    double g = 0;
    for (int d = 2; d < x.size(); ++d) g += (x(d) - 0.5) * (x(d) - 0.5);
    const double a = x(0) * M_PI / 2, b = x(1) * M_PI / 2;
    Eigen::VectorXd r(3);
    r(0) = -(1 + g) * std::cos(a) * std::cos(b);
    r(1) = -(1 + g) * std::cos(a) * std::sin(b);
    r(2) = -(1 + g) * std::sin(a);
    return r;
}

static bool in_box(const Eigen::VectorXd& x)
{
    for (int d = 0; d < x.size(); ++d)
        if (!(x(d) >= 0.0 && x(d) <= 1.0)) return false;
    return true;
}

// BatchedCmaes over f, and the best value f takes over the random pass (recorded while no device search runs)
template <typename F>
static int check(const char* name, F&& eval, int D, bool expect_search)
{
    double pass_best = -INFINITY;
    long calls = 0;
    auto f = [&](const Eigen::VectorXd& x, bool) {
        ++calls;
        const double v = eval(x);
        if (!limbo_b200::opt::current_cmaes() && v > pass_best) pass_best = v;
        return opt::no_grad(v);
    };
    limbo_b200::opt::BatchedCmaes<Params> bc;
    const Eigen::VectorXd x = bc(f, Eigen::VectorXd::Constant(D, 0.5), true);
    const double vx = eval(x);
    const bool searched = bc.n_evals() > 0;
    const bool ok = in_box(x) && searched == expect_search && vx >= pass_best - 1e-12 * std::fabs(pass_best)
        && (expect_search ? calls == 2 : calls == Params::opt_batchedcmaes::candidates());
    std::printf("%s: %ld calls of f, %lld search evaluations, value %.6e (random pass best %.6e): %s\n", name, calls,
        (long long)bc.n_evals(), vx, pass_best, ok ? "ok" : "FAILED");
    return ok ? 0 : 1;
}

int main()
{
    unsigned long long seed = 11;
    int fails = 0;
    const int D = 4;
    std::vector<Eigen::VectorXd> X, obs[3], single;
    for (int i = 0; i < 60; ++i) {
        Eigen::VectorXd x((Eigen::Index)D);
        for (int d = 0; d < D; ++d) x(d) = u01(seed);
        const Eigen::VectorXd y = dtlz2(x);
        X.push_back(x);
        for (int j = 0; j < 3; ++j) obs[j].push_back(Eigen::VectorXd::Constant(1, y(j)));
    }
    GP_t gp(D, 1);
    gp.compute(X, obs[2]);
    FirstElem afun;
    {
        limbo_b200::acqui::UCB<Params, GP_t> ucb(gp, 0);
        fails += check("BatchedCmaes over limbo_b200::acqui::UCB", [&](const Eigen::VectorXd& x) { return opt::fun(ucb(x, afun, false)); }, D,
            true);
        limbo_b200::acqui::EI<Params, GP_t> ei(gp, 0);
        fails += check("BatchedCmaes over limbo_b200::acqui::EI", [&](const Eigen::VectorXd& x) { return opt::fun(ei(x, afun, false)); }, D,
            true);
        acqui::UCB<Params, GP_t> ref_ucb(gp, 0);
        fails += check("BatchedCmaes over the reference's acqui::UCB", [&](const Eigen::VectorXd& x) { return opt::fun(ref_ucb(x, afun, false)); },
            D, false);
    }
    {
        std::vector<GP_t> gps;
        for (int j = 0; j < 3; ++j) gps.emplace_back(D, 1);
        std::vector<std::tuple<Eigen::VectorXd, Eigen::VectorXd, Eigen::VectorXd>> packed;
        for (size_t i = 0; i < X.size(); ++i) packed.emplace_back(X[i], dtlz2(X[i]), Eigen::VectorXd::Zero(3));
        for (int j = 0; j < 3; ++j) gps[(size_t)j].compute(X, obs[j]);
        auto front = pareto::pareto_set<1>(packed);
        std::vector<individual> store(front.size());
        std::deque<individual*> pop;
        for (size_t i = 0; i < front.size(); ++i) {
            for (int d = 0; d < 3; ++d) store[i].f[d] = std::get<1>(front[i])(d);
            pop.push_back(&store[i]);
        }
        Eigen::VectorXd r(3);
        r << -11.0, -11.0, -11.0;
        acqui::Ehvi<Params, GP_t> ehvi(gps, pop, r);
        fails += check("BatchedCmaes over acqui::Ehvi (three device models)", [&](const Eigen::VectorXd& x) { return ehvi(x); }, D, true);
    }
    if (fails == 0) std::printf("CMAES DROPIN OK\n");
    return fails ? 1 : 0;
}
