// tests/cpp/cmaes_eci_spgp_dropin_test.cpp — the batched CMA-ES over ECI and over SPGP through the C++ drop-ins, compiled against
// the reference's own headers and the Eigen stand-in of oracle/ref_shim/spgp_eigen:
//   (1) limbo_b200::opt::BatchedCmaes in experimental::bayes_opt::CBOptimizer's inner loop (cboptimizer.hpp:171-176: a fresh
//       acquisition per iteration, acqui(x, afun, g) handed to the acquisition optimiser) over the batch-aware
//       limbo_b200::acqui::ECI answers its CmaesRequest with one lb_eci_cmaes in every iteration (two calls of f, n_evals > 0)
//       and returns a point in the box no worse than the best of its random pass;
//   (2) BatchedCmaes over the batch-aware limbo_b200::acqui::UCB and EI on limbo_b200::model::SPGP does the same through one
//       lb_spgp_acq_cmaes.
// CBOptimizer itself needs Boost.Parameter (bayes_opt/bo_base.hpp), which the stand-in does not provide, so its inner loop is
// restated here with the reference's own lambda.  Needs a GPU to run; prints "CMAES ECI SPGP DROPIN OK".
#include <Eigen/Core>
#include <cmath>
#include <cstdio>
#include <vector>
#include "dropin_common.hpp"

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
    struct acqui_eci {
        BO_PARAM(double, jitter, 0.0);
    };
    struct acqui_ucb {
        BO_PARAM(double, alpha, 0.5);
    };
    struct acqui_ei {
        BO_PARAM(double, jitter, 0.01);
    };
    struct mean_constant {
        BO_PARAM(double, constant, 0.5);
    };
    struct opt_batchedcmaes : public limbo_b200::defaults::opt_batchedcmaes {
        BO_PARAM(int, candidates, 500);
        BO_PARAM(int, starts, 8);
        BO_PARAM(int, generations, 30);
    };
};

using ObjGP = limbo_b200::model::GP<Params, kernel::SquaredExpARD<Params>, mean::Data<Params>, model::gp::NoLFOpt<Params>>;
using ConGP = limbo_b200::model::GP<Params, kernel::Exp<Params>, mean::Constant<Params>, model::gp::NoLFOpt<Params>>;
using ECI_t = limbo_b200::acqui::ECI<Params, ObjGP, ConGP>;
using SPGP_t = limbo_b200::model::SPGP<Params, kernel::SquaredExpARD<Params>, mean::Data<Params>, opt::Rprop<Params>>;

// the acquisitions are instantiated over SPGP_t itself (their device paths are selected on the model type); SPGPX only reaches
// the protected set-up
struct SPGPX : SPGP_t {
    void init(const std::vector<Eigen::VectorXd>& s, const std::vector<Eigen::VectorXd>& o) { this->_init(s, o); }
    void compute_at(const Eigen::VectorXd& w)
    {
        this->_optimized = true;
        this->_compute_at(w);
    }
    size_t m() const { return this->_m; }
};

static Eigen::VectorXd objective(const Eigen::VectorXd& x)
{
    return Eigen::VectorXd::Constant(1, std::sin(5.0 * x(0)) * std::cos(3.0 * x(1)) + 0.3 * x(0));
}
// feasible (> 1) on a band only, so that part of the box is infeasible
static Eigen::VectorXd constraint(const Eigen::VectorXd& x) { return Eigen::VectorXd::Constant(1, 1.0 + std::cos(4.0 * x(0) + x(1))); }

static bool in_box(const Eigen::VectorXd& x)
{
    for (int d = 0; d < x.size(); ++d)
        if (!(x(d) >= 0.0 && x(d) <= 1.0)) return false;
    return true;
}

// BatchedCmaes over f (value only) from `start`: the search must answer with one device search (two calls of f: the announced
// random pass and the announced search) and return a point in the box no worse than the best value of its random pass
template <typename F>
static bool cmaes_answers(F&& eval, const Eigen::VectorXd& start, int64_t* n_evals, double* value, double* pass_best_out)
{
    double pass_best = -INFINITY;
    long calls = 0;
    auto f = [&](const Eigen::VectorXd& x, bool g) {
        ++calls;
        const double v = eval(x, g);
        limbo_b200::opt::BatchRequest* req = limbo_b200::opt::current_batch();
        if (req && req->answered) pass_best = std::max(pass_best, req->best_value);
        return opt::no_grad(v);
    };
    limbo_b200::opt::BatchedCmaes<Params> bc;
    const Eigen::VectorXd x = bc(f, start, true);
    *n_evals = bc.n_evals();
    *value = eval(x, false);
    *pass_best_out = pass_best;
    return in_box(x) && calls == 2 && bc.n_evals() > 0 && *value >= pass_best - 1e-12 * std::fabs(pass_best);
}

static int eci_cb_loop(unsigned long long& seed)
{
    const int D = 2;
    ObjGP o(D, 1);
    ConGP c(D, 1);
    std::vector<Eigen::VectorXd> S, Yo, Yc;
    for (int i = 0; i < 20; ++i) {
        Eigen::VectorXd x(D);
        for (int d = 0; d < D; ++d) x(d) = u01(seed);
        S.push_back(x);
        Yo.push_back(objective(x));
        Yc.push_back(constraint(x));
    }
    o.compute(S, Yo);
    c.compute(S, Yc);
    FirstElem afun;
    int bad = 0;
    for (int it = 0; it < 4; ++it) {
        ECI_t acqui(o, c, it);
        auto acqui_optimization = [&](const Eigen::VectorXd& x, bool g) { return opt::fun(acqui(x, afun, g)); };
        Eigen::VectorXd start(D);
        for (int d = 0; d < D; ++d) start(d) = u01(seed);
        int64_t n = 0;
        double v = 0, pass = 0;
        const bool ok = cmaes_answers(acqui_optimization, start, &n, &v, &pass);
        std::printf("BatchedCmaes over limbo_b200::acqui::ECI in CBOptimizer's inner loop, iteration %d: %lld search evaluations, "
                    "value %.6e (random pass best %.6e): %s\n", it, (long long)n, v, pass, ok ? "ok" : "FAILED");
        if (!ok) ++bad;
        // the new sample, as eval_and_add and the two add_sample calls of cboptimizer.hpp:178-183 leave the models
        Eigen::VectorXd nx(D);
        for (int d = 0; d < D; ++d) nx(d) = u01(seed);
        o.add_sample(nx, objective(nx));
        c.add_sample(nx, constraint(nx));
    }
    return bad;
}

template <typename Acq>
static int spgp_case(const SPGP_t& model, const char* name)
{
    Acq acq(model, 0);
    FirstElem afun;
    int64_t n = 0;
    double v = 0, pass = 0;
    const bool ok = cmaes_answers([&](const Eigen::VectorXd& x, bool g) { return opt::fun(acq(x, afun, g)); },
        Eigen::VectorXd::Constant(model.dim_in(), 0.5), &n, &v, &pass);
    std::printf("BatchedCmaes over limbo_b200::acqui::%s<SPGP>: %lld search evaluations, value %.6e (random pass best %.6e): %s\n",
        name, (long long)n, v, pass, ok ? "ok" : "FAILED");
    return ok ? 0 : 1;
}

int main()
{
    unsigned long long seed = 23;
    int fails = eci_cb_loop(seed);

    const int N = 300, D = 3;
    std::vector<Eigen::VectorXd> s, o;
    for (int i = 0; i < N; ++i) {
        Eigen::VectorXd x(D);
        double y = 0.0;
        for (int d = 0; d < D; ++d) { x(d) = u01(seed); y += std::sin(3.0 * x(d)); }
        s.push_back(x);
        o.push_back(Eigen::VectorXd::Constant(1, y));
    }
    SPGPX sp;
    sp.init(s, o);
    const size_t M = sp.m();
    Eigen::VectorXd w((M + 1) * D + 2);
    for (size_t i = 0; i < M; ++i)
        for (int d = 0; d < D; ++d) w(d * M + i) = s[(7 * i) % N](d);
    for (int d = 0; d < D; ++d) w(M * D + d) = 2.0 + 0.1 * d;
    w((M + 1) * D) = std::log(0.8);
    w((M + 1) * D + 1) = std::log(0.05);
    sp.compute_at(w);
    fails += spgp_case<limbo_b200::acqui::UCB<Params, SPGP_t>>(sp, "UCB");
    fails += spgp_case<limbo_b200::acqui::EI<Params, SPGP_t>>(sp, "EI");
    if (fails == 0) std::printf("CMAES ECI SPGP DROPIN OK\n");
    return fails ? 1 : 0;
}
