// tests/cpp/parego_dropin_test.cpp — ParEGO through the C++ drop-ins (include/limbo_b200/model/gp_parego.hpp), compiled against
// the reference's own headers, the Eigen stand-in of oracle/ref_shim and the replaying tools::random_vector of
// oracle/ref_shim/parego_shim, so that the reference's GPParego and the specialisation draw the same weight vectors:
//   (1) GPParego<Params, limbo_b200::model::GP> against the reference's GPParego<Params, limbo::model::GP> under the same weight
//       sequence, after compute() and each of several add_sample() calls, K = 2 (MOP2) and K = 3 (a third, negative objective):
//       the scalarised observations bit for bit, mu and sigma^2 at query points within 1e-9, and every add_sample on the
//       incremental path (lb_append);
//   (2) experimental::bayes_opt::Parego's loop over that model with acquiopt<limbo_b200::opt::BatchedRandom> and the batch-aware
//       limbo_b200::acqui::UCB runs MOP2: every proposal in [0, 1]^2 and every update incremental.  Parego (a BOptimizer) needs
//       Boost.Parameter (bayes_opt/bo_base.hpp), which the stand-in does not provide, so BOptimizer::optimize's inner loop
//       (boptimizer.hpp:139-170) is restated here over the model Parego builds;
//   (3) GP::acq_argmax_cols: with one column it equals GP::acq_argmax bit for bit; with three, each column's record is the first
//       maximum of its values.
// Needs a GPU to run; prints "PAREGO DROPIN OK".
#include <limbo/tools/random_generator.hpp> // first: the replaying tools::random_vector of oracle/ref_shim/parego_shim
#include <cmath>
#include <cstdio>
#include <vector>
#include "dropin_common.hpp"

#include <limbo/acqui/ucb.hpp>
#include <limbo/kernel/matern_five_halves.hpp>
#include <limbo/mean/data.hpp>
#include <limbo/model/gp.hpp>

#include <limbo_b200/model/gp.hpp>
#include <limbo_b200/model/gp_parego.hpp>
#include <limbo_b200/opt/batched_random.hpp>

extern "C" long long lb_debug_append_count(const lb_gp* h);

using namespace limbo;

struct Params {
    struct kernel : public defaults::kernel {};
    struct kernel_maternfivehalves : public defaults::kernel_maternfivehalves {};
    struct model_gp_parego : public experimental::defaults::model_gp_parego {};
    struct acqui_ucb : public defaults::acqui_ucb {};
    struct opt_batchedrandom : public limbo_b200::defaults::opt_batchedrandom {
        BO_PARAM(int, candidates, 4000);
    };
};

using Kernel = kernel::MaternFiveHalves<Params>;
using RefGP = experimental::model::GPParego<Params, model::GP<Params, Kernel, mean::Data<Params>>>;
using NewGP = experimental::model::GPParego<Params, limbo_b200::model::GP<Params, Kernel, mean::Data<Params>, model::gp::NoLFOpt<Params>>>;

struct Probe : NewGP { // the handle is protected: the append counter is read through a derived class
    using NewGP::NewGP;
    long long appends() const { return lb_debug_append_count(this->_h); }
};

static Eigen::VectorXd objectives(const Eigen::VectorXd& x, int K)
{ // examples/experimental/multi.cpp's mop2 (maximised), and -(f1 + f2) as a third objective
    const double d = (double)x.size();
    double a = 0, b = 0;
    for (int i = 0; i < x.size(); ++i) {
        const double xi = 4.0 * x(i) - 2.0;
        a += (xi - 1.0 / std::sqrt(d)) * (xi - 1.0 / std::sqrt(d));
        b += (xi + 1.0 / std::sqrt(d)) * (xi + 1.0 / std::sqrt(d));
    }
    Eigen::VectorXd f((Eigen::Index)K);
    f(0) = std::exp(-a);
    f(1) = std::exp(-b);
    if (K == 3) f(2) = -(f(0) + f(1));
    return f;
}

static int check_against_reference(int K)
{
    const int D = 2, N0 = 40, ADD = 6;
    unsigned long long seed = 7 + K;
    std::vector<Eigen::VectorXd> X, F, Q;
    for (int i = 0; i < N0 + ADD; ++i) {
        Eigen::VectorXd x((Eigen::Index)D);
        for (int d = 0; d < D; ++d) x(d) = u01(seed);
        X.push_back(x);
        F.push_back(objectives(x, K));
    }
    for (int i = 0; i < 50; ++i) {
        Eigen::VectorXd x((Eigen::Index)D);
        for (int d = 0; d < D; ++d) x(d) = u01(seed);
        Q.push_back(x);
    }
    std::vector<double> draws((size_t)(K * (1 + ADD)));
    for (double& w : draws) w = u01(seed);
    RefGP ref(D, K);
    Probe gp(D, K);
    int bad = 0;
    double dmu = 0, ds = 0;
    for (int pass = 0; pass < 2; ++pass) { // the same weight sequence for each model
        limbo_parego_replay(draws.data(), draws.size());
        const std::vector<Eigen::VectorXd> X0(X.begin(), X.begin() + N0), F0(F.begin(), F.begin() + N0);
        if (pass == 0) {
            ref.compute(X0, F0);
            for (int i = N0; i < N0 + ADD; ++i) ref.add_sample(X[(size_t)i], F[(size_t)i]);
        } else {
            gp.compute(X0, F0);
            for (int i = N0; i < N0 + ADD; ++i) gp.add_sample(X[(size_t)i], F[(size_t)i]);
        }
    }
    const auto ro = ref.observations();
    const Eigen::MatrixXd& go = gp.observations_matrix();
    for (int i = 0; i < N0 + ADD; ++i) bad += ro[(size_t)i](0) != go(i, 0);
    for (const auto& q : Q) {
        Eigen::VectorXd m1, m2;
        double s1, s2;
        std::tie(m1, s1) = ref.query(q);
        std::tie(m2, s2) = gp.query(q);
        dmu = std::max(dmu, std::abs(m1(0) - m2(0)));
        ds = std::max(ds, std::abs(s1 - s2));
    }
    const bool ok = bad == 0 && dmu < 1e-9 && ds < 1e-9 && gp.appends() == ADD && (int)gp.raw_observations().size() == N0 + ADD;
    std::printf("GPParego<limbo_b200::model::GP> vs the reference's GPParego<model::GP>, K=%d: %d scalarised rows differ, dmu=%.3e "
                "dsigma2=%.3e, %lld of %d add_sample calls incremental: %s\n",
        K, bad, dmu, ds, gp.appends(), ADD, ok ? "ok" : "FAILED");
    return ok ? 0 : 1;
}

static int parego_loop()
{
    using Acq_t = limbo_b200::acqui::UCB<Params, Probe>;
    const int D = 2, K = 2, ITERS = 15;
    unsigned long long seed = 123;
    std::vector<double> draws((size_t)(K * (1 + ITERS)));
    for (double& w : draws) w = u01(seed);
    limbo_parego_replay(draws.data(), draws.size());
    std::vector<Eigen::VectorXd> S, O;
    for (int i = 0; i < 10; ++i) { // init::RandomSampling
        Eigen::VectorXd x((Eigen::Index)D);
        for (int d = 0; d < D; ++d) x(d) = u01(seed);
        S.push_back(x);
        O.push_back(objectives(x, K));
    }
    Probe model(D, K); // what Parego's modelfun builds: GPParego<Params, model_t>
    model.compute(S, O);
    limbo_b200::opt::BatchedRandom<Params> acqui_optimizer;
    FirstElem afun;
    bool inside = true;
    for (int it = 0; it < ITERS; ++it) {
        Acq_t acqui(model, it);
        auto acqui_optimization = [&](const Eigen::VectorXd& x, bool g) { return acqui(x, afun, g); };
        Eigen::VectorXd start((Eigen::Index)D);
        for (int d = 0; d < D; ++d) start(d) = u01(seed);
        Eigen::VectorXd nx = acqui_optimizer(acqui_optimization, start, true);
        inside = inside && nx.minCoeff() >= 0.0 && nx.maxCoeff() <= 1.0;
        S.push_back(nx);
        O.push_back(objectives(nx, K));
        model.add_sample(S.back(), O.back());
    }
    const bool ok = inside && model.appends() == ITERS && model.nb_samples() == 10 + ITERS;
    std::printf("Parego loop over GPParego<limbo_b200::model::GP> + BatchedRandom on MOP2: %d iterations, %lld incremental, in box %d: %s\n",
        ITERS, model.appends(), (int)inside, ok ? "ok" : "FAILED");
    return ok ? 0 : 1;
}

static int argmax_cols()
{
    using GP_t = limbo_b200::model::GP<Params, Kernel, mean::Data<Params>, model::gp::NoLFOpt<Params>>;
    const int D = 2;
    unsigned long long seed = 5;
    std::vector<Eigen::VectorXd> X, F1, F3, Q;
    for (int i = 0; i < 60; ++i) {
        Eigen::VectorXd x((Eigen::Index)D);
        for (int d = 0; d < D; ++d) x(d) = u01(seed);
        X.push_back(x);
        F3.push_back(objectives(x, 3));
        F1.push_back(F3.back().head(1));
    }
    for (int i = 0; i < 700; ++i) {
        Eigen::VectorXd x((Eigen::Index)D);
        for (int d = 0; d < D; ++d) x(d) = u01(seed);
        Q.push_back(x);
    }
    GP_t one(D, 1), three(D, 3);
    one.compute(X, F1);
    three.compute(X, F3);
    std::vector<double> v1, vc, best;
    std::vector<long> idx;
    const auto r1 = one.acq_argmax(LB_ACQ_UCB, 0.5, 0.0, Q, &v1);
    one.acq_argmax_cols(LB_ACQ_UCB, {0.5, 0.0}, Q, best, idx, &vc);
    bool ok = vc == v1 && best[0] == r1.first && idx[0] == r1.second;
    three.acq_argmax_cols(LB_ACQ_UCB, {0.5, 0.0, 1.0, 0.0, 2.0, 0.0}, Q, best, idx, &vc);
    for (int r = 0; r < 3; ++r) {
        std::vector<double> col;
        for (size_t m = 0; m < Q.size(); ++m) col.push_back(vc[m * 3 + (size_t)r]);
        ok = ok && idx[(size_t)r] == first_max(col) && best[(size_t)r] == col[(size_t)idx[(size_t)r]];
    }
    std::printf("GP::acq_argmax_cols: one column equals acq_argmax, three columns' records are their first maxima: %s\n", ok ? "ok" : "FAILED");
    return ok ? 0 : 1;
}

int main()
{
    int fails = check_against_reference(2) + check_against_reference(3) + parego_loop() + argmax_cols();
    if (fails == 0) std::printf("PAREGO DROPIN OK\n");
    return fails;
}
