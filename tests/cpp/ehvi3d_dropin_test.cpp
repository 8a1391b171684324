// tests/cpp/ehvi3d_dropin_test.cpp — three-objective EHVI in C++, compiled: three Matern-5/2 / mean::Data models per side on a
// three-objective DTLZ2, the front from the reference's pareto::pareto_set<1> of the observations, and on one fixed candidate set
//   (1) the reference's ehvi3d_sliceupdate over three of the reference's limbo::model::GP (mu(v)(0) and sigma(v) of each), one
//       point at a time,
//   (2) the three-model specialisation acqui::Ehvi<Params, limbo_b200::model::GP<...>> (include/limbo_b200/acqui/ehvi.hpp), one
//       point at a time (a batch of one on the device each),
//   (3) the same specialisation answering a BatchRequest as BatchedRandom issues it (one lb_ehvi3d_argmax),
//   (4) the specialisation with an aggregator that is not FirstElem-like (the host path: ehvi3d_sliceupdate over the device GP's
//       mu and sigma), against (1) with the same aggregator,
// must agree to 1e-10 with the same argmax.  Then limbo_b200::opt::BatchedRandom drives (2) as opt::no_grad(acqui(x)): it must
// reach f once per round, and (1) must agree with it at the point it returns, which is no worse than the candidate set's best it
// started from.  A GradRequest stays unanswered.  Needs a GPU to run; prints "EHVI3D DROPIN OK".
// (Eigen is the stand-in from oracle/ref_shim so that no Eigen install is needed.)
#include <cmath>
#include <cstdio>
#include <deque>
#include <vector>

#include <Eigen/Core>

#include "dropin_common.hpp"

#include <limbo/experimental/tools/pareto.hpp>
#include <limbo/kernel/matern_five_halves.hpp>
#include <limbo/mean/data.hpp>
#include <limbo/model/gp.hpp>

#include <limbo_b200/acqui/ehvi.hpp>

using namespace limbo;

struct Params {
    struct kernel : public defaults::kernel {};
    struct kernel_maternfivehalves : public defaults::kernel_maternfivehalves {};
    struct opt_batchedrandom {
        BO_PARAM(int, candidates, 2000);
        BO_PARAM(int, refinements, 2);
        BO_PARAM(double, shrink, 0.1);
    };
};

using RefGP = model::GP<Params, kernel::MaternFiveHalves<Params>, mean::Data<Params>>;
using NewGP = limbo_b200::model::GP<Params, kernel::MaternFiveHalves<Params>, mean::Data<Params>, model::gp::NoLFOpt<Params>>;

struct Scaled { // not FirstElem-like: the host path
    double operator()(const Eigen::VectorXd& x) const { return 0.5 * x(0); }
};

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

template <typename Agg>
static double ref_value(const std::vector<RefGP>& gps, std::deque<individual*>& pop, double* r, const Eigen::VectorXd& v, const Agg& afun)
{
    double mu[3], s[3];
    for (int j = 0; j < 3; ++j) {
        mu[j] = afun(gps[(size_t)j].mu(v));
        s[j] = gps[(size_t)j].sigma(v);
    }
    return ehvi3d_sliceupdate(pop, r, mu, s);
}

static int run_case(int N, int D, double rv)
{
    unsigned long long seed = 17 + N;
    std::vector<Eigen::VectorXd> X, Q;
    std::vector<std::vector<Eigen::VectorXd>> obs(3);
    std::vector<std::tuple<Eigen::VectorXd, Eigen::VectorXd, Eigen::VectorXd>> packed;
    for (int i = 0; i < N; ++i) {
        Eigen::VectorXd x((Eigen::Index)D);
        for (int d = 0; d < D; ++d) x(d) = u01(seed);
        const Eigen::VectorXd y = dtlz2(x);
        X.push_back(x);
        for (int j = 0; j < 3; ++j) obs[(size_t)j].push_back(Eigen::VectorXd::Constant(1, y(j)));
        packed.push_back(std::make_tuple(x, y, Eigen::VectorXd::Zero(3)));
    }
    for (int i = 0; i < 300; ++i) {
        Eigen::VectorXd q((Eigen::Index)D);
        for (int d = 0; d < D; ++d) q(d) = u01(seed);
        Q.push_back(q);
    }
    std::vector<RefGP> ref(3, RefGP(D, 1));
    std::vector<NewGP> gpu;
    for (int j = 0; j < 3; ++j) gpu.emplace_back(D, 1);
    for (int j = 0; j < 3; ++j) {
        ref[(size_t)j].compute(X, obs[(size_t)j]);
        gpu[(size_t)j].compute(X, obs[(size_t)j]);
    }
    auto front = pareto::pareto_set<1>(packed);
    std::vector<individual> store(front.size());
    std::deque<individual*> pop;
    for (size_t i = 0; i < front.size(); ++i) {
        for (int d = 0; d < 3; ++d) store[i].f[d] = std::get<1>(front[i])(d);
        pop.push_back(&store[i]);
    }
    double rr[3] = {rv, rv, rv};
    Eigen::VectorXd r(3);
    r << rv, rv, rv;
    acqui::Ehvi<Params, NewGP> ehvi_dev(gpu, pop, r);
    std::vector<double> v1, v2;
    double d4 = 0;
    for (size_t k = 0; k < Q.size(); ++k) {
        v1.push_back(ref_value(ref, pop, rr, Q[k], FirstElem()));
        v2.push_back(ehvi_dev(Q[k]));
        if (k < 20) {
            const double a = ref_value(ref, pop, rr, Q[k], Scaled()), b = ehvi_dev(Q[k], Scaled());
            d4 = std::max(d4, std::fabs(a - b));
        }
    }
    const long i1 = first_max(v1);
    limbo_b200::opt::BatchRequest req; // what BatchedRandom announces before calling f
    std::vector<double> vals;
    req.candidates = &Q;
    req.values = &vals;
    limbo_b200::opt::GradRequest greq; // left unanswered with three models
    greq.points = &Q;
    limbo_b200::opt::current_batch() = &req;
    limbo_b200::opt::current_grad_batch() = &greq;
    const double v0 = ehvi_dev(Q[0]);
    limbo_b200::opt::current_batch() = nullptr;
    limbo_b200::opt::current_grad_batch() = nullptr;
    double d2 = 0, d3 = 0;
    for (size_t k = 0; k < Q.size(); ++k) {
        d2 = std::max(d2, std::fabs(v1[k] - v2[k]));
        if (vals.size() == Q.size()) d3 = std::max(d3, std::fabs(v1[k] - vals[k]));
    }
    const double dbest = std::fabs(req.best_value - v1[(size_t)i1]);

    long calls = 0;
    auto f = [&](const Eigen::VectorXd& x, bool) { ++calls; return opt::no_grad(ehvi_dev(x)); };
    const Eigen::VectorXd x = limbo_b200::opt::BatchedRandom<Params>()(f, Q[(size_t)i1], true); // starts at, and keeps, Q's best
    const double at_x = ref_value(ref, pop, rr, x, FirstElem()), at_x_dev = ehvi_dev(x);
    std::printf("N=%d D=%d k=%zu best=%.6e@%ld |ref - specialisation|=%.3e host path |d|=%.3e batch: answered=%d best=%.6e@%ld "
                "|d|=%.3e |values - ref|=%.3e |v0|=%.3e grad answered=%d; BatchedRandom: %ld calls of f, ehvi(x)=%.6e |ref - dev|=%.3e\n",
        N, D, front.size(), v1[(size_t)i1], i1, d2, d4, (int)req.answered, req.best_value, req.best_index, dbest, d3,
        std::fabs(v0 - v1[0]), (int)greq.answered, calls, at_x, std::fabs(at_x - at_x_dev));
    const double tol = 1e-10 * std::max(1.0, std::fabs(v1[(size_t)i1]));
    const bool ok = v1[(size_t)i1] > 0 && d2 <= tol && first_max(v2) == i1 && d4 <= tol && req.answered && req.best_index == i1
        && dbest <= tol && vals.size() == Q.size() && d3 <= tol && std::fabs(v0 - v1[0]) <= tol && !greq.answered
        && calls == 1 + Params::opt_batchedrandom::refinements() && at_x >= v1[(size_t)i1] - tol && std::fabs(at_x - at_x_dev) <= tol;
    return ok ? 0 : 1;
}

int main()
{
    int bad = 0;
    bad += run_case(60, 3, -11.0);
    bad += run_case(150, 4, -2.0);
    if (bad) {
        std::printf("EHVI3D DROPIN FAILED (%d)\n", bad);
        return 1;
    }
    std::printf("EHVI3D DROPIN OK\n");
    return 0;
}
