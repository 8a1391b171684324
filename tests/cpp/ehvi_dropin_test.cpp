// tests/cpp/ehvi_dropin_test.cpp — multi-objective BO's acquisition, compiled: two Matern-5/2 / mean::Data models per side on
// mop2 data, the front from the reference's pareto::pareto_set<1> of the observations, and on one fixed candidate set
//   (1) the reference's primary acqui::Ehvi over two of the reference's limbo::model::GP, one point at a time,
//   (2) the specialisation acqui::Ehvi<Params, limbo_b200::model::GP<...>> (include/limbo_b200/acqui/ehvi.hpp), one point at a
//       time (a batch of one on the device each),
//   (3) the same specialisation answering a BatchRequest as BatchedRandom issues it (one lb_ehvi_argmax),
// must agree to 1e-10 with the same argmax.  Then limbo_b200::opt::BatchedRandom drives (2) as the reference's
// experimental::bayes_opt::Ehvi does (opt::no_grad(acqui(x))): it must reach f once per round, and the reference's functor must
// agree with it at the point it returns, which is no worse than the candidate set's best it started from.  Needs a GPU to run; prints "EHVI DROPIN OK".
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

static Eigen::VectorXd mop2(const Eigen::VectorXd& x) // examples/experimental/multi.cpp
{
    const double c = 1.0 / std::sqrt((double)x.size());
    double v1 = 0, v2 = 0;
    for (int d = 0; d < x.size(); ++d) {
        const double xx = x(d) * 4.0 - 2.0;
        v1 += (xx - c) * (xx - c);
        v2 += (xx + c) * (xx + c);
    }
    Eigen::VectorXd r(2);
    r(0) = std::exp(-v1);
    r(1) = std::exp(-v2);
    return r;
}

static int run_case(int N, int D, double ref0, double ref1)
{
    unsigned long long seed = 11 + N;
    std::vector<Eigen::VectorXd> X, Q;
    std::vector<std::vector<Eigen::VectorXd>> obs(2);
    std::vector<std::tuple<Eigen::VectorXd, Eigen::VectorXd, Eigen::VectorXd>> packed;
    for (int i = 0; i < N; ++i) {
        Eigen::VectorXd x((Eigen::Index)D);
        for (int d = 0; d < D; ++d) x(d) = u01(seed);
        const Eigen::VectorXd y = mop2(x);
        X.push_back(x);
        for (int j = 0; j < 2; ++j) obs[(size_t)j].push_back(Eigen::VectorXd::Constant(1, y(j)));
        packed.push_back(std::make_tuple(x, y, Eigen::VectorXd::Zero(2)));
    }
    for (int i = 0; i < 1000; ++i) {
        Eigen::VectorXd q((Eigen::Index)D);
        for (int d = 0; d < D; ++d) q(d) = u01(seed);
        Q.push_back(q);
    }
    std::vector<RefGP> ref(2, RefGP(D, 1));
    std::vector<NewGP> gpu;
    gpu.emplace_back(D, 1);
    gpu.emplace_back(D, 1);
    for (int j = 0; j < 2; ++j) {
        ref[(size_t)j].compute(X, obs[(size_t)j]);
        gpu[(size_t)j].compute(X, obs[(size_t)j]);
    }
    auto front = pareto::pareto_set<1>(packed);
    std::vector<individual> store(front.size());
    std::deque<individual*> pop;
    for (size_t i = 0; i < front.size(); ++i) {
        store[i].f[0] = std::get<1>(front[i])(0);
        store[i].f[1] = std::get<1>(front[i])(1);
        store[i].f[2] = 0;
        pop.push_back(&store[i]);
    }
    Eigen::VectorXd r(3);
    r(0) = ref0;
    r(1) = ref1;
    r(2) = 0;
    acqui::Ehvi<Params, RefGP> ehvi_ref(ref, pop, r);
    acqui::Ehvi<Params, NewGP> ehvi_dev(gpu, pop, r);
    std::vector<double> v1, v2;
    for (auto& q : Q) {
        v1.push_back(ehvi_ref(q));
        v2.push_back(ehvi_dev(q));
    }
    const long i1 = first_max(v1);
    limbo_b200::opt::BatchRequest req; // what BatchedRandom announces before calling f
    req.candidates = &Q;
    limbo_b200::opt::current_batch() = &req;
    const double v0 = ehvi_dev(Q[0]);
    limbo_b200::opt::current_batch() = nullptr;
    double d2 = 0;
    for (size_t k = 0; k < Q.size(); ++k) d2 = std::max(d2, std::fabs(v1[k] - v2[k]));
    const double dbest = std::fabs(req.best_value - v1[(size_t)i1]);

    // BatchedRandom over the specialisation, as experimental::bayes_opt::Ehvi calls it (ehvi.hpp:134-138)
    long calls = 0;
    auto f = [&](const Eigen::VectorXd& x, bool) { ++calls; return opt::no_grad(ehvi_dev(x)); };
    const Eigen::VectorXd x = limbo_b200::opt::BatchedRandom<Params>()(f, Q[(size_t)i1], true); // starts at, and keeps, Q's best
    const double at_x = ehvi_ref(x), at_x_dev = ehvi_dev(x);
    std::printf("N=%d D=%d k=%zu best=%.6e@%ld |ref - specialisation|=%.3e batch: answered=%d best=%.6e@%ld |d|=%.3e |v0|=%.3e; "
                "BatchedRandom: %ld calls of f, ehvi(x)=%.6e |ref - dev|=%.3e\n",
        N, D, front.size(), v1[(size_t)i1], i1, d2, (int)req.answered, req.best_value, req.best_index, dbest, std::fabs(v0 - v1[0]), calls,
        at_x, std::fabs(at_x - at_x_dev));
    const bool ok = v1[(size_t)i1] > 0 && d2 <= 1e-10 && first_max(v2) == i1 && req.answered && req.best_index == i1 && dbest <= 1e-10
        && std::fabs(v0 - v1[0]) <= 1e-10 && calls == 1 + Params::opt_batchedrandom::refinements() && at_x >= v1[(size_t)i1] - 1e-10
        && std::fabs(at_x - at_x_dev) <= 1e-10;
    return ok ? 0 : 1;
}

int main()
{
    int bad = 0;
    bad += run_case(60, 2, -11.0, -11.0);
    bad += run_case(200, 2, -1.0, -1.0);
    bad += run_case(120, 3, 0.0, 0.0);
    if (bad) {
        std::printf("EHVI DROPIN FAILED (%d)\n", bad);
        return 1;
    }
    std::printf("EHVI DROPIN OK\n");
    return 0;
}
