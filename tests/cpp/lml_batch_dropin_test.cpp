// tests/cpp/lml_batch_dropin_test.cpp — the batched hyper-parameter fit through the C++ drop-in, compiled against the reference's
// own headers:
//   (1) limbo_b200::model::GP::lml_grad_batch (one lb_lml_grad_batch) against the reference's limbo::model::GP refitted at every
//       row (set_h_params, recompute(false), compute_log_lik, compute_kernel_grad_log_lik): lik within 1e-11 relative, grad
//       within 1e-9 max(1, |g|inf), SE-ARD and Matern-5/2;
//   (2) every lane of limbo_b200::opt::BatchedRprop against the reference's opt::Rprop from the same start over the reference
//       GP's likelihood (KernelLFOptimization's evaluation), within 1e-9;
//   (3) a GP typedef with limbo_b200::model::gp::BatchedKernelLFOpt compiles, and optimize_hyperparams raises the log-likelihood.
// Needs a GPU to run; prints "LML BATCH DROPIN OK".  (Eigen is the stand-in from oracle/ref_shim.)
#include <cmath>
#include <cstdio>
#include <vector>

#include <Eigen/Core>
#include "dropin_common.hpp"

#include <limbo/kernel/matern_five_halves.hpp>
#include <limbo/kernel/squared_exp_ard.hpp>
#include <limbo/mean/data.hpp>
#include <limbo/model/gp.hpp>
#include <limbo/model/gp/no_lf_opt.hpp>
#include <limbo/opt/rprop.hpp>

#include <limbo_b200/model/gp.hpp>
#include <limbo_b200/opt/batched_rprop.hpp>

using namespace limbo;

struct Params {
    struct kernel : public defaults::kernel {};
    struct kernel_squared_exp_ard : public defaults::kernel_squared_exp_ard {};
    struct kernel_maternfivehalves : public defaults::kernel_maternfivehalves {};
    struct opt_rprop {
        BO_PARAM(int, iterations, 20);
        BO_PARAM(double, eps_stop, 0.0);
    };
    struct opt_parallelrepeater {
        BO_PARAM(int, repeats, 6);
        BO_PARAM(double, epsilon, 1e-2);
    };
};

static void data(int N, int D, std::vector<Eigen::VectorXd>& X, std::vector<Eigen::VectorXd>& Y)
{
    unsigned long long seed = 7;
    for (int i = 0; i < N; ++i) {
        Eigen::VectorXd x((Eigen::Index)D), y((Eigen::Index)1);
        double s = 0;
        for (int d = 0; d < D; ++d) {
            x(d) = u01(seed);
            s += std::sin(3.0 * x(d));
        }
        y(0) = s;
        X.push_back(x);
        Y.push_back(y);
    }
}

template <typename GP>
struct RefObjective { // kernel_lf_opt.hpp:77-92 over the reference GP
    const GP& g0;
    limbo::opt::eval_t operator()(const Eigen::VectorXd& p, bool compute_grad) const
    {
        GP g(g0);
        g.kernel_function().set_h_params(p);
        g.recompute(false);
        double lik = g.compute_log_lik();
        if (!compute_grad) return limbo::opt::no_grad(lik);
        return {lik, g.compute_kernel_grad_log_lik()};
    }
};

static int fails = 0;
#define CHECK(c, ...)                          \
    do {                                       \
        if (!(c)) {                            \
            std::printf("FAIL: " __VA_ARGS__); \
            std::printf("\n");                 \
            ++fails;                           \
        }                                      \
    } while (0)

template <typename Kernel>
void check_kernel(const char* name, int N, int D)
{
    using RefGP = model::GP<Params, Kernel, mean::Data<Params>, model::gp::NoLFOpt<Params>>;
    using NewGP = limbo_b200::model::GP<Params, Kernel, mean::Data<Params>, model::gp::NoLFOpt<Params>>;
    std::vector<Eigen::VectorXd> X, Y;
    data(N, D, X, Y);
    RefGP ref(D, 1);
    NewGP gp(D, 1);
    ref.compute(X, Y);
    gp.compute(X, Y);
    const Eigen::VectorXd h0 = ref.kernel_function().h_params();
    const int nh = (int)h0.size(), R = 5;
    Eigen::MatrixXd H(R, nh);
    unsigned long long seed = 99;
    for (int r = 0; r < R; ++r)
        for (int j = 0; j < nh; ++j) H(r, j) = h0(j) - 1.2 + 2.0 * u01(seed);
    // (1) the batched rows against the reference GP
    Eigen::VectorXd lik;
    Eigen::MatrixXd G;
    std::vector<int> info;
    gp.lml_grad_batch(H, lik, &G, &info);
    RefObjective<RefGP> f{ref};
    for (int r = 0; r < R; ++r) {
        Eigen::VectorXd p(nh);
        for (int j = 0; j < nh; ++j) p(j) = H(r, j);
        auto e = f(p, true);
        const double l = e.first;
        const Eigen::VectorXd& g = e.second.get();
        double gmax = 1.0, dg = 0.0;
        for (int j = 0; j < nh; ++j) {
            gmax = std::max(gmax, std::abs(g(j)));
            dg = std::max(dg, std::abs(G(r, j) - g(j)));
        }
        CHECK(info[(size_t)r] == 0, "%s row %d: info %d", name, r, info[(size_t)r]);
        CHECK(std::abs(lik(r) - l) <= 1e-11 * std::max(1.0, std::abs(l)), "%s row %d: lik %.17g vs %.17g", name, r, lik(r), l);
        CHECK(dg <= 1e-9 * gmax, "%s row %d: grad off by %g", name, r, dg);
    }
    // (2) BatchedRprop lanes against the reference's Rprop from the same starts
    limbo_b200::model::gp::BatchedLFObjective<NewGP> fb{gp};
    Eigen::MatrixXd starts(4, nh);
    for (int r = 0; r < 4; ++r)
        for (int j = 0; j < nh; ++j) starts(r, j) = h0(j) - 0.3 + 0.6 * u01(seed);
    Eigen::MatrixXd V = limbo_b200::opt::BatchedRprop<Params>()(fb, starts, false);
    for (int r = 0; r < 4; ++r) {
        Eigen::VectorXd s(nh);
        for (int j = 0; j < nh; ++j) s(j) = starts(r, j);
        Eigen::VectorXd want = limbo::opt::Rprop<Params>()(f, s, false);
        double d = 0.0;
        for (int j = 0; j < nh; ++j) d = std::max(d, std::abs(V(r, j) - want(j)));
        CHECK(d <= 1e-9, "%s lane %d: BatchedRprop off the reference Rprop by %g", name, r, d);
    }
    std::printf("%s N=%d D=%d: %d rows, 4 Rprop lanes checked\n", name, N, D, R);
}

int main()
{
    check_kernel<kernel::SquaredExpARD<Params>>("SquaredExpARD", 60, 3);
    check_kernel<kernel::MaternFiveHalves<Params>>("MaternFiveHalves", 150, 2);
    // (3) the HyperParamsOptimizer in a GP typedef
    using FitGP = limbo_b200::model::GP<Params, kernel::SquaredExpARD<Params>, mean::Data<Params>,
        limbo_b200::model::gp::BatchedKernelLFOpt<Params>>;
    std::vector<Eigen::VectorXd> X, Y;
    data(80, 2, X, Y);
    FitGP gp(2, 1);
    gp.compute(X, Y);
    const double before = gp.compute_log_lik();
    gp.optimize_hyperparams();
    const double after = gp.get_log_lik();
    std::printf("BatchedKernelLFOpt: log-lik %.6f -> %.6f\n", before, after);
    CHECK(after > before, "BatchedKernelLFOpt did not raise the log-likelihood (%g -> %g)", before, after);
    if (fails) return 1;
    std::printf("LML BATCH DROPIN OK\n");
    return 0;
}
