// oracle/ref_shim/ref_driver.cpp — TEST INFRASTRUCTURE ONLY.
//
// Runs the REFERENCE'S OWN hot-path code (headers included from
// the reference's src/ where they lie: limbo/model/gp.hpp, kernel/*.hpp,
// mean/data.hpp, acqui/ucb.hpp, acqui/ei.hpp, model/gp/kernel_lf_opt.hpp,
// opt/rprop.hpp) with the dense linear algebra supplied by the stand-in in
// ./Eigen.  Used to pin oracle/limbo_oracle.hpp (tests/test_oracle_vs_ref.py)
// and to generate tests/golden/*.npz (tests/golden/make_golden.py).
// No reference source is copied: this file only instantiates its templates.
#define protected public // same trick as src/tests/test_gp.cpp:48 to read _kernel
#include <limbo/acqui/ei.hpp>
#include <limbo/acqui/ucb.hpp>
#include <limbo/kernel/exp.hpp>
#include <limbo/kernel/matern_five_halves.hpp>
#include <limbo/kernel/matern_three_halves.hpp>
#include <limbo/kernel/squared_exp_ard.hpp>
#include <limbo/mean/constant.hpp>
#include <limbo/mean/data.hpp>
#include <limbo/mean/function_ard.hpp>
#include <limbo/model/gp.hpp>
#include <limbo/model/gp/kernel_lf_opt.hpp>
#include <limbo/opt/rprop.hpp>
#undef protected
#include <chrono>
#include <cstring>
#include <thread>

using namespace limbo;

struct Params {
    struct kernel {
        BO_DYN_PARAM(double, noise);
        BO_PARAM(bool, optimize_noise, false);
    };
    struct kernel_squared_exp_ard : public defaults::kernel_squared_exp_ard {};
    struct kernel_maternfivehalves : public defaults::kernel_maternfivehalves {};
    struct kernel_maternthreehalves : public defaults::kernel_maternthreehalves {};
    struct kernel_exp : public defaults::kernel_exp {};
    struct opt_rprop {
        BO_DYN_PARAM(int, iterations);
        BO_PARAM(double, eps_stop, 0.0);
    };
    struct acqui_ucb : public defaults::acqui_ucb {};
    struct acqui_ei : public defaults::acqui_ei {};
    struct mean_constant {
        BO_PARAM(double, constant, 0.25);
    };
};
BO_DECLARE_DYN_PARAM(double, Params::kernel, noise);
BO_DECLARE_DYN_PARAM(int, Params::opt_rprop, iterations);

// Params::kernel_squared_exp_ard::k() = 2: SE-ARD with two Lambda columns (squared_exp_ard.hpp:109-126,142-146)
struct ParamsLambda : Params {
    struct kernel_squared_exp_ard {
        BO_PARAM(int, k, 2);
        BO_PARAM(double, sigma_sq, 1);
    };
};

struct ParamsNoise : Params {
    struct kernel {
        BO_DYN_PARAM(double, noise);
        BO_PARAM(bool, optimize_noise, true);
    };
};
BO_DECLARE_DYN_PARAM(double, ParamsNoise::kernel, noise);

// bayes_opt/bo_base.hpp:99-105 (FirstElem) restated: bo_base.hpp itself needs Boost.Parameter/Fusion
struct FirstElem {
    double operator()(const Eigen::VectorXd& x) const { return x(0); }
};

namespace {

std::vector<Eigen::VectorXd> rows_of(const double* a, long n, int d)
{
    std::vector<Eigen::VectorXd> v;
    for (long i = 0; i < n; ++i) {
        Eigen::VectorXd x((Eigen::Index)d);
        for (int k = 0; k < d; ++k) x(k) = a[i * d + k];
        v.push_back(x);
    }
    return v;
}

void put(const Eigen::MatrixXd& m, double* dst)
{
    if (dst) std::memcpy(dst, m.data(), sizeof(double) * (size_t)m.size());
}

template <typename P, typename Kernel>
int run(long N, int D, int Pout, const double* X, const double* Y, double noise, const double* hp, int nh, long N0, long M,
    const double* Xq, int rprop_iters, double* K, double* L, double* alpha, double* mu, double* s2, double* loglik, double* grad,
    double* ucb, double* ei, double* hp_out)
{
    P::kernel::set_noise(noise);
    using GP_t = model::GP<P, Kernel, mean::Data<P>, model::gp::KernelLFOpt<P, opt::Rprop<P>>>;
    auto samples = rows_of(X, N, D);
    auto obs = rows_of(Y, N, Pout);
    GP_t gp(D, Pout);
    if (hp) {
        Eigen::VectorXd h((Eigen::Index)nh);
        for (int i = 0; i < nh; ++i) h(i) = hp[i];
        gp.kernel_function().set_h_params(h);
    }
    if (N0 > 0 && N0 < N) { // gp.hpp:126-152 incremental path for the last N - N0 samples
        std::vector<Eigen::VectorXd> s0(samples.begin(), samples.begin() + N0), o0(obs.begin(), obs.begin() + N0);
        gp.compute(s0, o0);
        for (long i = N0; i < N; ++i) gp.add_sample(samples[i], obs[i]);
    }
    else
        gp.compute(samples, obs);
    if (rprop_iters > 0) {
        Params::opt_rprop::set_iterations(rprop_iters);
        gp.optimize_hyperparams();
    }
    if (hp_out) {
        Eigen::VectorXd h = gp.kernel_function().h_params();
        for (Eigen::Index i = 0; i < h.size(); ++i) hp_out[i] = h(i);
    }
    put(gp._kernel, K);
    put(gp.matrixL(), L);
    put(gp.alpha(), alpha);
    if (loglik) *loglik = gp.compute_log_lik();
    if (grad) {
        Eigen::VectorXd g = gp.compute_kernel_grad_log_lik();
        for (Eigen::Index i = 0; i < g.size(); ++i) grad[i] = g(i);
    }
    acqui::UCB<P, GP_t> a_ucb(gp);
    acqui::EI<P, GP_t> a_ei(gp);
    FirstElem afun;
    for (long q = 0; q < M; ++q) {
        Eigen::VectorXd v((Eigen::Index)D);
        for (int k = 0; k < D; ++k) v(k) = Xq[q * D + k];
        Eigen::VectorXd m;
        double s;
        std::tie(m, s) = gp.query(v);
        for (int p = 0; p < Pout; ++p) mu[q * Pout + p] = m(p);
        s2[q] = s;
        // the reference's own consistency property (test_gp.cpp:506-507)
        if (!(gp.sigma(v) == s)) return 2;
        if (ucb) ucb[q] = opt::fun(a_ucb(v, afun, false));
        if (ei) ei[q] = opt::fun(a_ei(v, afun, false));
    }
    return 0;
}

// LOO-CV objective and its gradient (gp.hpp:339-399), kernel gradient of the likelihood for comparison
template <typename P, typename Kernel>
int run_loo(long N, int D, int Pout, const double* X, const double* Y, double noise, const double* hp, int nh, double* loo, double* loo_grad)
{
    P::kernel::set_noise(noise);
    using GP_t = model::GP<P, Kernel, mean::Data<P>, model::gp::KernelLFOpt<P, opt::Rprop<P>>>;
    auto samples = rows_of(X, N, D);
    auto obs = rows_of(Y, N, Pout);
    GP_t gp(D, Pout);
    if (hp) {
        Eigen::VectorXd h((Eigen::Index)nh);
        for (int i = 0; i < nh; ++i) h(i) = hp[i];
        gp.kernel_function().set_h_params(h);
    }
    gp.compute(samples, obs);
    *loo = gp.compute_log_loo_cv();
    if (loo_grad) {
        Eigen::VectorXd g = gp.compute_kernel_grad_log_loo_cv();
        for (Eigen::Index i = 0; i < g.size(); ++i) loo_grad[i] = g(i);
    }
    return 0;
}

// mean-parameter gradient of the likelihood (gp.hpp:313-330) with mean::FunctionARD<mean::Constant> (tunable affine map of
// a tunable constant): h-params = [tr (P x (P+1), row-major), constant]
template <typename P, typename Kernel>
int run_mean_grad(long N, int D, int Pout, const double* X, const double* Y, double noise, const double* hp, int nh, const double* mean_hp,
    int n_mean_hp, double* loglik, double* mean_grad, double* mu_at_x0)
{
    P::kernel::set_noise(noise);
    using Mean_t = mean::FunctionARD<P, mean::Constant<P>>;
    using GP_t = model::GP<P, Kernel, Mean_t, model::gp::KernelLFOpt<P, opt::Rprop<P>>>;
    auto samples = rows_of(X, N, D);
    auto obs = rows_of(Y, N, Pout);
    GP_t gp(D, Pout);
    if (hp) {
        Eigen::VectorXd h((Eigen::Index)nh);
        for (int i = 0; i < nh; ++i) h(i) = hp[i];
        gp.kernel_function().set_h_params(h);
    }
    if ((int)gp.mean_function().h_params_size() != n_mean_hp) return 3;
    Eigen::VectorXd mh((Eigen::Index)n_mean_hp);
    for (int i = 0; i < n_mean_hp; ++i) mh(i) = mean_hp[i];
    gp.mean_function().set_h_params(mh);
    gp.compute(samples, obs);
    *loglik = gp.compute_log_lik();
    Eigen::VectorXd g = gp.compute_mean_grad_log_lik();
    for (Eigen::Index i = 0; i < g.size(); ++i) mean_grad[i] = g(i);
    Eigen::VectorXd m = gp.mu(samples[0]);
    for (int p = 0; p < Pout; ++p) mu_at_x0[p] = m(p);
    return 0;
}

// Timing entry (bench.py --impl reference / cpu_baseline): the reference's own GP::compute (gp.hpp:88-116: kernel loops,
// LLT, alpha) once on the calling thread - Eigen's LLT is single-threaded - then acqui::UCB (ucb.hpp:83-90 -> GP::query,
// gp.hpp:159-167) over M candidates, one at a time as the reference does, fanned over `nthreads` host threads the way
// tools::par / opt::ParallelRepeater spread evaluations (query() is const).  Returns seconds for both parts.
template <typename P, typename Kernel>
int run_bench(long N, int D, const double* X, const double* Y, double noise, long M, const double* Xq, int nthreads, double* t_fit,
    double* t_query, double* best, long* best_idx)
{
    using clk = std::chrono::steady_clock;
    P::kernel::set_noise(noise);
    using GP_t = model::GP<P, Kernel, mean::Data<P>, model::gp::KernelLFOpt<P, opt::Rprop<P>>>;
    auto samples = rows_of(X, N, D);
    auto obs = rows_of(Y, N, 1);
    GP_t gp(D, 1);
    auto t0 = clk::now();
    gp.compute(samples, obs);
    *t_fit = std::chrono::duration<double>(clk::now() - t0).count();
    auto cands = rows_of(Xq, M, D);
    std::vector<double> val((size_t)M);
    acqui::UCB<P, GP_t> a_ucb(gp);
    t0 = clk::now();
    {
        std::vector<std::thread> th;
        const int nt = nthreads < 1 ? 1 : nthreads;
        for (int t = 0; t < nt; ++t)
            th.emplace_back([&, t] {
                FirstElem afun;
                for (long q = t; q < M; q += nt) val[(size_t)q] = opt::fun(a_ucb(cands[(size_t)q], afun, false));
            });
        for (auto& x : th) x.join();
    }
    long bi = 0;
    for (long q = 1; q < M; ++q)
        if (val[(size_t)q] > val[(size_t)bi]) bi = q;
    *t_query = std::chrono::duration<double>(clk::now() - t0).count();
    if (best) *best = M > 0 ? val[(size_t)bi] : 0.0;
    if (best_idx) *best_idx = bi;
    return 0;
}

} // namespace

extern "C" {

int ref_gp_bench(int kernel_id, long N, int D, const double* X, const double* Y, double noise, long M, const double* Xq, int nthreads,
    double* t_fit, double* t_query, double* best, long* best_idx)
{
    switch (kernel_id) {
    case 0: return run_bench<Params, kernel::SquaredExpARD<Params>>(N, D, X, Y, noise, M, Xq, nthreads, t_fit, t_query, best, best_idx);
    case 1: return run_bench<Params, kernel::MaternFiveHalves<Params>>(N, D, X, Y, noise, M, Xq, nthreads, t_fit, t_query, best, best_idx);
    default: return 1;
    }
}

int ref_gp_mean_grad(int kernel_id, long N, int D, int P, const double* X, const double* Y, double noise, const double* hp, int nh,
    const double* mean_hp, int n_mean_hp, double* loglik, double* mean_grad, double* mu_at_x0)
{
#define RUN(KK) return run_mean_grad<Params, kernel::KK<Params>>(N, D, P, X, Y, noise, hp, nh, mean_hp, n_mean_hp, loglik, mean_grad, mu_at_x0)
    switch (kernel_id) {
    case 0: RUN(SquaredExpARD);
    case 1: RUN(MaternFiveHalves);
    case 2: RUN(MaternThreeHalves);
    default: RUN(Exp);
    }
#undef RUN
}

int ref_gp_loo(int kernel_id, int optimize_noise, long N, int D, int P, const double* X, const double* Y, double noise,
    const double* hp, int nh, double* loo, double* loo_grad)
{
#define RUN(PP, KK) return run_loo<PP, kernel::KK<PP>>(N, D, P, X, Y, noise, hp, nh, loo, loo_grad)
    if (optimize_noise) {
        switch (kernel_id) {
        case 0: RUN(ParamsNoise, SquaredExpARD);
        case 1: RUN(ParamsNoise, MaternFiveHalves);
        case 2: RUN(ParamsNoise, MaternThreeHalves);
        default: RUN(ParamsNoise, Exp);
        }
    }
    switch (kernel_id) {
    case 0: RUN(Params, SquaredExpARD);
    case 1: RUN(Params, MaternFiveHalves);
    case 2: RUN(Params, MaternThreeHalves);
    case 4: RUN(ParamsLambda, SquaredExpARD); // k = 2
    default: RUN(Params, Exp);
    }
#undef RUN
}

// kernel_id: 0 SquaredExpARD, 1 MaternFiveHalves, 2 MaternThreeHalves, 3 Exp.  Y is N x P row-major observations
// (NOT mean-subtracted: mean::Data is the reference's own).  optimize_noise selects ParamsNoise (grad gets +1 entry).
int ref_gp_run(int kernel_id, int optimize_noise, long N, int D, int P, const double* X, const double* Y, double noise,
    const double* hp, int nh, long N0, long M, const double* Xq, int rprop_iters, double* K, double* L, double* alpha, double* mu,
    double* s2, double* loglik, double* grad, double* ucb, double* ei, double* hp_out)
{
#define RUN(PP, KK) return run<PP, kernel::KK<PP>>(N, D, P, X, Y, noise, hp, nh, N0, M, Xq, rprop_iters, K, L, alpha, mu, s2, loglik, grad, ucb, ei, hp_out)
    if (optimize_noise) {
        switch (kernel_id) {
        case 0: RUN(ParamsNoise, SquaredExpARD);
        case 1: RUN(ParamsNoise, MaternFiveHalves);
        case 2: RUN(ParamsNoise, MaternThreeHalves);
        default: RUN(ParamsNoise, Exp);
        }
    }
    switch (kernel_id) {
    case 0: RUN(Params, SquaredExpARD);
    case 1: RUN(Params, MaternFiveHalves);
    case 2: RUN(Params, MaternThreeHalves);
    case 4: RUN(ParamsLambda, SquaredExpARD); // k = 2
    default: RUN(Params, Exp);
    }
#undef RUN
}
}
