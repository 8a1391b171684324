// include/limbo_b200/opt/batched_rprop.hpp — every hyper-parameter restart at once.
//
//   limbo_b200::opt::BatchedRprop<Params>
//       opt::Rprop (rprop.hpp:82-145) on the R rows of a start matrix in lockstep: each lane follows exactly the iterates
//       Rprop follows from its start (best-seen point, the eps_stop break and the bounded clipping per lane); every iteration
//       hands the lanes still running to one f.batch(X, compute_grad, lik, grad) call.  A lane that has stopped is no longer
//       evaluated.  Returns the R best points (R x n).
//   limbo_b200::model::gp::BatchedKernelLFOpt<Params>
//       the HyperParamsOptimizer of limbo_b200::model::GP that replaces
//       model::gp::KernelLFOpt<Params, opt::ParallelRepeater<Params, opt::Rprop<Params>>>: the R = opt_parallelrepeater::repeats()
//       deviations are drawn from tools::random_vector in restart order, the restarts run under BatchedRprop, one batched
//       evaluation without gradient scores the results, the first strictly larger value wins from (init, -FLT_MAX), and the GP is
//       refitted there (set_h_params, recompute(false), compute_log_lik), as KernelLFOpt does.  The likelihood goes through
//       GP::lml_grad_batch (lb_lml_grad_batch) where one call beats the evaluations it replaces (batch_pays), otherwise through
//       GP copies, as the reference's KernelLFOptimization does.
#ifndef LIMBO_B200_OPT_BATCHED_RPROP_HPP
#define LIMBO_B200_OPT_BATCHED_RPROP_HPP

#include <algorithm>
#include <cassert>
#include <cmath>
#include <limits>
#include <vector>

#include <Eigen/Core>

#include <limbo/tools/math.hpp>
#include <limbo/tools/random_generator.hpp>

#include "../../limbo_b200.h"

namespace limbo_b200 {
    namespace opt {
        template <typename Params>
        struct BatchedRprop {
            template <typename F>
            Eigen::MatrixXd operator()(const F& f, const Eigen::MatrixXd& init, bool bounded) const
            {
                assert(Params::opt_rprop::eps_stop() >= 0.);
                const long R = (long)init.rows();
                const int n = (int)init.cols();
                const double delta0 = 0.1, deltamin = 1e-6, deltamax = 50, etaminus = 0.5, etaplus = 1.2;
                const double eps_stop = Params::opt_rprop::eps_stop();
                std::vector<Eigen::VectorXd> delta, grad_old, params, best_params;
                std::vector<double> best((size_t)R, std::log(0.0));
                for (long r = 0; r < R; ++r) {
                    Eigen::VectorXd p(n);
                    for (int j = 0; j < n; ++j) {
                        p(j) = init(r, j);
                        if (bounded && p(j) < 0) p(j) = 0;
                        if (bounded && p(j) > 1) p(j) = 1;
                    }
                    params.push_back(p);
                    best_params.push_back(p);
                    delta.push_back(Eigen::VectorXd::Ones(n) * delta0);
                    grad_old.push_back(Eigen::VectorXd::Zero(n));
                }
                std::vector<long> live((size_t)R);
                for (long r = 0; r < R; ++r) live[(size_t)r] = r;
                for (int it = 0; it < Params::opt_rprop::iterations() && !live.empty(); ++it) {
                    Eigen::MatrixXd X((Eigen::Index)live.size(), n);
                    for (size_t q = 0; q < live.size(); ++q)
                        for (int j = 0; j < n; ++j) X((Eigen::Index)q, j) = params[(size_t)live[q]](j);
                    Eigen::VectorXd lik;
                    Eigen::MatrixXd G;
                    f.batch(X, true, lik, G);
                    std::vector<long> next;
                    for (size_t q = 0; q < live.size(); ++q) { // rprop.hpp:113-142, lane r
                        const long r = live[q];
                        if (lik((Eigen::Index)q) > best[(size_t)r]) {
                            best[(size_t)r] = lik((Eigen::Index)q);
                            best_params[(size_t)r] = params[(size_t)r];
                        }
                        Eigen::VectorXd grad(n);
                        for (int j = 0; j < n; ++j) grad(j) = -G((Eigen::Index)q, j);
                        Eigen::VectorXd go = grad_old[(size_t)r].cwiseProduct(grad);
                        Eigen::VectorXd& d = delta[(size_t)r];
                        Eigen::VectorXd& p = params[(size_t)r];
                        for (int j = 0; j < n; ++j) {
                            if (go(j) > 0)
                                d(j) = std::min(d(j) * etaplus, deltamax);
                            else if (go(j) < 0) {
                                d(j) = std::max(d(j) * etaminus, deltamin);
                                grad(j) = 0;
                            }
                            p(j) += -limbo::tools::signum(grad(j)) * d(j);
                            if (bounded && p(j) < 0) p(j) = 0;
                            if (bounded && p(j) > 1) p(j) = 1;
                        }
                        grad_old[(size_t)r] = grad;
                        if (!(grad.norm() < eps_stop)) next.push_back(r);
                    }
                    live.swap(next);
                }
                Eigen::MatrixXd out(R, n);
                for (long r = 0; r < R; ++r)
                    for (int j = 0; j < n; ++j) out(r, j) = best_params[(size_t)r](j);
                return out;
            }
        };
    } // namespace opt

    namespace model {
        namespace gp {
            // Whether one lb_lml_grad_batch call of `rows` vectors at n samples beats `rows` single evaluations: n within
            // LB_LML_BATCH_MAX_N and rows >= (n / 90)^2, the crossover measured on an H100 (DESIGN.md §4.12).
            inline bool batch_pays(long n, long rows) { return n <= LB_LML_BATCH_MAX_N && rows * 8100 >= n * n; }

            template <typename GP>
            struct BatchedLFObjective {
                const GP& gp;
                void batch(const Eigen::MatrixXd& X, bool compute_grad, Eigen::VectorXd& lik, Eigen::MatrixXd& grad) const
                {
                    if (batch_pays(gp.nb_samples(), (long)X.rows())) {
                        gp.lml_grad_batch(X, lik, compute_grad ? &grad : nullptr);
                        return;
                    }
                    lik.resize(X.rows());
                    if (compute_grad) grad.resize(X.rows(), X.cols());
                    for (Eigen::Index r = 0; r < X.rows(); ++r) { // kernel_lf_opt.hpp:77-92: a copy of the GP per evaluation
                        Eigen::VectorXd p(X.cols());
                        for (Eigen::Index j = 0; j < X.cols(); ++j) p(j) = X(r, j);
                        GP g(gp);
                        g.kernel_function().set_h_params(p);
                        g.recompute(false);
                        lik(r) = g.compute_log_lik();
                        if (compute_grad) {
                            Eigen::VectorXd gr = g.compute_kernel_grad_log_lik();
                            for (Eigen::Index j = 0; j < X.cols(); ++j) grad(r, j) = gr(j);
                        }
                    }
                }
            };

            template <typename Params>
            struct BatchedKernelLFOpt {
                template <typename GP>
                void operator()(GP& gp)
                {
                    _called = true;
                    const int R = Params::opt_parallelrepeater::repeats();
                    const double eps = Params::opt_parallelrepeater::epsilon();
                    assert(R > 0 && eps > 0.);
                    const Eigen::VectorXd init = gp.kernel_function().h_params();
                    const int n = (int)init.size();
                    Eigen::MatrixXd starts(R, n);
                    for (int r = 0; r < R; ++r) { // parallel_repeater.hpp:87, in restart order
                        Eigen::VectorXd dev = limbo::tools::random_vector(n).array() * 2. * eps - eps;
                        for (int j = 0; j < n; ++j) starts(r, j) = init(j) + dev(j);
                    }
                    BatchedLFObjective<GP> f{gp};
                    Eigen::MatrixXd V = opt::BatchedRprop<Params>()(f, starts, false);
                    Eigen::VectorXd vals;
                    Eigen::MatrixXd unused;
                    f.batch(V, false, vals, unused);
                    Eigen::VectorXd best = init;
                    double best_val = -std::numeric_limits<float>::max(); // parallel_repeater.hpp:102
                    for (int r = 0; r < R; ++r)
                        if (vals(r) > best_val) {
                            best_val = vals(r);
                            for (int j = 0; j < n; ++j) best(j) = V(r, j);
                        }
                    gp.kernel_function().set_h_params(best); // kernel_lf_opt.hpp:67-70
                    gp.recompute(false);
                    gp.compute_log_lik();
                }
                bool called() const { return _called; }

            private:
                bool _called = false;
            };
        } // namespace gp
    } // namespace model
} // namespace limbo_b200

#endif
