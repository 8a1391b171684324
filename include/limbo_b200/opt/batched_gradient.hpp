// include/limbo_b200/opt/batched_gradient.hpp — a multi-start gradient acquisition optimiser for the UNMODIFIED bayes_opt::BOptimizer,
// the C++ twin of bayes_opt.BatchedGradientSearch:
//
//     bayes_opt::BOptimizer<Params, modelfun<GP_t>, acquifun<limbo_b200::acqui::UCB<Params, GP_t>>,
//                           acquiopt<limbo_b200::opt::BatchedGradient<Params>>> opt;
//
// 1. one random pass of `candidates` points in [0, 1]^D, announced through BatchedRandom's BatchRequest (one lb_acq_argmax with
//    every value when a batch-aware UCB / EI answers it);
// 2. the best `starts` distinct points climb the acquisition in lockstep for `iterations` steps of Adam with the reference's update
//    (opt/adam.hpp: b1 = 0.9, b2 = 0.999, epsilon = 1e-8, step `alpha`, clipped to [0, 1] when bounded); each step announces the
//    start points through a thread-local GradRequest and calls f once, and the batch-aware functor files every point's value and
//    gradient (one lb_acq_grad per step);
// 3. the best point seen is returned, the random pass included.
// With a functor that is not batch-aware (the reference's acqui::UCB) the random pass runs one point at a time, as BatchedRandom
// does, no gradient is ever requested (f is never called with gradient = true), and the random pass's best point is returned.
//
// Parameters (struct Params::opt_batchedgradient): candidates (10000), starts (32), iterations (30), alpha (0.01); DESIGN.md §4.10.
#ifndef LIMBO_B200_OPT_BATCHED_GRADIENT_HPP
#define LIMBO_B200_OPT_BATCHED_GRADIENT_HPP

#include <algorithm>
#include <cmath>
#include <numeric>
#include <random>
#include <set>
#include <vector>

#include "batched_random.hpp"

namespace limbo_b200 {
    namespace defaults {
        struct opt_batchedgradient {
            BO_PARAM(int, candidates, 10000);
            BO_PARAM(int, starts, 32);
            BO_PARAM(int, iterations, 30);
            BO_PARAM(double, alpha, 0.01);
        };
    }

    namespace opt {
        template <typename Params>
        struct BatchedGradient {
            // opt/optimizer.hpp:84-96: maximise f from `init`; bounded = search inside [0, 1]^D
            template <typename F>
            Eigen::VectorXd operator()(const F& f, const Eigen::VectorXd& init, bool bounded) const
            {
                const int D = (int)init.size();
                const int M = Params::opt_batchedgradient::candidates();
                static thread_local std::mt19937_64 rng{std::random_device{}()};
                std::uniform_real_distribution<double> u01(0.0, 1.0);
                std::vector<Eigen::VectorXd> cands((size_t)M, Eigen::VectorXd((Eigen::Index)D));
                for (auto& c : cands)
                    for (int d = 0; d < D; ++d) c(d) = bounded ? u01(rng) : init(d) + (2.0 * u01(rng) - 1.0);
                cands[0] = init;
                _grad_steps = 0;

                // 1. the random pass
                std::vector<double> values;
                BatchRequest req;
                req.candidates = &cands;
                req.values = &values;
                {
                    Scope<BatchRequest> s(current_batch(), &req);
                    const double v0 = limbo::opt::eval(f, cands[0]);
                    if (!req.answered) { // not batch-aware: the reference's one-point contract, no gradients
                        double best = v0;
                        size_t idx = 0;
                        for (size_t i = 1; i < cands.size(); ++i) {
                            const double v = limbo::opt::eval(f, cands[i]);
                            if (v > best) { best = v; idx = i; }
                        }
                        return cands[idx];
                    }
                }
                double best = req.best_value;
                Eigen::VectorXd x_best = cands[(size_t)req.best_index];
                if (!req.gradients || values.size() != cands.size()) return x_best;

                // 2. the best `starts` distinct points
                std::vector<size_t> order(cands.size());
                std::iota(order.begin(), order.end(), (size_t)0);
                std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) {
                    const double va = std::isnan(values[a]) ? -INFINITY : values[a], vb = std::isnan(values[b]) ? -INFINITY : values[b];
                    return va > vb;
                });
                std::vector<Eigen::VectorXd> x;
                std::set<std::vector<double>> seen;
                for (size_t i : order) {
                    std::vector<double> key(cands[i].data(), cands[i].data() + D);
                    if (seen.insert(key).second) x.push_back(cands[i]);
                    if ((int)x.size() == Params::opt_batchedgradient::starts()) break;
                }
                const double b1 = 0.9, b2 = 0.999, eps = 1e-8, alpha = Params::opt_batchedgradient::alpha();
                double b1_t = b1, b2_t = b2;
                std::vector<Eigen::VectorXd> m(x.size(), Eigen::VectorXd::Zero((Eigen::Index)D)), v(m);
                for (int it = 0; it < Params::opt_batchedgradient::iterations(); ++it) {
                    GradRequest g;
                    g.points = &x;
                    {
                        Scope<GradRequest> s(current_grad_batch(), &g);
                        limbo::opt::eval(f, x[0]);
                    }
                    if (!g.answered) break;
                    ++_grad_steps;
                    for (size_t k = 0; k < x.size(); ++k) {
                        if (g.values(k) > best) { best = g.values(k); x_best = x[k]; }
                        for (int d = 0; d < D; ++d) {
                            const double gr = g.grads(k, d);
                            m[k](d) = b1 * m[k](d) + (1.0 - b1) * gr;
                            v[k](d) = b2 * v[k](d) + (1.0 - b2) * gr * gr;
                            double xn = x[k](d) + alpha * (m[k](d) / (1.0 - b1_t)) / (std::sqrt(v[k](d) / (1.0 - b2_t)) + eps);
                            if (bounded) xn = xn < 0.0 ? 0.0 : (xn > 1.0 ? 1.0 : xn);
                            x[k](d) = xn;
                        }
                    }
                    b1_t *= b1;
                    b2_t *= b2;
                }
                return x_best;
            }

            // gradient steps the last call took (each one lb_acq_grad call for all starts)
            int grad_steps() const { return _grad_steps; }

        protected:
            mutable int _grad_steps = 0;

            template <typename R>
            struct Scope { // announces *req for the duration of one call of f (nested requests restore the outer one)
                R*& slot;
                R* outer;
                Scope(R*& s, R* req) : slot(s), outer(s) { slot = req; }
                ~Scope() { slot = outer; }
            };
        };
    } // namespace opt
} // namespace limbo_b200

#endif
