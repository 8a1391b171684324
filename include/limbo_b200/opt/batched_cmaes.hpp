// include/limbo_b200/opt/batched_cmaes.hpp — a derivative-free acquisition optimiser for the UNMODIFIED bayes_opt::BOptimizer and
// experimental::bayes_opt::Ehvi, the C++ twin of bayes_opt.BatchedCmaesSearch:
//
//     bayes_opt::BOptimizer<Params, modelfun<GP_t>, acquifun<limbo_b200::acqui::UCB<Params, GP_t>>,
//                           acquiopt<limbo_b200::opt::BatchedCmaes<Params>>> opt;
//
// 1. one random pass of `candidates` points in [0, 1]^D, announced through BatchedRandom's BatchRequest (one lb_acq_argmax /
//    lb_ehvi*_argmax with every value when a batch-aware functor answers it);
// 2. the best `starts` distinct points start one batched CMA-ES on the device (DESIGN.md §4.15), announced through a thread-local
//    CmaesRequest and one call of f: a batch-aware UCB / EI over limbo_b200::model::GP or model::SPGP, the batch-aware ECI over
//    two limbo_b200::model::GP (experimental::bayes_opt::CBOptimizer), or the acqui::Ehvi specialisation with two or three models,
//    answers it with one lb_acq_cmaes / lb_spgp_acq_cmaes / lb_eci_cmaes / lb_ehvi_cmaes when the means do not depend on the input;
// 3. the better of the search's best point and the random pass's is returned (the random pass's on ties).
// With a functor that is not batch-aware (the reference's acqui::UCB) the random pass runs one point at a time, as BatchedRandom
// does, and its best point is returned; so is it when the CmaesRequest stays unanswered.
//
// Parameters (struct Params::opt_batchedcmaes): candidates (10000), starts (32), lambda (0: 4 + floor(3 ln D)), sigma (0.1),
// generations (50), tolx (1e-6); DESIGN.md §4.15.
#ifndef LIMBO_B200_OPT_BATCHED_CMAES_HPP
#define LIMBO_B200_OPT_BATCHED_CMAES_HPP

#include <algorithm>
#include <cmath>
#include <numeric>
#include <random>
#include <set>
#include <vector>

#include "batched_random.hpp"

namespace limbo_b200 {
    namespace defaults {
        struct opt_batchedcmaes {
            BO_PARAM(int, candidates, 10000);
            BO_PARAM(int, starts, 32);
            BO_PARAM(int, lambda, 0);
            BO_PARAM(double, sigma, 0.1);
            BO_PARAM(int, generations, 50);
            BO_PARAM(double, tolx, 1e-6);
        };
    }

    namespace opt {
        template <typename Params>
        struct BatchedCmaes {
            // opt/optimizer.hpp:84-96: maximise f from `init`; bounded = search inside [0, 1]^D
            template <typename F>
            Eigen::VectorXd operator()(const F& f, const Eigen::VectorXd& init, bool bounded) const
            {
                const int D = (int)init.size();
                const int M = Params::opt_batchedcmaes::candidates();
                static thread_local std::mt19937_64 rng{std::random_device{}()};
                std::uniform_real_distribution<double> u01(0.0, 1.0);
                std::vector<Eigen::VectorXd> cands((size_t)M, Eigen::VectorXd((Eigen::Index)D));
                for (auto& c : cands)
                    for (int d = 0; d < D; ++d) c(d) = bounded ? u01(rng) : init(d) + (2.0 * u01(rng) - 1.0);
                cands[0] = init;
                _n_evals = 0;

                // 1. the random pass
                std::vector<double> values;
                BatchRequest req;
                req.candidates = &cands;
                req.values = &values;
                {
                    Scope<BatchRequest> s(current_batch(), &req);
                    const double v0 = limbo::opt::eval(f, cands[0]);
                    if (!req.answered) { // not batch-aware: the reference's one-point contract
                        double best = v0;
                        size_t idx = 0;
                        for (size_t i = 1; i < cands.size(); ++i) {
                            const double v = limbo::opt::eval(f, cands[i]);
                            if (v > best) { best = v; idx = i; }
                        }
                        return cands[idx];
                    }
                }
                const double best = req.best_value;
                const Eigen::VectorXd x_best = cands[(size_t)req.best_index];
                if (values.size() != cands.size()) return x_best;

                // 2. the best `starts` distinct points
                std::vector<size_t> order(cands.size());
                std::iota(order.begin(), order.end(), (size_t)0);
                std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) {
                    const double va = std::isnan(values[a]) ? -INFINITY : values[a], vb = std::isnan(values[b]) ? -INFINITY : values[b];
                    return va > vb;
                });
                std::vector<Eigen::VectorXd> starts;
                std::set<std::vector<double>> seen;
                for (size_t i : order) {
                    std::vector<double> key(cands[i].data(), cands[i].data() + D);
                    if (seen.insert(key).second) starts.push_back(cands[i]);
                    if ((int)starts.size() == Params::opt_batchedcmaes::starts()) break;
                }
                CmaesRequest c;
                c.starts = &starts;
                c.opts.lambda = Params::opt_batchedcmaes::lambda();
                c.opts.sigma0 = Params::opt_batchedcmaes::sigma();
                c.opts.generations = Params::opt_batchedcmaes::generations();
                c.opts.tolx = Params::opt_batchedcmaes::tolx();
                c.opts.seed = rng();
                c.opts.bounded = bounded ? 1 : 0;
                {
                    Scope<CmaesRequest> s(current_cmaes(), &c);
                    limbo::opt::eval(f, starts[0]);
                }
                if (!c.answered) return x_best;
                _n_evals = c.n_evals;
                return c.best_value > best ? c.best_x : x_best;
            }

            // candidates the last call's device search scored (0: no search ran)
            int64_t n_evals() const { return _n_evals; }

        protected:
            mutable int64_t _n_evals = 0;

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
