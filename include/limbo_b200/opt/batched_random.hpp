// include/limbo_b200/opt/batched_random.hpp — a device-aware inner acquisition optimiser and the batch-aware acquisition
// functors it drives, both usable with the UNMODIFIED bayes_opt::BOptimizer:
//
//     using GP_t   = limbo_b200::model::GP<Params, kernel::SquaredExpARD<Params>, mean::Data<Params>, ...>;
//     using Acq_t  = limbo_b200::acqui::UCB<Params, GP_t>;            // or EI
//     bayes_opt::BOptimizer<Params, modelfun<GP_t>, acquifun<Acq_t>, acquiopt<limbo_b200::opt::BatchedRandom<Params>>> opt;
//
// and, for constrained BO, limbo_b200::acqui::ECI<Params, GP_t, GPc_t> with experimental::bayes_opt::CBOptimizer (INTEGRATION.md).
//
// Why: the reference's optimiser contract (opt/optimizer.hpp:84-96; call site bayes_opt/boptimizer.hpp:151-156) hands the
// policy nothing but a closure `f(x, gradient)` that evaluates ONE point, so every reference policy (RandomPoint,
// GridSearch, NLOpt, CMA-ES) reaches the model one query() at a time, which leaves a GPU idle.  BatchedRandom keeps the
// contract - it only calls f - but announces the whole candidate set through a thread-local BatchRequest before the call;
// a batch-aware acquisition functor (the classes below, drop-ins for acqui::UCB / acqui::EI with the same constructor and
// operator()) sees the request inside f, scores all candidates in one device pass (GP::acq_argmax -> lb_acq_argmax) and
// files (best value, best index) in the request.  With an acquisition functor that is not batch-aware (e.g. the
// reference's acqui::UCB) the request stays unanswered and BatchedRandom evaluates the candidates one by one through f:
// same result, one device query per candidate.
//
// Parameters (struct Params::opt_batchedrandom): candidates (default 20000), refinements (2), shrink (0.1).
#ifndef LIMBO_B200_OPT_BATCHED_RANDOM_HPP
#define LIMBO_B200_OPT_BATCHED_RANDOM_HPP

#include <algorithm>
#include <cmath>
#include <limits>
#include <random>
#include <tuple>
#include <type_traits>
#include <vector>

#include <Eigen/Core>

#include <limbo/opt/optimizer.hpp>
#include <limbo/tools/macros.hpp>

#include "../../limbo_b200.h"

namespace limbo_b200 {
    namespace defaults {
        struct opt_batchedrandom {
            BO_PARAM(int, candidates, 20000);
            BO_PARAM(int, refinements, 2);
            BO_PARAM(double, shrink, 0.1);
        };
    }

    namespace model {
        template <typename Params, typename KernelFunction, typename MeanFunction, typename HyperParamsOptimizer>
        class GP;
    }

    namespace opt {
        // The candidate set announced by BatchedRandom for the duration of one call of f.
        struct BatchRequest {
            const std::vector<Eigen::VectorXd>* candidates = nullptr;
            bool answered = false;
            double best_value = 0.0;
            long best_index = -1;
        };
        inline BatchRequest*& current_batch()
        {
            static thread_local BatchRequest* req = nullptr;
            return req;
        }

        template <typename Params>
        struct BatchedRandom {
            // opt/optimizer.hpp:84-96: maximise f from `init`; bounded = search inside [0, 1]^D
            template <typename F>
            Eigen::VectorXd operator()(const F& f, const Eigen::VectorXd& init, bool bounded) const
            {
                const int D = (int)init.size();
                const int M = Params::opt_batchedrandom::candidates();
                static thread_local std::mt19937_64 rng{std::random_device{}()};
                std::uniform_real_distribution<double> u01(0.0, 1.0);
                std::vector<Eigen::VectorXd> cands((size_t)M, Eigen::VectorXd((Eigen::Index)D));
                for (auto& c : cands)
                    for (int d = 0; d < D; ++d) c(d) = bounded ? u01(rng) : init(d) + (2.0 * u01(rng) - 1.0);
                cands[0] = init; // the starting point takes part
                double best;
                long idx;
                std::tie(best, idx) = _argmax(f, cands);
                Eigen::VectorXd x = cands[(size_t)idx];
                double radius = 1.0;
                for (int r = 0; r < Params::opt_batchedrandom::refinements(); ++r) {
                    radius *= Params::opt_batchedrandom::shrink();
                    for (auto& c : cands)
                        for (int d = 0; d < D; ++d) {
                            double v = x(d) + (2.0 * u01(rng) - 1.0) * radius;
                            if (bounded) v = v < 0.0 ? 0.0 : (v > 1.0 ? 1.0 : v);
                            c(d) = v;
                        }
                    cands[0] = x; // keep the incumbent in the set
                    double b2;
                    long i2;
                    std::tie(b2, i2) = _argmax(f, cands);
                    if (b2 >= best) { best = b2; x = cands[(size_t)i2]; }
                }
                return x;
            }

        protected:
            template <typename F>
            static std::pair<double, long> _argmax(const F& f, const std::vector<Eigen::VectorXd>& cands)
            {
                BatchRequest req;
                req.candidates = &cands;
                BatchRequest*& slot = current_batch();
                BatchRequest* outer = slot;
                slot = &req;
                const double v0 = limbo::opt::eval(f, cands[0]); // a batch-aware functor answers the request in here
                slot = outer;
                if (req.answered) return std::make_pair(req.best_value, req.best_index);
                double best = v0;
                long idx = 0;
                for (size_t i = 1; i < cands.size(); ++i) { // not batch-aware: the reference's one-point contract
                    const double v = limbo::opt::eval(f, cands[i]);
                    if (v > best) { best = v; idx = (long)i; }
                }
                return std::make_pair(best, idx);
            }
        };
    } // namespace opt

    namespace acqui {
        namespace detail {
            // the device argmax implements the FirstElem aggregator (bayes_opt/bo_base.hpp:99-105); accept any aggregator
            // that acts like it on probe vectors
            template <typename A>
            inline bool acts_like_first_elem(const A& afun, int dim_out)
            {
                Eigen::VectorXd a((Eigen::Index)dim_out), b((Eigen::Index)dim_out);
                for (int i = 0; i < dim_out; ++i) { a(i) = 0.37 + 1.3 * i; b(i) = -2.5 - 0.7 * i; }
                return afun(a) == a(0) && afun(b) == b(0);
            }
            // files argmax(candidates) -> (best value, best index) in the pending request, if any
            template <typename Argmax>
            inline void answer_batch(const Argmax& argmax)
            {
                opt::BatchRequest* req = opt::current_batch();
                if (!req || req->answered || !req->candidates || req->candidates->empty()) return;
                auto res = argmax(*req->candidates);
                req->best_value = res.first;
                req->best_index = res.second;
                req->answered = true;
            }
            template <typename Model>
            inline void answer_batch(const Model& model, int acq_id, double p0, double p1)
            {
                answer_batch([&](const std::vector<Eigen::VectorXd>& c) { return model.acq_argmax(acq_id, p0, p1, c); });
            }
            template <typename M> struct is_device_gp : std::false_type {};
            template <typename P, typename K, typename Mf, typename H> struct is_device_gp<model::GP<P, K, Mf, H>> : std::true_type {};
        }

        // acqui::UCB (acqui/ucb.hpp:83-90), batch-aware
        template <typename Params, typename Model>
        class UCB {
        public:
            UCB(const Model& model, int iteration = 0) : _model(model) {}
            size_t dim_in() const { return _model.dim_in(); }
            size_t dim_out() const { return _model.dim_out(); }

            template <typename AggregatorFunction>
            limbo::opt::eval_t operator()(const Eigen::VectorXd& v, const AggregatorFunction& afun, bool gradient) const
            {
                assert(!gradient);
                if (opt::current_batch() && _model.nb_samples() > 0 && detail::acts_like_first_elem(afun, (int)_model.dim_out()))
                    detail::answer_batch(_model, LB_ACQ_UCB, Params::acqui_ucb::alpha(), 0.0);
                Eigen::VectorXd mu;
                double sigma;
                std::tie(mu, sigma) = _model.query(v);
                return limbo::opt::no_grad(afun(mu) + Params::acqui_ucb::alpha() * std::sqrt(sigma));
            }

        protected:
            const Model& _model;
        };

        // acqui::EI (acqui/ei.hpp:85-116), batch-aware; f_max = max_i afun(mu(x_i)) is refreshed in one batched pass
        template <typename Params, typename Model>
        class EI {
        public:
            EI(const Model& model, int iteration = 0) : _model(model), _nb_samples(-1), _f_max(0.0) {}
            size_t dim_in() const { return _model.dim_in(); }
            size_t dim_out() const { return _model.dim_out(); }

            template <typename AggregatorFunction>
            limbo::opt::eval_t operator()(const Eigen::VectorXd& v, const AggregatorFunction& afun, bool gradient) const
            {
                assert(!gradient);
                if (_model.samples().size() < 1) return limbo::opt::no_grad(0.0);
                if (_nb_samples != (int)_model.nb_samples()) { // ei.hpp:100-108
                    Eigen::MatrixXd mus;
                    Eigen::VectorXd s2;
                    _model.query_batch(_model.samples(), mus, s2);
                    _f_max = -std::numeric_limits<double>::max();
                    for (long i = 0; i < (long)mus.rows(); ++i) {
                        Eigen::VectorXd m((Eigen::Index)mus.cols());
                        for (long p = 0; p < (long)mus.cols(); ++p) m(p) = mus(i, p);
                        const double val = afun(m);
                        if (val > _f_max) _f_max = val;
                    }
                    _nb_samples = (int)_model.nb_samples();
                }
                if (opt::current_batch() && detail::acts_like_first_elem(afun, (int)_model.dim_out()))
                    detail::answer_batch(_model, LB_ACQ_EI, _f_max, Params::acqui_ei::jitter());
                Eigen::VectorXd mu;
                double sigma_sq;
                std::tie(mu, sigma_sq) = _model.query(v);
                const double sigma = std::sqrt(sigma_sq);
                if (sigma < 1e-10) return limbo::opt::no_grad(0.0);
                const double X = afun(mu) - _f_max - Params::acqui_ei::jitter();
                const double Z = X / sigma;
                const double phi = std::exp(-0.5 * std::pow(Z, 2.0)) / std::sqrt(2.0 * M_PI);
                const double Phi = 0.5 * std::erfc(-Z / std::sqrt(2));
                return limbo::opt::no_grad(X * Phi + sigma * phi);
            }

        protected:
            const Model& _model;
            mutable int _nb_samples;
            mutable double _f_max;
        };

        // experimental::acqui::ECI (experimental/acqui/eci.hpp:76-130), with the reference's constructor so that
        // experimental::bayes_opt::CBOptimizer builds it.  When both models are limbo_b200::model::GP and afun acts like FirstElem,
        // it answers BatchedRandom's request with one fused device pass over both models (GP::eci_argmax -> lb_eci_argmax);
        // otherwise it evaluates one point at a time, exactly as eci.hpp does.
        template <typename Params, typename Model, typename ConstraintModel>
        class ECI {
        public:
            ECI(const Model& model, const ConstraintModel& constraint_model, int iteration = 0)
                : _model(model), _constraint_model(constraint_model), _nb_samples(-1), _f_max(0.0) {}
            size_t dim_in() const { return _model.dim_in(); }
            size_t dim_out() const { return _model.dim_out(); }

            template <typename AggregatorFunction>
            limbo::opt::eval_t operator()(const Eigen::VectorXd& v, const AggregatorFunction& afun, bool gradient) const
            {
                assert(!gradient);
                if constexpr (detail::is_device_gp<Model>::value && detail::is_device_gp<ConstraintModel>::value) {
                    if (opt::current_batch() && _model.nb_samples() > 0 && detail::acts_like_first_elem(afun, (int)_model.dim_out())) {
                        _update_f_max(afun);
                        detail::answer_batch([&](const std::vector<Eigen::VectorXd>& c) {
                            return _model.eci_argmax(_constraint_model, _f_max, Params::acqui_eci::jitter(), c);
                        });
                    }
                }
                Eigen::VectorXd mu;
                double sigma_sq;
                std::tie(mu, sigma_sq) = _model.query(v);
                const double sigma = std::sqrt(sigma_sq);
                if (sigma < 1e-10 || _model.samples().size() < 1) return limbo::opt::no_grad(0.0);
                _update_f_max(afun);
                const double X = afun(mu) - _f_max - Params::acqui_eci::jitter();
                const double Z = X / sigma;
                const double phi = std::exp(-0.5 * std::pow(Z, 2.0)) / std::sqrt(2.0 * M_PI);
                const double Phi = 0.5 * std::erfc(-Z / std::sqrt(2));
                return limbo::opt::no_grad(_pf(v, afun) * (X * Phi + sigma * phi));
            }

        protected:
            const Model& _model;
            const ConstraintModel& _constraint_model;
            mutable int _nb_samples;
            mutable double _f_max;

            // f_max = max_i afun(mu(x_i)) (eci.hpp:91-99); one batched query on a device GP, one mu() per sample otherwise
            template <typename AggregatorFunction>
            void _update_f_max(const AggregatorFunction& afun) const
            {
                if (_nb_samples == (int)_model.nb_samples()) return;
                _f_max = -std::numeric_limits<double>::max();
                if constexpr (detail::is_device_gp<Model>::value) {
                    Eigen::MatrixXd mus;
                    Eigen::VectorXd s2;
                    _model.query_batch(_model.samples(), mus, s2);
                    for (long i = 0; i < (long)mus.rows(); ++i) {
                        Eigen::VectorXd m((Eigen::Index)mus.cols());
                        for (long p = 0; p < (long)mus.cols(); ++p) m(p) = mus(i, p);
                        _f_max = std::max(_f_max, (double)afun(m));
                    }
                }
                else
                    for (const auto& s : _model.samples()) _f_max = std::max(_f_max, (double)afun(_model.mu(s)));
                _nb_samples = (int)_model.nb_samples();
            }

            // eci.hpp:116-130
            template <typename AggregatorFunction>
            double _pf(const Eigen::VectorXd& v, const AggregatorFunction& afun) const
            {
                Eigen::VectorXd mu;
                double sigma_sq;
                std::tie(mu, sigma_sq) = _constraint_model.query(v);
                const double sigma = std::sqrt(sigma_sq);
                if (sigma < 1e-10 || _constraint_model.samples().size() < 1) return 1.0;
                const double Z = (afun(mu) - 1.0) / sigma;
                return 0.5 * std::erfc(-Z / std::sqrt(2));
            }
        };
    } // namespace acqui
} // namespace limbo_b200

#endif
