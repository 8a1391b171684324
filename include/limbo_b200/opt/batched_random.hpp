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
#include "../model/mean_traits.hpp"

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
        template <typename Params, typename KernelFunction, typename MeanFunction, class HyperParamsOptimizer>
        class SPGP;
    }

    namespace opt {
        // The candidate set announced by BatchedRandom for the duration of one call of f.
        struct BatchRequest {
            const std::vector<Eigen::VectorXd>* candidates = nullptr;
            bool answered = false;
            double best_value = 0.0;
            long best_index = -1;
            std::vector<double>* values = nullptr; // when set, the answer also files every candidate's value here
            bool gradients = false;                // the answering functor also answers a GradRequest (BatchedGradient)
        };
        inline BatchRequest*& current_batch()
        {
            static thread_local BatchRequest* req = nullptr;
            return req;
        }

        // The start points announced by BatchedGradient (opt/batched_gradient.hpp) for one call of f: a batch-aware UCB / EI over
        // limbo_b200::model::GP or model::SPGP files every point's value and gradient (one lb_acq_grad or lb_spgp_acq_grad).
        struct GradRequest {
            const std::vector<Eigen::VectorXd>* points = nullptr;
            bool answered = false;
            Eigen::VectorXd values;
            Eigen::MatrixXd grads;
        };
        inline GradRequest*& current_grad_batch()
        {
            static thread_local GradRequest* req = nullptr;
            return req;
        }

        // The start points announced by BatchedCmaes (opt/batched_cmaes.hpp) for one call of f: a batch-aware UCB / EI over
        // limbo_b200::model::GP or model::SPGP, ECI over two limbo_b200::model::GP, or the acqui::Ehvi specialisation
        // (acqui/ehvi.hpp), runs one device CMA-ES from them (lb_acq_cmaes / lb_spgp_acq_cmaes / lb_eci_cmaes / lb_ehvi_cmaes) and
        // files its best point, value and evaluations.  Means must not depend on the input.
        struct CmaesRequest {
            const std::vector<Eigen::VectorXd>* starts = nullptr;
            lb_cmaes_opts opts{};
            bool answered = false;
            Eigen::VectorXd best_x;
            double best_value = 0.0;
            int64_t n_evals = 0;
        };
        inline CmaesRequest*& current_cmaes()
        {
            static thread_local CmaesRequest* req = nullptr;
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
                opt::BatchRequest* req = opt::current_batch();
                std::vector<double>* values = req ? req->values : nullptr;
                answer_batch([&](const std::vector<Eigen::VectorXd>& c) { return model.acq_argmax(acq_id, p0, p1, c, values); });
                if (req && req->answered) req->gradients = true;
            }
            // files every start point's value and gradient in the pending GradRequest, if any (one lb_acq_grad)
            template <typename Model>
            inline void answer_grad_batch(const Model& model, int acq_id, double p0, double p1)
            {
                opt::GradRequest* req = opt::current_grad_batch();
                if (!req || req->answered || !req->points || req->points->empty()) return;
                model.acq_grad(acq_id, p0, p1, *req->points, req->values, req->grads);
                req->answered = true;
            }
            // runs the pending CmaesRequest, if any, through run(starts, opts, best_x, n_evals) -> best value
            template <typename Run>
            inline void answer_cmaes(const Run& run)
            {
                opt::CmaesRequest* req = opt::current_cmaes();
                if (!req || req->answered || !req->starts || req->starts->empty()) return;
                req->best_value = run(*req->starts, req->opts, req->best_x, req->n_evals);
                req->answered = true;
            }
            template <typename Model>
            inline void answer_cmaes(const Model& model, int acq_id, double p0, double p1)
            {
                answer_cmaes([&](const std::vector<Eigen::VectorXd>& st, const lb_cmaes_opts& o, Eigen::VectorXd& x, int64_t& n) {
                    return model.acq_cmaes(acq_id, p0, p1, st, o, x, n);
                });
            }
            // value and gradient at one point from one lb_acq_grad call
            template <typename Model>
            inline limbo::opt::eval_t one_point_grad(const Model& model, int acq_id, double p0, double p1, const Eigen::VectorXd& v)
            {
                Eigen::VectorXd vals;
                Eigen::MatrixXd grads;
                model.acq_grad(acq_id, p0, p1, std::vector<Eigen::VectorXd>{v}, vals, grads);
                Eigen::VectorXd g((Eigen::Index)v.size());
                for (int d = 0; d < (int)v.size(); ++d) g(d) = grads(0, d);
                return limbo::opt::eval_t{vals(0), g};
            }
            template <typename M> struct is_device_gp : std::false_type {};
            template <typename P, typename K, typename Mf, typename H> struct is_device_gp<model::GP<P, K, Mf, H>> : std::true_type {};
            template <typename M> struct has_candidate_grad : std::false_type {};
            template <typename P, typename K, typename Mf, typename H>
            struct has_candidate_grad<model::GP<P, K, Mf, H>> : model::mean_is_input_free<Mf> {};
            template <typename P, typename K, typename Mf, typename H>
            struct has_candidate_grad<model::SPGP<P, K, Mf, H>> : model::mean_is_input_free<Mf> {};
            // a device model with an input-free mean: the device CMA-ES (lb_acq_cmaes, lb_eci_cmaes and lb_ehvi_cmaes for a GP,
            // lb_spgp_acq_cmaes for an SPGP) takes it
            template <typename M> struct has_device_cmaes : std::false_type {};
            template <typename P, typename K, typename Mf, typename H>
            struct has_device_cmaes<model::GP<P, K, Mf, H>> : model::mean_is_input_free<Mf> {};
            template <typename P, typename K, typename Mf, typename H>
            struct has_device_cmaes<model::SPGP<P, K, Mf, H>> : model::mean_is_input_free<Mf> {};
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
                if constexpr (detail::has_candidate_grad<Model>::value) {
                    if (gradient) { // one lb_acq_grad call, FirstElem aggregator only
                        assert(detail::acts_like_first_elem(afun, (int)_model.dim_out()));
                        return detail::one_point_grad(_model, LB_ACQ_UCB, Params::acqui_ucb::alpha(), 0.0, v);
                    }
                    if (opt::current_grad_batch() && detail::acts_like_first_elem(afun, (int)_model.dim_out()))
                        detail::answer_grad_batch(_model, LB_ACQ_UCB, Params::acqui_ucb::alpha(), 0.0);
                }
                else
                    assert(!gradient);
                if constexpr (detail::has_device_cmaes<Model>::value)
                    if (opt::current_cmaes() && _model.nb_samples() > 0 && detail::acts_like_first_elem(afun, (int)_model.dim_out()))
                        detail::answer_cmaes(_model, LB_ACQ_UCB, Params::acqui_ucb::alpha(), 0.0);
                if (opt::current_batch() && _model.nb_samples() > 0 && detail::acts_like_first_elem(afun, (int)_model.dim_out())) {
                    detail::answer_batch(_model, LB_ACQ_UCB, Params::acqui_ucb::alpha(), 0.0);
                    if (!detail::has_candidate_grad<Model>::value) opt::current_batch()->gradients = false;
                }
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
                if constexpr (!detail::has_candidate_grad<Model>::value)
                    assert(!gradient);
                if (_model.samples().size() < 1) // ei.hpp:88-89; the gradient is 0 too
                    return gradient ? limbo::opt::eval_t{0.0, Eigen::VectorXd(Eigen::VectorXd::Zero((Eigen::Index)v.size()))} : limbo::opt::no_grad(0.0);
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
                if constexpr (detail::has_candidate_grad<Model>::value) {
                    if (gradient) { // one lb_acq_grad call, FirstElem aggregator only
                        assert(detail::acts_like_first_elem(afun, (int)_model.dim_out()));
                        return detail::one_point_grad(_model, LB_ACQ_EI, _f_max, Params::acqui_ei::jitter(), v);
                    }
                    if (opt::current_grad_batch() && detail::acts_like_first_elem(afun, (int)_model.dim_out()))
                        detail::answer_grad_batch(_model, LB_ACQ_EI, _f_max, Params::acqui_ei::jitter());
                }
                if constexpr (detail::has_device_cmaes<Model>::value)
                    if (opt::current_cmaes() && detail::acts_like_first_elem(afun, (int)_model.dim_out()))
                        detail::answer_cmaes(_model, LB_ACQ_EI, _f_max, Params::acqui_ei::jitter());
                if (opt::current_batch() && detail::acts_like_first_elem(afun, (int)_model.dim_out())) {
                    detail::answer_batch(_model, LB_ACQ_EI, _f_max, Params::acqui_ei::jitter());
                    if (!detail::has_candidate_grad<Model>::value) opt::current_batch()->gradients = false;
                }
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
        // otherwise it evaluates one point at a time, exactly as eci.hpp does.  When, in addition, both means do not depend on the
        // input, it answers operator()(v, afun, true) and BatchedGradient's GradRequest with one lb_eci_grad (GP::eci_grad), files
        // every candidate's value in BatchedGradient's random pass so that the optimiser climbs, and answers BatchedCmaes's
        // CmaesRequest with one lb_eci_cmaes (GP::eci_cmaes) once the objective has samples.
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
                if constexpr (has_grad) {
                    const bool first = detail::acts_like_first_elem(afun, (int)_model.dim_out());
                    if (gradient) { // one lb_eci_grad call, FirstElem aggregator only
                        assert(first);
                        Eigen::VectorXd vals;
                        Eigen::MatrixXd grads;
                        _grad(afun, std::vector<Eigen::VectorXd>{v}, vals, grads);
                        return limbo::opt::eval_t{vals(0), Eigen::VectorXd(grads.row(0).transpose())};
                    }
                    opt::GradRequest* greq = opt::current_grad_batch();
                    if (greq && first && !greq->answered && greq->points && !greq->points->empty()) { // BatchedGradient's start points
                        _grad(afun, *greq->points, greq->values, greq->grads);
                        greq->answered = true;
                    }
                }
                else
                    assert(!gradient);
                if constexpr (has_cmaes) {
                    if (opt::current_cmaes() && _model.nb_samples() > 0 && detail::acts_like_first_elem(afun, (int)_model.dim_out())) {
                        _update_f_max(afun);
                        detail::answer_cmaes([&](const std::vector<Eigen::VectorXd>& st, const lb_cmaes_opts& o, Eigen::VectorXd& x, int64_t& n) {
                            return _model.eci_cmaes(_constraint_model, _f_max, Params::acqui_eci::jitter(), st, o, x, n);
                        });
                    }
                }
                if constexpr (detail::is_device_gp<Model>::value && detail::is_device_gp<ConstraintModel>::value) {
                    opt::BatchRequest* req = opt::current_batch();
                    if (req && _model.nb_samples() > 0 && detail::acts_like_first_elem(afun, (int)_model.dim_out())) {
                        _update_f_max(afun);
                        detail::answer_batch([&](const std::vector<Eigen::VectorXd>& c) {
                            return _model.eci_argmax(_constraint_model, _f_max, Params::acqui_eci::jitter(), c, req->values);
                        });
                        if (req->answered) req->gradients = has_grad;
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
            // both models are device GPs whose means do not depend on the input: gradients from lb_eci_grad
            static constexpr bool has_grad = detail::has_candidate_grad<Model>::value && detail::has_candidate_grad<ConstraintModel>::value;
            // both models are device GPs whose means do not depend on the input: the search from lb_eci_cmaes
            static constexpr bool has_cmaes = detail::is_device_gp<Model>::value && detail::is_device_gp<ConstraintModel>::value
                && detail::has_device_cmaes<Model>::value && detail::has_device_cmaes<ConstraintModel>::value;

            const Model& _model;
            const ConstraintModel& _constraint_model;
            mutable int _nb_samples;
            mutable double _f_max;

            // values and gradients at the points vs (one lb_eci_grad; 0 before the objective has samples, eci.hpp:86)
            template <typename AggregatorFunction>
            void _grad(const AggregatorFunction& afun, const std::vector<Eigen::VectorXd>& vs, Eigen::VectorXd& values, Eigen::MatrixXd& grads) const
            {
                if (_model.nb_samples() > 0) _update_f_max(afun);
                _model.eci_grad(_constraint_model, _f_max, Params::acqui_eci::jitter(), vs, values, grads);
            }

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
