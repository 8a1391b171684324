// include/limbo_b200/model/spgp.hpp — header-only drop-in for limbo's experimental::model::SPGP
// (src/limbo/experimental/model/spgp.hpp:85-718): Snelson and Ghahramani's sparse GP with M learned pseudo-inputs, whose
// likelihood, gradient, factorisation and prediction run on the device through the C ABI (lb_spgp_*, include/limbo_b200.h).
// The host side keeps the reference's own code paths: the initial vector (srand(time) + std::random_shuffle, the row-major write
// of the pseudo-inputs into the column-major xb block), the HyperParamsOptimizer call, the mean functor.  Single output, SE-ARD.
// Differences: without USE_NLOPT the default optimiser is opt::Rprop<Params> (the reference's default names NLopt); a
// non-positive pivot of Q or A scores (-inf, zero gradient) instead of reading an unchecked LLT.
#ifndef LIMBO_B200_MODEL_SPGP_HPP
#define LIMBO_B200_MODEL_SPGP_HPP

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <ctime>
#include <limits>
#include <stdexcept>
#include <tuple>
#include <vector>

#include <Eigen/Core>

#include <limbo/opt.hpp>
#include <limbo/tools/macros.hpp>

#include "../../limbo_b200.h"
#include "batch_args.hpp"
#include "mean_traits.hpp" // mean_is_input_free

#ifndef LIMBO_MODEL_SPGP_HPP // the reference's header defines the same defaults
namespace limbo {
    namespace defaults {
        struct model_spgp { // experimental/model/spgp.hpp:64-73
            BO_PARAM(double, jitter, 0.000001);
            BO_PARAM(double, samples_percent, 10);
            BO_PARAM(int, min_m, 1);
            BO_PARAM(double, sig, 0.01);
            BO_PARAM(double, pred_kernel_sigma_sq, 0.5);
            BO_PARAM(double, pred_kernel_l, 0.5);
        };
    } // namespace defaults
} // namespace limbo
#endif

namespace limbo_b200 {
    namespace model {
#ifdef USE_NLOPT
        template <typename Params>
        using SPGPDefaultOpt = limbo::opt::NLOptGrad<Params, nlopt::LD_LBFGS>;
#else
        template <typename Params>
        using SPGPDefaultOpt = limbo::opt::Rprop<Params>;
#endif

        template <typename Params, typename KernelFunction, typename MeanFunction, class HyperParamsOptimizer = SPGPDefaultOpt<Params>>
        class SPGP {
        public:
            SPGP() : _dim_in(-1), _dim_out(-1) { _create(); }
            SPGP(int dim_in, int dim_out) : _dim_in(dim_in), _dim_out(dim_out), _mean_function(dim_out), _kernel_function(dim_in) { _create(); }
            SPGP(const std::vector<Eigen::VectorXd>& samples, const std::vector<Eigen::VectorXd>& observations) : SPGP()
            {
                _init(samples, observations);
            }
            SPGP(const SPGP&) = delete;
            SPGP& operator=(const SPGP&) = delete;
            ~SPGP() { lb_spgp_destroy(_h); }

            void optimize_hyperparams() // spgp.hpp:125-129
            {
                _optimize_init = true;
                _optimize_hyperparams();
                _compute_at(_w);
            }
            void compute(const std::vector<Eigen::VectorXd>& samples, const std::vector<Eigen::VectorXd>& observations) // :132-152
            {
                assert(samples.size() != 0 && samples.size() == observations.size());
                _optimize_init = true;
                _init(samples, observations);
                _compute();
            }
            void add_sample(const Eigen::VectorXd& sample, const Eigen::VectorXd& observation) // :155-186
            {
                _samples.push_back(sample);
                _observations.push_back(observation);
                _init(_samples, _observations);
                _optimize_init = true;
                _compute();
            }
            void recompute(bool = true) // :283-287
            {
                _optimize_init = true;
                _compute();
            }

            std::tuple<Eigen::VectorXd, double> query(const Eigen::VectorXd& v) const // :193-197
            {
                Eigen::MatrixXd mu;
                Eigen::VectorXd s2;
                query_batch(std::vector<Eigen::VectorXd>(1, v), mu, s2);
                return std::make_tuple(Eigen::VectorXd(mu.row(0)), s2(0));
            }
            // :204-207 and _predict :582-610; xt holds one point per row
            std::pair<Eigen::MatrixXd, Eigen::MatrixXd> predict(const Eigen::MatrixXd& xt) const
            {
                std::vector<Eigen::VectorXd> vs;
                for (Eigen::Index i = 0; i < xt.rows(); ++i) vs.push_back(Eigen::VectorXd(xt.row(i)));
                Eigen::MatrixXd mu;
                Eigen::VectorXd s2;
                query_batch(vs, mu, s2);
                Eigen::MatrixXd s2m(s2.size(), 1);
                for (Eigen::Index i = 0; i < s2.size(); ++i) s2m(i, 0) = s2(i);
                return {mu, s2m};
            }
            Eigen::MatrixXd mu(const Eigen::MatrixXd& v) const { return predict(v).first; }

            // ---- batched extensions with GP's signatures (not in the reference): what the batch-aware acquisitions of
            // opt/batched_random.hpp call under BatchedRandom, BatchedGradient and BatchedCmaes ----
            // mu: M x dim_out (mean function included), sigma2: M
            void query_batch(const std::vector<Eigen::VectorXd>& vs, Eigen::MatrixXd& mu, Eigen::VectorXd& sigma2) const
            {
                const int64_t nq = (int64_t)vs.size();
                mu = Eigen::MatrixXd(nq, std::max(_dim_out, 1));
                for (int64_t i = 0; i < nq; ++i) mu.row(i) = _mean_function(vs[(size_t)i], *this).transpose();
                if (_samples.empty()) {
                    sigma2 = Eigen::VectorXd(nq);
                    for (int64_t i = 0; i < nq; ++i) sigma2(i) = _kernel_function(vs[(size_t)i], vs[(size_t)i]);
                    return;
                }
                std::vector<double> q = detail::pack_rows(vs), m((size_t)nq), s((size_t)nq);
                _check(lb_spgp_query(_h, nq, q.data(), _optimized ? 1 : 0, m.data(), s.data()), "lb_spgp_query");
                for (int64_t i = 0; i < nq; ++i) mu(i, 0) += m[(size_t)i];
                detail::unpack(s, sigma2);
            }
            // fused UCB / EI + argmax on the device with the FirstElem aggregator (lb_spgp_acq_argmax)
            std::pair<double, long> acq_argmax(int acq_id, double p0, double p1, const std::vector<Eigen::VectorXd>& vs,
                std::vector<double>* values = nullptr) const
            {
                const std::vector<double> xq = detail::pack_rows(vs), mean0 = detail::first_means(*this, vs);
                double params[2] = {p0, p1}, best = 0;
                int64_t idx = 0;
                if (values) values->resize(vs.size());
                _check(lb_spgp_acq_argmax(_h, acq_id, params, (int64_t)vs.size(), xq.data(), _optimized ? 1 : 0, mean0.data(), 0.0,
                           values ? values->data() : nullptr, &best, &idx),
                    "lb_spgp_acq_argmax");
                return std::make_pair(best, (long)idx);
            }
            // UCB / EI values (M) and gradients (M x D) with the FirstElem aggregator in one device pass (lb_spgp_acq_grad)
            void acq_grad(int acq_id, double p0, double p1, const std::vector<Eigen::VectorXd>& vs, Eigen::VectorXd& values,
                Eigen::MatrixXd& grads) const
            {
                static_assert(mean_is_input_free<MeanFunction>::value, "acq_grad: the mean function has no input gradient");
                const long M = (long)vs.size();
                const int D = (int)vs[0].size();
                const std::vector<double> xq = detail::pack_rows(vs), mean0 = detail::first_means(*this, vs);
                std::vector<double> v((size_t)M), g((size_t)M * D);
                double params[2] = {p0, p1};
                _check(lb_spgp_acq_grad(_h, acq_id, params, M, xq.data(), _optimized ? 1 : 0, mean0.data(), 0.0, nullptr, v.data(), g.data()),
                    "lb_spgp_acq_grad");
                detail::unpack(v, values);
                detail::unpack(g, M, D, grads);
            }
            // mu (M x dim_out, mean added), sigma^2 (M) and their candidate gradients dmu, dsigma2 (M x D) in one device pass
            // (lb_spgp_query_grad)
            void query_grad(const std::vector<Eigen::VectorXd>& vs, Eigen::MatrixXd& mu, Eigen::VectorXd& sigma2, Eigen::MatrixXd& dmu,
                Eigen::MatrixXd& dsigma2) const
            {
                static_assert(mean_is_input_free<MeanFunction>::value, "query_grad: the mean function has no input gradient");
                const long M = (long)vs.size();
                const int D = (int)vs[0].size(), P = std::max(_dim_out, 1);
                const std::vector<double> xq = detail::pack_rows(vs);
                std::vector<double> m((size_t)M), s((size_t)M), gm((size_t)M * D), gs((size_t)M * D);
                _check(lb_spgp_query_grad(_h, M, xq.data(), _optimized ? 1 : 0, m.data(), s.data(), gm.data(), gs.data()), "lb_spgp_query_grad");
                mu = Eigen::MatrixXd((Eigen::Index)M, (Eigen::Index)P);
                for (long i = 0; i < M; ++i) {
                    mu.row(i) = _mean_function(vs[(size_t)i], *this).transpose();
                    mu(i, 0) += m[(size_t)i];
                }
                detail::unpack(s, sigma2);
                detail::unpack(gm, M, D, dmu);
                detail::unpack(gs, M, D, dsigma2);
            }
            // Batched CMA-ES on the device (lb_spgp_acq_cmaes) over UCB / EI (acq_id, p0, p1 as acq_argmax), one instance from each
            // start; the mean must not depend on the input (its first output is passed as a constant).  Returns the best value; best_x
            // and n_evals (candidates scored) are filled in.
            double acq_cmaes(int acq_id, double p0, double p1, const std::vector<Eigen::VectorXd>& starts, const lb_cmaes_opts& opts,
                Eigen::VectorXd& best_x, int64_t& n_evals) const
            {
                static_assert(mean_is_input_free<MeanFunction>::value, "acq_cmaes: the mean function depends on the input");
                const int D = (int)starts[0].size();
                const std::vector<double> st = detail::pack_rows(starts);
                double params[2] = {p0, p1}, best = 0;
                best_x.resize(D);
                _check(lb_spgp_acq_cmaes(_h, acq_id, params, _optimized ? 1 : 0, _mean_function(Eigen::VectorXd::Zero(D), *this)(0), &opts,
                           (int64_t)starts.size(), st.data(), best_x.data(), &best, &n_evals),
                    "lb_spgp_acq_cmaes");
                return best;
            }
            double sigma(const Eigen::VectorXd& v) const { return std::get<1>(query(v)); }

            int dim_in() const { assert(_dim_in != -1); return _dim_in; }
            int dim_out() const { assert(_dim_out != -1); return _dim_out; }
            const MeanFunction& mean_function() const { return _mean_function; }
            MeanFunction& mean_function() { return _mean_function; }
            Eigen::VectorXd max_observation() const
            {
                double m = -std::numeric_limits<double>::infinity();
                for (const auto& o : _observations) m = std::max(m, o.maxCoeff());
                return Eigen::VectorXd::Constant(1, m);
            }
            Eigen::VectorXd mean_observation() const { return _samples.empty() ? Eigen::VectorXd::Zero(std::max(_dim_out, 1)) : _obs_mean; }
            int nb_samples() const { return (int)_samples.size(); }
            int nb_pseudo_samples() const { return _w.size() ? (int)_m : 0; }
            std::vector<Eigen::VectorXd> samples() const { return _samples; }
            std::vector<Eigen::VectorXd> pseudo_samples() const // HyperParams' column-major xb (:99-100)
            {
                std::vector<Eigen::VectorXd> r;
                for (size_t j = 0; j < (_w.size() ? _m : 0); ++j) {
                    Eigen::VectorXd p(_dim_in);
                    for (int d = 0; d < _dim_in; ++d) p(d) = _w(d * _m + j);
                    r.push_back(p);
                }
                return r;
            }

        protected:
            lb_spgp* _h = nullptr;
            int _dim_in, _dim_out;
            size_t _m = 0;
            std::vector<Eigen::VectorXd> _samples, _observations;
            Eigen::VectorXd _obs_mean;
            std::vector<double> _X, _y_zm; // row-major samples, first output minus the mean
            MeanFunction _mean_function;
            KernelFunction _kernel_function;
            HyperParamsOptimizer _hp_optimize;
            bool _optimize_init = true, _optimized = false;
            Eigen::VectorXd _w_init, _w;

            static void _check(int rc, const char* where)
            {
                if (rc != LB_OK) throw std::runtime_error(std::string(where) + ": " + lb_strerror(rc));
            }
            void _create() { _check(lb_spgp_create(&_h, 0), "lb_spgp_create"); }

            void _init(const std::vector<Eigen::VectorXd>& samples, const std::vector<Eigen::VectorXd>& observations) // :353-379
            {
                _samples = samples;
                _observations = observations;
                _dim_in = (int)samples[0].size();
                _dim_out = (int)observations[0].size();
                _mean_function = MeanFunction(_dim_out);
                _kernel_function = KernelFunction(_dim_in);
                const size_t n = samples.size();
                _obs_mean = Eigen::VectorXd::Zero(_dim_out);
                for (const auto& o : observations) _obs_mean = _obs_mean + o;
                _obs_mean = _obs_mean / (double)n;
                _X.assign(n * _dim_in, 0.0);
                _y_zm.assign(n, 0.0);
                for (size_t i = 0; i < n; ++i) {
                    for (int d = 0; d < _dim_in; ++d) _X[i * _dim_in + d] = samples[i](d);
                    _y_zm[i] = observations[i](0) - _mean_function(samples[i], *this)(0);
                }
                _update_m();
                _check(lb_spgp_set_data(_h, (int64_t)n, _dim_in, _X.data(), _y_zm.data()), "lb_spgp_set_data");
                _optimize_init = true;
                srand(time(NULL));
            }
            void _update_m() // :381-387
            {
                _m = Params::model_spgp::samples_percent() * _samples.size() / 100;
                if (_m < (size_t)Params::model_spgp::min_m())
                    _m = Params::model_spgp::min_m();
            }
            void _compute()
            {
                _optimize_hyperparams();
                _compute_at(_w);
            }
            void _optimize_hyperparams() // :409-444
            {
                if (_optimize_init) {
                    _update_m();
                    const size_t n = _samples.size();
                    _w_init = Eigen::VectorXd((_m + 1) * _dim_in + 2);
                    Eigen::VectorXd positions = Eigen::VectorXd::LinSpaced(n, 0, n - 1);
                    std::random_shuffle(positions.data(), positions.data() + positions.size());
                    for (size_t i = 0; i < _m; ++i)
                        for (int d = 0; d < _dim_in; ++d) _w_init(i * _dim_in + d) = _samples[(size_t)positions(i)](d); // row-major
                    double y2 = 0.0;
                    for (double v : _y_zm) y2 += v * v;
                    y2 /= (double)n;
                    for (int d = 0; d < _dim_in; ++d) {
                        double lo = _samples[0](d), hi = lo;
                        for (const auto& s : _samples) { lo = std::min(lo, s(d)); hi = std::max(hi, s(d)); }
                        _w_init(_m * _dim_in + d) = -2 * std::log((hi - lo) / 2);
                    }
                    _w_init((_m + 1) * _dim_in) = std::log(y2);
                    _w_init((_m + 1) * _dim_in + 1) = std::log(y2 / 4);
                    _optimize_init = false;
                }
                auto f = [&](const Eigen::VectorXd& x, bool g) { return this->_likelihood(x, g); };
                _w = _hp_optimize(f, _w_init, false);
                _optimized = true;
            }
            // _likelihood(w, eval_grad) (:446-451): (-fw, -dfw)
            limbo::opt::eval_t _likelihood(const Eigen::VectorXd& w, bool eval_grad = false) const
            {
                double f = 0.0;
                std::vector<double> g(eval_grad ? (size_t)w.size() : 0);
                const int rc = lb_spgp_lik(_h, (int64_t)_m, (int64_t)w.size(), w.data(), Params::model_spgp::jitter(), &f, eval_grad ? g.data() : nullptr);
                if (rc > 0) {
                    if (!eval_grad) return limbo::opt::no_grad(-std::numeric_limits<double>::infinity());
                    return {-std::numeric_limits<double>::infinity(), Eigen::VectorXd(Eigen::VectorXd::Zero(w.size()))};
                }
                _check(rc, "lb_spgp_lik");
                if (!eval_grad) return limbo::opt::no_grad(f);
                Eigen::VectorXd gv(w.size());
                for (int i = 0; i < (int)w.size(); ++i) gv(i) = g[(size_t)i];
                return {f, gv};
            }
            // _compute(false) at HyperParams(w) (:389-407)
            void _compute_at(const Eigen::VectorXd& w)
            {
                _check(lb_spgp_compute(_h, (int64_t)_m, (int64_t)w.size(), w.data(), Params::model_spgp::jitter()), "lb_spgp_compute");
                _w = w;
            }
        };
    } // namespace model
} // namespace limbo_b200

#endif
