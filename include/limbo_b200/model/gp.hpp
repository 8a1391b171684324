// include/limbo_b200/model/gp.hpp — header-only drop-in for limbo::model::GP.
//
//   limbo_b200::model::GP<Params, KernelFunction, MeanFunction, HyperParamsOptimizer>
//
// has the public member set and signatures of the reference's
// limbo::model::GP (src/limbo/model/gp.hpp:81-511), so it can be used wherever a
// "Model" is expected: bayes_opt::BOptimizer<Params, modelfun<...>>,
// acqui::UCB / EI / GP_UCB, model::gp::KernelLFOpt, stat::*, stop::MaxPredictedValue,
// MultiGP<Params, limbo_b200::model::GP, ...>.  The kernel / mean / hp-opt policy
// types stay the reference's own (kernel::SquaredExpARD<Params>, mean::Data<Params>,
// gp::KernelLFOpt<Params> ...); only their public state (h_params(), noise()) is read
// and handed to the CUDA library through the C ABI (include/limbo_b200.h).
// Mean functions and aggregators remain host functors, exactly as in the reference.
//
// A kernel type without a trait specialisation below is a compile-time error: there
// is no CPU fallback.
#ifndef LIMBO_B200_MODEL_GP_HPP
#define LIMBO_B200_MODEL_GP_HPP

#include <cassert>
#include <cmath>
#include <iostream>
#include <limits>
#include <stdexcept>
#include <string>
#include <tuple>
#include <vector>

#include <Eigen/Core>

#include "../../limbo_b200.h"

namespace limbo {
    namespace kernel {
        template <typename Params> struct SquaredExpARD;
        template <typename Params> struct MaternFiveHalves;
        template <typename Params> struct MaternThreeHalves;
        template <typename Params> struct Exp;
    }
}

namespace limbo_b200 {
    namespace model {

        // kernel policy type -> device kernel id (kernel/*.hpp)
        template <typename K> struct kernel_traits; // no definition: unsupported kernels do not compile
        template <typename P> struct kernel_traits<limbo::kernel::SquaredExpARD<P>> {
            static constexpr int id = LB_KERNEL_SQUARED_EXP_ARD;
            // k > 0 (Lambda columns, squared_exp_ard.hpp:109-126): the h-params carry the D x k matrix, lb_set_kernel reads k from their count
            static void check() { assert(P::kernel_squared_exp_ard::k() >= 0 && P::kernel_squared_exp_ard::k() <= 4 && "SquaredExpARD: 0 <= k <= 4"); }
        };
        template <typename P> struct kernel_traits<limbo::kernel::MaternFiveHalves<P>> {
            static constexpr int id = LB_KERNEL_MATERN_FIVE_HALVES;
            static void check() {}
        };
        template <typename P> struct kernel_traits<limbo::kernel::MaternThreeHalves<P>> {
            static constexpr int id = LB_KERNEL_MATERN_THREE_HALVES;
            static void check() {}
        };
        template <typename P> struct kernel_traits<limbo::kernel::Exp<P>> {
            static constexpr int id = LB_KERNEL_EXP;
            static void check() {}
        };

        inline void lb_check(int rc, const char* where)
        {
            if (rc < 0) throw std::runtime_error(std::string(where) + ": " + lb_strerror(rc) + " " + lb_last_cuda_error());
        }

        template <typename Params, typename KernelFunction, typename MeanFunction, typename HyperParamsOptimizer>
        class GP {
        public:
            // gp.hpp:84-88
            GP() : _dim_in(-1), _dim_out(-1), _inv_kernel_updated(false) { _create(); }
            GP(int dim_in, int dim_out)
                : _dim_in(dim_in), _dim_out(dim_out), _kernel_function(dim_in), _mean_function(dim_out), _inv_kernel_updated(false) { _create(); }

            // value semantics: KernelLFOptimization copies the GP per evaluation (kernel_lf_opt.hpp:79)
            GP(const GP& o)
                : _dim_in(o._dim_in), _dim_out(o._dim_out), _kernel_function(o._kernel_function), _mean_function(o._mean_function),
                  _samples(o._samples), _observations(o._observations), _mean_vector(o._mean_vector), _obs_mean(o._obs_mean),
                  _mean_observation(o._mean_observation), _log_lik(o._log_lik), _log_loo_cv(o._log_loo_cv),
                  _inv_kernel_updated(false), _hp_optimize(o._hp_optimize)
            {
                lb_check(lb_clone(o._h, &_h), "lb_clone");
            }
            GP& operator=(const GP& o)
            {
                if (this != &o) {
                    GP tmp(o);
                    swap(tmp);
                }
                return *this;
            }
            ~GP() { if (_h) lb_destroy(_h); }

            // Same contract as limbo::model::GP::compute (gp.hpp:88-116): takes ownership of a copy of the data, (re)builds
            // the policy functors when a dimension changed, forms obs_mean on the host (the mean is a host functor) and,
            // unless told otherwise, runs the device fit.
            void compute(const std::vector<Eigen::VectorXd>& samples, const std::vector<Eigen::VectorXd>& observations,
                bool compute_kernel = true)
            {
                assert(!samples.empty() && !observations.empty() && samples.size() == observations.size());
                _adopt_dims(samples.front().size(), observations.front().size());
                _samples = samples;
                _pack_rows(observations, _observations);
                _refresh_means();
                if (compute_kernel) _compute_full_kernel();
            }

            void optimize_hyperparams() { _hp_optimize(*this); } // gp.hpp:119-122

            // Incremental update (gp.hpp:126-152): one kernel row, one forward solve and a new alpha on the device
            // (lb_append) instead of a refit.
            void add_sample(const Eigen::VectorXd& sample, const Eigen::VectorXd& observation)
            {
                if (_samples.empty())
                    _adopt_dims(sample.size(), observation.size());
                else
                    assert(sample.size() == _dim_in && observation.size() == _dim_out);
                _samples.push_back(sample);
                const long n = (long)_samples.size();
                _observations.conservativeResize(n, _dim_out);
                for (int p = 0; p < _dim_out; ++p) _observations(n - 1, p) = observation(p);
                _refresh_means();
                _compute_incremental_kernel();
            }

            // gp.hpp:159-191 — one point; the batched extensions below are what a device-aware optimiser calls
            std::tuple<Eigen::VectorXd, double> query(const Eigen::VectorXd& v) const
            {
                Eigen::MatrixXd mu;
                Eigen::VectorXd s2;
                std::vector<Eigen::VectorXd> one(1, v);
                query_batch(one, mu, s2);
                Eigen::VectorXd m(_dim_out);
                for (int p = 0; p < _dim_out; ++p) m(p) = mu(0, p);
                return std::make_tuple(m, s2(0));
            }
            Eigen::VectorXd mu(const Eigen::VectorXd& v) const { return std::get<0>(query(v)); }
            double sigma(const Eigen::VectorXd& v) const { return std::get<1>(query(v)); }

            // ---- batched extensions (not in the reference) ----
            // mu: M x dim_out (mean function included), sigma2: M
            void query_batch(const std::vector<Eigen::VectorXd>& vs, Eigen::MatrixXd& mu, Eigen::VectorXd& sigma2) const
            {
                const long M = (long)vs.size();
                const int P = _dim_out > 0 ? _dim_out : 1;
                const int D = (int)vs[0].size();
                if (_samples.empty()) _push_prior(D);
                std::vector<double> xq((size_t)M * D), m((size_t)M * P), s((size_t)M);
                for (long i = 0; i < M; ++i)
                    for (int d = 0; d < D; ++d) xq[(size_t)i * D + d] = vs[i](d);
                lb_check(lb_query(_h, M, xq.data(), m.data(), s.data()), "lb_query");
                mu.resize(M, P);
                sigma2.resize(M);
                for (long i = 0; i < M; ++i) {
                    Eigen::VectorXd mv = _mean_function(vs[i], *this); // gp.hpp:615 (host functor)
                    for (int p = 0; p < P; ++p) mu(i, p) = m[(size_t)i * P + p] + mv(p);
                    sigma2(i) = s[(size_t)i];
                }
            }
            // fused UCB / EI + argmax on the device with the FirstElem aggregator (bo_base.hpp:99-105)
            std::pair<double, long> acq_argmax(int acq_id, double p0, double p1, const std::vector<Eigen::VectorXd>& vs) const
            {
                const long M = (long)vs.size();
                const int D = (int)vs[0].size();
                std::vector<double> xq((size_t)M * D), mean0((size_t)M);
                for (long i = 0; i < M; ++i) {
                    for (int d = 0; d < D; ++d) xq[(size_t)i * D + d] = vs[i](d);
                    mean0[(size_t)i] = _mean_function(vs[i], *this)(0);
                }
                double params[2] = {p0, p1}, best = 0;
                int64_t idx = 0;
                lb_check(lb_acq_argmax(_h, acq_id, params, M, xq.data(), mean0.data(), 0.0, nullptr, &best, &idx), "lb_acq_argmax");
                return std::make_pair(best, (long)idx);
            }
            // fused ECI + argmax on the device (experimental/acqui/eci.hpp:76-130, FirstElem aggregator): this GP is the objective,
            // `con` the constraint model, whose first output gives Pf (Pf = 1 while it has no samples).  Both mean functors run on
            // the host.  Without objective samples every value is 0 and the first candidate wins (eci.hpp:86).
            template <typename ConstraintGP>
            std::pair<double, long> eci_argmax(const ConstraintGP& con, double f_max, double jitter, const std::vector<Eigen::VectorXd>& vs) const
            {
                if (_samples.empty()) return std::make_pair(0.0, 0L);
                const long M = (long)vs.size();
                const int D = (int)vs[0].size();
                const bool use_con = !con._samples.empty();
                std::vector<double> xq((size_t)M * D), mean0((size_t)M), cmean0(use_con ? (size_t)M : 0);
                for (long i = 0; i < M; ++i) {
                    for (int d = 0; d < D; ++d) xq[(size_t)i * D + d] = vs[i](d);
                    mean0[(size_t)i] = _mean_function(vs[i], *this)(0);
                    if (use_con) cmean0[(size_t)i] = con._mean_function(vs[i], con)(0);
                }
                double params[2] = {f_max, jitter}, best = 0;
                int64_t idx = 0;
                lb_check(lb_eci_argmax(_h, con._h, params, M, xq.data(), mean0.data(), 0.0, use_con ? cmean0.data() : nullptr, 0.0, nullptr,
                             &best, &idx),
                    "lb_eci_argmax");
                return std::make_pair(best, (long)idx);
            }

            int dim_in() const { assert(_dim_in != -1); return _dim_in; }
            int dim_out() const { assert(_dim_out != -1); return _dim_out; }
            const KernelFunction& kernel_function() const { return _kernel_function; }
            KernelFunction& kernel_function() { return _kernel_function; }
            const MeanFunction& mean_function() const { return _mean_function; }
            MeanFunction& mean_function() { return _mean_function; }

            Eigen::VectorXd max_observation() const // gp.hpp:207-214 (meaningful for dim_out == 1 only)
            {
                if (_observations.cols() > 1) std::cout << "WARNING max_observation with multi dimensional observations doesn't make sense" << std::endl;
                Eigen::VectorXd best(1);
                best(0) = _observations.maxCoeff();
                return best;
            }
            Eigen::VectorXd mean_observation() const // gp.hpp:217-222: zero until there is data
            {
                assert(_dim_out > 0);
                if (_samples.empty()) return Eigen::VectorXd::Zero(_dim_out);
                return _mean_observation;
            }
            const Eigen::MatrixXd& mean_vector() const { return _mean_vector; }
            const Eigen::MatrixXd& obs_mean() const { return _obs_mean; }
            int nb_samples() const { return _samples.size(); }

            void recompute(bool update_obs_mean = true, bool update_full_kernel = true) // gp.hpp:241-252
            {
                assert(!_samples.empty());
                if (update_obs_mean) this->_compute_obs_mean();
                if (update_full_kernel) this->_compute_full_kernel();
                else this->_compute_alpha();
            }

            void compute_inv_kernel() // gp.hpp:254-264
            {
                lb_check(lb_compute_inv_kernel(_h), "lb_compute_inv_kernel");
                _inv_kernel_updated = true;
            }
            double compute_log_lik() // gp.hpp:267-282
            {
                lb_check(lb_log_lik(_h, &_log_lik), "lb_log_lik");
                return _log_lik;
            }
            Eigen::VectorXd compute_kernel_grad_log_lik() // gp.hpp:285-311
            {
                const int nh = (int)_kernel_function.h_params_size();
                std::vector<double> g((size_t)nh);
                lb_check(lb_kernel_grad_log_lik(_h, Params::kernel::optimize_noise() ? 1 : 0, g.data()), "lb_kernel_grad_log_lik");
                _inv_kernel_updated = true;
                Eigen::VectorXd grad(nh);
                for (int i = 0; i < nh; ++i) grad(i) = g[(size_t)i];
                return grad;
            }
            Eigen::VectorXd compute_mean_grad_log_lik() // gp.hpp:313-330; obs_mean^T K^-1 on the device, functor gradient on the host
            {
                const long n = (long)_samples.size();
                std::vector<double> w((size_t)n * _dim_out);
                lb_check(lb_kinv_obs_mean(_h, w.data()), "lb_kinv_obs_mean");
                _inv_kernel_updated = true;
                Eigen::VectorXd grad = Eigen::VectorXd::Zero(_mean_function.h_params_size());
                for (long n_obs = 0; n_obs < n; n_obs++) {
                    Eigen::MatrixXd mg = _mean_function.grad(_samples[n_obs], *this);
                    for (int i_obs = 0; i_obs < _dim_out; ++i_obs)
                        for (long q = 0; q < (long)grad.size(); ++q) grad(q) += w[(size_t)i_obs * n + n_obs] * mg(i_obs, q);
                }
                return grad;
            }
            double get_log_lik() const { return _log_lik; }
            void set_log_lik(double v) { _log_lik = v; }
            double compute_log_loo_cv() // gp.hpp:339-351
            {
                lb_check(lb_log_loo_cv(_h, &_log_loo_cv), "lb_log_loo_cv");
                _inv_kernel_updated = true;
                return _log_loo_cv;
            }
            Eigen::VectorXd compute_kernel_grad_log_loo_cv() // gp.hpp:353-399
            {
                const int nh = (int)_kernel_function.h_params_size();
                std::vector<double> g((size_t)nh);
                lb_check(lb_kernel_grad_log_loo_cv(_h, Params::kernel::optimize_noise() ? 1 : 0, g.data()), "lb_kernel_grad_log_loo_cv");
                _inv_kernel_updated = true;
                Eigen::VectorXd grad(nh);
                for (int i = 0; i < nh; ++i) grad(i) = g[(size_t)i];
                return grad;
            }
            double get_log_loo_cv() const { return _log_loo_cv; }
            void set_log_loo_cv(double v) { _log_loo_cv = v; }

            // host mirrors, refreshed from the device on access (gp.hpp:404-436)
            const Eigen::MatrixXd& matrixL() const { return _fetch(LB_GET_L, _matrixL, (long)_samples.size(), (long)_samples.size()); }
            const Eigen::MatrixXd& alpha() const { return _fetch(LB_GET_ALPHA, _alpha, (long)_samples.size(), _dim_out); }
            const Eigen::MatrixXd& inv_kernel() const
            {
                const Eigen::MatrixXd& r = _fetch(LB_GET_KINV, _inv_kernel, (long)_samples.size(), (long)_samples.size());
                _inv_kernel_updated = true;
                return r;
            }
            const Eigen::MatrixXd& kernel_matrix() const { return _fetch(LB_GET_K, _kernel, (long)_samples.size(), (long)_samples.size()); }
            const std::vector<Eigen::VectorXd>& samples() const { return _samples; }
            std::vector<Eigen::VectorXd> observations() const
            {
                std::vector<Eigen::VectorXd> obs;
                for (int i = 0; i < _observations.rows(); i++) {
                    Eigen::VectorXd o(_dim_out);
                    for (int p = 0; p < _dim_out; ++p) o(p) = _observations(i, p);
                    obs.push_back(o);
                }
                return obs;
            }
            const Eigen::MatrixXd& observations_matrix() const { return _observations; }
            bool inv_kernel_computed() { return _inv_kernel_updated; }
            /// LAPACK-style info of the last factorisation (0 ok, > 0 failing pivot); the reference never checks LLT::info()
            int cholesky_info() const { return _info; }

            // Same six archive objects as the reference (gp.hpp:448-460), so directories written by either side load in the
            // other; matrixL / alpha are fetched from the device when saving.
            template <typename A> void save(const std::string& directory) const { save(A(directory)); }
            template <typename A> void save(const A& archive) const
            {
                const bool has_k = _kernel_function.h_params_size() > 0, has_m = _mean_function.h_params_size() > 0;
                if (has_k) archive.save(_kernel_function.h_params(), "kernel_params");
                if (has_m) archive.save(_mean_function.h_params(), "mean_params");
                archive.save(_samples, "samples");
                archive.save(_observations, "observations");
                archive.save(matrixL(), "matrixL");
                archive.save(alpha(), "alpha");
            }
            template <typename A> void load(const std::string& directory, bool recompute = true) { load(A(directory), recompute); }
            // recompute == false adopts the stored factor (lb_load_factor) instead of refactorising (gp.hpp:505-509)
            template <typename A> void load(const A& archive, bool recompute = true)
            {
                _samples.clear();
                archive.load(_samples, "samples");
                archive.load(_observations, "observations");
                _dim_in = -1;
                _dim_out = -1;
                _adopt_dims(_samples.front().size(), _observations.cols());
                _restore_params(archive, _kernel_function, "kernel_params");
                _restore_params(archive, _mean_function, "mean_params");
                _refresh_means();
                if (recompute) { _compute_full_kernel(); return; }
                Eigen::MatrixXd L, a;
                archive.load(L, "matrixL");
                archive.load(a, "alpha");
                _upload_data();
                _push_kernel();
                lb_check(lb_load_factor(_h, L.data(), a.data()), "lb_load_factor");
                _inv_kernel_updated = false;
            }

            void swap(GP& o)
            {
                using std::swap;
                swap(_h, o._h); swap(_dim_in, o._dim_in); swap(_dim_out, o._dim_out);
                swap(_kernel_function, o._kernel_function); swap(_mean_function, o._mean_function);
                swap(_samples, o._samples); swap(_observations, o._observations); swap(_mean_vector, o._mean_vector);
                swap(_obs_mean, o._obs_mean); swap(_mean_observation, o._mean_observation);
                swap(_log_lik, o._log_lik); swap(_log_loo_cv, o._log_loo_cv); swap(_inv_kernel_updated, o._inv_kernel_updated);
                swap(_info, o._info);
            }

        protected:
            template <typename, typename, typename, typename> friend class GP; // eci_argmax reads the constraint GP's handle and mean
            lb_gp* _h = nullptr;
            int _dim_in;
            int _dim_out;
            KernelFunction _kernel_function;
            MeanFunction _mean_function;
            std::vector<Eigen::VectorXd> _samples;
            Eigen::MatrixXd _observations;
            Eigen::MatrixXd _mean_vector;
            Eigen::MatrixXd _obs_mean;
            Eigen::VectorXd _mean_observation;
            mutable Eigen::MatrixXd _alpha, _kernel, _inv_kernel, _matrixL; // host mirrors
            double _log_lik = 0, _log_loo_cv = 0;
            mutable bool _inv_kernel_updated;
            int _info = 0;
            HyperParamsOptimizer _hp_optimize;

            void _create()
            {
                kernel_traits<KernelFunction>::check();
                lb_check(lb_create(&_h, 0, LB_PREC_FP64), "lb_create");
            }
            const Eigen::MatrixXd& _fetch(int what, Eigen::MatrixXd& dst, long r, long c) const
            {
                dst.resize(r, c);
                lb_check(lb_get(_h, what, dst.data()), "lb_get");
                return dst;
            }
            void _push_kernel() const
            {
                Eigen::VectorXd hp = _kernel_function.h_params(); // log-space, noise last when optimised (kernel.hpp:105-113)
                const int own = (int)hp.size() - (Params::kernel::optimize_noise() ? 1 : 0);
                std::vector<double> p((size_t)own);
                for (int i = 0; i < own; ++i) p[(size_t)i] = hp(i);
                lb_check(lb_set_kernel(_h, kernel_traits<KernelFunction>::id, p.data(), own, _kernel_function.noise()), "lb_set_kernel");
            }
            void _push_prior(int D) const
            {
                lb_check(lb_set_data(_h, 0, D, _dim_out > 0 ? _dim_out : 1, nullptr, nullptr), "lb_set_data");
                _push_kernel();
            }
            // (re)build the policy functors when a dimension changes (what gp.hpp:95-103 / 127-136 do inline)
            void _adopt_dims(long d_in, long d_out)
            {
                if (_dim_in != d_in) { _dim_in = (int)d_in; _kernel_function = KernelFunction(_dim_in); }
                if (_dim_out != d_out) { _dim_out = (int)d_out; _mean_function = MeanFunction(_dim_out); }
            }
            static void _pack_rows(const std::vector<Eigen::VectorXd>& rows, Eigen::MatrixXd& out)
            {
                out.resize(rows.size(), rows.front().size());
                for (size_t i = 0; i < rows.size(); ++i)
                    for (long c = 0; c < (long)rows[i].size(); ++c) out(i, c) = rows[i](c);
            }
            // column means of the observations, then the host mean functor at every sample: obs_mean = Y - M
            void _refresh_means()
            {
                _mean_observation = _observations.colwise().mean();
                _compute_obs_mean();
            }
            void _compute_obs_mean() // gp.hpp:537-548
            {
                const long n = (long)_samples.size();
                assert(n > 0);
                _mean_vector.resize(n, _dim_out);
                for (long i = 0; i < n; ++i) {
                    const Eigen::VectorXd m = _mean_function(_samples[i], *this);
                    for (int p = 0; p < _dim_out; ++p) _mean_vector(i, p) = m(p);
                }
                _obs_mean = _observations - _mean_vector;
            }
            template <typename A, typename Functor>
            static void _restore_params(const A& archive, Functor& fn, const char* name)
            {
                if (fn.h_params_size() == 0) return;
                Eigen::VectorXd hp;
                archive.load(hp, name);
                assert((size_t)hp.size() == (size_t)fn.h_params_size());
                fn.set_h_params(hp);
            }
            void _upload_data()
            {
                const long n = (long)_samples.size();
                std::vector<double> X((size_t)n * _dim_in);
                for (long i = 0; i < n; ++i)
                    for (int d = 0; d < _dim_in; ++d) X[(size_t)i * _dim_in + d] = _samples[i](d);
                lb_check(lb_set_data(_h, n, _dim_in, _dim_out, X.data(), _obs_mean.data()), "lb_set_data");
            }
            void _compute_full_kernel() // gp.hpp:550-571: K -> L -> alpha, all on the device
            {
                _upload_data();
                _push_kernel();
                _info = lb_fit(_h);
                lb_check(_info, "lb_fit");
                _inv_kernel_updated = false;
            }
            void _compute_incremental_kernel() // gp.hpp:573-603
            {
                const long n = (long)_samples.size();
                if (n == 1 || lb_nb_samples(_h) != n - 1) { _compute_full_kernel(); return; }
                _push_kernel();
                std::vector<double> x((size_t)_dim_in);
                for (int d = 0; d < _dim_in; ++d) x[(size_t)d] = _samples.back()(d);
                int rc = lb_append(_h, x.data(), _obs_mean.data());
                if (rc == LB_ERR_STATE) { _compute_full_kernel(); return; }
                lb_check(rc, "lb_append");
                _info = rc;
                _inv_kernel_updated = false;
            }
            void _compute_alpha() // gp.hpp:605-611
            {
                lb_check(lb_refit_alpha(_h, _obs_mean.data()), "lb_refit_alpha");
            }
        };
    } // namespace model
} // namespace limbo_b200

#endif
