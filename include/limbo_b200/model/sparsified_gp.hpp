// include/limbo_b200/model/sparsified_gp.hpp — header-only drop-in for limbo::model::SparsifiedGP.
//
//   limbo_b200::model::SparsifiedGP<Params, KernelFunction, MeanFunction, HyperParamsOptimizer>
//
// has the reference's template signature and defaults (src/limbo/model/sparsified_gp.hpp:71-72) and its compute / add_sample
// contract: with more than Params::model_sparse_gp::max_points() samples, the densest samples (smallest sum of the distances to
// their D nearest remaining samples) are removed first, and the remaining ones are fitted by limbo_b200::model::GP.  The
// sparsification runs on the device (lb_sparsify); so it can be used in model::MultiGP<Params, limbo_b200::model::SparsifiedGP, ...>.
#ifndef LIMBO_B200_MODEL_SPARSIFIED_GP_HPP
#define LIMBO_B200_MODEL_SPARSIFIED_GP_HPP

#include <cstdint>
#include <vector>

#include "gp.hpp"

namespace limbo {
    namespace mean {
        template <typename Params> struct Data;
    }
    namespace model {
        namespace gp {
            template <typename Params> struct NoLFOpt;
        }
    }
}

namespace limbo_b200 {
    namespace model {

        template <typename Params, typename KernelFunction = limbo::kernel::MaternFiveHalves<Params>,
            typename MeanFunction = limbo::mean::Data<Params>, typename HyperParamsOptimizer = limbo::model::gp::NoLFOpt<Params>>
        class SparsifiedGP : public GP<Params, KernelFunction, MeanFunction, HyperParamsOptimizer> {
        public:
            using base_gp_t = GP<Params, KernelFunction, MeanFunction, HyperParamsOptimizer>;

            SparsifiedGP() : base_gp_t() {}
            SparsifiedGP(int dim_in, int dim_out) : base_gp_t(dim_in, dim_out) {}

            // sparsified_gp.hpp:84-100
            void compute(const std::vector<Eigen::VectorXd>& samples, const std::vector<Eigen::VectorXd>& observations,
                bool compute_kernel = true)
            {
                if (samples.size() <= (size_t)Params::model_sparse_gp::max_points()) {
                    base_gp_t::compute(samples, observations, compute_kernel);
                    return;
                }
                std::vector<Eigen::VectorXd> samp, obs;
                for (int64_t i : sparsify(samples)) {
                    samp.push_back(samples[(size_t)i]);
                    obs.push_back(observations[(size_t)i]);
                }
                base_gp_t::compute(samp, obs, compute_kernel);
            }

            // sparsified_gp.hpp:104-118.  Past max_points the reference appends, then re-sparsifies and refits the whole set; the
            // append is skipped here, with the same result.
            void add_sample(const Eigen::VectorXd& sample, const Eigen::VectorXd& observation)
            {
                if (this->_samples.size() + 1 <= (size_t)Params::model_sparse_gp::max_points()) {
                    base_gp_t::add_sample(sample, observation);
                    return;
                }
                std::vector<Eigen::VectorXd> samples = this->_samples, observations = this->observations();
                samples.push_back(sample);
                observations.push_back(observation);
                compute(samples, observations, true);
            }

            // indices (ascending) of the samples _sparsify keeps (sparsified_gp.hpp:157-183)
            std::vector<int64_t> sparsify(const std::vector<Eigen::VectorXd>& samples) const
            {
                const int64_t N = (int64_t)samples.size();
                const int D = (int)samples[0].size();
                std::vector<double> X((size_t)N * D);
                for (int64_t i = 0; i < N; ++i)
                    for (int d = 0; d < D; ++d) X[(size_t)(i * D + d)] = samples[(size_t)i](d);
                std::vector<int64_t> kept((size_t)N);
                int64_t n_kept = 0;
                lb_check(lb_sparsify(this->_h, N, D, X.data(), Params::model_sparse_gp::max_points(), kept.data(), &n_kept, nullptr, nullptr),
                    "lb_sparsify");
                kept.resize((size_t)n_kept);
                return kept;
            }
        };
    } // namespace model
} // namespace limbo_b200

#endif
