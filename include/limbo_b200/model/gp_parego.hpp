// include/limbo_b200/model/gp_parego.hpp — experimental::model::GPParego over limbo_b200::model::GP, for the UNMODIFIED
// experimental::bayes_opt::Parego:
//
//     using GP_t = limbo_b200::model::GP<Params, kernel::MaternFiveHalves<Params>, mean::Data<Params>, ...>;
//     experimental::bayes_opt::Parego<Params, parego_modelfun<GP_t>, acquiopt<limbo_b200::opt::BatchedRandom<Params>>> opt;
//
// Parego wraps its model in GPParego<Params, model_t> (experimental/bayes_opt/parego.hpp:73-86), so this header provides the
// partial specialisation of limbo::experimental::model::GPParego for limbo_b200::model::GP.  compute() and the scalarisation are
// the primary template's (gp_parego.hpp:83-90, 103-117): a new weight vector per call, divided by its sum, then y = max(lambda f) +
// rho sum(lambda f) with rho = Params::model_gp_parego::rho().  add_sample() differs: the reference refits the whole model
// (gp_parego.hpp:92-98), while the factor depends only on the samples and the kernel, so here every observation is rescalarised
// with the new weights, the factor grows by one row and alpha is re-solved against the rescalarised observations (lb_append, as
// limbo_b200::model::GP::add_sample does).  The weights come from tools::random_vector (the reference's auto-seeded generator) unless
// set_lambda_source() supplies a generator: a callable int K -> Eigen::VectorXd of K raw weights, e.g. a seeded one that can be
// replayed.  DESIGN.md §4.16.
//
// Include order: as for the reference's experimental/model/gp_parego.hpp, which is included here.
#ifndef LIMBO_B200_MODEL_GP_PAREGO_HPP
#define LIMBO_B200_MODEL_GP_PAREGO_HPP

#include <functional>
#include <vector>

#include <Eigen/Core>

#include <limbo/tools/macros.hpp>
#include <limbo/tools/math.hpp>
#include <limbo/tools/random_generator.hpp>
#include <limbo/experimental/model/gp_parego.hpp>

#include "gp.hpp"

namespace limbo {
    namespace experimental {
        namespace model {
            template <typename Params, typename P, typename K, typename Mf, typename H>
            class GPParego<Params, limbo_b200::model::GP<P, K, Mf, H>> : public limbo_b200::model::GP<P, K, Mf, H> {
            public:
                using Model = limbo_b200::model::GP<P, K, Mf, H>;
                using LambdaSource = std::function<Eigen::VectorXd(int)>;

                GPParego() {}
                GPParego(int dim_in, int dim_out) : Model(dim_in, 1), _nb_objs(dim_out) {}

                // the generator of the raw weights (K values in [0, 1) per call); empty: tools::random_vector
                void set_lambda_source(LambdaSource source) { _lambda_source = std::move(source); }

                void compute(const std::vector<Eigen::VectorXd>& samples, const std::vector<Eigen::VectorXd>& observations)
                {
                    _raw_observations = observations;
                    _nb_objs = observations[0].size();
                    Model::compute(samples, _scalarize_obs(observations));
                }

                // incremental: every observation rescalarised with new weights, one factor row appended, alpha re-solved
                void add_sample(const Eigen::VectorXd& sample, const Eigen::VectorXd& observation)
                {
                    if (this->_samples.empty()) {
                        compute(std::vector<Eigen::VectorXd>(1, sample), std::vector<Eigen::VectorXd>(1, observation));
                        return;
                    }
                    _raw_observations.push_back(observation);
                    const std::vector<Eigen::VectorXd> scalarized = _scalarize_obs(_raw_observations);
                    this->_samples.push_back(sample);
                    Model::_pack_rows(scalarized, this->_observations);
                    this->_refresh_means();
                    this->_compute_incremental_kernel();
                }

                const std::vector<Eigen::VectorXd>& raw_observations() const { return _raw_observations; }

            protected:
                size_t _nb_objs = 0;
                std::vector<Eigen::VectorXd> _raw_observations;
                LambdaSource _lambda_source;

                // gp_parego.hpp:103-117, expression for expression
                std::vector<Eigen::VectorXd> _scalarize_obs(const std::vector<Eigen::VectorXd>& observations)
                {
                    Eigen::VectorXd lambda = _lambda_source ? _lambda_source((int)_nb_objs) : tools::random_vector(_nb_objs);
                    double sum = lambda.sum();
                    lambda = lambda / sum;
                    std::vector<Eigen::VectorXd> scalarized;
                    for (auto x : observations) {
                        double y = (lambda.array() * x.array()).maxCoeff();
                        double s = (lambda.array() * x.array()).sum();
                        scalarized.push_back(tools::make_vector(y + Params::model_gp_parego::rho() * s));
                    }
                    return scalarized;
                }
            };
        } // namespace model
    } // namespace experimental
} // namespace limbo

#endif
