// include/limbo_b200/model/batch_args.hpp — host-side arguments and results of the device models' batched calls into the C ABI
// (gp.hpp, spgp.hpp): candidates packed row-major, the first mean of a model at each candidate, row-major results into Eigen.
#ifndef LIMBO_B200_MODEL_BATCH_ARGS_HPP
#define LIMBO_B200_MODEL_BATCH_ARGS_HPP

#include <vector>

#include <Eigen/Core>

namespace limbo_b200 {
    namespace model {
        namespace detail {
            // the candidates as a row-major M x D array
            inline std::vector<double> pack_rows(const std::vector<Eigen::VectorXd>& vs)
            {
                const size_t D = vs.empty() ? 0 : (size_t)vs[0].size();
                std::vector<double> xq(vs.size() * D);
                for (size_t i = 0; i < vs.size(); ++i)
                    for (size_t d = 0; d < D; ++d) xq[i * D + d] = vs[i]((Eigen::Index)d);
                return xq;
            }
            // the first component of the model's mean functor at every candidate (a host functor, as in the reference)
            template <typename Model>
            std::vector<double> first_means(const Model& model, const std::vector<Eigen::VectorXd>& vs)
            {
                std::vector<double> m(vs.size());
                for (size_t i = 0; i < vs.size(); ++i) m[i] = model.mean_function()(vs[i], model)(0);
                return m;
            }
            // M values, and a row-major M x C array, from the device into Eigen
            inline void unpack(const std::vector<double>& a, Eigen::VectorXd& out)
            {
                out = Eigen::VectorXd((Eigen::Index)a.size());
                for (size_t i = 0; i < a.size(); ++i) out((Eigen::Index)i) = a[i];
            }
            inline void unpack(const std::vector<double>& a, long M, long C, Eigen::MatrixXd& out)
            {
                out = Eigen::MatrixXd((Eigen::Index)M, (Eigen::Index)C);
                for (long i = 0; i < M; ++i)
                    for (long c = 0; c < C; ++c) out(i, c) = a[(size_t)(i * C + c)];
            }
        } // namespace detail
    } // namespace model
} // namespace limbo_b200

#endif
