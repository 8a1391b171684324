// include/limbo_b200/acqui/ehvi.hpp — experimental::acqui::Ehvi on the device, for the UNMODIFIED
// experimental::bayes_opt::Ehvi:
//
//     using GP_t = limbo_b200::model::GP<Params, kernel::MaternFiveHalves<Params>, mean::Data<Params>, ...>;
//     experimental::bayes_opt::Ehvi<Params, modelfun<GP_t>, acquiopt<limbo_b200::opt::BatchedRandom<Params>>> opt;
//
// The reference's optimiser hard-codes acqui::Ehvi<Params, model_t> (experimental/bayes_opt/ehvi.hpp:123), so a new
// acquisition class cannot be injected; this header provides the partial specialisation of limbo::acqui::Ehvi for
// limbo_b200::model::GP instead.  It keeps the reference's constructor and call.  Inside BatchedRandom's call of the
// acquisition it answers the announced BatchRequest with one lb_ehvi_argmax over the whole candidate set; outside a batch it
// scores the one point as a batch of one.  Inside limbo_b200::opt::BatchedGradient's call it also files every candidate's value
// and answers the GradRequest of the start points with one lb_ehvi_grad (means that do not depend on the input), so the unmodified
// loop, which only ever calls opt::no_grad(acqui(x)), climbs the acquisition.  Aggregators that do not act like FirstElem take the
// reference's host path.
// The reference's tools::par::max may call it from several threads at once: lb_ehvi_argmax locks both handles.
//
// Three models (three objectives; the reference has no three-objective functor, so this path is for callers who build the
// functor themselves: the reference's experimental::bayes_opt::Ehvi writes f[2] = 0 and z_ref = 0 and stays two-objective).  The
// value is ehvi3d_sliceupdate (src/ehvi/ehvi_sliceupdate.cc) at (mu_i(v)[0]) and (sigma_i(v)), read from pop's f[0..2] and
// ref_point(0..2).  A BatchRequest is answered with one lb_ehvi3d_argmax, and a point outside a batch is a batch of one.  The
// GradRequest is left unanswered (there is no three-objective gradient on the device), so limbo_b200::opt::BatchedGradient stops
// after scoring its start points (batched_gradient.hpp:103); limbo_b200::opt::BatchedCmaes climbs it instead: with two or three
// models and input-free means, its CmaesRequest is answered by one lb_ehvi_cmaes.  Aggregators that do not act like FirstElem run the reference's
// ehvi3d_sliceupdate on the host, one point at a time: an aggregator type other than limbo::FirstElem instantiates that path, and
// then src/ehvi/ehvi_sliceupdate.cc must be linked too (with FirstElem it is never referenced).
//
// Include order: limbo::FirstElem (bayes_opt/bo_base.hpp) must be visible first, as for the reference's own
// experimental/acqui/ehvi.hpp, which is included here; link the reference's src/ehvi/*.cc as for the reference.
#ifndef LIMBO_B200_ACQUI_EHVI_HPP
#define LIMBO_B200_ACQUI_EHVI_HPP

#include <cassert>
#include <deque>
#include <type_traits>
#include <vector>

#include <Eigen/Core>

#include <limbo/experimental/acqui/ehvi.hpp>
#include <ehvi/ehvi_sliceupdate.h>

#include "../model/gp.hpp"
#include "../opt/batched_random.hpp"

namespace limbo {
    namespace acqui {
        template <typename Params, typename P, typename K, typename Mf, typename H>
        class Ehvi<Params, limbo_b200::model::GP<P, K, Mf, H>> {
        public:
            using Model = limbo_b200::model::GP<P, K, Mf, H>;

            Ehvi(const std::vector<Model>& models, const std::deque<individual*>& pop, const Eigen::VectorXd& ref_point)
                : _models(models), _pop(pop), _ref_point(ref_point)
            {
                assert(_models.size() == 2 || _models.size() == 3);
            }

            size_t dim() const { return _models[0].dim_in(); }

            template <typename AggregatorFunction = FirstElem>
            double operator()(const Eigen::VectorXd& v, const AggregatorFunction& afun = AggregatorFunction()) const
            {
                if (_models.size() == 3) return _ehvi3d(v, afun);
                assert(_models.size() == 2);
                const double r[2] = {_ref_point(0), _ref_point(1)};
                if (limbo_b200::acqui::detail::acts_like_first_elem(afun, _models[0].dim_out())) {
                    const std::vector<double> front = _front();
                    if constexpr (has_grad) { // BatchedGradient's start points: values and gradients in one lb_ehvi_grad
                        limbo_b200::opt::GradRequest* greq = limbo_b200::opt::current_grad_batch();
                        if (greq && !greq->answered && greq->points && !greq->points->empty()) {
                            _models[0].ehvi_grad(_models[1], r, front, *greq->points, greq->values, greq->grads);
                            greq->answered = true;
                        }
                    }
                    _answer_cmaes(r, front, nullptr);
                    limbo_b200::opt::BatchRequest* req = limbo_b200::opt::current_batch();
                    limbo_b200::acqui::detail::answer_batch([&](const std::vector<Eigen::VectorXd>& c) {
                        return _models[0].ehvi_argmax(_models[1], r, front, c, req ? req->values : nullptr);
                    });
                    if (req && req->answered) req->gradients = has_grad;
                    return _models[0].ehvi_argmax(_models[1], r, front, std::vector<Eigen::VectorXd>{v}).first;
                }
                // experimental/acqui/ehvi.hpp:73-78
                double rr[3] = {r[0], r[1], 0};
                double mu[3] = {afun(_models[0].mu(v)), afun(_models[1].mu(v)), 0};
                double s[3] = {_models[0].sigma(v), _models[1].sigma(v), 0};
                return ehvi2d(_pop, rr, mu, s);
            }

        protected:
            // three models: one lb_ehvi3d_argmax per BatchRequest (or per point), the GradRequest left unanswered; other aggregators
            // take ehvi3d_sliceupdate on the host
            template <typename AggregatorFunction>
            double _ehvi3d(const Eigen::VectorXd& v, const AggregatorFunction& afun) const
            {
                double r[3] = {_ref_point(0), _ref_point(1), _ref_point(2)};
                if constexpr (!std::is_same<AggregatorFunction, FirstElem>::value) { // FirstElem never instantiates the host path
                    if (!limbo_b200::acqui::detail::acts_like_first_elem(afun, _models[0].dim_out())) {
                        double mu[3], s[3];
                        for (int i = 0; i < 3; ++i) {
                            mu[i] = afun(_models[(size_t)i].mu(v));
                            s[i] = _models[(size_t)i].sigma(v);
                        }
                        return ehvi3d_sliceupdate(_pop, r, mu, s);
                    }
                }
                const std::vector<double> front = _front(3);
                _answer_cmaes(r, front, &_models[2]);
                limbo_b200::opt::BatchRequest* req = limbo_b200::opt::current_batch();
                limbo_b200::acqui::detail::answer_batch([&](const std::vector<Eigen::VectorXd>& c) {
                    return _models[0].ehvi3d_argmax(_models[1], _models[2], r, front, c, req ? req->values : nullptr);
                });
                return _models[0].ehvi3d_argmax(_models[1], _models[2], r, front, std::vector<Eigen::VectorXd>{v}).first;
            }

            // means that do not depend on the input: gradients from lb_ehvi_grad
            static constexpr bool has_grad = limbo_b200::acqui::detail::has_candidate_grad<Model>::value;

            // BatchedCmaes's start points: one lb_ehvi_cmaes over two (m2 NULL) or three models (means that do not depend on the input)
            void _answer_cmaes(const double* r, const std::vector<double>& front, const Model* m2) const
            {
                if constexpr (limbo_b200::acqui::detail::has_device_cmaes<Model>::value)
                    limbo_b200::acqui::detail::answer_cmaes(
                        [&](const std::vector<Eigen::VectorXd>& st, const lb_cmaes_opts& o, Eigen::VectorXd& x, int64_t& n) {
                            return _models[0].ehvi_cmaes(_models[1], m2, r, front, st, o, x, n);
                        });
            }

            const std::vector<Model>& _models;
            const std::deque<individual*>& _pop;
            Eigen::VectorXd _ref_point;

            // pop's first n_obj objectives, row-major
            std::vector<double> _front(int n_obj = 2) const
            {
                std::vector<double> f;
                f.reserve((size_t)n_obj * _pop.size());
                for (const individual* p : _pop)
                    for (int d = 0; d < n_obj; ++d) f.push_back(p->f[d]);
                return f;
            }
        };
    } // namespace acqui
} // namespace limbo

#endif
