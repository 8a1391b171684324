// oracle/ref_shim/ehvi_driver.cpp — TEST INFRASTRUCTURE ONLY.
//
// Runs the REFERENCE'S OWN two-objective EHVI (src/ehvi/ehvi_calculations.cc: ehvi2d, through experimental/acqui/ehvi.hpp over
// two of the reference's model::GP) and its Pareto filter (experimental/tools/pareto.hpp), with the dense linear algebra supplied
// by the stand-in in ./Eigen.  Used to pin oracle/ehvi.py (tests/test_ehvi_host.py) and to generate tests/golden/ehvi/*.npz
// (tests/golden/make_golden_ehvi.py).  No reference source is copied: this file only instantiates its templates and links the
// reference's src/ehvi/*.cc (Makefile: libref_ehvi.so).
#include <deque>
#include <tuple>
#include <vector>
#include <Eigen/Core>

// experimental/acqui/ehvi.hpp names limbo::FirstElem (bayes_opt/bo_base.hpp:99-105, which needs Boost.Parameter) as its
// default aggregator: restated here, before the include
namespace limbo {
    struct FirstElem {
        double operator()(const Eigen::VectorXd& x) const { return x(0); }
    };
} // namespace limbo

#include <limbo/experimental/acqui/ehvi.hpp>
#include <limbo/experimental/tools/pareto.hpp>
#include <limbo/kernel/matern_five_halves.hpp>
#include <limbo/mean/data.hpp>
#include <limbo/model/gp.hpp>

using namespace limbo;

struct Params {
    struct kernel {
        BO_DYN_PARAM(double, noise);
        BO_PARAM(bool, optimize_noise, false);
    };
    struct kernel_maternfivehalves : public defaults::kernel_maternfivehalves {};
};
BO_DECLARE_DYN_PARAM(double, Params::kernel, noise);

namespace {

Eigen::VectorXd vec(const double* a, int d)
{
    Eigen::VectorXd x((Eigen::Index)d);
    for (int i = 0; i < d; ++i) x(i) = a[i];
    return x;
}

using pareto_point_t = std::tuple<Eigen::VectorXd, Eigen::VectorXd, Eigen::VectorXd>;

// pareto::pareto_set<1> over n points of K objectives; the point slot carries the input index
std::vector<pareto_point_t> ref_front(long n, int K, const double* objs)
{
    std::vector<pareto_point_t> v;
    for (long i = 0; i < n; ++i) {
        Eigen::VectorXd id(1);
        id(0) = (double)i;
        v.push_back(std::make_tuple(id, vec(objs + i * K, K), Eigen::VectorXd::Zero(K)));
    }
    return pareto::pareto_set<1>(v);
}

} // namespace

extern "C" {

// ehvi2d(front, r, mu_q, s_q) for M candidates (mu, s: M x 2 row-major)
int ref_ehvi2d(long k, const double* front, const double* r, long M, const double* mu, const double* s, double* out)
{
    std::deque<individual*> pop;
    std::vector<individual> store((size_t)k);
    for (long i = 0; i < k; ++i) {
        store[(size_t)i].f[0] = front[2 * i];
        store[(size_t)i].f[1] = front[2 * i + 1];
        store[(size_t)i].f[2] = 0;
        pop.push_back(&store[(size_t)i]);
    }
    double rr[3] = {r[0], r[1], 0};
    for (long q = 0; q < M; ++q) {
        double m[3] = {mu[2 * q], mu[2 * q + 1], 0}, sd[3] = {s[2 * q], s[2 * q + 1], 0};
        out[q] = ehvi2d(pop, rr, m, sd);
    }
    return 0;
}

// pareto::pareto_set<1>: the kept input indices in the reference's order
int ref_pareto_set(long n, int K, const double* objs, long* idx, long* n_front)
{
    auto f = ref_front(n, K, objs);
    for (size_t i = 0; i < f.size(); ++i) idx[i] = (long)std::get<0>(f[i])(0);
    *n_front = (long)f.size();
    return 0;
}

// experimental::bayes_opt::Ehvi's acquisition step (ehvi.hpp:110-125, bo_multi.hpp:173-180, 233-245): one Matern-5/2 / mean::Data
// GP per objective on (X, Y[:, i]) with default hyper-parameters, the Pareto set of the observations, and acqui::Ehvi at each
// candidate.  Y: N x 2 row-major; mu, s: M x 2 (each model's mu(v)(0) and sigma(v)); front: the Pareto objectives (room for N x 2).
int ref_gp_ehvi(long N, int D, const double* X, const double* Y, double noise, const double* r, long M, const double* Xq, double* ehvi,
    double* mu, double* s, double* front, long* n_front)
{
    Params::kernel::set_noise(noise);
    using GP_t = model::GP<Params, kernel::MaternFiveHalves<Params>, mean::Data<Params>>;
    std::vector<Eigen::VectorXd> samples;
    std::vector<std::vector<Eigen::VectorXd>> obs(2);
    for (long i = 0; i < N; ++i) {
        samples.push_back(vec(X + i * D, D));
        for (int j = 0; j < 2; ++j) obs[(size_t)j].push_back(Eigen::VectorXd::Constant(1, Y[2 * i + j]));
    }
    std::vector<GP_t> models(2, GP_t(D, 1));
    for (int j = 0; j < 2; ++j) models[(size_t)j].compute(samples, obs[(size_t)j]);
    auto f = ref_front(N, 2, Y);
    std::deque<individual*> pop;
    std::vector<individual> store(f.size());
    for (size_t i = 0; i < f.size(); ++i) {
        store[i].f[0] = front[2 * i] = std::get<1>(f[i])(0);
        store[i].f[1] = front[2 * i + 1] = std::get<1>(f[i])(1);
        store[i].f[2] = 0;
        pop.push_back(&store[i]);
    }
    *n_front = (long)f.size();
    Eigen::VectorXd ref(3);
    ref(0) = r[0];
    ref(1) = r[1];
    ref(2) = 0;
    acqui::Ehvi<Params, GP_t> acq(models, pop, ref);
    for (long q = 0; q < M; ++q) {
        Eigen::VectorXd v = vec(Xq + q * D, D);
        for (int j = 0; j < 2; ++j) {
            mu[2 * q + j] = models[(size_t)j].mu(v)(0);
            s[2 * q + j] = models[(size_t)j].sigma(v);
        }
        ehvi[q] = acq(v, FirstElem());
    }
    return 0;
}
}
