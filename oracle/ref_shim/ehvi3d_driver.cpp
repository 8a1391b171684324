// oracle/ref_shim/ehvi3d_driver.cpp — TEST INFRASTRUCTURE ONLY.
//
// Runs the REFERENCE'S OWN three-objective EHVI schemes (src/ehvi/ehvi_sliceupdate.cc: ehvi3d_sliceupdate;
// src/ehvi/ehvi_calculations.cc: ehvi3d_5term, ehvi3d_8term) and its 3-D hypervolume (src/ehvi/ehvi_hvol.cc: hvol3d; calculateS
// there is the 2-D one) behind C entries, and ehvi3d_sliceupdate over three of the reference's model::GP with the dense linear
// algebra supplied by the stand-in in ./Eigen.  Used to pin oracle/ehvi3d.py (tests/test_ehvi3d_host.py) and to generate
// tests/golden/ehvi3d/*.npz (tests/golden/make_golden_ehvi3d.py).  No reference source is copied: this file only instantiates
// its templates and calls the functions of the reference's src/ehvi/*.cc, which the Makefile links into libref_ehvi3d.so.
//
// The front is handed over in the order given.  The reference sorts it with std::sort, which is not stable;
// tests/test_ehvi3d_host.py checks that the tested fronts' sums do not depend on their input order.
#include <algorithm>
#include <cmath>
#include <deque>
#include <tuple>
#include <vector>

#include <Eigen/Core>

#include <ehvi/helper.h>
#include <ehvi/ehvi_calculations.h>
#include <ehvi/ehvi_hvol.h>
#include <ehvi/ehvi_sliceupdate.h>

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

struct Front {
    std::vector<individual> store;
    std::deque<individual*> pop;
    Front(long k, const double* f) : store((size_t)k)
    {
        for (long i = 0; i < k; ++i) {
            for (int d = 0; d < 3; ++d) store[(size_t)i].f[d] = f[3 * i + d];
            pop.push_back(&store[(size_t)i]);
        }
    }
};

template <typename Scheme>
int run(Scheme scheme, long k, const double* front, const double* r, long M, const double* mu, const double* s, double* out)
{
    Front F(k, front);
    double rr[3] = {r[0], r[1], r[2]};
    for (long q = 0; q < M; ++q) {
        double m[3] = {mu[3 * q], mu[3 * q + 1], mu[3 * q + 2]}, sd[3] = {s[3 * q], s[3 * q + 1], s[3 * q + 2]};
        out[q] = scheme(F.pop, rr, m, sd);
    }
    return 0;
}

} // namespace

extern "C" {

// ehvi3d_sliceupdate(front, r, mu_q, s_q) for M candidates (front k x 3, mu and s M x 3, all row-major)
int ref_ehvi3d_sliceupdate(long k, const double* front, const double* r, long M, const double* mu, const double* s, double* out)
{
    return run(ehvi3d_sliceupdate, k, front, r, M, mu, s, out);
}
int ref_ehvi3d_5term(long k, const double* front, const double* r, long M, const double* mu, const double* s, double* out)
{
    return run(ehvi3d_5term, k, front, r, M, mu, s, out);
}
int ref_ehvi3d_8term(long k, const double* front, const double* r, long M, const double* mu, const double* s, double* out)
{
    return run(ehvi3d_8term, k, front, r, M, mu, s, out);
}

// hvol3d of the front between r and +inf (the points sorted by f[2] ascending, as hvol3d requires)
int ref_hv3d(long k, const double* front, const double* r, double* out)
{
    Front F(k, front);
    std::stable_sort(F.pop.begin(), F.pop.end(), [](individual* a, individual* b) { return a->f[2] < b->f[2]; });
    double cl[3] = {r[0], r[1], r[2]}, fmax[3] = {INFINITY, INFINITY, INFINITY};
    *out = hvol3d(F.pop, cl, fmax);
    return 0;
}

// One Matern-5/2 / mean::Data GP per objective on (X, Y[:, j]) with default hyper-parameters (N may be 0: prior models), the
// reference's pareto::pareto_set<1> of Y as the front, and ehvi3d_sliceupdate(front, r, (mu_j(v)(0)), (sigma_j(v))) at every
// candidate: sigma() where a deviation is expected, the convention of the two-objective acqui::Ehvi.  Y: N x 3 row-major; mu, s:
// M x 3; front: the Pareto objectives in the reference's order (room for N x 3).
int ref_gp_ehvi3d(long N, int D, const double* X, const double* Y, double noise, const double* r, long M, const double* Xq, double* ehvi,
    double* mu, double* s, double* front, long* n_front)
{
    Params::kernel::set_noise(noise);
    using GP_t = model::GP<Params, kernel::MaternFiveHalves<Params>, mean::Data<Params>>;
    auto vec = [](const double* a, int d) {
        Eigen::VectorXd x((Eigen::Index)d);
        for (int i = 0; i < d; ++i) x(i) = a[i];
        return x;
    };
    std::vector<Eigen::VectorXd> samples;
    std::vector<std::vector<Eigen::VectorXd>> obs(3);
    std::vector<std::tuple<Eigen::VectorXd, Eigen::VectorXd, Eigen::VectorXd>> packed;
    for (long i = 0; i < N; ++i) {
        samples.push_back(vec(X + i * D, D));
        for (int j = 0; j < 3; ++j) obs[(size_t)j].push_back(Eigen::VectorXd::Constant(1, Y[3 * i + j]));
        Eigen::VectorXd id(1);
        id(0) = (double)i;
        packed.push_back(std::make_tuple(id, vec(Y + 3 * i, 3), Eigen::VectorXd::Zero(3)));
    }
    std::vector<GP_t> models(3, GP_t(D, 1));
    if (N > 0)
        for (int j = 0; j < 3; ++j) models[(size_t)j].compute(samples, obs[(size_t)j]);
    auto f = pareto::pareto_set<1>(packed);
    std::vector<individual> store(f.size());
    std::deque<individual*> pop;
    for (size_t i = 0; i < f.size(); ++i) {
        for (int d = 0; d < 3; ++d) store[i].f[d] = front[3 * i + d] = std::get<1>(f[i])(d);
        pop.push_back(&store[i]);
    }
    *n_front = (long)f.size();
    double rr[3] = {r[0], r[1], r[2]};
    for (long q = 0; q < M; ++q) {
        Eigen::VectorXd v = vec(Xq + q * D, D);
        double m[3], sd[3];
        for (int j = 0; j < 3; ++j) {
            m[j] = mu[3 * q + j] = models[(size_t)j].mu(v)(0);
            sd[j] = s[3 * q + j] = models[(size_t)j].sigma(v);
        }
        ehvi[q] = ehvi3d_sliceupdate(pop, rr, m, sd);
    }
    return 0;
}

} // extern "C"
