// tests/cpp/sparsified_dropin_test.cpp — the sparsified model, compiled: on the setups of the reference's test_gp.cpp:760-880
// (M = 100 one-dimensional samples, max_points M / 3 and M / 2) and on a 3-D set,
//   (1) the reference's limbo::model::SparsifiedGP and (2) limbo_b200::model::SparsifiedGP
// must keep the same samples and predict within 1e-10; so must add_sample past max_points, and
// model::MultiGP<Params, ..SparsifiedGP..> over both.  Needs a GPU to run; prints "SPARSE DROPIN OK".
// (Eigen is the stand-in from oracle/ref_shim so that no Eigen install is needed.)
#include <Eigen/Core> // first: the stand-in with the writable VectorXd::Map (sparse_eigen/Eigen/Core)
#include <cmath>
#include <cstdio>
#include <limbo/kernel/matern_five_halves.hpp>
#include <limbo/kernel/squared_exp_ard.hpp>
#include <limbo/mean/constant.hpp>
#include <limbo/mean/data.hpp>
#include <limbo/model/gp.hpp>
#include <limbo/model/multi_gp.hpp>
#include <limbo/model/sparsified_gp.hpp>

#include <limbo_b200/model/sparsified_gp.hpp>

using namespace limbo;

struct Params {
    struct kernel : public defaults::kernel {};
    struct kernel_squared_exp_ard : public defaults::kernel_squared_exp_ard {};
    struct kernel_maternfivehalves : public defaults::kernel_maternfivehalves {};
    struct mean_constant : public defaults::mean_constant {};
    struct model_sparse_gp {
        BO_DYN_PARAM(int, max_points);
    };
};
BO_DECLARE_DYN_PARAM(int, Params::model_sparse_gp, max_points);

static double u01(unsigned long long& s)
{ // splitmix64, as limbo_b200/synth.py
    s += 0x9E3779B97F4A7C15ULL;
    unsigned long long z = s;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    z ^= z >> 31;
    return (double)(z >> 11) * (1.0 / 9007199254740992.0);
}

static int failures = 0;
static void check(bool ok, const char* what)
{
    if (!ok) {
        std::printf("FAIL %s\n", what);
        ++failures;
    }
}

static bool same_samples(const std::vector<Eigen::VectorXd>& a, const std::vector<Eigen::VectorXd>& b)
{
    if (a.size() != b.size()) return false;
    for (size_t i = 0; i < a.size(); ++i)
        for (long d = 0; d < a[i].size(); ++d)
            if (a[i](d) != b[i](d)) return false;
    return true;
}

template <typename RefM, typename NewM>
static double max_pred_diff(RefM& r, NewM& n, const std::vector<Eigen::VectorXd>& Q)
{
    double e = 0;
    for (auto& q : Q) {
        auto a = r.query(q);
        auto b = n.query(q);
        e = std::max(e, std::abs(std::get<0>(a)(0) - std::get<0>(b)(0)));
        e = std::max(e, std::abs(std::get<1>(a) - std::get<1>(b)));
    }
    return e;
}

int main()
{
    using Ref = model::SparsifiedGP<Params>;
    using New = limbo_b200::model::SparsifiedGP<Params>;
    using RefSE = model::SparsifiedGP<Params, kernel::SquaredExpARD<Params>, mean::Constant<Params>>;
    using NewSE = limbo_b200::model::SparsifiedGP<Params, kernel::SquaredExpARD<Params>, mean::Constant<Params>>;
    unsigned long long seed = 7;
    struct Setup { int D; int M; int max_points; double lo, hi; };
    for (Setup su : {Setup{1, 100, 33, 0.0, 10.0}, Setup{1, 100, 50, -2.0, 2.0}, Setup{3, 300, 120, -1.0, 1.0}}) {
        Params::model_sparse_gp::set_max_points(su.max_points);
        std::vector<Eigen::VectorXd> samples, obs, Q;
        for (int i = 0; i < su.M; ++i) {
            Eigen::VectorXd x(su.D), y(1);
            for (int d = 0; d < su.D; ++d) x(d) = su.lo + (su.hi - su.lo) * u01(seed);
            y(0) = std::cos(x(0)) + (su.D > 1 ? x(1) * x(1) : 0.0);
            samples.push_back(x);
            obs.push_back(y);
            Eigen::VectorXd q(su.D);
            for (int d = 0; d < su.D; ++d) q(d) = su.lo + (su.hi - su.lo) * u01(seed);
            Q.push_back(q);
        }
        Ref r;
        New n;
        r.compute(samples, obs);
        n.compute(samples, obs);
        check(same_samples(r.samples(), n.samples()), "compute: kept samples");
        check(max_pred_diff(r, n, Q) < 1e-10, "compute: predictions");
        RefSE rs;
        NewSE ns;
        rs.compute(samples, obs);
        ns.compute(samples, obs);
        check(same_samples(rs.samples(), ns.samples()), "SE-ARD / mean::Constant: kept samples");
        check(max_pred_diff(rs, ns, Q) < 1e-10, "SE-ARD / mean::Constant: predictions");
        // add_sample past max_points: the reference re-sparsifies max_points + 1 samples
        for (int i = 0; i < 3; ++i) {
            r.add_sample(Q[i], obs[i]);
            n.add_sample(Q[i], obs[i]);
        }
        check((int)n.nb_samples() == su.max_points && same_samples(r.samples(), n.samples()), "add_sample: kept samples");
        check(max_pred_diff(r, n, Q) < 1e-10, "add_sample: predictions");
        // model::MultiGP over both sparsified models (test_gp.cpp:1015)
        using RefMulti = model::MultiGP<Params, model::SparsifiedGP, kernel::SquaredExpARD<Params>, mean::Constant<Params>>;
        using NewMulti = model::MultiGP<Params, limbo_b200::model::SparsifiedGP, kernel::SquaredExpARD<Params>, mean::Constant<Params>>;
        RefMulti rm;
        NewMulti nm;
        rm.compute(samples, obs);
        nm.compute(samples, obs);
        double e = 0;
        for (auto& q : Q) {
            auto a = rm.query(q);
            auto b = nm.query(q);
            e = std::max(e, std::abs(std::get<0>(a)(0) - std::get<0>(b)(0)));
            e = std::max(e, std::abs(std::get<1>(a)(0) - std::get<1>(b)(0)));
        }
        check(same_samples(rm.gp_models()[0].samples(), nm.gp_models()[0].samples()), "MultiGP: kept samples");
        check(e < 1e-10, "MultiGP: predictions");
    }
    if (failures) return 1;
    std::printf("SPARSE DROPIN OK\n");
    return 0;
}
