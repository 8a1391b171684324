// tests/cpp/eci_dropin_test.cpp — constrained BO's acquisition, compiled: on one fixed candidate set,
//   (1) the reference's experimental::acqui::ECI over a pair of the reference's limbo::model::GP (objective, constraint),
//   (2) the same reference functor over a pair of limbo_b200::model::GP,
//   (3) limbo_b200::acqui::ECI over the limbo_b200 pair, answering a BatchRequest as BatchedRandom issues it (one fused device
//       pass, lb_eci_argmax) and, outside a batch, one point at a time,
// must agree to 1e-10 with the same argmax.  Needs a GPU to run; prints "ECI DROPIN OK".
// (Eigen is the stand-in from oracle/ref_shim so that no Eigen install is needed.)
#include <cstdio>
#include <limbo/acqui/ucb.hpp>
#include <limbo/experimental/acqui/eci.hpp>
#include <limbo/kernel/exp.hpp>
#include <limbo/kernel/squared_exp_ard.hpp>
#include <limbo/mean/constant.hpp>
#include <limbo/mean/data.hpp>
#include <limbo/model/gp.hpp>

#include <limbo_b200/model/gp.hpp>
#include <limbo_b200/opt/batched_random.hpp>

using namespace limbo;

struct Params {
    struct kernel : public defaults::kernel {};
    struct kernel_squared_exp_ard : public defaults::kernel_squared_exp_ard {};
    struct kernel_exp : public defaults::kernel_exp {};
    struct acqui_eci : public defaults::acqui_eci {};
    struct mean_constant {
        BO_PARAM(double, constant, 0.5);
    };
    struct opt_batchedrandom : public limbo_b200::defaults::opt_batchedrandom {};
};

struct FirstElem {
    double operator()(const Eigen::VectorXd& x) const { return x(0); }
};

static double u01(unsigned long long& s)
{ // splitmix64, as limbo_b200/synth.py
    s += 0x9E3779B97F4A7C15ULL;
    unsigned long long z = s;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    z ^= z >> 31;
    return (double)(z >> 11) * (1.0 / 9007199254740992.0);
}

using RefGP = model::GP<Params, kernel::SquaredExpARD<Params>, mean::Data<Params>>;
using RefGPc = model::GP<Params, kernel::Exp<Params>, mean::Constant<Params>>;
using NewGP = limbo_b200::model::GP<Params, kernel::SquaredExpARD<Params>, mean::Data<Params>, model::gp::NoLFOpt<Params>>;
using NewGPc = limbo_b200::model::GP<Params, kernel::Exp<Params>, mean::Constant<Params>, model::gp::NoLFOpt<Params>>;

template <typename Acq>
static std::vector<double> one_by_one(Acq& acq, const std::vector<Eigen::VectorXd>& Q)
{
    FirstElem afun;
    std::vector<double> v;
    for (auto& q : Q) v.push_back(opt::fun(acq(q, afun, false)));
    return v;
}

static long first_max(const std::vector<double>& v)
{
    long i = 0;
    for (long k = 1; k < (long)v.size(); ++k)
        if (v[(size_t)k] > v[(size_t)i]) i = k;
    return i;
}

// nc: constraint samples (0: a constraint model without samples, Pf = 1)
static int run_case(const char* name, int N, int D, int nc)
{
    unsigned long long seed = 7 + N;
    std::vector<Eigen::VectorXd> X, Y, Yc, Q;
    for (int i = 0; i < N; ++i) {
        Eigen::VectorXd x((Eigen::Index)D), y(1), c(2);
        double s = 0;
        for (int d = 0; d < D; ++d) { x(d) = u01(seed); s += std::cos(3.0 * x(d)); }
        y(0) = s;
        c(0) = 0.2 + 1.6 * x(0); // first column around the threshold 1
        c(1) = 2.0 - 1.5 * x(1);
        X.push_back(x);
        Y.push_back(y);
        Yc.push_back(c);
    }
    for (int i = 0; i < 1000; ++i) {
        Eigen::VectorXd q((Eigen::Index)D);
        for (int d = 0; d < D; ++d) q(d) = u01(seed);
        Q.push_back(q);
    }
    RefGP ref(D, 1);
    RefGPc refc(D, 2);
    NewGP gpu(D, 1);
    NewGPc gpuc(D, 2);
    ref.compute(X, Y);
    gpu.compute(X, Y);
    if (nc > 0) {
        std::vector<Eigen::VectorXd> Xc(X.begin(), X.begin() + nc), Ycc(Yc.begin(), Yc.begin() + nc);
        refc.compute(Xc, Ycc);
        gpuc.compute(Xc, Ycc);
    }
    experimental::acqui::ECI<Params, RefGP, RefGPc> eci_ref(ref, refc);
    experimental::acqui::ECI<Params, NewGP, NewGPc> eci_ref_on_b200(gpu, gpuc);
    limbo_b200::acqui::ECI<Params, NewGP, NewGPc> eci_b200(gpu, gpuc);
    const std::vector<double> v1 = one_by_one(eci_ref, Q), v2 = one_by_one(eci_ref_on_b200, Q), v3 = one_by_one(eci_b200, Q);
    const long i1 = first_max(v1);
    limbo_b200::opt::BatchRequest req; // what BatchedRandom announces before calling f
    req.candidates = &Q;
    limbo_b200::opt::current_batch() = &req;
    FirstElem afun;
    const double v0 = opt::fun(eci_b200(Q[0], afun, false));
    limbo_b200::opt::current_batch() = nullptr;
    double d2 = 0, d3 = 0;
    for (size_t k = 0; k < Q.size(); ++k) {
        d2 = std::max(d2, std::fabs(v1[k] - v2[k]));
        d3 = std::max(d3, std::fabs(v1[k] - v3[k]));
    }
    const double dbest = std::fabs(req.best_value - v1[(size_t)i1]);
    std::printf("%s N=%d D=%d nc=%d best=%.6e@%ld |ref-on-b200|=%.3e |b200 one-point|=%.3e batch: answered=%d best=%.6e@%ld |d|=%.3e "
                "|v0|=%.3e\n",
        name, N, D, nc, v1[(size_t)i1], i1, d2, d3, (int)req.answered, req.best_value, req.best_index, dbest, std::fabs(v0 - v1[0]));
    const bool ok = v1[(size_t)i1] > 0 && d2 <= 1e-10 && d3 <= 1e-10 && first_max(v2) == i1 && first_max(v3) == i1 && req.answered
        && req.best_index == i1 && dbest <= 1e-10 && std::fabs(v0 - v1[0]) <= 1e-10;
    return ok ? 0 : 1;
}

int main()
{
    int bad = 0;
    bad += run_case("se_ard+exp", 80, 3, 80);
    bad += run_case("se_ard+exp partial", 150, 4, 90);
    bad += run_case("se_ard, empty constraint", 60, 2, 0);
    if (bad) {
        std::printf("ECI DROPIN FAILED (%d)\n", bad);
        return 1;
    }
    std::printf("ECI DROPIN OK\n");
    return 0;
}
