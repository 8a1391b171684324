// tests/cpp/binding_calls_test.cpp — the batched methods of limbo_b200::model::GP and SPGP against a recording stand-in for the C
// library, without a GPU.  The lb_* entry points the methods reach are defined below: each records its arguments (handles,
// scalars, the contents of its input arrays, which pointers are NULL) and writes pattern(position, j) into its outputs.  For each
// method the test checks the entry point called, every argument, and that the outputs come back in the method's results.  It
// pins the client-side rules of each method: every mean goes as the array of first components, never as the constant; which
// methods push a model's prior; ECI without objective samples calls nothing; SPGP's _check throws on any non-zero code while
// lb_check throws only on negative ones.  Built by oracle/ref_shim/Makefile's binding_calls_test against the reference's headers,
// not linked to liblimbo_b200.so; prints "BINDING CALLS OK".
#include <cstdint>
#include <cstdio>
#include <stdexcept>
#include <string>
#include <vector>

#include <Eigen/Core>
#include "dropin_common.hpp"

namespace nlopt {
enum algorithm { LD_LBFGS = 11 };
}
namespace limbo {
namespace opt {
template <typename Params, nlopt::algorithm Algorithm>
struct NLOptGrad;
}
} // namespace limbo

#include <limbo/kernel/matern_five_halves.hpp>
#include <limbo/kernel/squared_exp_ard.hpp>
#include <limbo/mean/data.hpp>
#include <limbo/mean/function_ard.hpp>

#include <limbo_b200/model/gp.hpp>
#include <limbo_b200/model/spgp.hpp>

// ---- the recording stand-in ----
struct Arg {
    bool null = false, out = false;
    std::vector<double> v;
    bool operator==(const Arg& o) const { return null == o.null && out == o.out && v == o.v; }
};
struct Call {
    std::string fn;
    std::vector<Arg> a;
};
static std::vector<Call> calls;
static int next_rc = 0; // what the next recorded call returns
static uintptr_t next_handle = 0x1000;
static double last_handle = 0;
static const int64_t IDX = 5;
static int D_ = 3, P_ = 1;

static double pattern(int pos, long j) { return 1000.0 * pos + 0.5 + (double)j; }
static Arg NUL()
{
    Arg a;
    a.null = true;
    return a;
}
static Arg OUT()
{
    Arg a;
    a.out = true;
    return a;
}
static Arg S(double x)
{
    Arg a;
    a.v = {x};
    return a;
}
static Arg V(const std::vector<double>& v)
{
    Arg a;
    a.v = v;
    return a;
}
static Arg h(const void* p) { return p ? S((double)(uintptr_t)p) : NUL(); }
static Arg in(const double* p, long n) { return p ? V(std::vector<double>(p, p + n)) : NUL(); }
static Arg out(double* p, long n, int pos)
{
    if (!p) return NUL();
    for (long j = 0; j < n; ++j) p[j] = pattern(pos, j);
    return OUT();
}
static Arg idx(int64_t* p)
{
    *p = IDX;
    return OUT();
}
static int record(const char* fn, std::vector<Arg> a)
{
    calls.push_back({fn, a});
    const int rc = next_rc;
    next_rc = 0;
    return rc;
}
template <typename T> static T* create(const char* fn)
{
    next_handle += 0x10;
    last_handle = (double)next_handle;
    record(fn, {S(last_handle)});
    return (T*)next_handle;
}

extern "C" {
int lb_create(lb_gp** o, int, int) { return *o = create<lb_gp>("lb_create"), 0; }
int lb_destroy(lb_gp* g) { return record("lb_destroy", {h(g)}); }
int lb_set_data(lb_gp* g, int64_t N, int D, int P, const double* X, const double* Y)
{
    return record("lb_set_data", {h(g), S(N), S(D), S(P), in(X, N * D), in(Y, N * P)});
}
int lb_set_kernel(lb_gp* g, int id, const double* p, int n, double noise) { return record("lb_set_kernel", {h(g), S(id), in(p, n), S(noise)}); }
int lb_fit(lb_gp* g) { return record("lb_fit", {h(g)}); }
int lb_query(const lb_gp* g, int64_t M, const double* xq, double* mu, double* s2)
{
    return record("lb_query", {h(g), S(M), in(xq, M * D_), out(mu, M * P_, 3), out(s2, M, 4)});
}
int lb_acq_argmax(const lb_gp* g, int acq, const double* p, int64_t M, const double* xq, const double* m, double mc, double* vals, double* best,
    int64_t* i)
{
    return record("lb_acq_argmax", {h(g), S(acq), in(p, 2), S(M), in(xq, M * D_), in(m, M), S(mc), out(vals, M, 7), out(best, 1, 8), idx(i)});
}
int lb_query_grad(const lb_gp* g, int64_t M, const double* xq, double* mu, double* s2, double* dmu, double* ds2)
{
    return record("lb_query_grad",
        {h(g), S(M), in(xq, M * D_), out(mu, M * P_, 3), out(s2, M, 4), out(dmu, M * D_, 5), out(ds2, M * D_, 6)});
}
int lb_acq_grad(const lb_gp* g, int acq, const double* p, int64_t M, const double* xq, const double* m, double mc, const double* mg,
    double* vals, double* grads)
{
    return record("lb_acq_grad",
        {h(g), S(acq), in(p, 2), S(M), in(xq, M * D_), in(m, M), S(mc), in(mg, M * D_), out(vals, M, 8), out(grads, M * D_, 9)});
}
int lb_eci_argmax(const lb_gp* o, const lb_gp* c, const double* p, int64_t M, const double* xq, const double* m, double mc, const double* cm,
    double cc, double* vals, double* best, int64_t* i)
{
    return record("lb_eci_argmax", {h(o), h(c), in(p, 2), S(M), in(xq, M * D_), in(m, M), S(mc), in(cm, M), S(cc), out(vals, M, 9),
                                       out(best, 1, 10), idx(i)});
}
int lb_eci_grad(const lb_gp* o, const lb_gp* c, const double* p, int64_t M, const double* xq, const double* m, double mc, const double* mg,
    const double* cm, double cc, const double* cg, double* vals, double* grads)
{
    return record("lb_eci_grad", {h(o), h(c), in(p, 2), S(M), in(xq, M * D_), in(m, M), S(mc), in(mg, M * D_), in(cm, M), S(cc),
                                     in(cg, M * D_), out(vals, M, 11), out(grads, M * D_, 12)});
}
int lb_ehvi_argmax(const lb_gp* m0, const lb_gp* m1, const double* r, int64_t k, const double* F, int64_t M, const double* xq,
    const double* a0, double c0, const double* a1, double c1, double* vals, double* best, int64_t* i)
{
    return record("lb_ehvi_argmax", {h(m0), h(m1), in(r, 2), S(k), in(F, k * 2), S(M), in(xq, M * D_), in(a0, M), S(c0), in(a1, M), S(c1),
                                        out(vals, M, 11), out(best, 1, 12), idx(i)});
}
int lb_ehvi_grad(const lb_gp* m0, const lb_gp* m1, const double* r, int64_t k, const double* F, int64_t M, const double* xq,
    const double* a0, double c0, const double* g0, const double* a1, double c1, const double* g1, double* vals, double* grads)
{
    return record("lb_ehvi_grad", {h(m0), h(m1), in(r, 2), S(k), in(F, k * 2), S(M), in(xq, M * D_), in(a0, M), S(c0), in(g0, M * D_),
                                      in(a1, M), S(c1), in(g1, M * D_), out(vals, M, 13), out(grads, M * D_, 14)});
}
int lb_ehvi3d_argmax(const lb_gp* m0, const lb_gp* m1, const lb_gp* m2, const double* r, int64_t k, const double* F, int64_t M,
    const double* xq, const double* a0, double c0, const double* a1, double c1, const double* a2, double c2, double* vals, double* best,
    int64_t* i)
{
    return record("lb_ehvi3d_argmax", {h(m0), h(m1), h(m2), in(r, 3), S(k), in(F, k * 3), S(M), in(xq, M * D_), in(a0, M), S(c0), in(a1, M),
                                          S(c1), in(a2, M), S(c2), out(vals, M, 14), out(best, 1, 15), idx(i)});
}
int lb_spgp_create(lb_spgp** o, int) { return *o = create<lb_spgp>("lb_spgp_create"), 0; }
int lb_spgp_destroy(lb_spgp* s) { return record("lb_spgp_destroy", {h(s)}); }
int lb_spgp_set_data(lb_spgp* s, int64_t N, int D, const double* X, const double* y)
{
    return record("lb_spgp_set_data", {h(s), S(N), S(D), in(X, N * D), in(y, N)});
}
int lb_spgp_lik(lb_spgp* s, int64_t, int64_t, const double*, double, double*, double*) { return record("lb_spgp_lik", {h(s)}); }
int lb_spgp_compute(lb_spgp* s, int64_t m, int64_t nw, const double* w, double jitter)
{
    return record("lb_spgp_compute", {h(s), S(m), S(nw), in(w, nw), S(jitter)});
}
int lb_spgp_query(const lb_spgp* s, int64_t M, const double* xq, int opt, double* mu, double* s2)
{
    return record("lb_spgp_query", {h(s), S(M), in(xq, M * D_), S(opt), out(mu, M, 4), out(s2, M, 5)});
}
int lb_spgp_acq_argmax(const lb_spgp* s, int acq, const double* p, int64_t M, const double* xq, int opt, const double* m, double mc,
    double* vals, double* best, int64_t* i)
{
    return record("lb_spgp_acq_argmax",
        {h(s), S(acq), in(p, 2), S(M), in(xq, M * D_), S(opt), in(m, M), S(mc), out(vals, M, 8), out(best, 1, 9), idx(i)});
}
int lb_spgp_query_grad(const lb_spgp* s, int64_t M, const double* xq, int opt, double* mu, double* s2, double* dmu, double* ds2)
{
    return record("lb_spgp_query_grad",
        {h(s), S(M), in(xq, M * D_), S(opt), out(mu, M, 4), out(s2, M, 5), out(dmu, M * D_, 6), out(ds2, M * D_, 7)});
}
int lb_spgp_acq_grad(const lb_spgp* s, int acq, const double* p, int64_t M, const double* xq, int opt, const double* m, double mc,
    const double* mg, double* vals, double* grads)
{
    return record("lb_spgp_acq_grad", {h(s), S(acq), in(p, 2), S(M), in(xq, M * D_), S(opt), in(m, M), S(mc), in(mg, M * D_),
                                          out(vals, M, 9), out(grads, M * D_, 10)});
}
const char* lb_strerror(int) { return "recorded error"; }
const char* lb_last_cuda_error(void) { return ""; }
}

// ---- the models ----
using namespace limbo;

struct Params {
    struct kernel : public defaults::kernel {};
    struct kernel_maternfivehalves : public defaults::kernel_maternfivehalves {};
    struct kernel_squared_exp_ard : public defaults::kernel_squared_exp_ard {};
    struct model_spgp : public defaults::model_spgp {};
};

// a mean that depends on the input, so each candidate has its own value
struct XSum {
    XSum(size_t dim_out = 1) : _dim_out(dim_out) {}
    template <typename GP> Eigen::VectorXd operator()(const Eigen::VectorXd& x, const GP&) const
    {
        Eigen::VectorXd m((Eigen::Index)_dim_out);
        for (size_t p = 0; p < _dim_out; ++p) {
            m((Eigen::Index)p) = 0.25 * (double)p;
            for (Eigen::Index d = 0; d < x.size(); ++d) m((Eigen::Index)p) += (d + 1) * x(d);
        }
        return m;
    }
    size_t _dim_out;
};
struct NoOpt {
    template <typename G> void operator()(G&) const {}
};
struct KeepW { // SPGP's hyper-parameter optimiser: the starting vector as is
    template <typename F> Eigen::VectorXd operator()(const F&, const Eigen::VectorXd& w, bool) const { return w; }
};

using Matern = kernel::MaternFiveHalves<Params>;
using Ard = mean::FunctionARD<Params, mean::Data<Params>>;
using GPData = limbo_b200::model::GP<Params, Matern, mean::Data<Params>, NoOpt>;
using GPArd = limbo_b200::model::GP<Params, Matern, Ard, NoOpt>;
using GPX = limbo_b200::model::GP<Params, Matern, XSum, NoOpt>;
using SE = kernel::SquaredExpARD<Params>;
using SPGPData = limbo_b200::model::SPGP<Params, SE, mean::Data<Params>, KeepW>;
using SPGPArd = limbo_b200::model::SPGP<Params, SE, Ard, KeepW>;
using SPGPX = limbo_b200::model::SPGP<Params, SE, XSum, KeepW>;

// ---- the cases ----
static int fails = 0;
#define CHECK(c)                                                                  \
    do {                                                                          \
        if (!(c)) {                                                               \
            std::printf("FAILED %s:%d (%s): %s\n", __FILE__, __LINE__, ctx, #c); \
            ++fails;                                                              \
        }                                                                         \
    } while (0)
static const char* ctx = "";

static std::vector<Eigen::VectorXd> vecs(const std::vector<std::vector<double>>& rows)
{
    std::vector<Eigen::VectorXd> r;
    for (const auto& row : rows) {
        Eigen::VectorXd v((Eigen::Index)row.size());
        for (size_t d = 0; d < row.size(); ++d) v((Eigen::Index)d) = row[d];
        r.push_back(v);
    }
    return r;
}
static const std::vector<Eigen::VectorXd> VS = vecs({{0.1, 0.2, 0.3}, {0.4, 0.5, 0.6}, {0.7, 0.8, 0.9}, {0.15, 0.25, 0.35}});
static const long M = 4;
static const std::vector<double> XQ = {0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9, 0.15, 0.25, 0.35};
static const std::vector<Eigen::VectorXd> X = vecs({{0.0, 0.5, 1.0}, {1.0, 0.25, 0.0}, {0.5, 0.75, 0.5}});
static const std::vector<Eigen::VectorXd> Y = vecs({{1.0}, {2.0}, {4.5}});
static const std::vector<Eigen::VectorXd> YC = vecs({{-1.0}, {-2.0}, {-4.5}});
static const std::vector<double> FRONT2 = {1.0, 2.0, 2.0, 1.0, 1.5, 1.5}, FRONT3 = {1.0, 2.0, 3.0, 3.0, 2.0, 1.0};
static const double REF[4] = {3.0, 4.0, 5.0, 6.0};

static std::vector<double> pat(int pos, long n)
{
    std::vector<double> v((size_t)n);
    for (long j = 0; j < n; ++j) v[(size_t)j] = pattern(pos, j);
    return v;
}
static std::vector<double> vals_of(const Eigen::VectorXd& v) { return std::vector<double>(v.data(), v.data() + v.size()); }
static std::vector<double> rows_of(const Eigen::MatrixXd& m)
{
    std::vector<double> r;
    for (Eigen::Index i = 0; i < m.rows(); ++i)
        for (Eigen::Index j = 0; j < m.cols(); ++j) r.push_back(m(i, j));
    return r;
}
template <typename G> static std::vector<double> first_means(const G& g)
{
    std::vector<double> r;
    for (const auto& v : VS) r.push_back(g.mean_function()(v, g)(0));
    return r;
}
template <typename G> static std::vector<double> mean_rows(const G& g)
{
    std::vector<double> r;
    for (const auto& v : VS) {
        Eigen::VectorXd m = g.mean_function()(v, g);
        for (Eigen::Index p = 0; p < m.size(); ++p) r.push_back(m(p));
    }
    return r;
}
static std::vector<double> plus(std::vector<double> a, const std::vector<double>& b)
{
    for (size_t i = 0; i < a.size(); ++i) a[i] += b[i];
    return a;
}
static std::vector<std::string> names()
{
    std::vector<std::string> r;
    for (const auto& c : calls) r.push_back(c.fn);
    return r;
}
static const Call& only(const char* fn)
{
    static Call none;
    const Call* found = nullptr;
    int n = 0;
    for (const auto& c : calls)
        if (c.fn == fn) { found = &c; ++n; }
    CHECK(n == 1);
    return n == 1 ? *found : none;
}
// index of the lb_set_data(h, 0, D, 1, NULL, NULL) + lb_set_kernel(h, ...) pair that pushes a model's prior, or -1
static long prior_push(double handle)
{
    for (size_t i = 0; i + 1 < calls.size(); ++i)
        if (calls[i].fn == "lb_set_data" && calls[i].a[0] == S(handle)) {
            CHECK((calls[i].a == std::vector<Arg>{S(handle), S(0), S(D_), S(1), NUL(), NUL()}));
            CHECK(calls[i + 1].fn == "lb_set_kernel" && calls[i + 1].a[0] == S(handle));
            return (long)i;
        }
    return -1;
}
static long index_of(const char* fn)
{
    for (size_t i = 0; i < calls.size(); ++i)
        if (calls[i].fn == fn) return (long)i;
    return -1;
}
template <typename G> static double made(G& g, bool samples, const std::vector<Eigen::VectorXd>& y = Y)
{
    const double handle = last_handle;
    if (samples) g.compute(X, y);
    calls.clear();
    return handle;
}
static void check_argmax(const std::pair<double, long>& r, const std::vector<double>* vals, int vals_pos)
{
    CHECK(r.first == pattern(vals_pos + 1, 0) && r.second == IDX);
    if (vals) CHECK(*vals == pat(vals_pos, M));
}

template <typename G> static void gp_query_batch(bool samples)
{
    G g(D_, 1);
    const double hg = made(g, samples);
    Eigen::MatrixXd mu;
    Eigen::VectorXd s2;
    g.query_batch(VS, mu, s2);
    CHECK((only("lb_query").a == std::vector<Arg>{S(hg), S(M), V(XQ), OUT(), OUT()}));
    CHECK(rows_of(mu) == plus(pat(3, M), mean_rows(g)) && vals_of(s2) == pat(4, M));
    CHECK(samples ? index_of("lb_set_data") == -1 : prior_push(hg) == 0);
}

template <typename G> static void gp_acq_argmax(bool samples, bool with_values)
{
    G g(D_, 1);
    const double hg = made(g, samples);
    std::vector<double> vals;
    auto r = g.acq_argmax(1, 0.25, 3.0, VS, with_values ? &vals : nullptr);
    CHECK(names() == std::vector<std::string>{"lb_acq_argmax"});
    CHECK((only("lb_acq_argmax").a == std::vector<Arg>{S(hg), S(1), V({0.25, 3.0}), S(M), V(XQ), V(first_means(g)), S(0.0),
                                          with_values ? OUT() : NUL(), OUT(), OUT()}));
    check_argmax(r, with_values ? &vals : nullptr, 7);
}

template <typename G> static void gp_acq_grad(bool samples)
{
    G g(D_, 1);
    const double hg = made(g, samples);
    Eigen::VectorXd vals;
    Eigen::MatrixXd grads;
    g.acq_grad(0, 0.5, 0.0, VS, vals, grads);
    CHECK(names() == std::vector<std::string>{"lb_acq_grad"});
    CHECK((only("lb_acq_grad").a
           == std::vector<Arg>{S(hg), S(0), V({0.5, 0.0}), S(M), V(XQ), V(first_means(g)), S(0.0), NUL(), OUT(), OUT()}));
    CHECK(vals_of(vals) == pat(8, M) && rows_of(grads) == pat(9, M * D_) && grads.rows() == M && grads.cols() == D_);
}

template <typename G> static void gp_query_grad(bool samples)
{
    G g(D_, 1);
    const double hg = made(g, samples);
    Eigen::MatrixXd mu, dmu, ds2;
    Eigen::VectorXd s2;
    g.query_grad(VS, mu, s2, dmu, ds2);
    CHECK(names() == std::vector<std::string>{"lb_query_grad"});
    CHECK((only("lb_query_grad").a == std::vector<Arg>{S(hg), S(M), V(XQ), OUT(), OUT(), OUT(), OUT()}));
    CHECK(rows_of(mu) == plus(pat(3, M), mean_rows(g)) && vals_of(s2) == pat(4, M));
    CHECK(rows_of(dmu) == pat(5, M * D_) && rows_of(ds2) == pat(6, M * D_) && dmu.cols() == D_ && ds2.cols() == D_);
}

static void gp_eci_argmax(bool obj_samples, bool con_samples, bool with_values)
{
    GPArd g(D_, 1);
    const double hg = made(g, obj_samples);
    GPX c(D_, 1);
    const double hc = made(c, con_samples, YC);
    std::vector<double> vals(2, 7.0);
    auto r = g.eci_argmax(c, 1.5, 0.01, VS, with_values ? &vals : nullptr);
    if (!obj_samples) {
        CHECK(calls.empty() && r.first == 0.0 && r.second == 0);
        if (with_values) CHECK(vals == std::vector<double>((size_t)M, 0.0));
        return;
    }
    CHECK(names() == std::vector<std::string>{"lb_eci_argmax"});
    CHECK((only("lb_eci_argmax").a == std::vector<Arg>{S(hg), S(hc), V({1.5, 0.01}), S(M), V(XQ), V(first_means(g)), S(0.0),
                                          con_samples ? V(first_means(c)) : NUL(), S(0.0), with_values ? OUT() : NUL(), OUT(), OUT()}));
    check_argmax(r, with_values ? &vals : nullptr, 9);
}

static void gp_eci_grad(bool obj_samples, bool con_samples)
{
    GPArd g(D_, 1);
    const double hg = made(g, obj_samples);
    GPData c(D_, 1);
    const double hc = made(c, con_samples, YC);
    Eigen::VectorXd vals;
    Eigen::MatrixXd grads;
    g.eci_grad(c, 1.5, 0.01, VS, vals, grads);
    if (!obj_samples) {
        CHECK(calls.empty() && vals_of(vals) == std::vector<double>((size_t)M, 0.0));
        CHECK(rows_of(grads) == std::vector<double>((size_t)(M * D_), 0.0) && grads.rows() == M && grads.cols() == D_);
        return;
    }
    CHECK(names() == std::vector<std::string>{"lb_eci_grad"});
    CHECK((only("lb_eci_grad").a == std::vector<Arg>{S(hg), S(hc), V({1.5, 0.01}), S(M), V(XQ), V(first_means(g)), S(0.0), NUL(),
                                        con_samples ? V(first_means(c)) : NUL(), S(0.0), NUL(), OUT(), OUT()}));
    CHECK(vals_of(vals) == pat(11, M) && rows_of(grads) == pat(12, M * D_));
}

static void gp_ehvi_argmax(bool full_front, bool samples, bool with_values)
{
    GPData g(D_, 1);
    const double hg = made(g, samples);
    GPX o(D_, 1);
    const double ho = made(o, samples, YC);
    const std::vector<double> front = full_front ? FRONT2 : std::vector<double>();
    std::vector<double> vals;
    auto r = g.ehvi_argmax(o, REF, front, VS, with_values ? &vals : nullptr);
    CHECK((only("lb_ehvi_argmax").a == std::vector<Arg>{S(hg), S(ho), V({3.0, 4.0}), S(full_front ? 3 : 0), full_front ? V(FRONT2) : NUL(),
                                           S(M), V(XQ), V(first_means(g)), S(0.0), V(first_means(o)), S(0.0), with_values ? OUT() : NUL(),
                                           OUT(), OUT()}));
    check_argmax(r, with_values ? &vals : nullptr, 11);
    if (samples)
        CHECK(names() == std::vector<std::string>{"lb_ehvi_argmax"});
    else
        CHECK(prior_push(hg) == 0 && prior_push(ho) == 2 && calls.size() == 5);
}

static void gp_ehvi3d_argmax(bool full_front, bool samples, bool with_values)
{
    GPArd g(D_, 1);
    const double hg = made(g, samples);
    GPX m1(D_, 1);
    const double h1 = made(m1, samples, YC);
    GPData m2(D_, 1);
    const double h2 = made(m2, samples);
    const std::vector<double> front = full_front ? FRONT3 : std::vector<double>();
    std::vector<double> vals;
    auto r = g.ehvi3d_argmax(m1, m2, REF, front, VS, with_values ? &vals : nullptr);
    CHECK((only("lb_ehvi3d_argmax").a
           == std::vector<Arg>{S(hg), S(h1), S(h2), V({3.0, 4.0, 5.0}), S(full_front ? 2 : 0), full_front ? V(FRONT3) : NUL(), S(M), V(XQ),
               V(first_means(g)), S(0.0), V(first_means(m1)), S(0.0), V(first_means(m2)), S(0.0), with_values ? OUT() : NUL(), OUT(), OUT()}));
    check_argmax(r, with_values ? &vals : nullptr, 14);
    if (samples)
        CHECK(names() == std::vector<std::string>{"lb_ehvi3d_argmax"});
    else
        CHECK(prior_push(hg) == 0 && prior_push(h1) == 2 && prior_push(h2) == 4 && calls.size() == 7);
}

static void gp_ehvi_grad(bool full_front, bool samples)
{
    GPArd g(D_, 1);
    const double hg = made(g, samples);
    GPData o(D_, 1);
    const double ho = made(o, samples, YC);
    const std::vector<double> front = full_front ? FRONT2 : std::vector<double>();
    Eigen::VectorXd vals;
    Eigen::MatrixXd grads;
    g.ehvi_grad(o, REF, front, VS, vals, grads);
    CHECK((only("lb_ehvi_grad").a == std::vector<Arg>{S(hg), S(ho), V({3.0, 4.0}), S(full_front ? 3 : 0), full_front ? V(FRONT2) : NUL(), S(M),
                                         V(XQ), V(first_means(g)), S(0.0), NUL(), V(first_means(o)), S(0.0), NUL(), OUT(), OUT()}));
    CHECK(vals_of(vals) == pat(13, M) && rows_of(grads) == pat(14, M * D_) && grads.cols() == D_);
    if (samples)
        CHECK(names() == std::vector<std::string>{"lb_ehvi_grad"});
    else
        CHECK(prior_push(hg) == 0 && prior_push(ho) == 2 && calls.size() == 5);
}

template <typename G> static void spgp_query_batch(bool samples)
{
    G s(D_, 1);
    const double hs = made(s, samples);
    Eigen::MatrixXd mu, xt((Eigen::Index)M, (Eigen::Index)D_);
    Eigen::VectorXd s2;
    s.query_batch(VS, mu, s2);
    for (long i = 0; i < M; ++i)
        for (int d = 0; d < D_; ++d) xt(i, d) = VS[(size_t)i](d);
    auto p = s.predict(xt);
    if (!samples) {
        SE k(D_);
        std::vector<double> prior;
        for (const auto& v : VS) prior.push_back(k(v, v));
        CHECK(calls.empty() && rows_of(mu) == mean_rows(s) && vals_of(s2) == prior);
        CHECK(rows_of(p.first) == mean_rows(s) && rows_of(p.second) == prior);
        return;
    }
    CHECK((names() == std::vector<std::string>{"lb_spgp_query", "lb_spgp_query"}));
    CHECK((calls[0].a == std::vector<Arg>{S(hs), S(M), V(XQ), S(1), OUT(), OUT()}) && calls[1].a == calls[0].a);
    CHECK(rows_of(mu) == plus(pat(4, M), mean_rows(s)) && vals_of(s2) == pat(5, M));
    CHECK(rows_of(p.first) == rows_of(mu) && rows_of(p.second) == pat(5, M));
}

template <typename G> static void spgp_acq_argmax(bool with_values)
{
    G s(D_, 1);
    const double hs = made(s, true);
    std::vector<double> vals;
    auto r = s.acq_argmax(1, 0.25, 3.0, VS, with_values ? &vals : nullptr);
    CHECK(names() == std::vector<std::string>{"lb_spgp_acq_argmax"});
    CHECK((only("lb_spgp_acq_argmax").a == std::vector<Arg>{S(hs), S(1), V({0.25, 3.0}), S(M), V(XQ), S(1), V(first_means(s)), S(0.0),
                                               with_values ? OUT() : NUL(), OUT(), OUT()}));
    check_argmax(r, with_values ? &vals : nullptr, 8);
}

template <typename G> static void spgp_acq_grad()
{
    G s(D_, 1);
    const double hs = made(s, true);
    Eigen::VectorXd vals;
    Eigen::MatrixXd grads;
    s.acq_grad(0, 0.5, 0.0, VS, vals, grads);
    CHECK(names() == std::vector<std::string>{"lb_spgp_acq_grad"});
    CHECK((only("lb_spgp_acq_grad").a
           == std::vector<Arg>{S(hs), S(0), V({0.5, 0.0}), S(M), V(XQ), S(1), V(first_means(s)), S(0.0), NUL(), OUT(), OUT()}));
    CHECK(vals_of(vals) == pat(9, M) && rows_of(grads) == pat(10, M * D_) && grads.cols() == D_);
}

template <typename G> static void spgp_query_grad()
{
    G s(D_, 1);
    const double hs = made(s, true);
    Eigen::MatrixXd mu, dmu, ds2;
    Eigen::VectorXd s2;
    s.query_grad(VS, mu, s2, dmu, ds2);
    CHECK(names() == std::vector<std::string>{"lb_spgp_query_grad"});
    CHECK((only("lb_spgp_query_grad").a == std::vector<Arg>{S(hs), S(M), V(XQ), S(1), OUT(), OUT(), OUT(), OUT()}));
    CHECK(rows_of(mu) == plus(pat(4, M), mean_rows(s)) && vals_of(s2) == pat(5, M));
    CHECK(rows_of(dmu) == pat(6, M * D_) && rows_of(ds2) == pat(7, M * D_) && dmu.cols() == D_);
}

// lb_check throws on negative codes only (a positive one is a pivot the caller may read); SPGP's _check on any non-zero code
static void error_codes()
{
    GPData g(D_, 1);
    made(g, true);
    SPGPData s(D_, 1);
    made(s, true);
    bool threw = false;
    next_rc = 2;
    g.acq_argmax(0, 0.5, 0.0, VS);
    next_rc = -1;
    try { g.acq_argmax(0, 0.5, 0.0, VS); } catch (const std::runtime_error&) { threw = true; }
    CHECK(threw);
    threw = false;
    next_rc = 2;
    try { s.acq_argmax(0, 0.5, 0.0, VS); } catch (const std::runtime_error&) { threw = true; }
    CHECK(threw);
    next_rc = 0;
}

int main()
{
    for (bool samples : {true, false}) {
        ctx = samples ? "with samples" : "without samples";
        gp_query_batch<GPData>(samples);
        gp_query_batch<GPX>(samples);
        for (bool with_values : {true, false}) {
            gp_acq_argmax<GPData>(samples, with_values);
            gp_acq_argmax<GPArd>(samples, with_values);
            gp_acq_argmax<GPX>(samples, with_values);
            for (bool con_samples : {true, false}) gp_eci_argmax(samples, con_samples, with_values);
            for (bool full_front : {true, false}) {
                gp_ehvi_argmax(full_front, samples, with_values);
                gp_ehvi3d_argmax(full_front, samples, with_values);
            }
        }
        gp_acq_grad<GPData>(samples);
        gp_acq_grad<GPArd>(samples);
        gp_query_grad<GPData>(samples);
        gp_query_grad<GPArd>(samples);
        for (bool con_samples : {true, false}) gp_eci_grad(samples, con_samples);
        for (bool full_front : {true, false}) gp_ehvi_grad(full_front, samples);
        spgp_query_batch<SPGPData>(samples);
        spgp_query_batch<SPGPX>(samples);
    }
    ctx = "SPGP";
    for (bool with_values : {true, false}) {
        spgp_acq_argmax<SPGPData>(with_values);
        spgp_acq_argmax<SPGPArd>(with_values);
        spgp_acq_argmax<SPGPX>(with_values);
    }
    spgp_acq_grad<SPGPData>();
    spgp_acq_grad<SPGPArd>();
    spgp_query_grad<SPGPData>();
    spgp_query_grad<SPGPArd>();
    ctx = "error codes";
    error_codes();
    if (fails == 0) std::printf("BINDING CALLS OK\n");
    return fails ? 1 : 0;
}
