// oracle/ref_shim/sparse_driver.cpp — TEST INFRASTRUCTURE ONLY.
//
// Runs the REFERENCE'S OWN model::SparsifiedGP::_sparsify (model/sparsified_gp.hpp:157-183) with the dense linear algebra
// supplied by the stand-in in ./Eigen (sequential tools::par::loop: no USE_TBB).  Used to pin the restatement
// (oracle/sparsify.py, tests/test_sparsify_host.py) and to generate tests/golden/sparsify/*.npz
// (tests/golden/make_golden_sparsify.py).  No reference source is copied: this file only instantiates its templates.
#include <Eigen/Core> // first: the stand-in with the writable VectorXd::Map (sparse_eigen/Eigen/Core)
#include <algorithm>
#include <numeric>
#include <limbo/kernel/matern_five_halves.hpp>
#include <limbo/mean/data.hpp>
#include <limbo/model/sparsified_gp.hpp>

using namespace limbo;

struct Params {
    struct kernel : public defaults::kernel {};
    struct kernel_maternfivehalves : public defaults::kernel_maternfivehalves {};
    struct model_sparse_gp {
        BO_DYN_PARAM(int, max_points);
    };
};
BO_DECLARE_DYN_PARAM(int, Params::model_sparse_gp, max_points);

namespace {

// exposes the protected members of the reference's SparsifiedGP (default policies: MaternFiveHalves, mean::Data, NoLFOpt)
struct Exposed : public model::SparsifiedGP<Params> {
    std::pair<std::vector<Eigen::VectorXd>, std::vector<Eigen::VectorXd>> sparsify(const std::vector<Eigen::VectorXd>& s,
        const std::vector<Eigen::VectorXd>& o) const
    {
        return this->_sparsify(s, o);
    }

    // _sparsify's loop (sparsified_gp.hpp:160-180) with its own _get_most_dense_point / _remove_row / _remove_column, recording
    // the original index of every removed point and its density, i.e. min_dist of _get_most_dense_point (:129-151)
    void traced(const std::vector<Eigen::VectorXd>& samples, std::vector<long>& order, std::vector<double>& scores,
        std::vector<long>& kept) const
    {
        const size_t N = samples.size();
        const int D = (int)samples[0].size();
        Eigen::MatrixXd distances(N, N);
        for (size_t i = 0; i < N; ++i)
            for (size_t j = 0; j < N; ++j)
                if (i != j) distances(i, j) = (samples[i] - samples[j]).norm();
        kept.resize(N);
        std::iota(kept.begin(), kept.end(), 0L);
        while (kept.size() > (size_t)Params::model_sparse_gp::max_points()) {
            const int n = (int)kept.size();
            const int k = this->_get_most_dense_point(D, n, distances);
            if (k < 0) break;
            std::vector<double> nb(n);
            for (int j = 0; j < n; ++j) nb[j] = distances(k, j);
            nb.erase(nb.begin() + k);
            std::partial_sort(nb.begin(), nb.begin() + D, nb.end());
            double dist = 0.;
            for (int j = 0; j < D; ++j) dist += nb[j];
            scores.push_back(dist);
            order.push_back(kept[k]);
            kept.erase(kept.begin() + k);
            this->_remove_column(distances, k);
            this->_remove_row(distances, k);
        }
    }
};

} // namespace

extern "C" {

// X: row-major N x D.  kept: room for N; removed / removed_score: room for N.  Returns 0, or 2 when the traced loop and
// _sparsify disagree on the kept set.
int ref_sparsify(long N, int D, const double* X, long max_points, long* kept, long* n_kept, long* removed, double* removed_score,
    long* n_removed)
{
    Params::model_sparse_gp::set_max_points((int)max_points);
    std::vector<Eigen::VectorXd> samples, obs;
    for (long i = 0; i < N; ++i) {
        Eigen::VectorXd x((Eigen::Index)D);
        for (int d = 0; d < D; ++d) x(d) = X[i * D + d];
        samples.push_back(x);
        Eigen::VectorXd o(1);
        o(0) = (double)i; // the observation carries the original index through _sparsify
        obs.push_back(o);
    }
    Exposed gp;
    std::vector<long> order, k;
    std::vector<double> sc;
    gp.traced(samples, order, sc, k);
    if (N > max_points) {
        auto res = gp.sparsify(samples, obs);
        if (res.second.size() != k.size()) return 2;
        for (size_t i = 0; i < k.size(); ++i)
            if ((long)res.second[i](0) != k[i]) return 2;
    }
    for (size_t i = 0; i < k.size(); ++i) kept[i] = k[i];
    for (size_t i = 0; i < order.size(); ++i) {
        removed[i] = order[i];
        removed_score[i] = sc[i];
    }
    *n_kept = (long)k.size();
    *n_removed = (long)order.size();
    return 0;
}

// the reference's _sparsify alone (for timing); returns the number of kept points
long ref_sparsify_only(long N, int D, const double* X, long max_points)
{
    Params::model_sparse_gp::set_max_points((int)max_points);
    std::vector<Eigen::VectorXd> samples, obs;
    for (long i = 0; i < N; ++i) {
        Eigen::VectorXd x((Eigen::Index)D);
        for (int d = 0; d < D; ++d) x(d) = X[i * D + d];
        samples.push_back(x);
        obs.push_back(Eigen::VectorXd::Zero(1));
    }
    Exposed gp;
    return (long)gp.sparsify(samples, obs).first.size();
}
}
