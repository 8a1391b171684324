// tests/cpp/dropin_common.hpp — helpers shared by the compiled drop-in tests (tests/cpp/*dropin_test.cpp).  Include it before
// the reference's headers: some of them name limbo::FirstElem as their default aggregator.
#pragma once
#include <vector>

#include <Eigen/Core>

namespace limbo { // bayes_opt/bo_base.hpp:99-105, which needs Boost.Parameter
    struct FirstElem {
        double operator()(const Eigen::VectorXd& x) const { return x(0); }
    };
} // namespace limbo

static double u01(unsigned long long& s)
{ // splitmix64, as limbo_b200/synth.py
    s += 0x9E3779B97F4A7C15ULL;
    unsigned long long z = s;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    z ^= z >> 31;
    return (double)(z >> 11) * (1.0 / 9007199254740992.0);
}

static long first_max(const std::vector<double>& v)
{
    long i = 0;
    for (long k = 1; k < (long)v.size(); ++k)
        if (v[(size_t)k] > v[(size_t)i]) i = k;
    return i;
}
