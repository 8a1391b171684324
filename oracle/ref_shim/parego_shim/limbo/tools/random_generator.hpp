// oracle/ref_shim/parego_shim/limbo/tools/random_generator.hpp — TEST INFRASTRUCTURE ONLY.
//
// The reference's own tools/random_generator.hpp (found next on the include path), with tools::random_vector replaced by a
// replaying one: each call returns the next `size` values of the sequence set by limbo_parego_replay(), so that
// experimental::model::GPParego draws a given weight vector instead of an auto-seeded one.  The reference's function is kept
// under another name; its other users in that header (random_lhs) call the renamed one.
#ifndef LIMBO_B200_PAREGO_REPLAY_RANDOM_HPP
#define LIMBO_B200_PAREGO_REPLAY_RANDOM_HPP

#define random_vector random_vector_unreplayed
#include_next <limbo/tools/random_generator.hpp>
#undef random_vector

#include <cstdlib>
#include <vector>

namespace limbo {
namespace tools {
struct ParegoReplay {
    std::vector<double> values;
    size_t next = 0;
};
inline ParegoReplay& parego_replay()
{
    static thread_local ParegoReplay r;
    return r;
}
inline Eigen::VectorXd random_vector(int size, bool = true)
{
    ParegoReplay& r = parego_replay();
    if (r.next + (size_t)size > r.values.size()) std::abort(); // a draw the caller did not supply
    Eigen::VectorXd v(size);
    for (int i = 0; i < size; ++i) v(i) = r.values[r.next++];
    return v;
}
} // namespace tools
} // namespace limbo

inline void limbo_parego_replay(const double* values, size_t n)
{
    limbo::tools::parego_replay().values.assign(values, values + n);
    limbo::tools::parego_replay().next = 0;
}

#endif
