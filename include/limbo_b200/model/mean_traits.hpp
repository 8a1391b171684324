// include/limbo_b200/model/mean_traits.hpp — which of the reference's mean functors do not depend on the input, shared by the
// device models (gp.hpp, spgp.hpp) and the batch-aware acquisitions (opt/batched_random.hpp).
#ifndef LIMBO_B200_MODEL_MEAN_TRAITS_HPP
#define LIMBO_B200_MODEL_MEAN_TRAITS_HPP

#include <type_traits>

namespace limbo {
    namespace mean {
        template <typename Params> struct NullFunction;
        template <typename Params> struct Constant;
        template <typename Params> struct Data;
        template <typename Params, typename MeanFunction> struct FunctionARD;
    }
}

namespace limbo_b200 {
    namespace model {
        // Means whose value does not depend on the input: the candidate gradients (acq_grad, query_grad) add no mean term for them.
        // FunctionARD is an affine map of its inner mean's value (mean/function_ard.hpp:88-92).  Other means have no input
        // gradient here, and requesting one does not compile.
        template <typename M> struct mean_is_input_free : std::false_type {};
        template <typename P> struct mean_is_input_free<limbo::mean::NullFunction<P>> : std::true_type {};
        template <typename P> struct mean_is_input_free<limbo::mean::Constant<P>> : std::true_type {};
        template <typename P> struct mean_is_input_free<limbo::mean::Data<P>> : std::true_type {};
        template <typename P, typename M> struct mean_is_input_free<limbo::mean::FunctionARD<P, M>> : mean_is_input_free<M> {};
    }
}

#endif
