// dispatch.h -- run-time configuration to template arguments, host only.  Each visitor calls f with a std::integral_constant
// (usable as a template argument) for the value it is given, or returns otherwise() for a value outside its set.  A visitor
// instantiates f for every value of its set, so the range of each call is the set of kernels that exists: widen it only
// with a kernel that should be built.
#pragma once
#include <type_traits>

namespace lb {

// f(SF) for sf in LO..HI
template <int LO, int HI, class Otherwise, class F>
auto with_sf(int sf, Otherwise otherwise, F f) {
    if constexpr (LO > HI) return otherwise();
    else return sf == LO ? f(std::integral_constant<int, LO>{}) : with_sf<LO + 1, HI>(sf, otherwise, f);
}

// f(D) for the K1 oversampling osr = sps / N: 8, 2, 16 or 32 (fs/bw = 4 has no kernels)
template <class Otherwise, class F>
auto with_osr(int osr, Otherwise otherwise, F f) {
    return osr == 8    ? f(std::integral_constant<int, 8>{})
           : osr == 2  ? f(std::integral_constant<int, 2>{})
           : osr == 16 ? f(std::integral_constant<int, 16>{})
           : osr == 32 ? f(std::integral_constant<int, 32>{})
                       : otherwise();
}

// f(B) for a bool
template <class F>
auto with_bool(bool b, F f) {
    return b ? f(std::true_type{}) : f(std::false_type{});
}

// f(SF, D) over the K1 configurations: sf in 7..12 and osr 8, 2, 16 or 32
template <class Otherwise, class F>
auto with_sf_osr(int sf, int osr, Otherwise otherwise, F f) {
    return with_osr(osr, otherwise, [&](auto D) { return with_sf<7, 12>(sf, otherwise, [&](auto SF) { return f(SF, D); }); });
}

}  // namespace lb
