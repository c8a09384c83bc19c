// TEST INFRASTRUCTURE ONLY — stand-in for Boost.Math's digamma (see ../../../README): evaluated in double, rounded to T.
#ifndef REF_SHIM_VB_DIGAMMA_HPP
#define REF_SHIM_VB_DIGAMMA_HPP
#include <cmath>
namespace boost { namespace math {
namespace shim_detail {
inline double digamma_double(double x)
{
    double r = 0.0;
    if (x != x) return x;
    if (x <= 0.0) {
        if (x == std::floor(x)) return std::nan("");
        const double pi = 3.14159265358979323846;
        r = -pi / std::tan(pi * x);
        x = 1.0 - x;
    }
    while (x < 10.0) { r -= 1.0 / x; x += 1.0; }
    const double f = 1.0 / (x * x);
    const double t = f * (-1.0 / 12 + f * (1.0 / 120 + f * (-1.0 / 252 + f * (1.0 / 240 + f * (-1.0 / 132 + f * (691.0 / 32760 + f * (-1.0 / 12)))))));
    return r + std::log(x) - 0.5 / x + t;
}
}
template <typename T> inline T digamma(T x) { return static_cast<T>(shim_detail::digamma_double(static_cast<double>(x))); }
}}
#endif
