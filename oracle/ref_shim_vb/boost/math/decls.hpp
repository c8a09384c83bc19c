// TEST INFRASTRUCTURE ONLY — declarations of the Boost.Math names utils/maths.hpp mentions, with no definitions: the variational
// Bayes path never calls them (see ref_shim_vb/README).
#ifndef REF_SHIM_VB_MATH_DECLS_HPP
#define REF_SHIM_VB_MATH_DECLS_HPP
namespace boost { namespace math {
template <typename T> T factorial(unsigned);
template <typename T> T binomial_coefficient(unsigned, unsigned);
template <typename T> int sign(const T&);
template <typename T, typename U> T gamma_p(T, U);
template <typename T, typename U> T gamma_q(T, U);
template <typename T1, typename T2, typename T3> T1 ibeta_inv(T1, T2, T3);
template <typename RealType = double> struct beta_distribution { beta_distribution(RealType, RealType); };
template <typename RealType = double> struct geometric_distribution { geometric_distribution(RealType); };
template <typename RealType = double> struct binomial_distribution { binomial_distribution(RealType, RealType); };
template <typename RealType = double> struct normal_distribution { normal_distribution(RealType, RealType); };
template <typename D> struct complemented { };
template <typename D, typename T> complemented<D> complement(const D&, const T&);
template <typename D, typename T> T pdf(const D&, const T&);
template <typename D, typename T> T cdf(const D&, const T&);
template <typename D> double cdf(const complemented<D>&);
}}
#endif
