// TEST INFRASTRUCTURE ONLY — stand-in for <boost/functional/hash.hpp> as DeNovoModel's address-cache hash uses it (hash_value on
// pointers, hash_combine). Any well-defined hash will do (the cache is only looked up).
#ifndef REF_SHIM_MUT_BOOST_FUNCTIONAL_HASH_HPP
#define REF_SHIM_MUT_BOOST_FUNCTIONAL_HASH_HPP
#include <cstddef>
#include <functional>
namespace boost {
template <typename T>
inline std::size_t hash_value(const T& value) noexcept { return std::hash<T> {}(value); }
template <typename T>
inline void hash_combine(std::size_t& seed, const T& value) noexcept
{
    seed ^= hash_value(value) + 0x9e3779b97f4a7c15ull + (seed << 6) + (seed >> 2);
}
} // namespace boost
#endif
