// TEST INFRASTRUCTURE ONLY — the MemoryFootprint constructor variational_bayes_mixture_model.hpp uses (see ../README).
#ifndef REF_SHIM_VB_MEMORY_FOOTPRINT_HPP
#define REF_SHIM_VB_MEMORY_FOOTPRINT_HPP
#include <cstddef>
namespace octopus {
class MemoryFootprint
{
public:
    MemoryFootprint(std::size_t bytes) : bytes_ {bytes} {}
    std::size_t bytes() const noexcept { return bytes_; }
private:
    std::size_t bytes_;
};
}
#endif
