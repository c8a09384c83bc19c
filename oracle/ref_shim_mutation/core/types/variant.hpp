// TEST INFRASTRUCTURE ONLY — Variant as calculate_approx_log_probability names it (core/types/variant.hpp). The Haplotype stand-in's
// difference() returns no variants, so none of these is ever evaluated.
#ifndef REF_SHIM_MUT_VARIANT_HPP
#define REF_SHIM_MUT_VARIANT_HPP
#include <cstddef>
#include "basics/genomic_region.hpp"
#include "concepts/mappable.hpp"
namespace octopus {
class Variant
{
public:
    const GenomicRegion& mapped_region() const noexcept { return region_; }
private:
    GenomicRegion region_;
};
inline bool is_indel(const Variant&) noexcept { return false; }
inline bool is_simple_indel(const Variant&) noexcept { return false; }
inline std::size_t indel_size(const Variant&) noexcept { return 0; }
inline std::size_t ref_sequence_size(const Variant&) noexcept { return 0; }
inline std::size_t alt_sequence_size(const Variant&) noexcept { return 0; }
} // namespace octopus
#endif
