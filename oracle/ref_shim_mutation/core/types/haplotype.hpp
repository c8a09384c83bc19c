// TEST INFRASTRUCTURE ONLY — Haplotype as the mutation model sees it (core/types/haplotype.hpp): a sequence with a mapped GenomicRegion.
// difference() (the approximate path, calculate_approx_log_probability) reports its (target, given) pair to difference_hook and
// returns no variants: the driver learns exactly which pairs the reference sent to the approximate path.
#ifndef REF_SHIM_MUT_HAPLOTYPE_HPP
#define REF_SHIM_MUT_HAPLOTYPE_HPP
#include <cstddef>
#include <functional>
#include <string>
#include <utility>
#include <vector>
#include "basics/genomic_region.hpp"
#include "core/types/variant.hpp"
namespace octopus {
class Haplotype;
extern void (*difference_hook)(const Haplotype& target, const Haplotype& given);
class Haplotype
{
public:
    using NucleotideSequence = std::string;
    Haplotype(NucleotideSequence sequence, GenomicRegion::Position begin)
    : sequence_ {std::move(sequence)}, region_ {"1", begin, static_cast<GenomicRegion::Position>(begin + sequence_.size())} {}
    const NucleotideSequence& sequence() const noexcept { return sequence_; }
    const GenomicRegion& mapped_region() const noexcept { return region_; }
    std::vector<Variant> difference(const Haplotype& given) const
    {
        if (difference_hook) difference_hook(*this, given);
        return {};
    }
private:
    NucleotideSequence sequence_;
    GenomicRegion region_;
};
inline Haplotype::NucleotideSequence::size_type sequence_size(const Haplotype& haplotype) noexcept { return haplotype.sequence().size(); }
inline bool operator==(const Haplotype& lhs, const Haplotype& rhs) noexcept
{
    return lhs.mapped_region().begin() == rhs.mapped_region().begin() && lhs.sequence() == rhs.sequence();
}
inline bool operator!=(const Haplotype& lhs, const Haplotype& rhs) noexcept { return !(lhs == rhs); }
} // namespace octopus
namespace std {
template <> struct hash<octopus::Haplotype>
{
    size_t operator()(const octopus::Haplotype& haplotype) const noexcept { return hash<string> {}(haplotype.sequence()) ^ haplotype.mapped_region().begin(); }
};
} // namespace std
#endif
