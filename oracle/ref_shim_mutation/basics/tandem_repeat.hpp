// TEST INFRASTRUCTURE ONLY — TandemRepeat (basics/tandem_repeat.hpp:15-45): a region and its motif; period() is the motif length.
#ifndef REF_SHIM_MUT_TANDEM_REPEAT_HPP
#define REF_SHIM_MUT_TANDEM_REPEAT_HPP
#include <string>
#include <utility>
#include "basics/genomic_region.hpp"
namespace octopus {
class TandemRepeat
{
public:
    using NucleotideSequence = std::string;
    using SizeType = GenomicRegion::Size;
    template <typename R, typename S>
    TandemRepeat(R&& region, S&& motif) : region_ {std::forward<R>(region)}, motif_ {std::forward<S>(motif)} {}
    SizeType period() const noexcept { return motif_.size(); }
    const NucleotideSequence& motif() const noexcept { return motif_; }
    const GenomicRegion& mapped_region() const noexcept { return region_; }
private:
    GenomicRegion region_;
    NucleotideSequence motif_;
};
} // namespace octopus
#endif
