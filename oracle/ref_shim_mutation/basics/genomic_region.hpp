// TEST INFRASTRUCTURE ONLY — GenomicRegion as repeat_finder.hpp and IndelMutationModel use it (basics/genomic_region.hpp): a contig
// name and a half-open [begin, end).
#ifndef REF_SHIM_MUT_GENOMIC_REGION_HPP
#define REF_SHIM_MUT_GENOMIC_REGION_HPP
#include <string>
#include <utility>
#include "basics/contig_region.hpp"
namespace octopus {
class GenomicRegion
{
public:
    using ContigName = std::string;
    using Position   = ContigRegion::Position;
    using Size       = ContigRegion::Size;
    using Distance   = ContigRegion::Distance;
    GenomicRegion() = default;
    GenomicRegion(ContigName contig, Position begin, Position end) : contig_ {std::move(contig)}, region_ {begin, end} {}
    const ContigName& contig_name() const noexcept { return contig_; }
    Position begin() const noexcept { return region_.begin(); }
    Position end() const noexcept { return region_.end(); }
private:
    ContigName contig_;
    ContigRegion region_;
};
inline GenomicRegion::Distance begin_distance(const GenomicRegion& first, const GenomicRegion& second) noexcept
{
    return static_cast<GenomicRegion::Distance>(second.begin()) - first.begin();
}
// concepts/mappable.hpp: region_size of anything mappable
template <typename T>
auto region_size(const T& mappable) noexcept { return mappable.mapped_region().end() - mappable.mapped_region().begin(); }
} // namespace octopus
#endif
