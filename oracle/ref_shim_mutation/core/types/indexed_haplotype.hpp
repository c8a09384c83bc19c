// TEST INFRASTRUCTURE ONLY — IndexedHaplotype<> and index(block) as DeNovoModel::prime / evaluate use them
// (core/types/indexed_haplotype.hpp:25-135): a haplotype reference plus its position in the block, compared by position.
#ifndef REF_SHIM_MUT_INDEXED_HAPLOTYPE_HPP
#define REF_SHIM_MUT_INDEXED_HAPLOTYPE_HPP
#include <cstddef>
#include <vector>
#include "core/types/haplotype.hpp"
#include "containers/mappable_block.hpp"
namespace octopus {
template <typename IndexTp = std::size_t>
class IndexedHaplotype
{
public:
    using IndexType = IndexTp;
    IndexedHaplotype(const Haplotype& haplotype, IndexType index) noexcept : haplotype_ {&haplotype}, index_ {index} {}
    const Haplotype& haplotype() const noexcept { return *haplotype_; }
    operator const Haplotype&() const noexcept { return *haplotype_; }
    IndexType index() const noexcept { return index_; }
private:
    const Haplotype* haplotype_;
    IndexType index_;
};
template <typename IndexTp>
IndexTp index_of(const IndexedHaplotype<IndexTp>& haplotype) noexcept { return haplotype.index(); }
template <typename IndexTp>
bool operator==(const IndexedHaplotype<IndexTp>& lhs, const IndexedHaplotype<IndexTp>& rhs) noexcept { return lhs.index() == rhs.index(); }
template <typename IndexTp>
bool operator!=(const IndexedHaplotype<IndexTp>& lhs, const IndexedHaplotype<IndexTp>& rhs) noexcept { return !(lhs == rhs); }
template <typename IndexType = std::size_t>
std::vector<IndexedHaplotype<IndexType>> index(const MappableBlock<Haplotype>& haplotypes)
{
    std::vector<IndexedHaplotype<IndexType>> result {};
    result.reserve(haplotypes.size());
    for (std::size_t i = 0; i < haplotypes.size(); ++i) result.emplace_back(haplotypes[i], static_cast<IndexType>(i));
    return result;
}
} // namespace octopus
#endif
