// TEST INFRASTRUCTURE ONLY — the slice of the reference's basics/cigar_string.hpp that pair_hmm.hpp touches
// (make_cigar, pair_hmm.hpp:152-188, 335): an operation is (length, SAM flag), a CIGAR is a vector of them.
// The real header needs Boost; this one exists so that pair_hmm.hpp itself compiles unmodified from the reference checkout.
#ifndef REF_SHIM_CIGAR_STRING_HPP
#define REF_SHIM_CIGAR_STRING_HPP
#include <cstdint>
#include <vector>
namespace octopus {
class CigarOperation
{
public:
    using Size = std::uint_fast32_t;
    enum class Flag : char { alignmentMatch = 'M', sequenceMatch = '=', substitution = 'X', insertion = 'I', deletion = 'D',
                             softClipped = 'S', hardClipped = 'H', padding = 'P', skipped = 'N' };
    CigarOperation() = default;
    CigarOperation(Size size, Flag flag) noexcept : size_ {size}, flag_ {flag} {}
    Size size() const noexcept { return size_; }
    Flag flag() const noexcept { return flag_; }
private:
    Size size_ = 0;
    Flag flag_ = Flag::alignmentMatch;
};
using CigarString = std::vector<CigarOperation>;
// basics/cigar_string.hpp: operations that consume read / haplotype sequence (used by the SNV error model's substitution mask)
inline bool advances_sequence(const CigarOperation& op) noexcept
{
    using Flag = CigarOperation::Flag;
    return !(op.flag() == Flag::deletion || op.flag() == Flag::hardClipped);   // basics/cigar_string.cpp:89-98
}
} // namespace octopus
#endif
