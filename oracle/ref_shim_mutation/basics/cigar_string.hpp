// TEST INFRASTRUCTURE ONLY — ../ref_shim's CIGAR stand-in plus the predicates recalculate_log_probability uses
// (basics/cigar_string.hpp: is_indel, is_deletion; reference_size appears in an assert only).
#ifndef REF_SHIM_MUT_CIGAR_STRING_HPP
#define REF_SHIM_MUT_CIGAR_STRING_HPP
#include "../../ref_shim/basics/cigar_string.hpp"
namespace octopus {
inline bool is_insertion(const CigarOperation& op) noexcept { return op.flag() == CigarOperation::Flag::insertion; }
inline bool is_deletion(const CigarOperation& op) noexcept { return op.flag() == CigarOperation::Flag::deletion; }
inline bool is_indel(const CigarOperation& op) noexcept { return is_insertion(op) || is_deletion(op); }
inline CigarOperation::Size reference_size(const CigarString& cigar) noexcept
{
    CigarOperation::Size result {0};
    for (const auto& op : cigar) if (op.flag() != CigarOperation::Flag::insertion) result += op.size();
    return result;
}
} // namespace octopus
#endif
