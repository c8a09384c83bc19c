// TEST INFRASTRUCTURE ONLY — a minimal octopus::Error family so that the UNMODIFIED reference headers pair_hmm.hpp (HMMOverflow
// derives from ProgramError, :47-65) and simd_pair_hmm_wrapper.hpp (includes user_error.hpp) compile from the reference checkout.
// The real exceptions/*.hpp pull in Octopus's config and Boost. All three classes live here; program_error.hpp and
// user_error.hpp only forward to this file.
#ifndef REF_SHIM_ERROR_HPP
#define REF_SHIM_ERROR_HPP
#include <exception>
#include <string>
namespace octopus {

class Error : public std::exception
{
public:
    virtual ~Error() = default;
    std::string type() const { return do_type(); }
    std::string where() const { return do_where(); }
    std::string why() const { return do_why(); }
    std::string help() const { return do_help(); }
private:
    virtual std::string do_type() const = 0;
    virtual std::string do_where() const = 0;
    virtual std::string do_why() const = 0;
    virtual std::string do_help() const = 0;
};

namespace ref_shim_detail {
enum class Blame { program, user };
template <Blame B>
class BlamedError : public Error
{
    std::string do_type() const override { return B == Blame::program ? "program" : "user"; }
    std::string do_help() const override { return std::string {}; }
};
} // namespace ref_shim_detail

class ProgramError : public ref_shim_detail::BlamedError<ref_shim_detail::Blame::program> { public: virtual ~ProgramError() = default; };
class UserError : public ref_shim_detail::BlamedError<ref_shim_detail::Blame::user> { public: virtual ~UserError() = default; };

} // namespace octopus
#endif
