// TEST INFRASTRUCTURE ONLY — the names of HaplotypeLikelihoodArray that variational_bayes_mixture_model.hpp uses (see ../../README).
#ifndef REF_SHIM_VB_HAPLOTYPE_LIKELIHOOD_ARRAY_HPP
#define REF_SHIM_VB_HAPLOTYPE_LIKELIHOOD_ARRAY_HPP
#include <cstddef>
#include <string>
#include <vector>
namespace octopus {
using SampleName = std::string;
class HaplotypeLikelihoodArray
{
public:
    using LikelihoodVector = std::vector<double>;
    std::size_t num_likelihoods(const SampleName&) const;
};
}
#endif
