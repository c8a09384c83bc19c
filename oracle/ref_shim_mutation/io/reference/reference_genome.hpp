// TEST INFRASTRUCTURE ONLY — repeat_finder.hpp declares overloads over a ReferenceGenome that the mutation model never calls.
#ifndef REF_SHIM_MUT_REFERENCE_GENOME_HPP
#define REF_SHIM_MUT_REFERENCE_GENOME_HPP
namespace octopus { class ReferenceGenome; }
#endif
