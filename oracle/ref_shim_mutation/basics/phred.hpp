// TEST INFRASTRUCTURE ONLY — denovo_model.cpp includes basics/phred.hpp (Boost.Multiprecision) but uses nothing from it.
#ifndef REF_SHIM_MUT_PHRED_HPP
#define REF_SHIM_MUT_PHRED_HPP
#endif
