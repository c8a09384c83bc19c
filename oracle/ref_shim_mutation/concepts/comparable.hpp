// TEST INFRASTRUCTURE ONLY — included by repeat_finder.hpp; nothing of it is used on the mutation model's path.
#ifndef REF_SHIM_MUT_COMPARABLE_HPP
#define REF_SHIM_MUT_COMPARABLE_HPP
#endif
