// octopus_b200::MutationRepeatTable::from_reference(indel_prior) compiled against the reference's own indel_mutation_model_config.hpp
// (included first, as an Octopus build would): prints max_period max_periodicity max_indel_length, then the open and extend tables
// as hex floats. Built and run by tests/test_mutation_oracle.py where the reference checkout exists.
#include "core/models/mutation/indel_mutation_model_config.hpp"
#include "phmm_b200.hpp"
#include <cstdio>
int main(int argc, char** argv) {
    const auto t = octopus_b200::MutationRepeatTable::from_reference(std::atof(argv[1]));
    std::printf("%d %d %d\n", t.max_period, t.max_periodicity, t.max_indel_length);
    for (float x : t.open) std::printf("%a ", x);
    std::printf("\n");
    for (float x : t.extend) std::printf("%a ", x);
    std::printf("\n");
}
