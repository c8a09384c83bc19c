// DeNovoModel's mutation model as the engine holds it (include/phmm_b200.h, phmm_mutation_*): shared by the host context model
// (phmm_error_model.cpp), phmm_mutation_prime (phmm_engine.cu) and the batcher's merge key (phmm_batcher.cpp).
#ifndef PHMM_MUTATION_H
#define PHMM_MUTATION_H

#include <cstdint>
#include <string>
#include <vector>

struct phmm_mutation_model {
    double snv_prior = 0.0;
    double snv_log_prior = 0.0;        // std::log(snv_prior) (denovo_model.cpp:33)
    std::int8_t snv_penalty = 0;       // probability_to_penalty(snv_prior) (:35)
    int max_period = 0, max_periodicity = 0, max_indel_length = 0;
    // IndelMutationModel's repeat table, cell (period, periods) at period * (max_periodicity + 1) + periods
    std::vector<float> open;           // [cells]
    std::vector<float> extend;         // [cells][max_indel_length]
    // per cell: the HMM's penalties (set_penalties, denovo_model.cpp:184-197) and
    // logp[cell][k] = std::log(calculate_indel_probability(...)) for an indel of length k + 1 (indel_mutation_model.cpp:114-123)
    std::vector<std::int8_t> open_penalty, extend_penalty;
    std::vector<float> logp;           // [cells][max_indel_length]
    // the model's inputs as bytes (snv_prior, the three dimensions, open, extend): equal keys give equal results, so the batcher
    // merges the requests of separately created models by this key
    std::string key;
    int cells() const { return (max_period + 1) * (max_periodicity + 1); }
};

#endif
