// TEST INFRASTRUCTURE ONLY — never linked into or called from the product path.
//
// extern "C" driver around the UNMODIFIED reference mutation model, compiled from where it lies (oracle/mutation.mk):
//   src/core/models/mutation/indel_mutation_model.cpp   the repeat table (constructor) and the context indel model (evaluate)
//   src/core/models/mutation/denovo_model.cpp           prime / evaluate: PairHMM<VariableGapExtendMutationModel, 32, int>::align
//                                                       and recalculate_log_probability
//   utils/repeat_finder.hpp, lib/tandem                 the repeat finder evaluate calls
// Its headers' dependencies resolve to ref_shim_mutation/ and ref_shim/. The product's own implementation (phmm_mutation_context,
// phmm_mutation_prime) is checked against this.
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#define private public          // the driver reads IndelMutationModel's repeat table; the compiled model itself is unchanged
#include "core/models/mutation/indel_mutation_model.hpp"
#undef private
#include "core/models/mutation/denovo_model.hpp"

namespace octopus {
void (*difference_hook)(const Haplotype& target, const Haplotype& given) = nullptr;
}

namespace {

const octopus::Haplotype* g_block = nullptr;
int g_n = 0;
std::int32_t* g_approx = nullptr;

void record_difference(const octopus::Haplotype& target, const octopus::Haplotype& given)
{
    const long t = &target - g_block, g = &given - g_block;
    if (g_approx && t >= 0 && t < g_n && g >= 0 && g < g_n) g_approx[t * g_n + g] = 1;
}

} // namespace

extern "C" {

// IndelMutationModel({indel_prior}) (indel_mutation_model.cpp:40-55): dims = {max_period, max_periodicity, max_indel_length};
// open [(P+1)(Q+1)], extend [(P+1)(Q+1)][X] when non-NULL.
int ref_mutation_table(double indel_prior, int* dims, float* open, float* extend)
{
    const octopus::IndelMutationModel model {{indel_prior}};
    const auto& table = model.indel_repeat_model_;
    dims[0] = (int)table.size() - 1;
    dims[1] = (int)table.front().size() - 1;
    dims[2] = (int)table.front().front().extend.size();
    std::size_t c = 0;
    for (const auto& row : table) {
        for (const auto& cell : row) {
            if (open) open[c] = cell.open;
            if (extend) std::memcpy(extend + c * dims[2], cell.extend.data(), cell.extend.size() * sizeof(float));
            ++c;
        }
    }
    return 0;
}

// IndelMutationModel::evaluate(haplotype) (:67-98): gap_open [n], gap_extend [n][max_indel_length].
int ref_mutation_context(double indel_prior, const char* seq, int n, float* gap_open, float* gap_extend)
{
    const octopus::IndelMutationModel model {{indel_prior}};
    const octopus::Haplotype haplotype {std::string(seq, seq + n), 0};
    const auto result = model.evaluate(haplotype);
    if ((int)result.gap_open.size() != n) return -1;
    for (int i = 0; i < n; ++i) {
        gap_open[i] = result.gap_open[i];
        std::memcpy(gap_extend + (std::size_t)i * result.gap_extend[i].size(), result.gap_extend[i].data(), result.gap_extend[i].size() * sizeof(float));
    }
    return 0;
}

// DeNovoModel({snv_prior, indel_prior}).prime(block), then evaluate(target, given) for every ordered pair: out[t * n + g];
// approx[t * n + g] = 1 where Haplotype::difference was called for the pair (the approximate path).
int ref_mutation_prime(double snv_prior, double indel_prior, int n, const std::int64_t* off, const char* seq, double* out, std::int32_t* approx)
{
    octopus::MappableBlock<octopus::Haplotype> block {};
    block.reserve(n);
    for (int h = 0; h < n; ++h) block.emplace_back(std::string(seq + off[h], seq + off[h + 1]), 0);
    g_block = block.data(); g_n = n; g_approx = approx;
    std::memset(approx, 0, sizeof(std::int32_t) * (std::size_t)n * n);
    octopus::difference_hook = record_difference;
    octopus::DeNovoModel model {{snv_prior, indel_prior}};
    model.prime(block);
    const auto indexed = octopus::index(block);
    for (int t = 0; t < n; ++t) {
        for (int g = 0; g < n; ++g) out[(std::size_t)t * n + g] = model.evaluate(indexed[t], indexed[g]);
    }
    octopus::difference_hook = nullptr;
    g_block = nullptr; g_approx = nullptr;
    return 0;
}

} // extern "C"
