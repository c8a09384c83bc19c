// phmm_b200.hpp — C++ host-side adapter over the C ABI (include/phmm_b200.h), mirroring the reference's own
// interface for the pair-HMM path so that Octopus code compiles against it unchanged:
//
//   octopus_b200::GpuPairHMM<Band>   satisfies the duck-typed PairHMM concept that octopus::hmm::evaluate / align are
//                                    templated on (src/core/models/pairhmm/pair_hmm.hpp:373-380, 397-406, 441-451, 471-483,
//                                    542-551, 590-601; canonical signatures simd_pair_hmm.hpp:433-549):
//                                    band_size(), name(), 4 x align(), calculate_flank_score().
//   octopus_b200::HaplotypeLikelihoodArray  the batch seam: populate(reads, haplotypes, flank_state) fills the
//                                    [haplotype][read] matrix (haplotype_likelihood_array.hpp:65-72, .cpp:51-103) and throws
//                                    ShortHaplotypeError exactly where the reference does (haplotype_likelihood_model.cpp:238-256).
//
// Header-only; link with -lphmm_b200. All likelihood arithmetic runs on the GPU behind the C ABI; the only host
// arithmetic here is calculate_flank_score, which in the reference too is a scalar replay of two alignment strings
// (simd_pair_hmm.hpp:352-430), not part of the DP.
#ifndef PHMM_B200_HPP
#define PHMM_B200_HPP

#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <functional>
#include <memory>
#include <new>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "phmm_b200.h"

namespace octopus_b200 {

class Error : public std::runtime_error
{
public:
    Error(int code, const std::string& what) : std::runtime_error {what}, code_ {code} {}
    int code() const noexcept { return code_; }
private:
    int code_;
};

// HaplotypeLikelihoodModel::ShortHaplotypeError (haplotype_likelihood_model.hpp:123-139)
class ShortHaplotypeError : public std::runtime_error
{
public:
    ShortHaplotypeError(std::size_t haplotype_index, unsigned required_extension)
    : std::runtime_error {"Haplotype is too short for alignment"}, haplotype_index_ {haplotype_index}, required_extension_ {required_extension} {}
    std::size_t haplotype_index() const noexcept { return haplotype_index_; }
    unsigned required_extension() const noexcept { return required_extension_; }
private:
    std::size_t haplotype_index_;
    unsigned required_extension_;
};

// simd::PairHMMWrapper::TooLargeBandSizeError (simd_pair_hmm_wrapper.hpp:45-61)
class TooLargeBandSizeError : public std::runtime_error
{
public:
    explicit TooLargeBandSizeError(unsigned band) : std::runtime_error {"Band size too large"}, band_ {band} {}
    unsigned band() const noexcept { return band_; }
private:
    unsigned band_;
};

namespace detail {

// ReadRealigner::realign's per-read step for every pair (phmm_realign_reads / phmm_batcher_realign_reads). Statuses as
// phmm_align_reads (PHMM_STATUS_*; SHORT_HAP carries the required extension in the high 16 bits); host memory.
struct PairAlignments
{
    std::vector<std::int64_t> mapping_position;
    std::vector<double> likelihood;
    std::vector<std::string> cigar;
    std::vector<std::int32_t> status;
};

// The outputs of one realign call at the adapter's CIGAR stride (4 x the longest read + 64); call(stride, mapping_position,
// likelihood, text, status) makes the call and throws on failure.
template <typename Call>
PairAlignments realign_reads(const phmm_reads& reads, std::size_t n, Call&& call)
{
    std::int64_t longest = 1;
    for (std::int32_t r = 0; r < reads.n; ++r) longest = std::max<std::int64_t>(longest, reads.off[r + 1] - reads.off[r]);
    const auto stride = static_cast<std::int32_t>(4 * longest + 64);
    PairAlignments a;
    a.mapping_position.resize(n); a.likelihood.resize(n); a.status.resize(n);
    std::vector<char> text(std::max<std::size_t>(n, 1) * static_cast<std::size_t>(stride), 0);
    call(stride, a.mapping_position.data(), a.likelihood.data(), text.data(), a.status.data());
    a.cigar.reserve(n);
    for (std::size_t j = 0; j < n; ++j) a.cigar.emplace_back(text.data() + j * static_cast<std::size_t>(stride));
    return a;
}

// compute_haplotype_support's scoring and choice for many genotypes (phmm_assign_reads / phmm_batcher_assign_reads, or per template
// phmm_assign_templates / phmm_batcher_assign_templates); host memory. top[i] bit k = group-local haplotype k is in item i's
// find_map_haplotypes set, an item being a read (or a template). likelihood: the groups' [H_g][items_g] matrices back to back; status:
// the groups' [H_g][R_g] matrices, per read either way. A short haplotype does not throw here: the code is PHMM_ERR_SHORT_HAPLOTYPE
// and the statuses carry the extension.
struct ReadAssignment
{
    std::vector<std::uint64_t> top;
    std::vector<double> likelihood;
    std::vector<std::int32_t> status;
    std::vector<std::int32_t> read_first;      // the groups' first reads: the layout of status (for a template call, derived once
                                               // from template_off)
    int code = PHMM_OK;
};

// sum over the groups of H_g x (first[g + 1] - first[g])
inline std::size_t group_slots(const std::vector<std::int32_t>& hap_first, const std::vector<std::int32_t>& first)
{
    std::size_t slots = 0;
    for (std::size_t g = 0; g + 1 < hap_first.size(); ++g)
        slots += static_cast<std::size_t>(std::max(0, hap_first[g + 1] - hap_first[g])) * static_cast<std::size_t>(std::max(0, first[g + 1] - first[g]));
    return slots;
}

// The outputs of one assign call of n_items items, the groups' items starting at item_first (read_first for a read call);
// call(groups, priors, top, likelihood, status) returns the call's code.
template <typename Call>
ReadAssignment assign(const phmm_haplotypes& haplotypes, std::int64_t n_items, const std::vector<std::int32_t>& hap_first,
                      const std::vector<std::int32_t>& read_first, const std::vector<std::int32_t>& item_first, const std::vector<double>* log_priors,
                      bool want_likelihoods, Call&& call)
{
    if (hap_first.empty() || hap_first.size() != read_first.size() || hap_first.size() != item_first.size())
        throw Error {PHMM_ERR_INVALID, "group bounds need n + 1 entries each"};
    const auto n = static_cast<std::int32_t>(hap_first.size() - 1);
    if (log_priors && log_priors->size() != static_cast<std::size_t>(haplotypes.n)) throw Error {PHMM_ERR_INVALID, "one log prior per haplotype"};
    const phmm_regions groups {n, hap_first.data(), read_first.data(), nullptr};
    ReadAssignment a;
    a.top.resize(static_cast<std::size_t>(std::max<std::int64_t>(0, n_items)));
    a.status.resize(group_slots(hap_first, read_first));
    if (want_likelihoods) a.likelihood.resize(group_slots(hap_first, item_first));
    a.read_first = read_first;
    a.code = call(groups, log_priors ? log_priors->data() : nullptr, a.top.data(), want_likelihoods ? a.likelihood.data() : nullptr, a.status.data());
    return a;
}

// The groups' first reads of a template call whose groups start at the templates template_first (template_off: n_templates + 1
// read offsets).
inline std::vector<std::int32_t> template_read_first(const std::int64_t* template_off, std::int32_t n_templates, const std::vector<std::int32_t>& template_first)
{
    std::vector<std::int32_t> read_first;
    read_first.reserve(template_first.size());
    for (std::int32_t t : template_first) {
        if (!template_off || t < 0 || t > n_templates) throw Error {PHMM_ERR_INVALID, "template_first must index template_off"};
        read_first.push_back(static_cast<std::int32_t>(template_off[t]));
    }
    return read_first;
}

} // namespace detail

class Engine
{
public:
    explicit Engine(int device = -1)
    {
        phmm_engine* e = nullptr;
        const int rc = phmm_create(&e, device);
        if (rc != PHMM_OK) throw Error {rc, phmm_last_error(nullptr)};
        handle_.reset(e, [] (phmm_engine* p) { phmm_destroy(p); });
    }
    explicit Engine(std::nullptr_t) noexcept {}   // no engine (an array that runs on a SharedEngine)
    phmm_engine* get() const noexcept { return handle_.get(); }
    void check(int rc) const
    {
        if (rc == PHMM_OK) return;
        throw Error {rc, phmm_last_error(handle_.get())};
    }

    // map_query_to_target(read, haplotype) uncapped for every pair (phmm_map_pairs): pair j's mapping begins are
    // positions[offsets[j], offsets[j + 1]), ascending. Host memory.
    struct PairMapping { std::vector<std::int64_t> offsets; std::vector<std::int32_t> positions; };
    PairMapping map_pairs(const phmm_haplotypes& haplotypes, const phmm_reads& reads, const std::vector<phmm_pair>& pairs) const
    {
        PairMapping m;
        m.offsets.resize(pairs.size() + 1);
        m.positions.resize(4 * pairs.size() + 16);   // most pairs have one or a few maxima; a second call takes the exact size
        for (;;) {
            check(phmm_map_pairs(get(), &haplotypes, &reads, pairs.data(), static_cast<std::int64_t>(pairs.size()), m.offsets.data(),
                                 m.positions.data(), static_cast<std::int64_t>(m.positions.size()), PHMM_SPACE_HOST));
            const auto total = static_cast<std::size_t>(m.offsets.back());
            if (total <= m.positions.size()) { m.positions.resize(total); return m; }
            m.positions.resize(total);
        }
    }

    // ReadRealigner::realign's per-read step for every pair (phmm_realign_reads); detail::PairAlignments.
    using PairAlignments = detail::PairAlignments;
    PairAlignments realign_reads(const phmm_config& config, const phmm_haplotypes& haplotypes, const phmm_reads& reads,
                                 const std::vector<phmm_pair>& pairs, const phmm_flank_state* flank_state = nullptr) const
    {
        return detail::realign_reads(reads, pairs.size(), [&] (std::int32_t stride, std::int64_t* mp, double* lk, char* text, std::int32_t* st) {
            check(phmm_realign_reads(get(), &config, &haplotypes, &reads, pairs.data(), static_cast<std::int64_t>(pairs.size()), flank_state,
                                     mp, lk, text, stride, st, PHMM_SPACE_HOST));
        });
    }

    // compute_haplotype_support's scoring and choice for many genotypes (phmm_assign_reads); detail::ReadAssignment.
    using ReadAssignment = detail::ReadAssignment;
    ReadAssignment assign_reads(const phmm_config& config, const phmm_haplotypes& haplotypes, const phmm_reads& reads,
                                const std::vector<std::int32_t>& hap_first, const std::vector<std::int32_t>& read_first,
                                const std::vector<double>* log_priors = nullptr, bool want_likelihoods = false) const
    {
        ReadAssignment a = detail::assign(haplotypes, reads.n, hap_first, read_first, read_first, log_priors, want_likelihoods,
                                          [&] (const phmm_regions& groups, const double* priors, std::uint64_t* top, double* lnl, std::int32_t* st) {
            return phmm_assign_reads(get(), &config, &haplotypes, &reads, &groups, priors, top, lnl, st, PHMM_SPACE_HOST);
        });
        if (a.code != PHMM_ERR_SHORT_HAPLOTYPE) check(a.code);
        return a;
    }

    // The same per template (phmm_assign_templates): template t owns reads [template_off[t], template_off[t+1]); group g owns
    // haplotypes [hap_first[g], hap_first[g+1]) and templates [template_first[g], template_first[g+1]). top and likelihood are per
    // template, status per read.
    ReadAssignment assign_templates(const phmm_config& config, const phmm_haplotypes& haplotypes, const phmm_reads& reads,
                                    const std::int64_t* template_off, std::int32_t n_templates, const std::vector<std::int32_t>& hap_first,
                                    const std::vector<std::int32_t>& template_first, const std::vector<double>* log_priors = nullptr,
                                    bool want_likelihoods = false) const
    {
        const auto read_first = detail::template_read_first(template_off, n_templates, template_first);
        ReadAssignment a = detail::assign(haplotypes, n_templates, hap_first, read_first, template_first, log_priors, want_likelihoods,
                                          [&] (const phmm_regions& groups, const double* priors, std::uint64_t* top, double* lnl, std::int32_t* st) {
            return phmm_assign_templates(get(), &config, &haplotypes, &reads, &groups, template_off, n_templates, priors, top, lnl, st, PHMM_SPACE_HOST);
        });
        if (a.code != PHMM_ERR_SHORT_HAPLOTYPE) check(a.code);
        return a;
    }
private:
    std::shared_ptr<phmm_engine> handle_;
};

// One engine for a whole process's threads (phmm_batcher): the populate calls that concurrent threads have in flight run as one
// multi-region kernel chain, their read assignments and realignments as one assign / realign call, each with the result it would
// get on an Engine of its own. Copies share the batcher; every thread may call it at once. clients: the number of threads that submit (Octopus's --threads); a batch is sent once that many wait,
// or max_wait_us after its first request arrived.
class SharedEngine
{
public:
    explicit SharedEngine(int device = -1, int clients = 0, int max_wait_us = 500)
    {
        phmm_batcher* b = nullptr;
        const phmm_batcher_options opt {clients, max_wait_us};
        const int rc = phmm_batcher_create(&b, device, &opt);
        if (rc != PHMM_OK) throw Error {rc, phmm_batcher_last_error()};
        handle_.reset(b, [] (phmm_batcher* p) { phmm_batcher_destroy(p); });
    }
    explicit SharedEngine(std::nullptr_t) noexcept {}
    phmm_batcher* get() const noexcept { return handle_.get(); }
    void check(int rc) const
    {
        if (rc == PHMM_OK) return;
        throw Error {rc, phmm_batcher_last_error()};   // the calling thread's own last error
    }
    phmm_batcher_stats stats() const
    {
        phmm_batcher_stats s {};
        check(phmm_batcher_stats_get(handle_.get(), &s));
        return s;
    }
    std::int64_t reruns() const { return phmm_batcher_reruns(handle_.get()); }

    // Engine::realign_reads, Engine::assign_reads and Engine::assign_templates through the shared engine (phmm_batcher_realign_reads /
    // _assign_reads / _assign_templates)
    using PairAlignments = detail::PairAlignments;
    PairAlignments realign_reads(const phmm_config& config, const phmm_haplotypes& haplotypes, const phmm_reads& reads,
                                 const std::vector<phmm_pair>& pairs, const phmm_flank_state* flank_state = nullptr) const
    {
        return detail::realign_reads(reads, pairs.size(), [&] (std::int32_t stride, std::int64_t* mp, double* lk, char* text, std::int32_t* st) {
            check(phmm_batcher_realign_reads(get(), &config, &haplotypes, &reads, pairs.data(), static_cast<std::int64_t>(pairs.size()),
                                             flank_state, mp, lk, text, stride, st));
        });
    }
    using ReadAssignment = detail::ReadAssignment;
    ReadAssignment assign_reads(const phmm_config& config, const phmm_haplotypes& haplotypes, const phmm_reads& reads,
                                const std::vector<std::int32_t>& hap_first, const std::vector<std::int32_t>& read_first,
                                const std::vector<double>* log_priors = nullptr, bool want_likelihoods = false) const
    {
        ReadAssignment a = detail::assign(haplotypes, reads.n, hap_first, read_first, read_first, log_priors, want_likelihoods,
                                          [&] (const phmm_regions& groups, const double* priors, std::uint64_t* top, double* lnl, std::int32_t* st) {
            return phmm_batcher_assign_reads(get(), &config, &haplotypes, &reads, &groups, priors, top, lnl, st);
        });
        if (a.code != PHMM_ERR_SHORT_HAPLOTYPE) check(a.code);
        return a;
    }
    ReadAssignment assign_templates(const phmm_config& config, const phmm_haplotypes& haplotypes, const phmm_reads& reads,
                                    const std::int64_t* template_off, std::int32_t n_templates, const std::vector<std::int32_t>& hap_first,
                                    const std::vector<std::int32_t>& template_first, const std::vector<double>* log_priors = nullptr,
                                    bool want_likelihoods = false) const
    {
        const auto read_first = detail::template_read_first(template_off, n_templates, template_first);
        ReadAssignment a = detail::assign(haplotypes, n_templates, hap_first, read_first, template_first, log_priors, want_likelihoods,
                                          [&] (const phmm_regions& groups, const double* priors, std::uint64_t* top, double* lnl, std::int32_t* st) {
            return phmm_batcher_assign_templates(get(), &config, &haplotypes, &reads, &groups, template_off, n_templates, priors, top, lnl, st);
        });
        if (a.code != PHMM_ERR_SHORT_HAPLOTYPE) check(a.code);
        return a;
    }
private:
    std::shared_ptr<phmm_batcher> handle_;
};

// Page-locked storage for the batch blocks: a std::allocator over phmm_host_alloc (cudaHostAlloc) that falls back to malloc where
// no GPU is usable. The blocks below are vectors of this allocator, so a populate() copies straight from / to pinned memory.
template <typename T>
struct PinnedAllocator
{
    using value_type = T;
    PinnedAllocator() = default;
    template <typename U> PinnedAllocator(const PinnedAllocator<U>&) noexcept {}
    T* allocate(std::size_t n)
    {
        // one tag word in front of the block remembers where it came from
        const std::size_t bytes = n * sizeof(T) + kHeader;
        char* p = static_cast<char*>(phmm_host_alloc(bytes));
        const bool pinned = p != nullptr;
        if (!p) p = static_cast<char*>(std::malloc(bytes));
        if (!p) throw std::bad_alloc {};
        *reinterpret_cast<std::size_t*>(p) = pinned ? 1 : 0;
        return reinterpret_cast<T*>(p + kHeader);
    }
    void deallocate(T* q, std::size_t) noexcept
    {
        char* p = reinterpret_cast<char*>(q) - kHeader;
        if (*reinterpret_cast<std::size_t*>(p)) phmm_host_free(p); else std::free(p);
    }
    template <typename U> bool operator==(const PinnedAllocator<U>&) const noexcept { return true; }
    template <typename U> bool operator!=(const PinnedAllocator<U>&) const noexcept { return false; }
private:
    static constexpr std::size_t kHeader = 64;   // keeps the payload 64-byte aligned
};
template <typename T> using pinned_vector = std::vector<T, PinnedAllocator<T>>;

// The reference's sequencing-error models (core/models/error/error_model_factory.cpp:531-589), i.e. what
// HaplotypeLikelihoodModel::reset runs per haplotype (haplotype_likelihood_model.cpp:60-78) — bit-identical, in the library.
class ErrorModel
{
public:
    explicit ErrorModel(const std::string& label = "PCR-free.HiSeq-2500")
    {
        phmm_error_model* m = nullptr;
        const int rc = phmm_error_model_create(&m, label.c_str());
        if (rc != PHMM_OK) throw Error {rc, phmm_error_model_last_error()};
        handle_.reset(m, [] (phmm_error_model* p) { phmm_error_model_destroy(p); });
    }
    static ErrorModel from_custom_model_text(const std::string& text)   // the contents of a --sequence-error-model file
    {
        phmm_error_model* m = nullptr;
        const int rc = phmm_error_model_create_custom(&m, text.c_str());
        if (rc != PHMM_OK) throw Error {rc, phmm_error_model_last_error()};
        ErrorModel result {std::shared_ptr<phmm_error_model>(m, [] (phmm_error_model* p) { phmm_error_model_destroy(p); })};
        return result;
    }
    const phmm_error_model* get() const noexcept { return handle_.get(); }
private:
    explicit ErrorModel(std::shared_ptr<phmm_error_model> h) : handle_ {std::move(h)} {}
    std::shared_ptr<phmm_error_model> handle_;
};

// ---------------------------------------------------------------------------------------------------------------------
// Per-call seam
// ---------------------------------------------------------------------------------------------------------------------
// The kernel with a runtime band, like simd::PairHMMWrapper (simd_pair_hmm_wrapper.hpp:218-241: smallest of 8, 16, ..., 256 that
// holds the request; TooLargeBandSizeError beyond). GpuPairHMM<Band> below fixes the band at compile time.
class GpuPairHMMDyn
{
public:
    using ScoreType = int;
    constexpr static char gap_label = '-';

    GpuPairHMMDyn() = default;
    explicit GpuPairHMMDyn(unsigned min_band_size, Engine engine = Engine {}) : engine_ {std::move(engine)} { reset(min_band_size); }
    void reset(unsigned min_band_size)
    {
        for (int b = 8; b <= 256; b <<= 1) if (min_band_size <= static_cast<unsigned>(b)) { band_ = b; return; }
        throw TooLargeBandSizeError {min_band_size};
    }

    constexpr static const char* name() noexcept { return "H100"; }
    int band_size() const noexcept { return band_; }

    // score only, no SNV model (simd_pair_hmm.hpp:438-452)
    template <typename GapExtend>
    int align(const char* truth, const char* target, const std::int8_t* qualities, int truth_len, int target_len,
              const std::int8_t* gap_open, GapExtend gap_extend, short nuc_prior) const noexcept
    {
        int first_pos;
        return run(truth, target, qualities, truth_len, target_len, nullptr, nullptr, gap_open, gap_extend, nuc_prior, first_pos, nullptr, nullptr);
    }
    // score only, SNV model (:454-470)
    template <typename GapExtend>
    int align(const char* truth, const char* target, const std::int8_t* qualities, int truth_len, int target_len,
              const char* snv_mask, const std::int8_t* snv_prior, const std::int8_t* gap_open, GapExtend gap_extend, short nuc_prior) const noexcept
    {
        int first_pos;
        return run(truth, target, qualities, truth_len, target_len, snv_mask, snv_prior, gap_open, gap_extend, nuc_prior, first_pos, nullptr, nullptr);
    }
    // traceback, no SNV model (:472-489)
    template <typename GapExtend>
    int align(const char* truth, const char* target, const std::int8_t* qualities, int truth_len, int target_len,
              const std::int8_t* gap_open, GapExtend gap_extend, short nuc_prior, int& first_pos, char* align1, char* align2) const noexcept
    {
        return run(truth, target, qualities, truth_len, target_len, nullptr, nullptr, gap_open, gap_extend, nuc_prior, first_pos, align1, align2);
    }
    // traceback, SNV model (:491-509)
    template <typename GapExtend>
    int align(const char* truth, const char* target, const std::int8_t* qualities, int truth_len, int target_len,
              const char* snv_mask, const std::int8_t* snv_prior, const std::int8_t* gap_open, GapExtend gap_extend, short nuc_prior,
              int& first_pos, char* align1, char* align2) const noexcept
    {
        return run(truth, target, qualities, truth_len, target_len, snv_mask, snv_prior, gap_open, gap_extend, nuc_prior, first_pos, align1, align2);
    }

    // simd_pair_hmm.hpp:530-549 (SNV overload): replay of the alignment strings; scalar on the host in the reference too
    template <typename GapExtend>
    int calculate_flank_score(int truth_len, int lhs_flank_len, int rhs_flank_len, const char* target, const std::int8_t* quals,
                              const char* snv_mask, const std::int8_t* snv_prior, const std::int8_t* gap_open, GapExtend gap_extend,
                              short nuc_prior, int first_pos, const char* aln1, const char* aln2, int& target_mask_size) const noexcept
    {
        enum { M, I, D };
        int prev = M, truth_idx = first_pos, target_idx = 0, result = 0;
        const int rhs_begin = truth_len - rhs_flank_len;
        target_mask_size = 0;
        for (int a = 0; aln1[a]; ++a) {
            int st = M;
            if (aln1[a] == gap_label) st = I; else if (aln2[a] == gap_label) st = D;
            const bool in_flank = truth_idx < lhs_flank_len || truth_idx >= rhs_begin;
            if (st == M) {
                if (in_flank) {
                    if (aln1[a] != aln2[a]) {
                        if (aln1[a] != 'N') {
                            int q = quals[target_idx];
                            if (snv_mask[truth_idx] == target[target_idx] && snv_prior[truth_idx] < q) q = snv_prior[truth_idx];
                            result += q;
                        } else result += 2;
                    }
                    ++target_mask_size;
                }
                ++truth_idx; ++target_idx;
            } else if (st == I) {
                if (in_flank) { result += (prev == I ? get(gap_extend, truth_idx - 1) : gap_open[truth_idx - 1]) + nuc_prior; ++target_mask_size; }
                ++target_idx;
            } else {
                if (in_flank) result += prev == D ? get(gap_extend, truth_idx) : gap_open[truth_idx];
                ++truth_idx;
            }
            prev = st;
        }
        return result;
    }

protected:
    GpuPairHMMDyn(Engine engine, int band) : engine_ {std::move(engine)}, band_ {band} {}   // an exact band (GpuPairHMM<Band>)

private:
    Engine engine_;
    int band_ = 8;

    static int get(const std::int8_t* v, int i) noexcept { return v[i]; }
    template <typename T> static int get(T v, int) noexcept { return static_cast<int>(v); }
    static const std::int8_t* ext_ptr(const std::int8_t* p) noexcept { return p; }
    template <typename T> static const std::int8_t* ext_ptr(T) noexcept { return nullptr; }
    static int ext_scalar(const std::int8_t*) noexcept { return 0; }
    template <typename T> static int ext_scalar(T v) noexcept { return static_cast<int>(v); }

    template <typename GapExtend>
    int run(const char* truth, const char* target, const std::int8_t* quals, int truth_len, int target_len,
            const char* snv_mask, const std::int8_t* snv_prior, const std::int8_t* gap_open, GapExtend gap_extend, short nuc_prior,
            int& first_pos, char* align1, char* align2) const noexcept
    {
        int score = 0;
        std::vector<char> a1, a2;
        if (!align1) { a1.assign(2 * (target_len + band_) + 1, 0); a2 = a1; align1 = a1.data(); align2 = a2.data(); }
        const int rc = phmm_align_traceback(engine_.get(), band_, truth, target, quals, truth_len, target_len, snv_mask, snv_prior,
                                            gap_open, ext_ptr(gap_extend), ext_scalar(gap_extend), nuc_prior, &score, &first_pos, align1, align2);
        if (rc != PHMM_OK) first_pos = -1;   // the reference signals failure through first_pos (simd_pair_hmm.hpp:176-199)
        return score;
    }
};

template <int BandSize>
class GpuPairHMM : private GpuPairHMMDyn
{
public:
    using GpuPairHMMDyn::ScoreType;
    using GpuPairHMMDyn::gap_label;
    using GpuPairHMMDyn::name;
    using GpuPairHMMDyn::align;
    using GpuPairHMMDyn::calculate_flank_score;

    explicit GpuPairHMM(Engine engine = Engine {}) : GpuPairHMMDyn {std::move(engine), BandSize} {}
    constexpr static int band_size() noexcept { return BandSize; }
};

// ---------------------------------------------------------------------------------------------------------------------
// Batch seam
// ---------------------------------------------------------------------------------------------------------------------
struct HaplotypeBlock   // what HaplotypeLikelihoodModel::reset derives per haplotype (haplotype_likelihood_model.cpp:60-78)
{
    pinned_vector<std::int64_t> off {0};
    pinned_vector<char> seq, snv_mask_fwd, snv_mask_rev;
    pinned_vector<std::int8_t> snv_prior_fwd, snv_prior_rev, gap_open, gap_extend;
    pinned_vector<std::int64_t> begin;
    pinned_vector<std::uint8_t> is_substitution;   // only used by reset(): bases that are substitutions in Haplotype::cigar()

    // Sequences only; reset(model) then fills the penalty arrays (the reference's likelihood_model_.reset(haplotype) per haplotype).
    void add(const std::string& sequence, std::int64_t mapped_begin = 0, const std::vector<bool>* substitutions = nullptr)
    {
        seq.insert(seq.end(), sequence.begin(), sequence.end());
        is_substitution.resize(seq.size(), 0);
        if (substitutions) for (std::size_t i = 0; i < substitutions->size() && i < sequence.size(); ++i) is_substitution[seq.size() - sequence.size() + i] = (*substitutions)[i] ? 1 : 0;
        begin.push_back(mapped_begin);
        off.push_back(static_cast<std::int64_t>(seq.size()));
    }
    void reset(const ErrorModel& model, int n_threads = 0)
    {
        const std::size_t n = seq.size();
        snv_mask_fwd.resize(n); snv_mask_rev.resize(n); snv_prior_fwd.resize(n); snv_prior_rev.resize(n); gap_open.resize(n); gap_extend.resize(n);
        is_substitution.resize(n, 0);
        const int rc = phmm_reset_haplotypes(model.get(), static_cast<std::int32_t>(size()), off.data(), seq.data(), is_substitution.data(),
                                             snv_mask_fwd.data(), snv_prior_fwd.data(), snv_mask_rev.data(), snv_prior_rev.data(),
                                             gap_open.data(), gap_extend.data(), n_threads);
        if (rc != PHMM_OK) throw Error {rc, phmm_error_model_last_error()};
    }
    // The same arrays, byte for byte, computed on the engine's GPU (phmm_engine_reset_haplotypes).
    void reset(const ErrorModel& model, Engine& engine)
    {
        const std::size_t n = seq.size();
        snv_mask_fwd.resize(n); snv_mask_rev.resize(n); snv_prior_fwd.resize(n); snv_prior_rev.resize(n); gap_open.resize(n); gap_extend.resize(n);
        is_substitution.resize(n, 0);
        engine.check(phmm_engine_reset_haplotypes(engine.get(), model.get(), static_cast<std::int32_t>(size()), off.data(), seq.data(),
                                                  is_substitution.data(), snv_mask_fwd.data(), snv_prior_fwd.data(), snv_mask_rev.data(),
                                                  snv_prior_rev.data(), gap_open.data(), gap_extend.data(), PHMM_SPACE_HOST));
    }

    void add(const std::string& sequence, const std::vector<char>& fwd_mask, const std::vector<std::int8_t>& fwd_priors,
             const std::vector<char>& rev_mask, const std::vector<std::int8_t>& rev_priors,
             const std::vector<std::int8_t>& open, const std::vector<std::int8_t>& extend, std::int64_t mapped_begin = 0)
    {
        seq.insert(seq.end(), sequence.begin(), sequence.end());
        snv_mask_fwd.insert(snv_mask_fwd.end(), fwd_mask.begin(), fwd_mask.end());
        snv_mask_rev.insert(snv_mask_rev.end(), rev_mask.begin(), rev_mask.end());
        snv_prior_fwd.insert(snv_prior_fwd.end(), fwd_priors.begin(), fwd_priors.end());
        snv_prior_rev.insert(snv_prior_rev.end(), rev_priors.begin(), rev_priors.end());
        gap_open.insert(gap_open.end(), open.begin(), open.end());
        gap_extend.insert(gap_extend.end(), extend.begin(), extend.end());
        begin.push_back(mapped_begin);
        off.push_back(static_cast<std::int64_t>(seq.size()));
    }
    std::size_t size() const noexcept { return off.size() - 1; }
    // The sequences side only: what a populate with an error model reads (seq, off, begin and the substitution flags of add()).
    phmm_haplotype_sequences sequences_view() const noexcept
    {
        return phmm_haplotype_sequences {static_cast<std::int32_t>(size()), off.data(), seq.data(),
                                         is_substitution.size() == seq.size() ? is_substitution.data() : nullptr, begin.data()};
    }
    phmm_haplotypes view() const noexcept
    {
        return phmm_haplotypes {static_cast<std::int32_t>(size()), off.data(), seq.data(), snv_mask_fwd.data(), snv_prior_fwd.data(),
                                snv_mask_rev.data(), snv_prior_rev.data(), gap_open.data(), gap_extend.data(), begin.data()};
    }
};

struct ReadBlock   // AlignedRead fields on the path (basics/aligned_read.hpp:36-39,120-146)
{
    pinned_vector<std::int64_t> off {0};
    pinned_vector<char> bases;
    pinned_vector<std::uint8_t> quals, mapq, reverse;
    pinned_vector<std::int64_t> begin;

    void add(const std::string& sequence, const std::vector<std::uint8_t>& base_qualities, std::uint8_t mapping_quality,
             bool is_marked_reverse_mapped, std::int64_t mapped_begin)
    {
        bases.insert(bases.end(), sequence.begin(), sequence.end());
        quals.insert(quals.end(), base_qualities.begin(), base_qualities.end());
        mapq.push_back(mapping_quality);
        reverse.push_back(is_marked_reverse_mapped ? 1 : 0);
        begin.push_back(mapped_begin);
        off.push_back(static_cast<std::int64_t>(bases.size()));
    }
    void append(const ReadBlock& other)
    {
        const auto base = static_cast<std::int64_t>(bases.size());
        bases.insert(bases.end(), other.bases.begin(), other.bases.end());
        quals.insert(quals.end(), other.quals.begin(), other.quals.end());
        mapq.insert(mapq.end(), other.mapq.begin(), other.mapq.end());
        reverse.insert(reverse.end(), other.reverse.begin(), other.reverse.end());
        begin.insert(begin.end(), other.begin.begin(), other.begin.end());
        for (std::size_t i = 1; i < other.off.size(); ++i) off.push_back(base + other.off[i]);
    }
    std::size_t size() const noexcept { return off.size() - 1; }
    phmm_reads view() const noexcept
    {
        return phmm_reads {static_cast<std::int32_t>(size()), off.data(), bases.data(), quals.data(), mapq.data(), reverse.data(), begin.data()};
    }
};

struct TemplateBlock   // AlignedTemplate containers: template t owns the reads [off[t], off[t+1]) (basics/aligned_template.hpp)
{
    ReadBlock reads;
    pinned_vector<std::int64_t> off {0};
    void add(const ReadBlock& template_reads) { reads.append(template_reads); off.push_back(static_cast<std::int64_t>(reads.size())); }
    std::size_t size() const noexcept { return off.size() - 1; }
};

struct FlankState { std::int64_t lhs_flank, rhs_flank; };   // HaplotypeLikelihoodModel::FlankState

namespace detail {

inline phmm_flank_state flank_state(const FlankState* f) noexcept
{
    return phmm_flank_state {f ? 1 : 0, f ? f->lhs_flank : 0, f ? f->rhs_flank : 0};
}

// Throws ShortHaplotypeError for the first of n statuses whose code is PHMM_STATUS_SHORT_HAP (its high 16 bits: the required
// extension); haplotype_of(i) is the haplotype index of status i's pair.
template <typename HaplotypeOf>
void throw_first_short_haplotype(const std::int32_t* status, std::size_t n, HaplotypeOf haplotype_of)
{
    for (std::size_t i = 0; i < n; ++i) {
        if ((status[i] & 0xFFFF) == PHMM_STATUS_SHORT_HAP)
            throw ShortHaplotypeError {haplotype_of(i), static_cast<unsigned>(static_cast<std::uint32_t>(status[i]) >> 16)};
    }
}

} // namespace detail

// One read's result of ReadRealigner::realign (read_realigner.cpp:92-103, 128-130): HaplotypeLikelihoodModel::Alignment.
struct Realignment
{
    std::int64_t mapping_position;
    std::string cigar;
    double likelihood;
};

namespace detail {

// realign() on an Engine or a SharedEngine (both have realign_reads)
template <typename AnyEngine>
std::vector<Realignment> realign(const ReadBlock& reads, const HaplotypeBlock& haplotypes, std::size_t haplotype, const phmm_config& config,
                                 const AnyEngine& engine, const FlankState* flank_state)
{
    std::vector<phmm_pair> pairs(reads.size());
    for (std::size_t r = 0; r < reads.size(); ++r) pairs[r] = phmm_pair {static_cast<std::int32_t>(r), static_cast<std::int32_t>(haplotype)};
    const phmm_flank_state fs = detail::flank_state(flank_state);
    const auto a = engine.realign_reads(config, haplotypes.view(), reads.view(), pairs, &fs);
    std::vector<Realignment> result;
    result.reserve(pairs.size());
    for (std::size_t r = 0; r < pairs.size(); ++r) {
        detail::throw_first_short_haplotype(&a.status[r], 1, [haplotype] (std::size_t) { return haplotype; });
        const int code = a.status[r] & 0xFFFF;
        if (code == PHMM_STATUS_HMM_OVERFLOW) throw Error {PHMM_ERR_INVALID, "HMMOverflow"};
        if (code == PHMM_STATUS_CIGAR_TRUNCATED) throw Error {PHMM_ERR_INVALID, "CIGAR truncated"};
        result.push_back(Realignment {a.mapping_position[r], a.cigar[r], a.likelihood[r]});
    }
    return result;
}

} // namespace detail

// realign(reads, haplotype, model) (read_realigner.cpp:105-144) for haplotype `haplotype` of the block: every read mapped with the
// uncapped k-mer mapper and aligned there, on the GPU. When a read's haplotype is too short, throws ShortHaplotypeError for the first
// such read in read order — the reference's serial loop, whose required extension safe_realign (:196-207) applies.
inline std::vector<Realignment> realign(const ReadBlock& reads, const HaplotypeBlock& haplotypes, std::size_t haplotype,
                                        const phmm_config& config, const Engine& engine = Engine {}, const FlankState* flank_state = nullptr)
{
    return detail::realign(reads, haplotypes, haplotype, config, engine, flank_state);
}

// The same through a shared engine: a region thread's realignments merge with other threads' requests, with the same results and
// exceptions.
inline std::vector<Realignment> realign(const ReadBlock& reads, const HaplotypeBlock& haplotypes, std::size_t haplotype,
                                        const phmm_config& config, const SharedEngine& engine, const FlankState* flank_state = nullptr)
{
    return detail::realign(reads, haplotypes, haplotype, config, engine, flank_state);
}

// AssignmentConfig::AmbiguousAction (core/tools/read_assigner.hpp). random needs the caller's RNG: apply it to
// HaplotypeSupport::ambiguous yourself (the helper treats it as drop).
enum class AmbiguousAction { drop, first, all, random };

// One genotype's result of compute_haplotype_support(genotype, reads, log_priors, model, ambiguous, config): the reads (indices into
// the read block) supported by each of the genotype's haplotypes, in genotype order, and the ambiguous reads with their top sets
// (group-local haplotype indices, ascending: AmbiguousRecord::haplotypes, the default), in read order.
struct HaplotypeSupport
{
    std::vector<std::vector<std::size_t>> reads;
    std::vector<std::pair<std::size_t, std::vector<unsigned>>> ambiguous;
};

namespace detail {

// The groups' supports from an assignment whose items (reads or templates) start at item_first per group; the assignment's own
// read_first lays out its statuses. Throws ShortHaplotypeError for the first short pair in the reference's order.
inline std::vector<HaplotypeSupport> support(const ReadAssignment& a, const std::vector<std::int32_t>& hap_first,
                                             const std::vector<std::int32_t>& item_first, AmbiguousAction action)
{
    if (a.code == PHMM_ERR_SHORT_HAPLOTYPE) {
        const std::vector<std::int32_t>& read_first = a.read_first;
        std::size_t slot = 0;
        for (std::size_t g = 0; g + 1 < hap_first.size(); ++g) {
            const auto nh = static_cast<std::size_t>(hap_first[g + 1] - hap_first[g]), nr = static_cast<std::size_t>(read_first[g + 1] - read_first[g]);
            detail::throw_first_short_haplotype(a.status.data() + slot, nh * nr, [&] (std::size_t i) { return hap_first[g] + i / nr; });
            slot += nh * nr;
        }
        throw Error {a.code, "Haplotype is too short for alignment"};
    }
    std::vector<HaplotypeSupport> result(hap_first.size() - 1);
    for (std::size_t g = 0; g + 1 < hap_first.size(); ++g) {
        const auto nh = static_cast<std::size_t>(hap_first[g + 1] - hap_first[g]), nr = static_cast<std::size_t>(item_first[g + 1] - item_first[g]);
        HaplotypeSupport& s = result[g];
        s.reads.resize(nh);
        for (std::size_t i = 0; i < nr; ++i) {
            const std::size_t r = static_cast<std::size_t>(item_first[g]) + i;
            const std::uint64_t top = a.top[r];
            if ((top & (top - 1)) == 0) {                       // one haplotype
                for (unsigned k = 0; k < nh; ++k) if (top >> k & 1u) s.reads[k].push_back(r);
                continue;
            }
            std::vector<unsigned> set;
            for (unsigned k = 0; k < nh; ++k) if (top >> k & 1u) set.push_back(k);
            if (action == AmbiguousAction::first) s.reads[set.front()].push_back(r);
            else if (action == AmbiguousAction::all) for (unsigned k : set) s.reads[k].push_back(r);
            s.ambiguous.emplace_back(r, std::move(set));
        }
    }
    return result;
}

// compute_haplotype_support() on an Engine or a SharedEngine (both have assign_reads and assign_templates)
template <typename AnyEngine>
std::vector<HaplotypeSupport> haplotype_support(const ReadBlock& reads, const HaplotypeBlock& haplotypes, const std::vector<std::int32_t>& hap_first,
                                                const std::vector<std::int32_t>& read_first, const std::vector<double>* log_priors,
                                                AmbiguousAction action, const phmm_config& config, const AnyEngine& engine)
{
    return support(engine.assign_reads(config, haplotypes.view(), reads.view(), hap_first, read_first, log_priors), hap_first, read_first, action);
}

template <typename AnyEngine>
std::vector<HaplotypeSupport> template_support(const TemplateBlock& templates, const HaplotypeBlock& haplotypes, const std::vector<std::int32_t>& hap_first,
                                               const std::vector<std::int32_t>& template_first, const std::vector<double>* log_priors,
                                               AmbiguousAction action, const phmm_config& config, const AnyEngine& engine)
{
    const auto n_templates = static_cast<std::int32_t>(templates.size());
    const auto a = engine.assign_templates(config, haplotypes.view(), templates.reads.view(), templates.off.data(), n_templates, hap_first,
                                           template_first, log_priors);
    return support(a, hap_first, template_first, action);
}

} // namespace detail

// compute_haplotype_support (core/tools/read_assigner.cpp:322-459) for many genotypes in one GPU call: group g (one genotype, after the
// caller's collapse) owns haplotypes [hap_first[g], hap_first[g+1]) and reads [read_first[g], read_first[g+1]). log_priors: one per
// haplotype of the block, or null. When a haplotype is too short, throws ShortHaplotypeError for the first short (haplotype, read)
// pair in the reference's order (groups in turn, haplotypes in genotype order, then reads), with the block's haplotype index.
inline std::vector<HaplotypeSupport> compute_haplotype_support(const ReadBlock& reads, const HaplotypeBlock& haplotypes,
                                                               const std::vector<std::int32_t>& hap_first, const std::vector<std::int32_t>& read_first,
                                                               const std::vector<double>* log_priors, AmbiguousAction action,
                                                               const phmm_config& config, const Engine& engine = Engine {})
{
    return detail::haplotype_support(reads, haplotypes, hap_first, read_first, log_priors, action, config, engine);
}

// The same through a shared engine: a region thread's assignments merge with other threads' requests, with the same results and
// exceptions.
inline std::vector<HaplotypeSupport> compute_haplotype_support(const ReadBlock& reads, const HaplotypeBlock& haplotypes,
                                                               const std::vector<std::int32_t>& hap_first, const std::vector<std::int32_t>& read_first,
                                                               const std::vector<double>* log_priors, AmbiguousAction action,
                                                               const phmm_config& config, const SharedEngine& engine)
{
    return detail::haplotype_support(reads, haplotypes, hap_first, read_first, log_priors, action, config, engine);
}

// compute_haplotype_support over AlignedTemplates (read_assigner.cpp:322-459 with the template overload; BAMRealigner's call under
// --read-linkage paired, bam_realigner.cpp:241-300) for many genotypes in one GPU call: group g owns haplotypes [hap_first[g],
// hap_first[g+1]) and TEMPLATES [template_first[g], template_first[g+1]) of the block. Every read of a template is scored as
// compute_haplotype_support scores reads; a template's value is the sum of its reads', and the choice is per template. The returned
// HaplotypeSupport holds TEMPLATE indices (into the block), in its reads and in its ambiguous list. When a haplotype is too short,
// throws ShortHaplotypeError for the first short (haplotype, read) pair in the reference's order (groups in turn, haplotypes in
// genotype order, then reads: the template loop's order), with the block's haplotype index.
inline std::vector<HaplotypeSupport> compute_haplotype_support(const TemplateBlock& templates, const HaplotypeBlock& haplotypes,
                                                               const std::vector<std::int32_t>& hap_first, const std::vector<std::int32_t>& template_first,
                                                               const std::vector<double>* log_priors, AmbiguousAction action,
                                                               const phmm_config& config, const Engine& engine = Engine {})
{
    return detail::template_support(templates, haplotypes, hap_first, template_first, log_priors, action, config, engine);
}

// The same through a shared engine, with the same results and exceptions.
inline std::vector<HaplotypeSupport> compute_haplotype_support(const TemplateBlock& templates, const HaplotypeBlock& haplotypes,
                                                               const std::vector<std::int32_t>& hap_first, const std::vector<std::int32_t>& template_first,
                                                               const std::vector<double>* log_priors, AmbiguousAction action,
                                                               const phmm_config& config, const SharedEngine& engine)
{
    return detail::template_support(templates, haplotypes, hap_first, template_first, log_priors, action, config, engine);
}

using SampleName = std::string;

// ---------------------------------------------------------------------------------------------------------------------
// DeNovoModel (core/models/mutation/denovo_model.{hpp,cpp}) over phmm_mutation_prime
// ---------------------------------------------------------------------------------------------------------------------
// IndelMutationModel's repeat table for one indel prior: cell (period p, periods q) at p * (max_periodicity + 1) + q; open[cell],
// extend[cell * max_indel_length + gap]. The values are Octopus's: with the reference's indel_mutation_model_config.hpp included
// before this header, from_reference(indel_prior) computes them as IndelMutationModel's constructor does (indel_mutation_model.cpp:17-55).
struct MutationRepeatTable
{
    int max_period = 10, max_periodicity = 50, max_indel_length = 50;   // IndelMutationModel::Parameters defaults (.hpp:25-26)
    std::vector<float> open, extend;
#ifdef indel_mutation_model_config_hpp
    static MutationRepeatTable from_reference(const double indel_prior, const unsigned max_period = 10, const unsigned max_periodicity = 50,
                                              const unsigned max_indel_length = 50, const double max_open_probability = 0.9,
                                              const double max_extend_probability = 1.0)
    {
        using octopus::enrichment_model;
        using octopus::extension_model;
        MutationRepeatTable t;
        t.max_period = static_cast<int>(max_period);
        t.max_periodicity = static_cast<int>(max_periodicity);
        t.max_indel_length = static_cast<int>(max_indel_length);
        const unsigned e_period = static_cast<unsigned>(enrichment_model.size() - 1), e_periods = static_cast<unsigned>(enrichment_model.front().size() - 1);
        const unsigned x_period = static_cast<unsigned>(extension_model.size() - 1), x_periods = static_cast<unsigned>(extension_model.front().size() - 1);
        const unsigned x_gap = static_cast<unsigned>(extension_model.front().front().size() - 1);
        for (unsigned period = 0; period <= max_period; ++period) {
            for (unsigned periods = 0; periods <= max_periodicity; ++periods) {
                // calculate_gap_open_prior / calculate_gap_extend_prior (:17-37)
                const double open_prior = (period == 0 || periods == 0) ? indel_prior
                    : std::min(indel_prior * enrichment_model[std::min(period, e_period)][std::min(periods, e_periods)], 1.0);
                t.open.push_back(static_cast<float>(std::min(open_prior, max_open_probability)));
                for (unsigned gap = 0; gap < max_indel_length; ++gap) {
                    const double extend_prior = std::max(open_prior, extension_model[std::min(period, x_period)][std::min(periods, x_periods)][std::min(gap, x_gap)]);
                    t.extend.push_back(static_cast<float>(std::min(extend_prior, max_extend_probability)));
                }
            }
        }
        return t;
    }
#endif
};

// DeNovoModel: prime(sequences) scores every ordered (target, given) pair of one region's haplotypes in one GPU call
// (phmm_mutation_prime); evaluate(target, given) = ln p(target | given), the reference's evaluate(IndexedHaplotype, IndexedHaplotype).
// Pairs the reference sends to its approximate path (length distance >= 32, another alignment offset, HMMOverflow) need
// Haplotype::difference, which lives with the caller: evaluate calls approx(target, given) for them, once, and keeps the value. So does
// a pair whose alignment puts an indel past the given haplotype (PHMM_MUT_OUT_OF_MODEL: the reference's value is undefined there).
// SomaticMutationModel::prime (somatic_mutation_model.cpp:20-23) is the same model under the cancer caller's priors.
class DeNovoModel
{
public:
    using LogProbability = double;
    struct Parameters { double snv_prior, indel_prior; };
    using ApproxFunction = std::function<LogProbability(std::size_t target_idx, std::size_t given_idx)>;

    DeNovoModel(Parameters parameters, const MutationRepeatTable& table, Engine& engine, ApproxFunction approx = nullptr)
    : DeNovoModel {parameters, table, &engine, SharedEngine {nullptr}, std::move(approx)} {}
    // prime() through a process-wide SharedEngine: any number of threads, each with its own model object, may prime at once; their
    // sets run as one phmm_mutation_prime_sets call where the models are equal (trio_caller.cpp:406 builds one per region)
    DeNovoModel(Parameters parameters, const MutationRepeatTable& table, SharedEngine& shared, ApproxFunction approx = nullptr)
    : DeNovoModel {parameters, table, nullptr, shared, std::move(approx)} {}
#ifdef indel_mutation_model_config_hpp
    DeNovoModel(Parameters parameters, Engine& engine, ApproxFunction approx = nullptr)
    : DeNovoModel {parameters, MutationRepeatTable::from_reference(parameters.indel_prior), engine, std::move(approx)} {}
    DeNovoModel(Parameters parameters, SharedEngine& shared, ApproxFunction approx = nullptr)
    : DeNovoModel {parameters, MutationRepeatTable::from_reference(parameters.indel_prior), shared, std::move(approx)} {}
#endif

    Parameters parameters() const { return params_; }

    void prime(const std::vector<std::string>& haplotypes)
    {
        if (is_primed()) throw std::runtime_error {"DeNovoModel: already primed"};
        const std::size_t n = haplotypes.size();
        std::vector<std::int64_t> off(n + 1, 0);
        std::string seq;
        for (std::size_t h = 0; h < n; ++h) { seq += haplotypes[h]; off[h + 1] = static_cast<std::int64_t>(seq.size()); }
        values_.assign(n * n, 0.0);
        status_.assign(n * n, PHMM_MUT_SELF);
        settled_.assign(n * n, 0);
        const auto h = static_cast<std::int32_t>(n);
        if (n > 0 && engine_) engine_->check(phmm_mutation_prime(engine_->get(), model_.get(), h, off.data(), seq.data(), values_.data(), status_.data()));
        if (n > 0 && !engine_) shared_.check(phmm_batcher_mutation_prime(shared_.get(), model_.get(), h, off.data(), seq.data(), values_.data(), status_.data()));
        n_ = n;
    }
    void unprime() noexcept { values_ = {}; status_ = {}; settled_ = {}; n_ = 0; }
    bool is_primed() const noexcept { return n_ > 0; }

    // ln p(target | given) for haplotype indices of the primed set
    LogProbability evaluate(const std::size_t target_idx, const std::size_t given_idx) const
    {
        if (target_idx >= n_ || given_idx >= n_) throw std::out_of_range {"DeNovoModel::evaluate: haplotype index"};
        const std::size_t i = target_idx * n_ + given_idx;
        if (status_[i] == PHMM_MUT_HMM || status_[i] == PHMM_MUT_SELF || settled_[i]) return values_[i];
        if (!approx_) throw Error {PHMM_ERR_INVALID, "DeNovoModel: an approximate pair needs the approx function"};
        values_[i] = approx_(target_idx, given_idx);
        settled_[i] = 1;
        return values_[i];
    }
    // PHMM_MUT_* of a pair (PHMM_MUT_APPROX_* / OUT_OF_MODEL: evaluate asks approx)
    std::int32_t status(const std::size_t target_idx, const std::size_t given_idx) const { return status_.at(target_idx * n_ + given_idx); }

private:
    DeNovoModel(Parameters parameters, const MutationRepeatTable& table, Engine* engine, SharedEngine shared, ApproxFunction approx)
    : params_ {parameters}, engine_ {engine}, shared_ {std::move(shared)}, approx_ {std::move(approx)}
    {
        phmm_mutation_model* m = nullptr;
        const int rc = phmm_mutation_model_create(&m, parameters.snv_prior, table.open.data(), table.extend.data(), table.max_period,
                                                  table.max_periodicity, table.max_indel_length);
        if (rc != PHMM_OK) throw Error {rc, phmm_error_model_last_error()};
        model_.reset(m, [] (phmm_mutation_model* p) { phmm_mutation_model_destroy(p); });
    }

    Parameters params_;
    Engine* engine_;              // null: prime() goes through shared_
    SharedEngine shared_;
    ApproxFunction approx_;
    std::shared_ptr<phmm_mutation_model> model_;
    std::size_t n_ = 0;
    mutable std::vector<double> values_;
    std::vector<std::int32_t> status_;
    mutable std::vector<char> settled_;
};

using SomaticMutationModel = DeNovoModel;

// A read-only view of one likelihoods_[haplotype][sample] vector (the reference returns const std::vector<double>&).
struct LikelihoodSpan
{
    const double* first = nullptr;
    std::size_t count = 0;
    const double* begin() const noexcept { return first; }
    const double* end() const noexcept { return first + count; }
    std::size_t size() const noexcept { return count; }
    bool empty() const noexcept { return count == 0; }
    double operator[](std::size_t i) const noexcept { return first[i]; }
    operator std::vector<double>() const { return std::vector<double>(first, first + count); }
};

// HaplotypeLikelihoodArray (haplotype_likelihood_array.hpp:34-175): likelihoods_[haplotype][sample][read or template].
// All samples of a populate() go to the GPU as ONE batch (their reads are concatenated; one phmm_populate call fills one
// [H][R_total] matrix), a sample is a column range of that matrix.
class HaplotypeLikelihoodArray
{
public:
    using LogProbability = double;
    using LikelihoodVector = std::vector<LogProbability>;
    using ReadMap = std::vector<std::pair<SampleName, ReadBlock>>;                 // config/common.hpp:33-37, in sample order
    using TemplateMap = std::vector<std::pair<SampleName, TemplateBlock>>;

    explicit HaplotypeLikelihoodArray(phmm_config config, Engine engine = Engine {}) : engine_ {std::move(engine)}, config_ {checked(config)} {}
    // populate() goes through a process-wide SharedEngine: any number of threads, each with its own array, share one GPU engine
    HaplotypeLikelihoodArray(phmm_config config, SharedEngine shared) : engine_ {nullptr}, shared_ {std::move(shared)}, config_ {checked(config)} {}
    // With an error model, populate() runs likelihood_model_.reset(haplotype) itself, as the reference's populate does
    // (haplotype_likelihood_array.cpp:77-95): it reads only the HaplotypeBlock's sequences (add(sequence, begin, substitutions)) and
    // the GPU derives the penalty arrays in the same call (phmm_populate*_reset), with the values of HaplotypeBlock::reset(model).
    HaplotypeLikelihoodArray(phmm_config config, ErrorModel model, Engine engine = Engine {})
        : engine_ {std::move(engine)}, model_ {std::make_shared<const ErrorModel>(std::move(model))}, config_ {checked(config)} {}
    HaplotypeLikelihoodArray(phmm_config config, ErrorModel model, SharedEngine shared)
        : engine_ {nullptr}, shared_ {std::move(shared)}, model_ {std::make_shared<const ErrorModel>(std::move(model))}, config_ {checked(config)} {}
    static phmm_config default_config() noexcept { phmm_config c; phmm_default_config(&c); return c; }

    // populate(const ReadMap&, haplotypes, flank_state) — haplotype_likelihood_array.cpp:51-103.
    // positions: optional candidate mapping positions (CSR over [H][R_total]); without them the device k-mer mapper runs
    // (config.map_positions), as the reference maps inline (:89-92).
    void populate(const ReadMap& reads, const HaplotypeBlock& haplotypes, const FlankState* flank_state = nullptr,
                  const phmm_positions* positions = nullptr)
    {
        ReadBlock all;
        begin_samples(reads.size());
        for (const auto& p : reads) { add_sample(p.first, p.second.size()); all.append(p.second); }
        run(all, nullptr, haplotypes, flank_state, positions);
    }
    // single unnamed sample, primed (what the reference's single-sample callers see after prime())
    void populate(const ReadBlock& reads, const HaplotypeBlock& haplotypes, const FlankState* flank_state = nullptr,
                  const phmm_positions* positions = nullptr)
    {
        begin_samples(1);
        add_sample(SampleName {}, reads.size());
        run(reads, nullptr, haplotypes, flank_state, positions);
        primed_ = 0;
    }
    // populate(const TemplateMap&, ...) — haplotype_likelihood_array.cpp:105-199: one value per (haplotype, template)
    void populate(const TemplateMap& templates, const HaplotypeBlock& haplotypes, const FlankState* flank_state = nullptr)
    {
        ReadBlock all;
        pinned_vector<std::int64_t> template_off {0};
        begin_samples(templates.size());
        for (const auto& p : templates) {
            add_sample(p.first, p.second.size());
            const auto base = static_cast<std::int64_t>(all.size());
            all.append(p.second.reads);
            for (std::size_t t = 1; t < p.second.off.size(); ++t) template_off.push_back(base + p.second.off[t]);
        }
        run(all, &template_off, haplotypes, flank_state, nullptr);
    }

    // accessors (haplotype_likelihood_array.cpp:200-291)
    std::size_t num_likelihoods(const SampleName& sample) const { return width(sample_index(sample)); }
    std::size_t num_likelihoods() const { return width(primed()); }
    LikelihoodSpan operator()(const SampleName& sample, std::size_t haplotype_index) const { return span(haplotype_index, sample_index(sample)); }
    LikelihoodSpan operator[](std::size_t haplotype_index) const { return span(haplotype_index, primed()); }
    const std::vector<SampleName>& samples() const noexcept { return samples_; }
    std::size_t num_haplotypes() const noexcept { return num_haplotypes_; }
    std::vector<LikelihoodVector> extract_sample(const SampleName& sample) const
    {
        const auto s = sample_index(sample);
        std::vector<LikelihoodVector> result;
        for (std::size_t h = 0; h < num_haplotypes_; ++h) result.push_back(span(h, s));
        return result;
    }
    bool is_empty() const noexcept { return likelihoods_.empty(); }
    void clear() noexcept { likelihoods_.clear(); samples_.clear(); sample_off_.assign(1, 0); num_haplotypes_ = 0; unprime(); }
    bool is_primed() const noexcept { return primed_ >= 0; }
    void prime(const SampleName& sample) const { primed_ = static_cast<std::ptrdiff_t>(sample_index(sample)); }
    void unprime() const noexcept { primed_ = -1; }

    // reset(haplotypes) (:331-360): keep a subset of the haplotypes — here by their (ascending) old indices
    void reset(const std::vector<std::size_t>& haplotypes_to_keep)
    {
        if (haplotypes_to_keep.empty()) { clear(); return; }
        const std::size_t w = total_width();
        std::size_t dst = 0, prev = 0;
        for (const std::size_t h : haplotypes_to_keep) {
            if (h >= num_haplotypes_ || (dst > 0 && h <= prev)) throw std::invalid_argument {"reset: haplotype indices must be ascending and in range"};
            if (h != dst) std::copy_n(likelihoods_.begin() + static_cast<std::ptrdiff_t>(h * w), w, likelihoods_.begin() + static_cast<std::ptrdiff_t>(dst * w));
            prev = h; ++dst;
        }
        num_haplotypes_ = dst;
        likelihoods_.resize(dst * w);
    }
    // merge_samples (:362-409): one sample holding the chosen samples' likelihoods back to back; the result is primed
    HaplotypeLikelihoodArray merge_samples(const std::vector<SampleName>& samples, const SampleName* new_sample = nullptr) const
    {
        SampleName name;
        if (new_sample) name = *new_sample; else for (const auto& s : samples) name += s;
        HaplotypeLikelihoodArray result = shared_.get() ? HaplotypeLikelihoodArray {config_, shared_} : HaplotypeLikelihoodArray {config_, engine_};
        result.model_ = model_;
        std::vector<std::size_t> idx;
        std::size_t total = 0;
        for (const auto& s : samples) { idx.push_back(sample_index(s)); total += width(idx.back()); }
        result.begin_samples(1);
        result.add_sample(name, total);
        result.num_haplotypes_ = num_haplotypes_;
        result.likelihoods_.resize(num_haplotypes_ * total);
        auto dst = result.likelihoods_.begin();
        for (std::size_t h = 0; h < num_haplotypes_; ++h) {
            for (const std::size_t s : idx) { const auto src = span(h, s); dst = std::copy(src.begin(), src.end(), dst); }
        }
        result.primed_ = 0;
        return result;
    }
    HaplotypeLikelihoodArray merge_samples(const SampleName* new_sample = nullptr) const { return merge_samples(samples_, new_sample); }

    const double* data() const noexcept { return likelihoods_.data(); }   // [haplotype][all samples' columns], row-major

private:
    Engine engine_;
    SharedEngine shared_ {nullptr};   // set: populate() goes through the batcher instead of engine_
    std::shared_ptr<const ErrorModel> model_;   // set: populate() takes sequences and runs the model's reset() on the GPU
    phmm_config config_;
    pinned_vector<double> likelihoods_;
    pinned_vector<std::int32_t> status_;
    std::vector<SampleName> samples_;
    std::vector<std::size_t> sample_off_ {0};
    std::size_t num_haplotypes_ = 0;
    mutable std::ptrdiff_t primed_ = -1;

    static phmm_config checked(const phmm_config& config)
    {
        if (config.max_indel_error > 256) throw TooLargeBandSizeError {static_cast<unsigned>(config.max_indel_error)};
        return config;
    }
    void begin_samples(std::size_t n) { samples_.clear(); samples_.reserve(n); sample_off_.assign(1, 0); unprime(); }
    void add_sample(const SampleName& name, std::size_t n) { samples_.push_back(name); sample_off_.push_back(sample_off_.back() + n); }
    std::size_t total_width() const noexcept { return sample_off_.back(); }
    std::size_t width(std::size_t s) const noexcept { return sample_off_[s + 1] - sample_off_[s]; }
    std::size_t sample_index(const SampleName& sample) const
    {
        for (std::size_t s = 0; s < samples_.size(); ++s) if (samples_[s] == sample) return s;
        throw std::out_of_range {"HaplotypeLikelihoodArray: unknown sample " + sample};   // the reference's unordered_map::at
    }
    std::size_t primed() const
    {
        if (primed_ < 0) throw std::logic_error {"HaplotypeLikelihoodArray: not primed"};   // an assert in the reference
        return static_cast<std::size_t>(primed_);
    }
    LikelihoodSpan span(std::size_t h, std::size_t s) const
    {
        if (h >= num_haplotypes_) throw std::out_of_range {"HaplotypeLikelihoodArray: haplotype index"};
        return LikelihoodSpan {likelihoods_.data() + h * total_width() + sample_off_[s], width(s)};
    }
    void run(const ReadBlock& reads, const pinned_vector<std::int64_t>* template_off, const HaplotypeBlock& haplotypes,
             const FlankState* flank_state, const phmm_positions* positions)
    {
        const auto hv = haplotypes.view();         // unused with an error model
        const auto rv = reads.view();
        num_haplotypes_ = haplotypes.size();
        likelihoods_.resize(num_haplotypes_ * total_width());        // every element is written by the call (no zero fill; the storage is page-locked and kept)
        if (num_haplotypes_ == 0 || reads.size() == 0) return;
        pinned_vector<std::int32_t>& status = status_;               // page-locked scratch kept across calls: allocating pinned memory costs milliseconds
        status.resize(num_haplotypes_ * reads.size());
        phmm_flank_state fs = detail::flank_state(flank_state);
        const auto n_templates = template_off ? static_cast<std::int32_t>(template_off->size() - 1) : 0;
        int rc;
        if (model_) {
            const auto sv = haplotypes.sequences_view();
            const phmm_error_model* m = model_->get();
            if (shared_.get()) {
                rc = template_off
                    ? phmm_batcher_populate_templates_reset(shared_.get(), &config_, m, &sv, &rv, template_off->data(), n_templates, &fs,
                                                            likelihoods_.data(), status.data())
                    : phmm_batcher_populate_reset(shared_.get(), &config_, m, &sv, &rv, positions, &fs, likelihoods_.data(), status.data());
            } else {
                rc = template_off
                    ? phmm_populate_templates_reset(engine_.get(), &config_, m, &sv, &rv, template_off->data(), n_templates, positions, &fs,
                                                    likelihoods_.data(), status.data(), PHMM_SPACE_HOST)
                    : phmm_populate_reset(engine_.get(), &config_, m, &sv, &rv, positions, &fs, likelihoods_.data(), status.data(), PHMM_SPACE_HOST);
            }
        } else if (shared_.get()) {
            rc = template_off
                ? phmm_batcher_populate_templates(shared_.get(), &config_, &hv, &rv, template_off->data(), n_templates, &fs, likelihoods_.data(), status.data())
                : phmm_batcher_populate(shared_.get(), &config_, &hv, &rv, positions, &fs, likelihoods_.data(), status.data());
        } else {
            rc = template_off
                ? phmm_populate_templates(engine_.get(), &config_, &hv, &rv, template_off->data(), n_templates, positions, &fs, likelihoods_.data(),
                                          status.data(), PHMM_SPACE_HOST)
                : phmm_populate(engine_.get(), &config_, &hv, &rv, positions, &fs, likelihoods_.data(), status.data(), PHMM_SPACE_HOST);
        }
        if (rc == PHMM_ERR_SHORT_HAPLOTYPE)
            detail::throw_first_short_haplotype(status.data(), status.size(), [&reads] (std::size_t i) { return i / reads.size(); });
        if (shared_.get()) shared_.check(rc); else engine_.check(rc);
    }
};

// ---------------------------------------------------------------------------------------------------------------------
// hmm::PairHMM<Parameters, BandSize, Score> (src/core/models/pairhmm/pair_hmm.hpp:892-1032) over the GPU kernel
// ---------------------------------------------------------------------------------------------------------------------
// The reference's class bundles a kernel object with a `const Parameters*` and forwards to the free templates hmm::evaluate /
// hmm::align. Those templates are the reference's own code, so this type exists only where its header has been included before
// this one (Octopus's build; tests/cpp/test_dropin.cpp): it differs from octopus::hmm::PairHMM in the kernel member alone, a
// GpuPairHMMDyn (runtime band).
// SubcloneModel / SomaticSubcloneModel::evaluate's inference (run_variational_bayes, variational_bayes_mixture_model.hpp:653-669;
// subclone_model.hpp:303) on the GPU, every seed in one phmm_variational_bayes call, in double. genotypes[g][k]: haplotype index of
// component k (the germline haplotypes first for SomaticSubcloneModel); every genotype has the same K (1 to 100). prior_alphas holds
// one K-vector per sample; seeds[i] is seed i's initial genotype log posteriors. The result is shaped like
// SubcloneModelBase::InferredLatents. Throws Error for input phmm_variational_bayes refuses.
struct VariationalBayesParameters { double epsilon = 0.05; unsigned max_iterations = 1000; };

struct VBLatents
{
    std::vector<double> genotype_probabilities;
    std::vector<double> genotype_log_probabilities;
    std::unordered_map<SampleName, std::vector<double>> alphas;
};

struct InferredLatents
{
    VBLatents max_evidence_params;
    std::vector<double> genotype_log_priors;
    std::vector<double> weighted_genotype_posteriors;
    double approx_log_evidence = 0.0;
};

namespace detail {

// The samples' columns of the matrix back to back, in the given sample order ([H][R]); off receives the S + 1 column offsets.
inline std::vector<double> sample_columns(const HaplotypeLikelihoodArray& likelihoods, const std::vector<SampleName>& samples,
                                          std::vector<std::int64_t>& off)
{
    const std::size_t H = likelihoods.num_haplotypes(), S = samples.size();
    off.assign(1, 0);
    for (const auto& s : samples) off.push_back(off.back() + static_cast<std::int64_t>(likelihoods.num_likelihoods(s)));
    const auto R = static_cast<std::size_t>(off.back());
    std::vector<double> lnl(H * R);
    for (std::size_t h = 0; h < H; ++h)
        for (std::size_t s = 0; s < S; ++s) {
            const auto span = likelihoods(samples[s], h);
            std::copy(span.begin(), span.end(), lnl.begin() + static_cast<std::ptrdiff_t>(h * R + static_cast<std::size_t>(off[s])));
        }
    return lnl;
}

} // namespace detail

inline InferredLatents run_variational_bayes(Engine& engine, const HaplotypeLikelihoodArray& likelihoods, const std::vector<SampleName>& samples,
                                             const std::vector<std::vector<std::int32_t>>& genotypes,
                                             const std::unordered_map<SampleName, std::vector<double>>& prior_alphas,
                                             std::vector<double> genotype_log_priors, const VariationalBayesParameters& params,
                                             const std::vector<std::vector<double>>& seeds)
{
    const std::size_t G = genotypes.size(), H = likelihoods.num_haplotypes(), S = samples.size();
    const std::size_t K = G ? genotypes.front().size() : 0;
    std::vector<std::int64_t> off;
    const auto lnl = detail::sample_columns(likelihoods, samples, off);
    const auto R = static_cast<std::size_t>(off.back());
    std::vector<std::int32_t> gt;
    gt.reserve(G * K);
    for (const auto& g : genotypes) {
        if (g.size() != K) throw Error {PHMM_ERR_INVALID, "genotypes of different sizes"};
        gt.insert(gt.end(), g.begin(), g.end());
    }
    std::vector<double> pa;
    pa.reserve(S * K);
    for (const auto& s : samples) {
        const auto& a = prior_alphas.at(s);
        if (a.size() != K) throw Error {PHMM_ERR_INVALID, "prior alphas of the wrong size"};
        pa.insert(pa.end(), a.begin(), a.end());
    }
    std::vector<double> sd;
    sd.reserve(seeds.size() * G);
    for (const auto& v : seeds) {
        if (v.size() != G) throw Error {PHMM_ERR_INVALID, "seed of the wrong size"};
        sd.insert(sd.end(), v.begin(), v.end());
    }
    if (genotype_log_priors.size() != G) throw Error {PHMM_ERR_INVALID, "genotype_log_priors of the wrong size"};
    InferredLatents r;
    r.max_evidence_params.genotype_probabilities.resize(G);
    r.max_evidence_params.genotype_log_probabilities.resize(G);
    r.weighted_genotype_posteriors.resize(G);
    std::vector<double> alphas(S * K);
    std::int32_t max_seed = 0;
    engine.check(phmm_variational_bayes(engine.get(), lnl.data(), static_cast<std::int32_t>(H), static_cast<std::int32_t>(R), off.data(),
                                        static_cast<std::int32_t>(S), gt.data(), static_cast<std::int32_t>(G), static_cast<std::int32_t>(K),
                                        pa.data(), genotype_log_priors.data(), sd.data(), static_cast<std::int32_t>(seeds.size()), params.epsilon,
                                        static_cast<std::int32_t>(std::min<unsigned>(params.max_iterations, 0x7fffffffu)),
                                        r.max_evidence_params.genotype_probabilities.data(), r.max_evidence_params.genotype_log_probabilities.data(),
                                        alphas.data(), r.weighted_genotype_posteriors.data(), &r.approx_log_evidence, &max_seed, nullptr, nullptr,
                                        PHMM_SPACE_HOST));
    for (std::size_t s = 0; s < S; ++s)
        r.max_evidence_params.alphas.emplace(samples[s], std::vector<double>(alphas.begin() + static_cast<std::ptrdiff_t>(s * K),
                                                                              alphas.begin() + static_cast<std::ptrdiff_t>((s + 1) * K)));
    r.genotype_log_priors = std::move(genotype_log_priors);
    return r;
}

// SingleCellModel::evaluate_model's inference (VariationalBayesMixtureMixtureModel::evaluate,
// variational_bayes_mixture_mixture_model.hpp:89-132) on the GPU, every seed in one phmm_variational_bayes_mixture_mixture call, in
// double. Where the reference takes a HaplotypeLikelihoodMatrix, the overloads take what make_likelihood_matrix
// (single_cell_model.cpp:824-851) reads: the likelihood array and its samples (the cells, in order), the genotypes as
// haplotype-index vectors, and the combinations as one genotype index per group. Every combination's genotype of group t has
// the same ploidy K_t (1 to 100, sum at most 100, at most 32 groups). The scalar overloads expand their concentrations as the
// reference's do (:61-126). A sample's group priors are its entry of GroupOptionalPriorArray; an empty vector means none (the
// reference's boost::none). The result is shaped like the reference's Inferences, without the component responsibilities, which
// no caller reads. Throws Error for input phmm_variational_bayes_mixture_mixture refuses.
class VariationalBayesMixtureMixtureModel
{
public:
    struct Options { double epsilon = 0.05; unsigned max_iterations = 1000; };

    using ProbabilityVector = std::vector<double>;
    using LogProbabilityVector = std::vector<double>;
    using GroupConcentrationVector = std::vector<double>;                      // one per group
    using ComponentConcentrationVector = std::vector<double>;                  // one per component of the group
    using MixtureConcentrationVector = std::vector<ComponentConcentrationVector>;   // one per group
    using MixtureConcentrationArray = std::vector<MixtureConcentrationVector>;      // one per sample
    using Sigma = std::vector<double>;                                         // one per group
    using GroupResponsibilityVector = std::vector<Sigma>;                      // one per sample
    using GroupOptionalPriorArray = std::vector<ProbabilityVector>;            // one per sample; empty: no priors
    using GenotypeVector = std::vector<std::vector<std::int32_t>>;              // haplotype indices of each genotype
    using GenotypeCombinationVector = std::vector<std::vector<std::size_t>>;    // a genotype index per group

    struct Latents
    {
        ProbabilityVector genotype_posteriors;
        LogProbabilityVector genotype_log_posteriors;
        GroupConcentrationVector group_concentrations;
        MixtureConcentrationArray mixture_concentrations;
        GroupResponsibilityVector group_responsibilities;
    };
    struct PointInferences { Latents latents; double approx_log_evidence = 0.0; };
    struct Inferences
    {
        PointInferences map;
        ProbabilityVector weighted_genotype_posteriors;
        GroupResponsibilityVector weighted_group_responsibilities;
    };

    VariationalBayesMixtureMixtureModel(Options options, Engine& engine) : options_ {options}, engine_ {&engine} {}

    Inferences evaluate(const LogProbabilityVector& genotype_log_priors, const HaplotypeLikelihoodArray& likelihoods,
                        const std::vector<SampleName>& samples, const GenotypeVector& genotypes,
                        const GenotypeCombinationVector& genotype_combinations, const GroupOptionalPriorArray& group_priors,
                        const GroupConcentrationVector& group_concentrations, const MixtureConcentrationArray& mixture_concentrations,
                        const std::vector<LogProbabilityVector>& seeds) const
    {
        return run(genotype_log_priors, likelihoods, samples, genotypes, genotype_combinations, group_priors, group_concentrations,
                   mixture_concentrations, seeds);
    }
    Inferences evaluate(const LogProbabilityVector& genotype_log_priors, const HaplotypeLikelihoodArray& likelihoods,
                        const std::vector<SampleName>& samples, const GenotypeVector& genotypes,
                        const GenotypeCombinationVector& genotype_combinations, const GroupConcentrationVector& group_concentrations,
                        const MixtureConcentrationArray& mixture_concentrations, const std::vector<LogProbabilityVector>& seeds) const
    {
        return run(genotype_log_priors, likelihoods, samples, genotypes, genotype_combinations, GroupOptionalPriorArray(samples.size()),
                   group_concentrations, mixture_concentrations, seeds);
    }
    Inferences evaluate(const LogProbabilityVector& genotype_log_priors, const HaplotypeLikelihoodArray& likelihoods,
                        const std::vector<SampleName>& samples, const GenotypeVector& genotypes,
                        const GenotypeCombinationVector& genotype_combinations, const GroupOptionalPriorArray& group_priors,
                        double group_concentration, const std::vector<double>& mixture_concentrations,
                        const std::vector<LogProbabilityVector>& seeds) const
    {
        const auto sizes = group_sizes(genotypes, genotype_combinations);
        if (mixture_concentrations.size() != samples.size()) throw Error {PHMM_ERR_INVALID, "one mixture concentration per sample"};
        MixtureConcentrationArray m;
        for (double c : mixture_concentrations) m.push_back(expand(sizes, c));
        return run(genotype_log_priors, likelihoods, samples, genotypes, genotype_combinations, group_priors,
                   GroupConcentrationVector(sizes.size(), group_concentration), m, seeds);
    }
    Inferences evaluate(const LogProbabilityVector& genotype_log_priors, const HaplotypeLikelihoodArray& likelihoods,
                        const std::vector<SampleName>& samples, const GenotypeVector& genotypes,
                        const GenotypeCombinationVector& genotype_combinations, double group_concentration,
                        const std::vector<double>& mixture_concentrations, const std::vector<LogProbabilityVector>& seeds) const
    {
        return evaluate(genotype_log_priors, likelihoods, samples, genotypes, genotype_combinations, GroupOptionalPriorArray(samples.size()),
                        group_concentration, mixture_concentrations, seeds);
    }
    Inferences evaluate(const LogProbabilityVector& genotype_log_priors, const HaplotypeLikelihoodArray& likelihoods,
                        const std::vector<SampleName>& samples, const GenotypeVector& genotypes,
                        const GenotypeCombinationVector& genotype_combinations, const GroupOptionalPriorArray& group_priors,
                        double group_concentration, double mixture_concentration, const std::vector<LogProbabilityVector>& seeds) const
    {
        const auto sizes = group_sizes(genotypes, genotype_combinations);
        return run(genotype_log_priors, likelihoods, samples, genotypes, genotype_combinations, group_priors,
                   GroupConcentrationVector(sizes.size(), group_concentration),
                   MixtureConcentrationArray(samples.size(), expand(sizes, mixture_concentration)), seeds);
    }
    Inferences evaluate(const LogProbabilityVector& genotype_log_priors, const HaplotypeLikelihoodArray& likelihoods,
                        const std::vector<SampleName>& samples, const GenotypeVector& genotypes,
                        const GenotypeCombinationVector& genotype_combinations, double group_concentration, double mixture_concentration,
                        const std::vector<LogProbabilityVector>& seeds) const
    {
        return evaluate(genotype_log_priors, likelihoods, samples, genotypes, genotype_combinations, GroupOptionalPriorArray(samples.size()),
                        group_concentration, mixture_concentration, seeds);
    }

private:
    Options options_;
    Engine* engine_;

    // K_t: the ploidy of group t's genotype, the same in every combination.
    static std::vector<std::int32_t> group_sizes(const GenotypeVector& genotypes, const GenotypeCombinationVector& combinations)
    {
        if (combinations.empty()) throw Error {PHMM_ERR_INVALID, "no genotype combinations"};
        std::vector<std::int32_t> sizes;
        for (const auto g : combinations.front()) sizes.push_back(static_cast<std::int32_t>(genotypes.at(g).size()));
        for (const auto& c : combinations) {
            if (c.size() != sizes.size()) throw Error {PHMM_ERR_INVALID, "combinations of different group counts"};
            for (std::size_t t = 0; t < c.size(); ++t)
                if (genotypes.at(c[t]).size() != static_cast<std::size_t>(sizes[t])) throw Error {PHMM_ERR_INVALID, "a group's genotypes differ in ploidy"};
        }
        return sizes;
    }
    static MixtureConcentrationVector expand(const std::vector<std::int32_t>& sizes, double c)
    {
        MixtureConcentrationVector r;
        for (const auto k : sizes) r.emplace_back(static_cast<std::size_t>(k), c);
        return r;
    }

    Inferences run(const LogProbabilityVector& genotype_log_priors, const HaplotypeLikelihoodArray& likelihoods,
                   const std::vector<SampleName>& samples, const GenotypeVector& genotypes,
                   const GenotypeCombinationVector& genotype_combinations, const GroupOptionalPriorArray& group_priors,
                   const GroupConcentrationVector& group_concentrations, const MixtureConcentrationArray& mixture_concentrations,
                   const std::vector<LogProbabilityVector>& seeds) const
    {
        const auto sizes = group_sizes(genotypes, genotype_combinations);
        const std::size_t C = genotype_combinations.size(), S = samples.size(), T = sizes.size(), H = likelihoods.num_haplotypes();
        std::size_t K = 0;
        for (const auto k : sizes) K += static_cast<std::size_t>(k);
        std::vector<std::int64_t> off;
        const auto lnl = detail::sample_columns(likelihoods, samples, off);
        std::vector<std::int32_t> gt;
        gt.reserve(C * K);
        for (const auto& c : genotype_combinations)
            for (const auto g : c) gt.insert(gt.end(), genotypes[g].begin(), genotypes[g].end());
        if (genotype_log_priors.size() != C) throw Error {PHMM_ERR_INVALID, "genotype_log_priors of the wrong size"};
        if (group_concentrations.size() != T) throw Error {PHMM_ERR_INVALID, "group concentrations of the wrong size"};
        if (group_priors.size() != S || mixture_concentrations.size() != S) throw Error {PHMM_ERR_INVALID, "one entry per sample expected"};
        std::vector<double> mc, gp(S * T, 0.0);
        std::vector<std::int32_t> mask(S, 0);
        bool any_prior = false;
        for (std::size_t s = 0; s < S; ++s) {
            if (mixture_concentrations[s].size() != T) throw Error {PHMM_ERR_INVALID, "mixture concentrations of the wrong shape"};
            for (std::size_t t = 0; t < T; ++t) {
                if (mixture_concentrations[s][t].size() != static_cast<std::size_t>(sizes[t])) throw Error {PHMM_ERR_INVALID, "mixture concentrations of the wrong shape"};
                mc.insert(mc.end(), mixture_concentrations[s][t].begin(), mixture_concentrations[s][t].end());
            }
            if (!group_priors[s].empty()) {
                if (group_priors[s].size() != T) throw Error {PHMM_ERR_INVALID, "group priors of the wrong size"};
                std::copy(group_priors[s].begin(), group_priors[s].end(), gp.begin() + static_cast<std::ptrdiff_t>(s * T));
                mask[s] = 1;
                any_prior = true;
            }
        }
        std::vector<double> sd;
        sd.reserve(seeds.size() * C);
        for (const auto& v : seeds) {
            if (v.size() != C) throw Error {PHMM_ERR_INVALID, "seed of the wrong size"};
            sd.insert(sd.end(), v.begin(), v.end());
        }
        Inferences r;
        auto& L = r.map.latents;
        L.genotype_posteriors.resize(C);
        L.genotype_log_posteriors.resize(C);
        L.group_concentrations.resize(T);
        r.weighted_genotype_posteriors.resize(C);
        std::vector<double> mco(S * K), sigma(S * T), wsigma(S * T);
        std::int32_t max_seed = 0;
        engine_->check(phmm_variational_bayes_mixture_mixture(
            engine_->get(), lnl.data(), static_cast<std::int32_t>(H), static_cast<std::int32_t>(off.back()), off.data(),
            static_cast<std::int32_t>(S), sizes.data(), static_cast<std::int32_t>(T), gt.data(), static_cast<std::int32_t>(C),
            genotype_log_priors.data(), any_prior ? gp.data() : nullptr, mask.data(), group_concentrations.data(), mc.data(), sd.data(),
            static_cast<std::int32_t>(seeds.size()), options_.epsilon, static_cast<std::int32_t>(std::min<unsigned>(options_.max_iterations, 0x7fffffffu)),
            L.genotype_posteriors.data(), L.genotype_log_posteriors.data(), L.group_concentrations.data(), mco.data(), sigma.data(),
            r.weighted_genotype_posteriors.data(), wsigma.data(), &r.map.approx_log_evidence, &max_seed, nullptr, nullptr, PHMM_SPACE_HOST));
        for (std::size_t s = 0; s < S; ++s) {
            L.mixture_concentrations.emplace_back();
            for (std::size_t t = 0, o = s * K; t < T; o += static_cast<std::size_t>(sizes[t]), ++t)
                L.mixture_concentrations.back().emplace_back(mco.begin() + static_cast<std::ptrdiff_t>(o),
                                                             mco.begin() + static_cast<std::ptrdiff_t>(o + static_cast<std::size_t>(sizes[t])));
            L.group_responsibilities.emplace_back(sigma.begin() + static_cast<std::ptrdiff_t>(s * T), sigma.begin() + static_cast<std::ptrdiff_t>((s + 1) * T));
            r.weighted_group_responsibilities.emplace_back(wsigma.begin() + static_cast<std::ptrdiff_t>(s * T), wsigma.begin() + static_cast<std::ptrdiff_t>((s + 1) * T));
        }
        return r;
    }
};

#ifdef pair_hmm_hpp   // the include guard of the reference's src/core/models/pairhmm/pair_hmm.hpp
template <typename Parameters, int BandSize = 0>
class PairHMM
{
public:
    using ParameterType = Parameters;
    PairHMM() = default;
    explicit PairHMM(unsigned min_band_size) { reset(min_band_size); }
    PairHMM(const Parameters& params, unsigned min_band_size = 8) { reset(min_band_size); set(params); }
    int band_size() const noexcept { return hmm_.band_size(); }
    void set(const Parameters& params) noexcept { params_ = std::addressof(params); }
    template <typename Sequence1, typename Sequence2>
    double evaluate(const Sequence1& target, const Sequence2& truth, const std::vector<std::uint8_t>& target_base_qualities, const std::size_t target_offset) const noexcept
    { return octopus::hmm::evaluate(truth, target, target_base_qualities, target_offset, hmm_, *params_); }
    template <typename Sequence1, typename Sequence2>
    void align(const Sequence1& target, const Sequence2& truth, const std::vector<std::uint8_t>& target_base_qualities, const std::size_t target_offset,
               octopus::hmm::Alignment& result) const
    { octopus::hmm::align(truth, target, target_base_qualities, target_offset, hmm_, *params_, result); }
    template <typename Sequence1, typename Sequence2>
    octopus::hmm::Alignment align(const Sequence1& target, const Sequence2& truth, const std::vector<std::uint8_t>& target_base_qualities, const std::size_t target_offset) const
    { octopus::hmm::Alignment result {}; this->align(target, truth, target_base_qualities, target_offset, result); return result; }
private:
    GpuPairHMMDyn hmm_ {BandSize > 0 ? static_cast<unsigned>(BandSize) : 8u};
    const Parameters* params_ = nullptr;
    void reset(unsigned min_band_size) { if (BandSize == 0) hmm_.reset(min_band_size); }
};
#endif

} // namespace octopus_b200

#endif
