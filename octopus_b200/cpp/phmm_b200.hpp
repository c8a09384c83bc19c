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

    // ReadRealigner::realign's per-read step for every pair (phmm_realign_reads). Statuses as phmm_align_reads (PHMM_STATUS_*;
    // SHORT_HAP carries the required extension in the high 16 bits); host memory.
    struct PairAlignments
    {
        std::vector<std::int64_t> mapping_position;
        std::vector<double> likelihood;
        std::vector<std::string> cigar;
        std::vector<std::int32_t> status;
    };
    PairAlignments realign_reads(const phmm_config& config, const phmm_haplotypes& haplotypes, const phmm_reads& reads,
                                 const std::vector<phmm_pair>& pairs, const phmm_flank_state* flank_state = nullptr) const
    {
        const std::size_t n = pairs.size();
        std::int64_t longest = 1;
        for (std::int32_t r = 0; r < reads.n; ++r) longest = std::max<std::int64_t>(longest, reads.off[r + 1] - reads.off[r]);
        const auto stride = static_cast<std::int32_t>(4 * longest + 64);
        PairAlignments a;
        a.mapping_position.resize(n); a.likelihood.resize(n); a.status.resize(n);
        std::vector<char> text(std::max<std::size_t>(n, 1) * static_cast<std::size_t>(stride), 0);
        check(phmm_realign_reads(get(), &config, &haplotypes, &reads, pairs.data(), static_cast<std::int64_t>(n), flank_state,
                                 a.mapping_position.data(), a.likelihood.data(), text.data(), stride, a.status.data(), PHMM_SPACE_HOST));
        a.cigar.reserve(n);
        for (std::size_t j = 0; j < n; ++j) a.cigar.emplace_back(text.data() + j * static_cast<std::size_t>(stride));
        return a;
    }

    // compute_haplotype_support's scoring and choice for many genotypes (phmm_assign_reads); host memory. top[r] bit k = group-local
    // haplotype k is in read r's find_map_haplotypes set. likelihood / status: the groups' [H_g][R_g] matrices back to back. A short
    // haplotype does not throw here: the return code is PHMM_ERR_SHORT_HAPLOTYPE and the statuses carry the extension.
    struct ReadAssignment
    {
        std::vector<std::uint64_t> top;
        std::vector<double> likelihood;
        std::vector<std::int32_t> status;
        int code = PHMM_OK;
    };
    ReadAssignment assign_reads(const phmm_config& config, const phmm_haplotypes& haplotypes, const phmm_reads& reads,
                                const std::vector<std::int32_t>& hap_first, const std::vector<std::int32_t>& read_first,
                                const std::vector<double>* log_priors = nullptr, bool want_likelihoods = false) const
    {
        if (hap_first.empty() || hap_first.size() != read_first.size()) throw Error {PHMM_ERR_INVALID, "group bounds need n + 1 entries each"};
        const auto n = static_cast<std::int32_t>(hap_first.size() - 1);
        if (log_priors && log_priors->size() != static_cast<std::size_t>(haplotypes.n)) throw Error {PHMM_ERR_INVALID, "one log prior per haplotype"};
        std::size_t pairs = 0;
        for (std::int32_t g = 0; g < n; ++g)
            pairs += static_cast<std::size_t>(std::max(0, hap_first[g + 1] - hap_first[g])) * static_cast<std::size_t>(std::max(0, read_first[g + 1] - read_first[g]));
        const phmm_regions groups {n, hap_first.data(), read_first.data(), nullptr};
        ReadAssignment a;
        a.top.resize(static_cast<std::size_t>(std::max(0, reads.n)));
        a.status.resize(pairs);
        if (want_likelihoods) a.likelihood.resize(pairs);
        a.code = phmm_assign_reads(get(), &config, &haplotypes, &reads, &groups, log_priors ? log_priors->data() : nullptr, a.top.data(),
                                   want_likelihoods ? a.likelihood.data() : nullptr, a.status.data(), PHMM_SPACE_HOST);
        if (a.code != PHMM_ERR_SHORT_HAPLOTYPE) check(a.code);
        return a;
    }
private:
    std::shared_ptr<phmm_engine> handle_;
};

// One engine for a whole process's threads (phmm_batcher): the populate calls that concurrent threads have in flight run as one
// multi-region kernel chain, each with the result it would get on an Engine of its own. Copies share the batcher; every thread
// may call it at once. clients: the number of threads that submit (Octopus's --threads); a batch is sent once that many wait,
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
template <int BandSize>
class GpuPairHMM
{
public:
    using ScoreType = int;
    constexpr static char gap_label = '-';

    explicit GpuPairHMM(Engine engine = Engine {}) : engine_ {std::move(engine)} {}

    constexpr static const char* name() noexcept { return "H100"; }
    constexpr static int band_size() noexcept { return BandSize; }

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

private:
    Engine engine_;

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
        if (!align1) { a1.assign(2 * (target_len + BandSize) + 1, 0); a2 = a1; align1 = a1.data(); align2 = a2.data(); }
        const int rc = phmm_align_traceback(engine_.get(), BandSize, truth, target, quals, truth_len, target_len, snv_mask, snv_prior,
                                            gap_open, ext_ptr(gap_extend), ext_scalar(gap_extend), nuc_prior, &score, &first_pos, align1, align2);
        if (rc != PHMM_OK) first_pos = -1;   // the reference signals failure through first_pos (simd_pair_hmm.hpp:176-199)
        return score;
    }
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

// One read's result of ReadRealigner::realign (read_realigner.cpp:92-103, 128-130): HaplotypeLikelihoodModel::Alignment.
struct Realignment
{
    std::int64_t mapping_position;
    std::string cigar;
    double likelihood;
};

// realign(reads, haplotype, model) (read_realigner.cpp:105-144) for haplotype `haplotype` of the block: every read mapped with the
// uncapped k-mer mapper and aligned there, on the GPU. When a read's haplotype is too short, throws ShortHaplotypeError for the first
// such read in read order — the reference's serial loop, whose required extension safe_realign (:196-207) applies.
inline std::vector<Realignment> realign(const ReadBlock& reads, const HaplotypeBlock& haplotypes, std::size_t haplotype,
                                        const phmm_config& config, const Engine& engine = Engine {}, const FlankState* flank_state = nullptr)
{
    std::vector<phmm_pair> pairs(reads.size());
    for (std::size_t r = 0; r < reads.size(); ++r) pairs[r] = phmm_pair {static_cast<std::int32_t>(r), static_cast<std::int32_t>(haplotype)};
    const phmm_flank_state fs {flank_state ? 1 : 0, flank_state ? flank_state->lhs_flank : 0, flank_state ? flank_state->rhs_flank : 0};
    const auto a = engine.realign_reads(config, haplotypes.view(), reads.view(), pairs, &fs);
    std::vector<Realignment> result;
    result.reserve(pairs.size());
    for (std::size_t r = 0; r < pairs.size(); ++r) {
        const int code = a.status[r] & 0xFFFF;
        if (code == PHMM_STATUS_SHORT_HAP) throw ShortHaplotypeError {haplotype, static_cast<unsigned>(static_cast<std::uint32_t>(a.status[r]) >> 16)};
        if (code == PHMM_STATUS_HMM_OVERFLOW) throw Error {PHMM_ERR_INVALID, "HMMOverflow"};
        if (code == PHMM_STATUS_CIGAR_TRUNCATED) throw Error {PHMM_ERR_INVALID, "CIGAR truncated"};
        result.push_back(Realignment {a.mapping_position[r], a.cigar[r], a.likelihood[r]});
    }
    return result;
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

// compute_haplotype_support (core/tools/read_assigner.cpp:322-459) for many genotypes in one GPU call: group g (one genotype, after the
// caller's collapse) owns haplotypes [hap_first[g], hap_first[g+1]) and reads [read_first[g], read_first[g+1]). log_priors: one per
// haplotype of the block, or null. When a haplotype is too short, throws ShortHaplotypeError for the first short (haplotype, read)
// pair in the reference's order (groups in turn, haplotypes in genotype order, then reads), with the block's haplotype index.
inline std::vector<HaplotypeSupport> compute_haplotype_support(const ReadBlock& reads, const HaplotypeBlock& haplotypes,
                                                               const std::vector<std::int32_t>& hap_first, const std::vector<std::int32_t>& read_first,
                                                               const std::vector<double>* log_priors, AmbiguousAction action,
                                                               const phmm_config& config, const Engine& engine = Engine {})
{
    const auto a = engine.assign_reads(config, haplotypes.view(), reads.view(), hap_first, read_first, log_priors);
    std::vector<HaplotypeSupport> result(hap_first.size() - 1);
    std::size_t slot = 0;
    for (std::size_t g = 0; g + 1 < hap_first.size(); ++g) {
        const auto nh = static_cast<std::size_t>(hap_first[g + 1] - hap_first[g]), nr = static_cast<std::size_t>(read_first[g + 1] - read_first[g]);
        if (a.code == PHMM_ERR_SHORT_HAPLOTYPE) {
            for (std::size_t i = 0; i < nh * nr; ++i) {
                if ((a.status[slot + i] & 0xFFFF) == PHMM_STATUS_SHORT_HAP)
                    throw ShortHaplotypeError {hap_first[g] + i / nr, static_cast<unsigned>(static_cast<std::uint32_t>(a.status[slot + i]) >> 16)};
            }
            slot += nh * nr;
            continue;
        }
        HaplotypeSupport& s = result[g];
        s.reads.resize(nh);
        for (std::size_t i = 0; i < nr; ++i) {
            const std::size_t r = static_cast<std::size_t>(read_first[g]) + i;
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
    if (a.code == PHMM_ERR_SHORT_HAPLOTYPE) throw Error {a.code, "Haplotype is too short for alignment"};
    return result;
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
    : params_ {parameters}, engine_ {&engine}, approx_ {std::move(approx)}
    {
        phmm_mutation_model* m = nullptr;
        const int rc = phmm_mutation_model_create(&m, parameters.snv_prior, table.open.data(), table.extend.data(), table.max_period,
                                                  table.max_periodicity, table.max_indel_length);
        if (rc != PHMM_OK) throw Error {rc, phmm_error_model_last_error()};
        model_.reset(m, [] (phmm_mutation_model* p) { phmm_mutation_model_destroy(p); });
    }
#ifdef indel_mutation_model_config_hpp
    DeNovoModel(Parameters parameters, Engine& engine, ApproxFunction approx = nullptr)
    : DeNovoModel {parameters, MutationRepeatTable::from_reference(parameters.indel_prior), engine, std::move(approx)} {}
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
        if (n > 0) engine_->check(phmm_mutation_prime(engine_->get(), model_.get(), static_cast<std::int32_t>(n), off.data(), seq.data(),
                                                      values_.data(), status_.data()));
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
    Parameters params_;
    Engine* engine_;
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

    explicit HaplotypeLikelihoodArray(phmm_config config, Engine engine = Engine {}) : engine_ {std::move(engine)}, config_ {config}
    {
        if (config.max_indel_error > 256) throw TooLargeBandSizeError {static_cast<unsigned>(config.max_indel_error)};
    }
    // populate() goes through a process-wide SharedEngine: any number of threads, each with its own array, share one GPU engine
    HaplotypeLikelihoodArray(phmm_config config, SharedEngine shared) : engine_ {nullptr}, shared_ {std::move(shared)}, config_ {config}
    {
        if (config.max_indel_error > 256) throw TooLargeBandSizeError {static_cast<unsigned>(config.max_indel_error)};
    }
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
    phmm_config config_;
    pinned_vector<double> likelihoods_;
    pinned_vector<std::int32_t> status_;
    std::vector<SampleName> samples_;
    std::vector<std::size_t> sample_off_ {0};
    std::size_t num_haplotypes_ = 0;
    mutable std::ptrdiff_t primed_ = -1;

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
        const auto hv = haplotypes.view();
        const auto rv = reads.view();
        num_haplotypes_ = haplotypes.size();
        likelihoods_.resize(num_haplotypes_ * total_width());        // every element is written by the call (no zero fill; the storage is page-locked and kept)
        if (num_haplotypes_ == 0 || reads.size() == 0) return;
        pinned_vector<std::int32_t>& status = status_;               // page-locked scratch kept across calls: allocating pinned memory costs milliseconds
        status.resize(num_haplotypes_ * reads.size());
        phmm_flank_state fs {flank_state ? 1 : 0, flank_state ? flank_state->lhs_flank : 0, flank_state ? flank_state->rhs_flank : 0};
        const auto n_templates = template_off ? static_cast<std::int32_t>(template_off->size() - 1) : 0;
        int rc;
        if (shared_.get()) {
            rc = template_off
                ? phmm_batcher_populate_templates(shared_.get(), &config_, &hv, &rv, template_off->data(), n_templates, &fs, likelihoods_.data(), status.data())
                : phmm_batcher_populate(shared_.get(), &config_, &hv, &rv, positions, &fs, likelihoods_.data(), status.data());
        } else {
            rc = template_off
                ? phmm_populate_templates(engine_.get(), &config_, &hv, &rv, template_off->data(), n_templates, positions, &fs, likelihoods_.data(),
                                          status.data(), PHMM_SPACE_HOST)
                : phmm_populate(engine_.get(), &config_, &hv, &rv, positions, &fs, likelihoods_.data(), status.data(), PHMM_SPACE_HOST);
        }
        if (rc == PHMM_ERR_SHORT_HAPLOTYPE) {
            for (std::size_t i = 0; i < status.size(); ++i) {
                if ((status[i] & 0xFFFF) == PHMM_STATUS_SHORT_HAP) throw ShortHaplotypeError {i / reads.size(), static_cast<unsigned>(static_cast<std::uint32_t>(status[i]) >> 16)};
            }
        }
        if (shared_.get()) shared_.check(rc); else engine_.check(rc);
    }
};

// ---------------------------------------------------------------------------------------------------------------------
// hmm::PairHMM<Parameters, BandSize, Score> (src/core/models/pairhmm/pair_hmm.hpp:892-1032) over the GPU kernel
// ---------------------------------------------------------------------------------------------------------------------
// The reference's class bundles a kernel object with a `const Parameters*` and forwards to the free templates hmm::evaluate /
// hmm::align. Those templates are the reference's own code, so this type exists only where its header has been included before
// this one (Octopus's build; tests/cpp/test_dropin.cpp): it differs from octopus::hmm::PairHMM in the kernel member alone.
// The kernel is GpuPairHMM with a RUNTIME band, like simd::PairHMMWrapper (simd_pair_hmm_wrapper.hpp:218-241: smallest of
// 8, 16, ..., 256 that holds the request; TooLargeBandSizeError beyond).
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
    template <typename GapExtend>
    int align(const char* truth, const char* target, const std::int8_t* qualities, int truth_len, int target_len,
              const std::int8_t* gap_open, GapExtend gap_extend, short nuc_prior) const noexcept
    { int fp; return run(truth, target, qualities, truth_len, target_len, nullptr, nullptr, gap_open, gap_extend, nuc_prior, fp, nullptr, nullptr); }
    template <typename GapExtend>
    int align(const char* truth, const char* target, const std::int8_t* qualities, int truth_len, int target_len,
              const char* snv_mask, const std::int8_t* snv_prior, const std::int8_t* gap_open, GapExtend gap_extend, short nuc_prior) const noexcept
    { int fp; return run(truth, target, qualities, truth_len, target_len, snv_mask, snv_prior, gap_open, gap_extend, nuc_prior, fp, nullptr, nullptr); }
    template <typename GapExtend>
    int align(const char* truth, const char* target, const std::int8_t* qualities, int truth_len, int target_len,
              const std::int8_t* gap_open, GapExtend gap_extend, short nuc_prior, int& first_pos, char* align1, char* align2) const noexcept
    { return run(truth, target, qualities, truth_len, target_len, nullptr, nullptr, gap_open, gap_extend, nuc_prior, first_pos, align1, align2); }
    template <typename GapExtend>
    int align(const char* truth, const char* target, const std::int8_t* qualities, int truth_len, int target_len,
              const char* snv_mask, const std::int8_t* snv_prior, const std::int8_t* gap_open, GapExtend gap_extend, short nuc_prior,
              int& first_pos, char* align1, char* align2) const noexcept
    { return run(truth, target, qualities, truth_len, target_len, snv_mask, snv_prior, gap_open, gap_extend, nuc_prior, first_pos, align1, align2); }
    template <typename... Args>
    int calculate_flank_score(Args&&... args) const noexcept { return GpuPairHMM<8> {engine_}.calculate_flank_score(std::forward<Args>(args)...); }   // band-independent replay
private:
    Engine engine_;
    int band_ = 8;
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
        if (rc != PHMM_OK) first_pos = -1;
        return score;
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
