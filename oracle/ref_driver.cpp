// TEST INFRASTRUCTURE ONLY — never linked into or called from the product path.
//
// extern "C" driver around the UNMODIFIED reference SIMD pair-HMM kernel. The reference sources are
// compiled from the octopus checkout named by REF (nothing is copied into this repo):
//   src/core/models/pairhmm/simd_pair_hmm_factory.hpp  (selector, :55-130)
//   src/core/models/pairhmm/simd_pair_hmm.hpp          (align_helper :240-324, flank replay :352-430)
//   src/core/models/pairhmm/{sse2,avx2,avx512}_pair_hmm_impl.hpp, rolling_initializer.hpp
// The Makefile builds this file three times (SSE4.1 / AVX2 / AVX-512 flags) into oracle/_ref/.
// The kernel chosen is the reference's own compile-time selection for those flags
// (simd_pair_hmm_factory.hpp:57-101), reported by ref_isa_name().
//
// Used by: tests/ (to pin the C restatement in phmm_oracle.c and to check the CUDA path) and by
// bench.py's cpu_baseline / --impl reference legs (kind "reference").

#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>
#include <algorithm>

#include "core/models/pairhmm/simd_pair_hmm_factory.hpp"

namespace {

using namespace octopus::hmm::simd;

struct AlignArgs
{
    const char* truth; const char* target; const std::int8_t* quals;
    int truth_len, target_len;
    const char* snv_mask; const std::int8_t* snv_prior;   // snv_mask == nullptr → no-SNV overloads
    const std::int8_t* gap_open;
    const std::int8_t* gap_extend; int gap_extend_scalar;   // gap_extend == nullptr → scalar overloads
    int nuc_prior;
};

template <typename HMM>
int do_align(const AlignArgs& a)
{
    const HMM hmm {};
    const auto nuc = static_cast<short>(a.nuc_prior);
    if (a.snv_mask) {
        if (a.gap_extend) return hmm.align(a.truth, a.target, a.quals, a.truth_len, a.target_len, a.snv_mask, a.snv_prior, a.gap_open, a.gap_extend, nuc);
        return hmm.align(a.truth, a.target, a.quals, a.truth_len, a.target_len, a.snv_mask, a.snv_prior, a.gap_open,
                         static_cast<typename HMM::ScoreType>(a.gap_extend_scalar), nuc);
    } else {
        if (a.gap_extend) return hmm.align(a.truth, a.target, a.quals, a.truth_len, a.target_len, a.gap_open, a.gap_extend, nuc);
        return hmm.align(a.truth, a.target, a.quals, a.truth_len, a.target_len, a.gap_open,
                         static_cast<typename HMM::ScoreType>(a.gap_extend_scalar), nuc);
    }
}

template <typename HMM>
int do_align_tb(const AlignArgs& a, int& first_pos, char* a1, char* a2)
{
    const HMM hmm {};
    const auto nuc = static_cast<short>(a.nuc_prior);
    if (a.snv_mask) {
        if (a.gap_extend) return hmm.align(a.truth, a.target, a.quals, a.truth_len, a.target_len, a.snv_mask, a.snv_prior, a.gap_open, a.gap_extend, nuc, first_pos, a1, a2);
        return hmm.align(a.truth, a.target, a.quals, a.truth_len, a.target_len, a.snv_mask, a.snv_prior, a.gap_open,
                         static_cast<typename HMM::ScoreType>(a.gap_extend_scalar), nuc, first_pos, a1, a2);
    } else {
        if (a.gap_extend) return hmm.align(a.truth, a.target, a.quals, a.truth_len, a.target_len, a.gap_open, a.gap_extend, nuc, first_pos, a1, a2);
        return hmm.align(a.truth, a.target, a.quals, a.truth_len, a.target_len, a.gap_open,
                         static_cast<typename HMM::ScoreType>(a.gap_extend_scalar), nuc, first_pos, a1, a2);
    }
}

template <typename HMM>
int do_flank(const AlignArgs& a, int lhs, int rhs, int first_pos, const char* a1, const char* a2, int& mask_size)
{
    const HMM hmm {};
    const auto nuc = static_cast<short>(a.nuc_prior);
    if (a.snv_mask) {
        if (a.gap_extend) return hmm.calculate_flank_score(a.truth_len, lhs, rhs, a.target, a.quals, a.snv_mask, a.snv_prior, a.gap_open, a.gap_extend, nuc, first_pos, a1, a2, mask_size);
        return hmm.calculate_flank_score(a.truth_len, lhs, rhs, a.target, a.quals, a.snv_mask, a.snv_prior, a.gap_open,
                                         static_cast<std::int8_t>(a.gap_extend_scalar), nuc, first_pos, a1, a2, mask_size);
    }
    // The no-SNV calculate_flank_score overloads (simd_pair_hmm.hpp:511-528) do not compile when instantiated
    // (they pass NullType where get_mismatch_quality expects const char*, :388) and are dead code in the
    // reference (flank sizes are NullType for the no-SNV models, pair_hmm.hpp:630-641).
    mask_size = 0;
    return -1000000;
}

struct BatchArgs
{
    long n;
    const char* read_bases; const std::int8_t* read_quals; const long* read_off;
    const char* hap_seq; const char* hap_mask; const std::int8_t* hap_prior;
    const std::int8_t* hap_gap_open; const std::int8_t* hap_gap_extend; const long* hap_off;
    const int* read_idx; const int* hap_idx; const int* win_off;
    int nuc_prior, nthreads; int* scores;
};

template <typename HMM>
int do_batch(const BatchArgs& b)
{
    constexpr int band = HMM::band_size();
    const auto work = [&b] (long lo, long hi) {
        const HMM hmm {};
        const auto nuc = static_cast<short>(b.nuc_prior);
        for (long j = lo; j < hi; ++j) {
            const long ro = b.read_off[b.read_idx[j]];
            const int L = static_cast<int>(b.read_off[b.read_idx[j] + 1] - ro);
            const long ho = b.hap_off[b.hap_idx[j]] + b.win_off[j];
            b.scores[j] = hmm.align(b.hap_seq + ho, b.read_bases + ro, b.read_quals + ro, L + 2 * band - 1, L,
                                    b.hap_mask + ho, b.hap_prior + ho, b.hap_gap_open + ho, b.hap_gap_extend + ho, nuc);
        }
    };
    const int nthreads = std::max(1, b.nthreads);
    if (nthreads == 1) { work(0, b.n); return 0; }
    std::vector<std::thread> pool;
    const long chunk = (b.n + nthreads - 1) / nthreads;
    for (int t = 0; t < nthreads; ++t) {
        const long lo = std::min<long>(b.n, t * chunk), hi = std::min<long>(b.n, lo + chunk);
        if (lo < hi) pool.emplace_back(work, lo, hi);
    }
    for (auto& th : pool) th.join();
    return 0;
}

// isa: 0 = the reference's own selection for these compile flags (SimdPairHMM), 1 = force SSE2 policy
#define REF_DISPATCH(CALL_T)                                                          \
    switch (band * 100 + bits + (isa == 1 ? 10000 : 0)) {                             \
        case   816: { using H = SimdPairHMM<8, short>;   CALL_T }                     \
        case   832: { using H = SimdPairHMM<8, int>;     CALL_T }                     \
        case  1616: { using H = SimdPairHMM<16, short>;  CALL_T }                     \
        case  1632: { using H = SimdPairHMM<16, int>;    CALL_T }                     \
        case  3216: { using H = SimdPairHMM<32, short>;  CALL_T }                     \
        case  3232: { using H = SimdPairHMM<32, int>;    CALL_T }                     \
        case  6416: { using H = SimdPairHMM<64, short>;  CALL_T }                     \
        case  6432: { using H = SimdPairHMM<64, int>;    CALL_T }                     \
        case 10816: { using H = SSE2PairHMM<8, short>;   CALL_T }                     \
        case 10832: { using H = SSE2PairHMM<8, int>;     CALL_T }                     \
        case 11616: { using H = SSE2PairHMM<16, short>;  CALL_T }                     \
        case 11632: { using H = SSE2PairHMM<16, int>;    CALL_T }                     \
        case 13216: { using H = SSE2PairHMM<32, short>;  CALL_T }                     \
        case 13232: { using H = SSE2PairHMM<32, int>;    CALL_T }                     \
        case 16416: { using H = SSE2PairHMM<64, short>;  CALL_T }                     \
        case 16432: { using H = SSE2PairHMM<64, int>;    CALL_T }                     \
        default: break;                                                               \
    }

} // namespace

extern "C" {

// Name of the instruction-set policy the reference selected ("SSE2", "AVX2", "AVX512"), or "" if unsupported.
const char* ref_isa_name(int band, int bits, int isa)
{
    REF_DISPATCH(return H::name();)
    return "";
}

// == reference hmm.align(...) score-only overloads (simd_pair_hmm.hpp:438-470). Returns -1000000 if (band,bits) unsupported.
int ref_align(int band, int bits, int isa,
              const char* truth, const char* target, const std::int8_t* quals, int truth_len, int target_len,
              const char* snv_mask, const std::int8_t* snv_prior,
              const std::int8_t* gap_open, const std::int8_t* gap_extend, int gap_extend_scalar, int nuc_prior)
{
    const AlignArgs a {truth, target, quals, truth_len, target_len, snv_mask, snv_prior, gap_open, gap_extend, gap_extend_scalar, nuc_prior};
    REF_DISPATCH(return do_align<H>(a);)
    return -1000000;
}

// == reference hmm.align(..., first_pos, align1, align2) traceback overloads (simd_pair_hmm.hpp:472-509).
// align1/align2: caller-allocated, >= 2*(target_len+band)+1 bytes, zero-filled.
int ref_align_tb(int band, int bits, int isa,
                 const char* truth, const char* target, const std::int8_t* quals, int truth_len, int target_len,
                 const char* snv_mask, const std::int8_t* snv_prior,
                 const std::int8_t* gap_open, const std::int8_t* gap_extend, int gap_extend_scalar, int nuc_prior,
                 int* first_pos, char* align1, char* align2)
{
    const AlignArgs a {truth, target, quals, truth_len, target_len, snv_mask, snv_prior, gap_open, gap_extend, gap_extend_scalar, nuc_prior};
    REF_DISPATCH(return do_align_tb<H>(a, *first_pos, align1, align2);)
    return -1000000;
}

// == reference hmm.calculate_flank_score(...) (simd_pair_hmm.hpp:511-549).
int ref_flank_score(int band, int bits, int isa, int truth_len, int lhs_flank, int rhs_flank,
                    const char* target, const std::int8_t* quals,
                    const char* snv_mask, const std::int8_t* snv_prior,
                    const std::int8_t* gap_open, const std::int8_t* gap_extend, int gap_extend_scalar, int nuc_prior,
                    int first_pos, const char* align1, const char* align2, int* target_mask_size)
{
    const AlignArgs a {nullptr, target, quals, truth_len, 0, snv_mask, snv_prior, gap_open, gap_extend, gap_extend_scalar, nuc_prior};
    REF_DISPATCH(return do_flank<H>(a, lhs_flank, rhs_flank, first_pos, align1, align2, *target_mask_size);)
    return -1000000;
}

// Batch form used for the CPU baseline: n independent alignments described as struct-of-arrays over
// packed reads / haplotypes (same packing the CUDA engine consumes, include/phmm_b200.h).
//   alignment j: read r = read_idx[j], haplotype h = hap_idx[j], window start a = win_off[j] (in hap coords)
//   truth = hap_seq + hap_off[h] + a, window length = L + 2*band - 1, SNV-mask overload, per-base gap arrays
//   (the overload HaplotypeLikelihoodModel uses: pair_hmm.hpp:387-407).
// The kernel type is dispatched once; the loop body is one direct hmm.align() call per alignment.
// Static split over nthreads std::threads. Writes the integer score of each alignment.
int ref_align_batch(int band, int bits, int isa, long n,
                    const char* read_bases, const std::int8_t* read_quals, const long* read_off,
                    const char* hap_seq, const char* hap_mask, const std::int8_t* hap_prior,
                    const std::int8_t* hap_gap_open, const std::int8_t* hap_gap_extend, const long* hap_off,
                    const int* read_idx, const int* hap_idx, const int* win_off,
                    int nuc_prior, int nthreads, int* scores)
{
    const BatchArgs b {n, read_bases, read_quals, read_off, hap_seq, hap_mask, hap_prior, hap_gap_open, hap_gap_extend,
                       hap_off, read_idx, hap_idx, win_off, nuc_prior, nthreads, scores};
    REF_DISPATCH(return do_batch<H>(b);)
    return -1;
}

} // extern "C"
