// HaplotypeLikelihoodModel::reset's arithmetic, written once for the host and the device: lib/tandem's exact tandem-repeat
// finder, the repeat-based indel model (gap_open / gap_extend) and the repeat-based SNV model (masks / priors per strand).
// Every function works in buffers its caller provides (no allocation), so phmm_reset_haplotypes and phmm_mutation_context
// run it on host threads and k_reset_haplotypes runs it on the GPU, one haplotype per thread — the same code on both sides.
//
// Reference (paths in the octopus source tree):
//   src/core/models/haplotype_likelihood_model.cpp:60-78            reset: which model fills which array; the no-SNV-model default
//   src/core/models/error/repeat_based_indel_error_model.cpp:67-83  per-base open / extend penalties from exact tandem repeats (period 1..5)
//   src/core/models/error/basic_repeat_based_indel_error_model.cpp:51-103   penalty lookup by motif period and repeat count
//   src/core/models/error/custom_repeat_based_indel_error_model.cpp:68-158  motif-keyed custom model
//   src/core/models/error/repeat_based_snv_error_model.cpp:48-179   run-length counting with gaps, per-strand prior caps, neighbour-base masks
//   lib/tandem/tandem.hpp:232-477, tandem.cpp:77-112                the repeat finder both models call: what it EMITS (which runs, which
//                                                                   period label, in which order) is procedural, not "all maximal runs"
//                                                                   (runs touching the end of the string are dropped, some sub-runs are
//                                                                   kept, period-5 runs are found from one side only), so the finder is
//                                                                   restated stage by stage: suffix array → LCP → longest-previous-factor
//                                                                   with previous occurrence → LZ factors → Main's per-factor repetitions
//                                                                   → Kolpakov-Kucherov propagation.
#pragma once

#include <cstddef>
#include <cstdint>

#include <string>
#include <vector>

#if defined(__CUDACC__)
#define RESET_HD __host__ __device__
#else
#define RESET_HD
#endif

namespace phmm_reset {

using Penalty = std::int8_t;
constexpr std::uint32_t kNone = 0xFFFFFFFFu;

struct Run { std::uint32_t pos, len, period; };

// Status of a core call: the run buffers of the scratch were too small (nothing is written past them; retry with a larger cap).
constexpr int kOk = 0;
constexpr int kOverflow = -1;
constexpr int kBadPeriods = -2;

template <typename T> RESET_HD inline T min_of(const T a, const T b) { return b < a ? b : a; }
template <typename T> RESET_HD inline T max_of(const T a, const T b) { return a < b ? b : a; }
template <typename T> RESET_HD inline void swap_of(T& a, T& b) { T t = a; a = b; b = t; }

// ---------------------------------------------------------------------------------------------------------
// The model, flattened: fixed-size rows and, for a custom model, its motif maps as sorted key arrays
// ---------------------------------------------------------------------------------------------------------

template <int N>
struct PaddedRow     // a parameter row copied into a fixed-size table, the tail filled with the row's last value (basic_…:16-20)
{
    Penalty v[N];
    RESET_HD void set(const signed char* src, const std::size_t count) { for (int i = 0; i < N; ++i) v[i] = src[(std::size_t)i < count ? i : count - 1]; }
    RESET_HD Penalty at(const std::uint32_t i) const { return v[i < (std::uint32_t)N ? i : N - 1]; }
};

// A custom model's motif key: the motif's length (1..5, the finder's periods) above its bytes, first byte highest. Motifs longer
// than 5 bytes are never looked up, so they need no key; the order of the keys is the order of the integers.
RESET_HD inline std::uint64_t motif_key(const unsigned char* motif, const std::uint32_t len)
{
    std::uint64_t k = len;
    for (std::uint32_t i = 0; i < len; ++i) k = (k << 8) | motif[i];
    return k << (8 * (5 - len));
}

struct MotifTable    // std::unordered_map<std::string, std::vector<Penalty>> restricted to keys of 1..5 bytes
{
    const std::uint64_t* key = nullptr;   // ascending
    const std::uint32_t* row = nullptr;   // key i's row: data[row[i] .. row[i + 1])
    const Penalty* data = nullptr;
    std::int32_t n = 0;

    RESET_HD std::int32_t find(const std::uint64_t k) const
    {
        std::int32_t lo = 0, hi = n;
        while (lo < hi) { const std::int32_t mid = (lo + hi) / 2; if (key[mid] < k) lo = mid + 1; else hi = mid; }
        return lo < n && key[lo] == k ? lo : -1;
    }
    RESET_HD Penalty lookup(const std::int32_t i, const std::uint32_t count) const   // row[count], or its last value
    {
        const std::uint32_t a = row[i], len = row[i + 1] - a;
        return data[a + (count < len ? count : len - 1)];
    }
};

struct Model
{
    // indel model
    bool custom = false;
    bool custom_has_extend = false;
    PaddedRow<50> open_at, open_cg, open_di, open_tri, ext_homo, ext_di, ext_tri;
    MotifTable custom_open, custom_extend;
    Penalty default_open = 0, default_extend = 0;
    // SNV model
    bool has_snv = false;
    PaddedRow<51> caps[3];

    // custom: the exact motif, then the wildcard N…N of the same period, then the default (custom_…:68-102)
    RESET_HD Penalty custom_penalty(const MotifTable& t, const unsigned char* motif, const std::uint32_t period, const std::uint32_t count, const Penalty fallback) const
    {
        std::int32_t i = t.find(motif_key(motif, period));
        if (i < 0) {
            const unsigned char ns[5] = {'N', 'N', 'N', 'N', 'N'};
            i = t.find(motif_key(ns, period));
            if (i < 0) return fallback;
        }
        return t.lookup(i, count);
    }
    RESET_HD Penalty open_penalty(const unsigned char* motif, const std::uint32_t period, const std::uint32_t len) const
    {
        const std::uint32_t count = len / period;
        if (custom) return custom_penalty(custom_open, motif, period, count, default_open);
        switch (period) {
            case 1: return (motif[0] == 'A' || motif[0] == 'T') ? open_at.at(count) : open_cg.at(count);
            case 2: {
                Penalty r = open_di.at(count);
                if (r > 7 && ((motif[0] == 'C' && motif[1] == 'G') || (motif[0] == 'G' && motif[1] == 'C'))) r = (Penalty)(r - 2);
                return r;
            }
            default: return open_tri.at(count);
        }
    }
    RESET_HD Penalty extend_penalty(const unsigned char* motif, const std::uint32_t period, const std::uint32_t len) const
    {
        const std::uint32_t count = len / period;
        if (custom) return custom_has_extend ? custom_penalty(custom_extend, motif, period, count, default_extend) : default_extend;
        return period == 1 ? ext_homo.at(count) : period == 2 ? ext_di.at(count) : ext_tri.at(count);
    }
};

// ---------------------------------------------------------------------------------------------------------
// std::sort as the reference build's libstdc++ runs it (introsort), restated: the indel model orders its runs by length with
// this unstable sort and then paints gap_extend in that order, so the order of equal-length runs is part of the output.
//   threshold 16; pivot = median of (first+1, middle, last-1) moved to first; unguarded partition of [first+1, last);
//   recurse on the right part, loop on the left; depth limit 2*floor(log2 n), then heap sort of the part;
//   final insertion sort: guarded over the first 16 elements, unguarded after them.
// ---------------------------------------------------------------------------------------------------------

namespace sort_detail {

constexpr std::ptrdiff_t kThreshold = 16;

template <typename T, typename Less>
RESET_HD void sift_up(T* first, std::ptrdiff_t hole, const std::ptrdiff_t top, T value, Less less)
{
    std::ptrdiff_t parent = (hole - 1) / 2;
    while (hole > top && less(first[parent], value)) { first[hole] = first[parent]; hole = parent; parent = (hole - 1) / 2; }
    first[hole] = value;
}

// moves the larger child up into the hole down to a leaf, then sifts value up from there
template <typename T, typename Less>
RESET_HD void adjust_heap(T* first, std::ptrdiff_t hole, const std::ptrdiff_t len, T value, Less less)
{
    const std::ptrdiff_t top = hole;
    std::ptrdiff_t child = hole;
    while (child < (len - 1) / 2) {
        child = 2 * (child + 1);
        if (less(first[child], first[child - 1])) --child;
        first[hole] = first[child];
        hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
        child = 2 * (child + 1);
        first[hole] = first[child - 1];
        hole = child - 1;
    }
    sift_up(first, hole, top, value, less);
}

template <typename T, typename Less>
RESET_HD void heap_sort(T* first, T* last, Less less)
{
    const std::ptrdiff_t len = last - first;
    if (len < 2) return;
    for (std::ptrdiff_t parent = (len - 2) / 2;; --parent) {      // make the heap
        adjust_heap(first, parent, len, first[parent], less);
        if (parent == 0) break;
    }
    while (last - first > 1) {                                      // pop the largest to the back, one at a time
        --last;
        const T value = *last;
        *last = *first;
        adjust_heap(first, (std::ptrdiff_t)0, last - first, value, less);
    }
}

template <typename T, typename Less>
RESET_HD void move_median_to_first(T* result, T* a, T* b, T* c, Less less)
{
    if (less(*a, *b)) {
        if (less(*b, *c)) swap_of(*result, *b);
        else if (less(*a, *c)) swap_of(*result, *c);
        else swap_of(*result, *a);
    } else if (less(*a, *c)) swap_of(*result, *a);
    else if (less(*b, *c)) swap_of(*result, *c);
    else swap_of(*result, *b);
}

template <typename T, typename Less>
RESET_HD T* unguarded_partition(T* first, T* last, const T* pivot, Less less)
{
    for (;;) {
        while (less(*first, *pivot)) ++first;
        --last;
        while (less(*pivot, *last)) --last;
        if (!(first < last)) return first;
        swap_of(*first, *last);
        ++first;
    }
}

template <typename T, typename Less>
RESET_HD void unguarded_linear_insert(T* last, Less less)
{
    const T value = *last;
    T* next = last - 1;
    while (less(value, *next)) { *last = *next; last = next; --next; }
    *last = value;
}

template <typename T, typename Less>
RESET_HD void insertion_sort(T* first, T* last, Less less)
{
    if (first == last) return;
    for (T* i = first + 1; i != last; ++i) {
        if (less(*i, *first)) {
            const T value = *i;
            for (T* k = i; k != first; --k) *k = *(k - 1);
            *first = value;
        } else unguarded_linear_insert(i, less);
    }
}

// The recursion on the right part becomes an explicit stack: one entry per partition level, at most the depth limit
// (2 floor(log2 n) <= 62 for the run counts of a haplotype) plus one.
template <typename T, typename Less>
RESET_HD void introsort_loop(T* first, T* last, int depth_limit, Less less, int* depth_exhausted)
{
    struct Part { T* first; T* last; int depth; };
    Part stack[64];
    int top = 0;
    stack[top++] = Part {first, last, depth_limit};
    while (top > 0) {
        Part p = stack[--top];
        while (p.last - p.first > kThreshold) {
            if (p.depth == 0) {
                heap_sort(p.first, p.last, less);
                if (depth_exhausted) ++*depth_exhausted;
                break;
            }
            --p.depth;
            T* mid = p.first + (p.last - p.first) / 2;
            move_median_to_first(p.first, p.first + 1, mid, p.last - 1, less);
            T* cut = unguarded_partition(p.first + 1, p.last, p.first, less);
            // the right part is sorted before the left one continues: push the left remainder under it
            stack[top++] = Part {p.first, cut, p.depth};
            p.first = cut;
        }
        // the right part (now p) is done; the left remainders are popped in order
    }
}

} // namespace sort_detail

// Sorts [first, last) into the permutation std::sort(first, last, less) gives with libstdc++. depth_exhausted (optional) counts
// the parts that reached the depth limit and were heap-sorted.
template <typename T, typename Less>
RESET_HD void introsort(T* first, T* last, Less less, int* depth_exhausted = nullptr)
{
    const std::ptrdiff_t n = last - first;
    if (n <= 0) return;
    int lg = 0;
    while (((std::ptrdiff_t)2 << lg) <= n) ++lg;                  // floor(log2 n)
    sort_detail::introsort_loop(first, last, 2 * lg, less, depth_exhausted);
    if (n > sort_detail::kThreshold) {
        sort_detail::insertion_sort(first, first + sort_detail::kThreshold, less);
        for (T* i = first + sort_detail::kThreshold; i != last; ++i) sort_detail::unguarded_linear_insert(i, less);
    } else sort_detail::insertion_sort(first, last, less);
}

// ---------------------------------------------------------------------------------------------------------
// Scratch of one haplotype
// ---------------------------------------------------------------------------------------------------------

// 32-bit words the LZ route needs for a string of n bases with run capacity cap (the SNV model needs fewer).
RESET_HD inline std::size_t scratch_words(const std::uint32_t n, const std::uint32_t cap)
{
    const std::size_t m = n;
    return 8 * m + max_of<std::size_t>(m, 256) + 8 + cap;
}

struct Scratch
{
    std::uint32_t* w;     // scratch_words(n, cap) words
    Run* runs;            // the finder's output: cap entries
    Run* main;            // Main's repetitions before propagation / a second scanned list: cap entries
    std::uint32_t cap;
};

// ---------------------------------------------------------------------------------------------------------
// String indexes
// ---------------------------------------------------------------------------------------------------------

// Suffix array by prefix doubling with counting sorts. Bytes compare unsigned and a suffix that is a prefix of another sorts first;
// the array is unique, so how it is built is free. On return rank[i] is the rank of suffix i (the inverse of sa).
// Words: sa, rank, tmp, sa2 (n each) and cnt (max(n, 256) + 1).
RESET_HD inline void build_suffix_array(const unsigned char* s, const std::uint32_t n, std::uint32_t* sa, std::uint32_t* rank,
                                       std::uint32_t* tmp, std::uint32_t* sa2, std::uint32_t* cnt)
{
    if (n == 1) { sa[0] = 0; rank[0] = 0; return; }
    std::uint32_t classes = 256;
    for (std::uint32_t c = 0; c <= classes; ++c) cnt[c] = 0;
    for (std::uint32_t i = 0; i < n; ++i) { rank[i] = s[i]; ++cnt[s[i] + 1]; }
    for (std::uint32_t c = 1; c <= classes; ++c) cnt[c] += cnt[c - 1];
    for (std::uint32_t i = 0; i < n; ++i) sa[cnt[rank[i]]++] = i;
    // compress the byte ranks to 0..classes-1
    tmp[sa[0]] = 0;
    for (std::uint32_t r = 1; r < n; ++r) tmp[sa[r]] = tmp[sa[r - 1]] + (rank[sa[r]] != rank[sa[r - 1]] ? 1u : 0u);
    classes = tmp[sa[n - 1]] + 1;
    for (std::uint32_t i = 0; i < n; ++i) rank[i] = tmp[i];
    for (std::uint32_t k = 1; classes < n; k <<= 1) {
        // order by the second key (rank[i + k], missing first), then a stable counting sort by the first key
        std::uint32_t m = 0;
        for (std::uint32_t i = n - k; i < n; ++i) sa2[m++] = i;
        for (std::uint32_t r = 0; r < n; ++r) if (sa[r] >= k) sa2[m++] = sa[r] - k;
        for (std::uint32_t c = 0; c <= classes; ++c) cnt[c] = 0;
        for (std::uint32_t i = 0; i < n; ++i) ++cnt[rank[i] + 1];
        for (std::uint32_t c = 1; c <= classes; ++c) cnt[c] += cnt[c - 1];
        for (std::uint32_t r = 0; r < n; ++r) { const std::uint32_t i = sa2[r]; sa[cnt[rank[i]]++] = i; }
        tmp[sa[0]] = 0;
        for (std::uint32_t r = 1; r < n; ++r) {
            const std::uint32_t a = sa[r - 1], b = sa[r];
            const bool same = rank[a] == rank[b] && (a + k < n ? rank[a + k] : kNone) == (b + k < n ? rank[b + k] : kNone);
            tmp[b] = tmp[a] + (same ? 0u : 1u);
        }
        classes = tmp[sa[n - 1]] + 1;
        for (std::uint32_t i = 0; i < n; ++i) rank[i] = tmp[i];
    }
}

// lcp[r] = longest common prefix of the suffixes ranked r-1 and r (lcp[0] = 0), Kasai's sweep (tandem.hpp:139-156)
RESET_HD inline void build_lcp(const unsigned char* s, const std::uint32_t n, const std::uint32_t* sa, const std::uint32_t* rank, std::uint32_t* lcp)
{
    for (std::uint32_t r = 0; r < n; ++r) lcp[r] = 0;
    std::uint32_t h = 0;
    for (std::uint32_t i = 0; i < n; ++i) {
        if (rank[i] == 0) continue;              // h carries over (it is only decremented after a comparison)
        const std::uint32_t j = sa[rank[i] - 1];
        while (i + h < n && j + h < n && s[i + h] == s[j + h]) ++h;
        lcp[rank[i]] = h;
        if (h > 0) --h;
    }
}

// Longest previous factor and one previous occurrence per text position (Crochemore & Ilie's stack sweep over the suffix
// array, tandem.cpp:77-112). Which previous occurrence is reported is a property of this sweep, and the reference runs it
// over arrays that carry one extra slot (a second entry for text position 0 with lcp 0 behind the last rank, tandem.hpp:96-104,
// 160-183) — reproduced here, since the propagation step copies runs from exactly that occurrence. lpf / prev_occ: n + 1 words,
// stack: 2 (n + 2) words.
RESET_HD inline void build_lpf(const std::uint32_t n, const std::uint32_t* sa, const std::uint32_t* lcp, std::uint32_t* lpf, std::uint32_t* prev_occ,
                              std::uint32_t* stack)
{
    auto order = [&](const std::uint32_t r) { return r < n ? sa[r] : r == n ? 0u : kNone; };   // the extra slot, then the terminator
    auto common = [&](const std::uint32_t r) { return r < n ? lcp[r] : 0u; };
    for (std::uint32_t i = 0; i <= n; ++i) { lpf[i] = 0; prev_occ[i] = 0; }
    std::uint32_t top = 0;                       // entries (common prefix with what lies below, text position) at stack[2k], stack[2k+1]
    stack[0] = 0u; stack[1] = order(0); top = 1;
    for (std::uint32_t r = 1; r <= n + 1; ++r) {
        std::uint32_t u = common(r);
        const std::uint32_t o = order(r);
        while (top > 0 && (o == kNone || o < stack[2 * (top - 1) + 1])) {
            const std::uint32_t first = stack[2 * (top - 1)], pos = stack[2 * (top - 1) + 1];
            --top;
            lpf[pos] = max_of(first, u);
            u = min_of(first, u);
            if (lpf[pos] == 0u) prev_occ[pos] = kNone;
            else if (first > u) prev_occ[pos] = stack[2 * (top - 1) + 1];   // the bottom entry always has first == 0: never popped here
            else prev_occ[pos] = o;
        }
        if (r < n + 1) { stack[2 * top] = u; stack[2 * top + 1] = o; ++top; }
    }
}

// ---------------------------------------------------------------------------------------------------------
// Exact tandem repeats, periods min_period..max_period > 3: lib/tandem's LZ route (tandem.hpp:232-392)
// ---------------------------------------------------------------------------------------------------------

// matches of s[a-k] against s[b-k], k = 0, 1, ... while a-k >= floor
RESET_HD inline std::uint32_t match_left(const unsigned char* s, std::uint32_t a, std::uint32_t b, const std::uint32_t floor)
{
    std::uint32_t k = 0;
    while (a - k >= floor && s[a - k] == s[b - k]) { ++k; if (a < k) break; }
    return k;
}
// matches of s[a+k] against s[b+k] while a+k < limit
RESET_HD inline std::uint32_t match_right(const unsigned char* s, const std::uint32_t a, const std::uint32_t b, const std::uint32_t limit)
{
    std::uint32_t k = 0;
    while (a + k < limit && s[a + k] == s[b + k]) ++k;
    return k;
}

// std::lower_bound's probe sequence over runs by end (pos + len < v), as the reference runs it
RESET_HD inline std::uint32_t lower_bound_end(const Run* first, std::uint32_t len, const std::uint32_t v)
{
    std::uint32_t at = 0;
    while (len > 0) {
        const std::uint32_t half = len >> 1;
        if (first[at + half].pos + first[at + half].len < v) { at += half + 1; len -= half + 1; }
        else len = half;
    }
    return at;
}

// Returns the number of runs in sc.runs, or kOverflow.
RESET_HD inline int tandem_repeats_lz(const unsigned char* s, const std::uint32_t n, const std::uint32_t min_period, const std::uint32_t max_period,
                                     const Scratch& sc)
{
    std::uint32_t* w = sc.w;
    const std::uint32_t cnt_words = max_of<std::uint32_t>(n, 256u) + 1;
    std::uint32_t* sa = w;                       // region A: the suffix array phase, reused by the factors and buckets below
    std::uint32_t* rank = sa + n;
    std::uint32_t* tmp = rank + n;
    std::uint32_t* sa2 = tmp + n;
    std::uint32_t* cnt = sa2 + n;
    std::uint32_t* lpf = cnt + cnt_words;
    std::uint32_t* prev_occ = lpf + n + 1;
    std::uint32_t* stack = prev_occ + n + 1;
    std::uint32_t* idx = stack + 2 * (n + 2);    // cap words
    build_suffix_array(s, n, sa, rank, tmp, sa2, cnt);
    std::uint32_t* lcp = tmp;
    build_lcp(s, n, sa, rank, lcp);
    build_lpf(n, sa, lcp, lpf, prev_occ, stack);

    // LZ factors and the start of each one's earlier occurrence (kNone: a new letter)
    std::uint32_t* fpos = w;
    std::uint32_t* flen = w + n;
    std::uint32_t* fsrc = w + 2 * n;
    std::uint32_t nf = 0;
    fpos[nf] = 0; flen[nf] = 1; fsrc[nf] = kNone; ++nf;
    for (std::uint32_t end = 1; end < n;) {
        const std::uint32_t m = max_of<std::uint32_t>(1u, lpf[end]);
        fpos[nf] = end; flen[nf] = m; fsrc[nf] = prev_occ[end]; ++nf;
        end += m;
    }

    // Main's step: repetitions that end inside factor h and reach back over the factor boundary (tandem.hpp:232-262), in the
    // order found; a run seen again with the same (pos, len) is dropped whatever its period label (:283-297, operator== :76-79).
    // A run of factor h ends inside factor h or on the last base of factor h - 1, so the duplicates to look for are among the
    // runs of these two factors.
    std::uint32_t nm = 0, previous_first = 0;
    for (std::uint32_t h = 1; h < nf; ++h) {
        const std::uint32_t u = fpos[h], fl = flen[h];
        const std::uint32_t reach = min_of(u, 2 * flen[h - 1] + fl), floor = u - reach, end = u + fl;
        const std::uint32_t look_from = previous_first;
        previous_first = nm;
        auto emit = [&](const std::uint32_t pos, const std::uint32_t len, const std::uint32_t period) {
            for (std::uint32_t k = look_from; k < nm; ++k) if (sc.main[k].pos == pos && sc.main[k].len == len) return true;
            if (nm == sc.cap) return false;
            sc.main[nm++] = Run {pos, len, period};
            return true;
        };
        for (std::uint32_t p = min_period; p <= min_of(fl, max_period); ++p) {              // period seed to the right of the boundary
            const std::uint32_t ls = match_left(s, u - 1, u + p - 1, floor), lp = match_right(s, u + p, u, end);
            if (ls + lp >= p && p + lp < fl && !emit(u - ls, p + lp + ls, p)) return kOverflow;
        }
        for (std::uint32_t p = min_period; p < min_of(reach, max_period); ++p) {            // seed to the left (strictly below max_period, :254)
            const std::uint32_t ls = match_left(s, u - p - 1, u - 1, floor), lp = match_right(s, u, u - p, end);
            if (ls + lp >= p && !emit(u - (ls + p), p + lp + ls, p)) return kOverflow;
        }
    }

    // by_pos (:306-320): Main's runs per start, by ascending end, equal ends in the order found — a counting sort by start of
    // the runs in the order found, then an insertion sort by end within each start (the buckets are a few runs long)
    std::uint32_t* bstart = fsrc + n;            // n + 1 words, still inside region A
    for (std::uint32_t p = 0; p <= n; ++p) bstart[p] = 0;
    for (std::uint32_t k = 0; k < nm; ++k) ++bstart[sc.main[k].pos + 1];
    for (std::uint32_t p = 1; p <= n; ++p) bstart[p] += bstart[p - 1];
    {
        std::uint32_t* fill = lpf;               // lpf is dead: n + 1 words
        for (std::uint32_t p = 0; p <= n; ++p) fill[p] = bstart[p];
        for (std::uint32_t k = 0; k < nm; ++k) idx[fill[sc.main[k].pos]++] = k;
    }
    for (std::uint32_t p = 0; p < n; ++p) {
        for (std::uint32_t a = bstart[p] + 1; a < bstart[p + 1]; ++a) {
            const std::uint32_t v = idx[a], e = sc.main[v].pos + sc.main[v].len;
            std::uint32_t b = a;
            while (b > bstart[p] && sc.main[idx[b - 1]].pos + sc.main[idx[b - 1]].len > e) { idx[b] = idx[b - 1]; --b; }
            idx[b] = v;
        }
    }

    // Kolpakov-Kucherov propagation: a factor repeats an earlier stretch of text, so the runs lying strictly inside that stretch
    // recur inside the factor; they are copied in front of what the factor's positions already hold (:323-365). Position j's list
    // is only changed while j is processed, and positions are processed in increasing order, so every list is final when it is
    // read as a source (src < j) and the lists can be written one after the other: ostart[j] .. ostart[j + 1] in sc.runs.
    std::uint32_t* ostart = lpf;                 // the fill cursors are dead
    std::uint32_t no = 0;
    for (std::uint32_t f = 0; f < nf; ++f) {
        const std::uint32_t fend = fpos[f] + flen[f];
        const std::uint32_t delta = fpos[f] - (fsrc[f] != kNone ? fsrc[f] : 0u);
        const std::uint32_t src_end_max = fend - delta;
        for (std::uint32_t j = fpos[f]; j < fend; ++j) {
            ostart[j] = no;
            const std::uint32_t own = bstart[j], own_n = bstart[j + 1] - bstart[j];
            if (j > 0) {                         // position 0 has nothing to copy (its source is itself)
                const std::uint32_t src = j - delta;
                std::uint32_t src_end = src_end_max;
                if (own_n > 0) src_end = min_of(src + sc.main[idx[own]].len, src_end_max);
                const Run* from = sc.runs + ostart[src];
                const std::uint32_t lo = lower_bound_end(from, ostart[src + 1] - ostart[src], src_end);
                if (no + lo > sc.cap) return kOverflow;
                for (std::uint32_t k = 0; k < lo; ++k) { Run r = from[k]; r.pos += delta; sc.runs[no++] = r; }
            }
            if (no + own_n > sc.cap) return kOverflow;
            for (std::uint32_t k = 0; k < own_n; ++k) sc.runs[no++] = sc.main[idx[own + k]];
            ostart[j + 1] = no;
        }
    }
    return (int)no;
}

// ---------------------------------------------------------------------------------------------------------
// Periods <= 3: lib/tandem's scanning route (tandem.hpp:394-500)
// ---------------------------------------------------------------------------------------------------------

// emit(Run) returns false to stop the scan (out of room); the scans then return false too.
template <typename Emit>
RESET_HD bool homopolymer_runs(const unsigned char* s, const std::uint32_t n, Emit emit)
{
    for (std::uint32_t i = 0; i + 1 < n;) {
        if (s[i] != s[i + 1]) { ++i; continue; }
        std::uint32_t j = i + 1;
        while (j < n && s[j] == s[i]) ++j;
        if (!emit(Run {i, j - i, 1u})) return false;
        i = j;
    }
    return true;
}

// Period-P repeats as the scanner reports them: a candidate starts only where two neighbouring bases differ; after a hit the
// scan resumes P bases before the hit's end, after a miss one base on (:416-444).
template <typename Emit>
RESET_HD bool scanned_repeats(const std::uint32_t P, const unsigned char* s, const std::uint32_t n, Emit emit)
{
    if (n < 2 * P) return true;
    auto next_change = [&](std::uint32_t i) { while (i + 1 < n && s[i] == s[i + 1]) ++i; return i + 1 < n ? i : n; };   // first i' >= i with s[i'] != s[i'+1]
    std::uint32_t a = next_change(0);
    if (a == n) return true;
    for (std::uint32_t b = a + P; b < n;) {
        std::uint32_t k = 0;
        while (b + k < n && s[b + k] == s[a + k]) ++k;
        if (k >= P) { if (!emit(Run {a, b + k - a, P})) return false; a = a + k; }
        else ++a;
        a = next_change(a);
        if (a == n) break;
        b = a + P;
    }
    return true;
}

template <typename Emit>
RESET_HD bool scanned_period(const std::uint32_t p, const unsigned char* s, const std::uint32_t n, Emit emit)
{
    return p == 1 ? homopolymer_runs(s, n, emit) : scanned_repeats(p, s, n, emit);
}

// Each period's list is merged into the runs so far as std::inplace_merge merges them: on equal pos the earlier list first.
RESET_HD inline int tandem_repeats_scan(const unsigned char* s, const std::uint32_t n, const std::uint32_t min_period, const std::uint32_t max_period,
                                       const Scratch& sc)
{
    std::uint32_t total = 0;
    for (std::uint32_t p = min_period; p <= max_period; ++p) {
        std::uint32_t ne = 0;
        const bool room = scanned_period(p, s, n, [&](const Run& r) { if (total + ne == sc.cap) return false; sc.main[ne++] = r; return true; });
        if (!room) return kOverflow;
        // backward merge into sc.runs[0, total + ne): the last of the merged list is the extra run unless the earlier one starts later
        std::uint32_t i = total, j = ne, out = total + ne;
        while (j > 0) {
            if (i > 0 && sc.runs[i - 1].pos > sc.main[j - 1].pos) sc.runs[--out] = sc.runs[--i];
            else sc.runs[--out] = sc.main[--j];
        }
        total += ne;
    }
    return (int)total;
}

// tandem::extract_exact_tandem_repeats (tandem.hpp:504-521): the number of runs in sc.runs, kOverflow or kBadPeriods
RESET_HD inline int tandem_repeats(const unsigned char* s, const std::uint32_t n, std::uint32_t min_period, const std::uint32_t max_period, const Scratch& sc)
{
    if (min_period == 0) ++min_period;
    if (n == 0 || n < min_period) return 0;
    if (min_period > max_period) return kBadPeriods;
    return max_period <= 3 ? tandem_repeats_scan(s, n, min_period, max_period, sc) : tandem_repeats_lz(s, n, min_period, max_period, sc);
}

// ---------------------------------------------------------------------------------------------------------
// The models
// ---------------------------------------------------------------------------------------------------------

// repeat_based_indel_error_model.cpp:67-83. kOk or kOverflow (open / extend then hold garbage).
RESET_HD inline int indel_penalties(const Model& m, const unsigned char* s, const std::uint32_t n, Penalty* open, Penalty* extend, const Scratch& sc)
{
    for (std::uint32_t i = 0; i < n; ++i) { open[i] = m.default_open; extend[i] = m.default_extend; }
    const int count = tandem_repeats(s, n, 1, 5, sc);
    if (count < 0) return count;
    // the reference orders the runs with std::sort (not stable): the same sort on the same sequence reproduces its order
    introsort(sc.runs, sc.runs + count, [](const Run& a, const Run& b) { return a.len < b.len; });
    for (int k = 0; k < count; ++k) {
        const Run r = sc.runs[k];
        const Penalty o = m.open_penalty(s + r.pos, r.period, r.len);
        for (std::uint32_t i = r.pos; i < r.pos + r.len; ++i) if (o < open[i]) open[i] = o;
        const Penalty e = m.extend_penalty(s + r.pos, r.period, r.len);
        for (std::uint32_t i = r.pos; i < r.pos + r.len; ++i) extend[i] = e;
    }
    return kOk;
}

// Length of the repeat run ENDING just before each position, reported where the run ends or is first interrupted; a run
// survives gaps of up to max_gap unmarked bases (repeat_based_snv_error_model.cpp:48-91; note the gap counter is not
// cleared when a different motif starts). get(i) reads the i-th mark of the sweep, put(i, v) takes its result.
template <typename Get, typename Put>
RESET_HD void count_runs(const std::uint32_t n, const unsigned max_gap, Get get, Put put)
{
    if (n == 0) return;
    std::int8_t prev = get(0);
    int count = prev > 0 ? 1 : 0;
    unsigned gap = 0;
    put(0, 0u);
    for (std::uint32_t i = 1; i < n; ++i) {
        const std::int8_t x = get(i);
        unsigned v = 0;
        if (x == 0) {
            ++gap;
            if (count > 0) { if (gap == 1) v = (unsigned)count; else if (gap > max_gap) count = 0; }
        } else if (prev == x) { gap = 0; ++count; }
        else { prev = x; v = (unsigned)count; count = 1; }
        put(i, v);
    }
}

RESET_HD inline std::int8_t base_mark(const unsigned char b) { return b == 'A' ? 1 : b == 'C' ? 2 : b == 'G' ? 3 : b == 'T' ? 4 : 5; }

// repeat_based_snv_error_model.cpp:144-179. marks: 3 n bytes of scratch. The finder's periods 1-3 are scanned one period at a
// time: each period paints its own mark array, so the merged order of the finder's output does not matter here.
RESET_HD inline void snv_arrays(const Model& m, const unsigned char* s, const std::uint32_t n, const std::uint8_t* is_substitution,
                               char* mask_f, Penalty* prior_f, char* mask_r, Penalty* prior_r, std::int8_t* marks)
{
    for (std::uint32_t k = 0; k < 3 * n; ++k) marks[k] = 0;
    for (std::uint32_t p = 1; p <= 3; ++p) {
        std::int8_t* mk = marks + (p - 1) * n;
        scanned_period(p, s, n, [&](const Run& r) {
            std::int8_t mark = 0;
            for (std::uint32_t k = 0; k < r.period; ++k) mark = (std::int8_t)(mark + base_mark(s[r.pos + k]));
            for (std::uint32_t k = r.pos; k < r.pos + r.len; ++k) mk[k] = mark;
            return true;
        });
    }
    const Penalty max_quality = m.caps[0].v[0];
    for (std::uint32_t k = 0; k < n; ++k) { prior_f[k] = max_quality; prior_r[k] = max_quality; }
    for (unsigned i = 0; i < 3; ++i) {
        const std::int8_t* mk = marks + i * n;
        const PaddedRow<51>& cap = m.caps[i];
        count_runs(n, i + 2, [&](std::uint32_t k) { return mk[k]; }, [&](std::uint32_t k, unsigned v) { prior_f[k] = min_of(cap.at(v), prior_f[k]); });
        count_runs(n, i + 2, [&](std::uint32_t k) { return mk[n - 1 - k]; },
                   [&](std::uint32_t k, unsigned v) { prior_r[n - 1 - k] = min_of(cap.at(v), prior_r[n - 1 - k]); });
    }
    if (is_substitution) for (std::uint32_t k = 0; k < n; ++k) if (is_substitution[k]) { prior_f[k] = max_quality; prior_r[k] = max_quality; }
    for (std::uint32_t k = 0; k < n; ++k) {          // the base before / after, cyclically (:174-178)
        mask_f[k] = (char)s[k == 0 ? n - 1 : k - 1];
        mask_r[k] = (char)s[k + 1 == n ? 0 : k + 1];
    }
}

// HaplotypeLikelihoodModel::reset for one haplotype (haplotype_likelihood_model.cpp:60-78): kOk or kOverflow (retry with a larger
// sc.cap; the outputs then hold garbage).
RESET_HD inline int reset_haplotype(const Model& m, const unsigned char* s, const std::uint32_t n, const std::uint8_t* is_substitution,
                                   char* mask_f, Penalty* prior_f, char* mask_r, Penalty* prior_r, Penalty* open, Penalty* extend, const Scratch& sc)
{
    if (m.has_snv) snv_arrays(m, s, n, is_substitution, mask_f, prior_f, mask_r, prior_r, reinterpret_cast<std::int8_t*>(sc.w));
    else {                                           // haplotype_likelihood_model.cpp:68-74
        for (std::uint32_t k = 0; k < n; ++k) { prior_f[k] = 100; prior_r[k] = 100; mask_f[k] = (char)s[k]; mask_r[k] = (char)s[k]; }
    }
    return indel_penalties(m, s, n, open, extend, sc);
}

// Run capacity of a first attempt: most haplotypes hold far fewer runs than bases.
RESET_HD inline std::uint32_t first_cap(const std::uint32_t n) { return n + 64; }

} // namespace phmm_reset

// ---------------------------------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------------------------------
struct phmm_error_model;
namespace phmm_reset {
// The flattened model of a phmm_error_model (its arrays live as long as the model). Defined in phmm_error_model.cpp.
const Model& model_of(const phmm_error_model* m);
// The model's content as bytes: models with equal keys give equal arrays for every sequence, so the request batcher merges their
// requests. Empty when the model holds a penalty outside [0,127] (populate refuses such arrays): those requests run alone.
const std::string& model_key(const phmm_error_model* m);
// Host scratch that grows on demand: a haplotype whose runs overflow is recomputed with twice the capacity.
struct HostScratch
{
    std::vector<std::uint32_t> w;
    std::vector<Run> runs;
    Scratch get(const std::uint32_t n, const std::uint32_t cap)
    {
        w.resize(scratch_words(n, cap));
        runs.resize(2 * (std::size_t)cap);
        return Scratch {w.data(), runs.data(), runs.data() + cap, cap};
    }
};
// reset_haplotype with the retry; kOk.
inline int reset_haplotype_host(const Model& m, const unsigned char* s, const std::uint32_t n, const std::uint8_t* is_substitution,
                                char* mask_f, Penalty* prior_f, char* mask_r, Penalty* prior_r, Penalty* open, Penalty* extend, HostScratch& hs)
{
    for (std::uint32_t cap = first_cap(n);; cap *= 2) {
        const int rc = reset_haplotype(m, s, n, is_substitution, mask_f, prior_f, mask_r, prior_r, open, extend, hs.get(n, cap));
        if (rc != kOverflow) return rc;
    }
}
// tandem_repeats with the retry: the runs in out; kOk or kBadPeriods.
inline int tandem_repeats_host(const unsigned char* s, const std::uint32_t n, const std::uint32_t min_period, const std::uint32_t max_period,
                               HostScratch& hs, std::vector<Run>& out)
{
    for (std::uint32_t cap = first_cap(n);; cap *= 2) {
        const Scratch sc = hs.get(n, cap);
        const int count = tandem_repeats(s, n, min_period, max_period, sc);
        if (count == kOverflow) continue;
        if (count < 0) return count;
        out.assign(sc.runs, sc.runs + count);
        return kOk;
    }
}
} // namespace phmm_reset
