// HaplotypeLikelihoodModel::reset for the H100 pair-HMM engine: the per-haplotype penalty arrays the kernels consume
// (SNV mask / prior per strand, gap_open[], gap_extend[]) from the haplotype sequence alone. Host C++, one haplotype per
// task, bit-identical to the reference's error models so that the engine can be fed from sequences directly.
//
// Reference (paths in the octopus source tree):
//   src/core/models/haplotype_likelihood_model.cpp:60-78            reset: which model fills which array; the no-SNV-model default
//   src/core/models/error/repeat_based_indel_error_model.cpp:67-83  per-base open / extend penalties from exact tandem repeats (period 1..5)
//   src/core/models/error/basic_repeat_based_indel_error_model.cpp:51-103   penalty lookup by motif period and repeat count
//   src/core/models/error/custom_repeat_based_indel_error_model.cpp:68-158  motif-keyed custom model + its text format
//   src/core/models/error/repeat_based_snv_error_model.cpp:48-179   run-length counting with gaps, per-strand prior caps, neighbour-base masks
//   src/core/models/error/error_model_factory.cpp:220-589           built-in parameters (generated table include), label parsing
//   lib/tandem/tandem.hpp:232-477, tandem.cpp:77-112                the repeat finder both models call: what it EMITS (which runs, which
//                                                                   period label, in which order) is procedural, not "all maximal runs"
//                                                                   (runs touching the end of the string are dropped, some sub-runs are
//                                                                   kept, period-5 runs are found from one side only), so the finder is
//                                                                   restated stage by stage: suffix array → LCP → longest-previous-factor
//                                                                   with previous occurrence → LZ factors → Main's per-factor repetitions
//                                                                   → Kolpakov-Kucherov propagation.
#include "../../include/phmm_b200.h"
#include "phmm_mutation.h"

#include <algorithm>
#include <atomic>
#include <cctype>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <thread>
#include <unordered_map>
#include <utility>
#include <vector>

namespace {

#include "phmm_error_model_tables.inc"

using Penalty = std::int8_t;
constexpr std::uint32_t kNone = 0xFFFFFFFFu;

struct Run { std::uint32_t pos, len, period; };

// ---------------------------------------------------------------------------------------------------------
// String indexes
// ---------------------------------------------------------------------------------------------------------

// Suffix array by prefix doubling (haplotypes are a few hundred to a few thousand bases). Bytes compare unsigned and a
// suffix that is a prefix of another sorts first, as in any suffix array — the array is unique, so how it is built is free.
void build_suffix_array(const unsigned char* s, const int n, std::vector<int>& sa)
{
    sa.resize(n);
    std::vector<int> rank(n), tmp(n);
    for (int i = 0; i < n; ++i) { sa[i] = i; rank[i] = s[i]; }
    for (int k = 1;; k <<= 1) {
        auto key = [&](int i) { return std::make_pair(rank[i], i + k < n ? rank[i + k] : -1); };
        std::sort(sa.begin(), sa.end(), [&](int a, int b) { return key(a) < key(b); });
        tmp[sa[0]] = 0;
        for (int i = 1; i < n; ++i) tmp[sa[i]] = tmp[sa[i - 1]] + (key(sa[i - 1]) < key(sa[i]) ? 1 : 0);
        rank.swap(tmp);
        if (rank[sa[n - 1]] == n - 1) break;
    }
}

// lcp[r] = longest common prefix of the suffixes ranked r-1 and r (lcp[0] = 0), Kasai's sweep (tandem.hpp:139-156)
void build_lcp(const unsigned char* s, const int n, const std::vector<int>& sa, std::vector<std::uint32_t>& lcp)
{
    std::vector<int> rank(n);
    for (int r = 0; r < n; ++r) rank[sa[r]] = r;
    lcp.assign(n, 0u);
    int h = 0;
    for (int i = 0; i < n; ++i) {
        if (rank[i] == 0) continue;              // h carries over (it is only decremented after a comparison)
        const int j = sa[rank[i] - 1];
        while (i + h < n && j + h < n && s[i + h] == s[j + h]) ++h;
        lcp[rank[i]] = (std::uint32_t)h;
        if (h > 0) --h;
    }
}

// Longest previous factor and one previous occurrence per text position (Crochemore & Ilie's stack sweep over the suffix
// array, tandem.cpp:77-112). Which previous occurrence is reported is a property of this sweep, and the reference runs it
// over arrays that carry one extra slot (a second entry for text position 0 with lcp 0 behind the last rank, tandem.hpp:96-104,
// 160-183) — reproduced here, since the propagation step copies runs from exactly that occurrence.
void build_lpf(const std::vector<int>& sa, const std::vector<std::uint32_t>& lcp, std::vector<std::uint32_t>& lpf, std::vector<std::uint32_t>& prev_occ)
{
    const std::size_t n = sa.size();
    std::vector<std::uint32_t> order(n + 2), common(n + 2, 0u);
    for (std::size_t r = 0; r < n; ++r) { order[r] = (std::uint32_t)sa[r]; common[r] = lcp[r]; }
    order[n] = 0u;               // the extra slot
    order[n + 1] = kNone;        // terminator: smaller than everything on the stack
    lpf.assign(n + 1, 0u);
    prev_occ.assign(n + 1, 0u);
    std::vector<std::pair<std::uint32_t, std::uint32_t>> stack;   // (common prefix with what lies below, text position)
    stack.emplace_back(0u, order[0]);
    for (std::size_t r = 1; r <= n + 1; ++r) {
        std::uint32_t u = common[r];
        while (!stack.empty() && (order[r] == kNone || order[r] < stack.back().second)) {
            const auto top = stack.back();
            stack.pop_back();
            lpf[top.second] = std::max(top.first, u);
            u = std::min(top.first, u);
            if (lpf[top.second] == 0u) prev_occ[top.second] = kNone;
            else if (top.first > u) prev_occ[top.second] = stack.back().second;   // the bottom entry always has first == 0: never popped here
            else prev_occ[top.second] = order[r];
        }
        if (r < n + 1) stack.emplace_back(u, order[r]);
    }
}

struct Factor { std::uint32_t pos, len, source; };   // LZ factor and the start of its earlier occurrence (kNone: a new letter)

void lz_factorise(const std::uint32_t n, const std::vector<std::uint32_t>& lpf, const std::vector<std::uint32_t>& prev_occ, std::vector<Factor>& out)
{
    out.clear();
    out.push_back(Factor {0u, 1u, kNone});
    for (std::uint32_t end = 1; end < n;) {
        const std::uint32_t m = std::max<std::uint32_t>(1u, lpf[end]);
        out.push_back(Factor {end, m, prev_occ[end]});
        end += m;
    }
}

// ---------------------------------------------------------------------------------------------------------
// Exact tandem repeats, periods min_period..max_period > 3: lib/tandem's LZ route (tandem.hpp:232-392)
// ---------------------------------------------------------------------------------------------------------

// matches of s[a-k] against s[b-k], k = 0, 1, ... while a-k >= floor
inline std::uint32_t match_left(const unsigned char* s, std::uint32_t a, std::uint32_t b, const std::uint32_t floor)
{
    std::uint32_t k = 0;
    while (a - k >= floor && s[a - k] == s[b - k]) { ++k; if (a < k) break; }
    return k;
}
// matches of s[a+k] against s[b+k] while a+k < limit
inline std::uint32_t match_right(const unsigned char* s, const std::uint32_t a, const std::uint32_t b, const std::uint32_t limit)
{
    std::uint32_t k = 0;
    while (a + k < limit && s[a + k] == s[b + k]) ++k;
    return k;
}

void tandem_repeats_lz(const unsigned char* s, const std::uint32_t n, const std::uint32_t min_period, const std::uint32_t max_period, std::vector<Run>& out)
{
    out.clear();
    std::vector<int> sa;
    std::vector<std::uint32_t> lcp, lpf, prev_occ;
    std::vector<Factor> factors;
    build_suffix_array(s, (int)n, sa);
    build_lcp(s, (int)n, sa, lcp);
    build_lpf(sa, lcp, lpf, prev_occ);
    lz_factorise(n, lpf, prev_occ, factors);

    // Main's step: repetitions that end inside factor h and reach back over the factor boundary (tandem.hpp:232-262), in
    // the order found; a run seen again with the same (pos, len) is dropped whatever its period label (:283-297, operator== :76-79)
    std::vector<std::vector<Run>> by_end(n), by_pos(n);
    auto emit = [&](const std::uint32_t pos, const std::uint32_t len, const std::uint32_t period) {
        std::vector<Run>& bucket = by_end[pos + len - 1];
        for (const Run& r : bucket) if (r.pos == pos && r.len == len) return;
        bucket.push_back(Run {pos, len, period});
    };
    for (std::size_t h = 1; h < factors.size(); ++h) {
        const std::uint32_t u = factors[h].pos, flen = factors[h].len;
        const std::uint32_t reach = std::min(u, 2 * factors[h - 1].len + flen), floor = u - reach, end = u + flen;
        for (std::uint32_t p = min_period; p <= std::min(flen, max_period); ++p) {          // period seed to the right of the boundary
            const std::uint32_t ls = match_left(s, u - 1, u + p - 1, floor), lp = match_right(s, u + p, u, end);
            if (ls + lp >= p && p + lp < flen) emit(u - ls, p + lp + ls, p);
        }
        for (std::uint32_t p = min_period; p < std::min(reach, max_period); ++p) {          // seed to the left (strictly below max_period, :254)
            const std::uint32_t ls = match_left(s, u - p - 1, u - 1, floor), lp = match_right(s, u, u - p, end);
            if (ls + lp >= p) emit(u - (ls + p), p + lp + ls, p);
        }
    }
    for (std::uint32_t e = 0; e < n; ++e) for (const Run& r : by_end[e]) by_pos[r.pos].push_back(r);   // per start, by ascending end (:306-320)

    // Kolpakov-Kucherov propagation: a factor repeats an earlier stretch of text, so the runs lying strictly inside that
    // stretch recur inside the factor; they are copied in front of what the factor's positions already hold (:323-365)
    std::vector<Run> copied;
    for (const Factor& f : factors) {
        const std::uint32_t fend = f.pos + f.len;
        const std::uint32_t delta = f.pos - (f.source != kNone ? f.source : 0u);
        const std::uint32_t src_end_max = fend - delta;
        for (std::uint32_t j = f.pos; j < fend; ++j) {
            const std::uint32_t src = j - delta;
            std::uint32_t src_end = src_end_max;
            if (!by_pos[j].empty()) src_end = std::min(src + by_pos[j].front().len, src_end_max);
            const std::vector<Run>& from = by_pos[src];
            // runs of the source position that end before src_end (the bucket is ordered by end)
            const std::size_t lo = (std::size_t)(std::lower_bound(from.begin(), from.end(), src_end, [](const Run& r, const std::uint32_t v) { return r.pos + r.len < v; }) - from.begin());
            if (lo == 0) continue;
            copied.assign(from.begin(), from.begin() + (std::ptrdiff_t)lo);
            for (Run& r : copied) r.pos += delta;
            by_pos[j].insert(by_pos[j].begin(), copied.begin(), copied.end());
        }
    }
    for (std::uint32_t p = 0; p < n; ++p) out.insert(out.end(), by_pos[p].begin(), by_pos[p].end());
}

// ---------------------------------------------------------------------------------------------------------
// Periods <= 3: lib/tandem's scanning route (tandem.hpp:394-500)
// ---------------------------------------------------------------------------------------------------------

void homopolymer_runs(const unsigned char* s, const std::uint32_t n, std::vector<Run>& out)
{
    for (std::uint32_t i = 0; i + 1 < n;) {
        if (s[i] != s[i + 1]) { ++i; continue; }
        std::uint32_t j = i + 1;
        while (j < n && s[j] == s[i]) ++j;
        out.push_back(Run {i, j - i, 1u});
        i = j;
    }
}

// Period-P repeats as the scanner reports them: a candidate starts only where two neighbouring bases differ; after a hit the
// scan resumes P bases before the hit's end, after a miss one base on (:416-444).
template <std::uint32_t P>
void scanned_repeats(const unsigned char* s, const std::uint32_t n, std::vector<Run>& out)
{
    if (n < 2 * P) return;
    auto next_change = [&](std::uint32_t i) { while (i + 1 < n && s[i] == s[i + 1]) ++i; return i + 1 < n ? i : n; };   // first i' >= i with s[i'] != s[i'+1]
    std::uint32_t a = next_change(0);
    if (a == n) return;
    for (std::uint32_t b = a + P; b < n;) {
        std::uint32_t k = 0;
        while (b + k < n && s[b + k] == s[a + k]) ++k;
        if (k >= P) { out.push_back(Run {a, b + k - a, P}); a = a + k; }
        else ++a;
        a = next_change(a);
        if (a == n) break;
        b = a + P;
    }
}

void merge_by_pos(std::vector<Run>& into, const std::vector<Run>& extra)   // std::inplace_merge's order: on equal pos the earlier list first
{
    std::vector<Run> merged;
    merged.reserve(into.size() + extra.size());
    std::size_t i = 0, j = 0;
    while (i < into.size() && j < extra.size()) merged.push_back(extra[j].pos < into[i].pos ? extra[j++] : into[i++]);
    merged.insert(merged.end(), into.begin() + (std::ptrdiff_t)i, into.end());
    merged.insert(merged.end(), extra.begin() + (std::ptrdiff_t)j, extra.end());
    into.swap(merged);
}

void tandem_repeats_scan(const unsigned char* s, const std::uint32_t n, const std::uint32_t min_period, const std::uint32_t max_period, std::vector<Run>& out)
{
    out.clear();
    std::vector<Run> extra;
    bool first = true;
    for (std::uint32_t p = min_period; p <= max_period; ++p) {
        extra.clear();
        if (p == 1) homopolymer_runs(s, n, extra);
        else if (p == 2) scanned_repeats<2>(s, n, extra);
        else scanned_repeats<3>(s, n, extra);
        if (first) { out.swap(extra); first = false; }
        else merge_by_pos(out, extra);
    }
}

// tandem::extract_exact_tandem_repeats (tandem.hpp:504-521)
bool tandem_repeats(const unsigned char* s, const std::uint32_t n, std::uint32_t min_period, const std::uint32_t max_period, std::vector<Run>& out)
{
    out.clear();
    if (min_period == 0) ++min_period;
    if (n == 0 || n < min_period) return true;
    if (min_period > max_period) return false;
    if (max_period <= 3) tandem_repeats_scan(s, n, min_period, max_period, out);
    else tandem_repeats_lz(s, n, min_period, max_period, out);
    return true;
}

// ---------------------------------------------------------------------------------------------------------
// The models
// ---------------------------------------------------------------------------------------------------------

using MotifMap = std::unordered_map<std::string, std::vector<Penalty>>;   // the reference's container: its iteration order picks the defaults

template <std::size_t N>
struct PaddedRow     // a parameter row copied into a fixed-size table, the tail filled with the row's last value (basic_…:16-20)
{
    Penalty v[N];
    void set(const signed char* src, const std::size_t count) { for (std::size_t i = 0; i < N; ++i) v[i] = src[i < count ? i : count - 1]; }
    Penalty at(const std::uint32_t i) const { return v[i < N ? i : N - 1]; }
};

PaddedRow<50> row50(const int id) { PaddedRow<50> r; r.set(kRowData + kRowStart[id][0], kRowStart[id][1]); return r; }
PaddedRow<51> row51(const int id) { PaddedRow<51> r; r.set(kRowData + kRowStart[id][0], kRowStart[id][1]); return r; }

Penalty lookup(const std::vector<Penalty>& row, const std::uint32_t i) { return i < row.size() ? row[i] : row.back(); }

} // namespace

struct phmm_error_model {
    // indel model
    bool custom = false;
    PaddedRow<50> open_at, open_cg, open_di, open_tri, ext_homo, ext_di, ext_tri;
    MotifMap custom_open, custom_extend;
    bool custom_has_extend = false;
    std::vector<std::string> ns;                 // "", "N", "NN", ... wildcard motifs of the custom model
    Penalty default_open = 0, default_extend = 0;
    // SNV model
    bool has_snv = false;
    PaddedRow<51> caps[3];

    Penalty open_penalty(const unsigned char* motif, const std::uint32_t period, const std::uint32_t len) const
    {
        const std::uint32_t count = len / period;
        if (custom) {
            auto it = custom_open.find(std::string((const char*)motif, period));
            if (it == custom_open.end()) { it = custom_open.find(ns[std::min<std::size_t>(period, ns.size() - 1)]); if (it == custom_open.end()) return default_open; }
            return lookup(it->second, count);
        }
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
    Penalty extend_penalty(const unsigned char* motif, const std::uint32_t period, const std::uint32_t len) const
    {
        const std::uint32_t count = len / period;
        if (custom) {
            if (!custom_has_extend) return default_extend;
            auto it = custom_extend.find(std::string((const char*)motif, period));
            if (it == custom_extend.end()) { it = custom_extend.find(ns[std::min<std::size_t>(period, ns.size() - 1)]); if (it == custom_extend.end()) return default_extend; }
            return lookup(it->second, count);
        }
        return period == 1 ? ext_homo.at(count) : period == 2 ? ext_di.at(count) : ext_tri.at(count);
    }
};

namespace {

thread_local std::string g_error;

void upper(std::string& s) { for (char& c : s) c = (char)std::toupper((unsigned char)c); }

// error_model_factory.cpp:94-112 / 174-200 (names are capitalised before comparison)
int library_index(std::string name)
{
    upper(name);
    if (name == "PCR") return 0;
    if (name == "PCR-FREE" || name == "PCRF") return 1;
    if (name == "10X") return 2;
    if (name == "MDA") return 3;
    return -1;
}
int sequencer_index(std::string name)
{
    upper(name);
    static const char* names[] = {"HISEQ-2000", "HISEQ-2500", "HISEQ-4000", "X10", "NOVASEQ", "BGISEQ-500", "PACBIO", "PACBIOCCS"};
    for (int i = 0; i < 8; ++i) if (name == names[i]) return i;
    return -1;
}
// operator>> reads one whitespace-delimited token (:94-97): leading blanks skipped, the rest of the name ignored
std::string first_token(const std::string& s)
{
    std::size_t a = 0;
    while (a < s.size() && std::isspace((unsigned char)s[a])) ++a;
    std::size_t b = a;
    while (b < s.size() && !std::isspace((unsigned char)s[b])) ++b;
    return s.substr(a, b - a);
}

void set_snv(phmm_error_model& m, const int library)
{
    m.has_snv = true;
    for (int i = 0; i < 3; ++i) m.caps[i] = row51(kSnvRows[library][i]);
}

// repeat_based_indel_error_model.cpp:67-83
void indel_penalties(const phmm_error_model& m, const unsigned char* s, const std::uint32_t n, Penalty* open, Penalty* extend, std::vector<Run>& runs)
{
    std::fill(open, open + n, m.default_open);
    std::fill(extend, extend + n, m.default_extend);
    tandem_repeats(s, n, 1, 5, runs);
    if (runs.empty()) return;
    // the reference orders the runs with std::sort (not stable): the same call on the same sequence reproduces its order
    std::sort(runs.begin(), runs.end(), [](const Run& a, const Run& b) { return a.len < b.len; });
    for (const Run& r : runs) {
        const Penalty o = m.open_penalty(s + r.pos, r.period, r.len);
        for (std::uint32_t i = r.pos; i < r.pos + r.len; ++i) if (o < open[i]) open[i] = o;
        const Penalty e = m.extend_penalty(s + r.pos, r.period, r.len);
        std::fill(extend + r.pos, extend + r.pos + r.len, e);
    }
}

// Length of the repeat run ENDING just before each position, reported where the run ends or is first interrupted; a run
// survives gaps of up to max_gap unmarked bases (repeat_based_snv_error_model.cpp:48-91; note the gap counter is not
// cleared when a different motif starts). get(i) reads the i-th mark of the sweep, put(i, v) stores its result.
template <typename Get, typename Put>
void count_runs(const std::uint32_t n, const unsigned max_gap, Get get, Put put)
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

std::int8_t base_mark(const unsigned char b) { return b == 'A' ? 1 : b == 'C' ? 2 : b == 'G' ? 3 : b == 'T' ? 4 : 5; }

// repeat_based_snv_error_model.cpp:144-179
void snv_arrays(const phmm_error_model& m, const unsigned char* s, const std::uint32_t n, const std::uint8_t* is_substitution,
                char* mask_f, Penalty* prior_f, char* mask_r, Penalty* prior_r, std::vector<Run>& runs)
{
    tandem_repeats(s, n, 1, 3, runs);
    std::vector<std::int8_t> marks[3];
    for (auto& v : marks) v.assign(n, 0);
    for (const Run& r : runs) {
        std::int8_t mark = 0;
        for (std::uint32_t k = 0; k < r.period; ++k) mark = (std::int8_t)(mark + base_mark(s[r.pos + k]));
        std::fill(marks[r.period - 1].begin() + r.pos, marks[r.period - 1].begin() + r.pos + r.len, mark);
    }
    const Penalty max_quality = m.caps[0].v[0];
    std::fill(prior_f, prior_f + n, max_quality);
    std::fill(prior_r, prior_r + n, max_quality);
    std::vector<unsigned> run_len(n);
    for (unsigned i = 0; i < 3; ++i) {
        const std::vector<std::int8_t>& mk = marks[i];
        count_runs(n, i + 2, [&](std::uint32_t k) { return mk[k]; }, [&](std::uint32_t k, unsigned v) { run_len[k] = v; });
        for (std::uint32_t k = 0; k < n; ++k) prior_f[k] = std::min(m.caps[i].at(run_len[k]), prior_f[k]);
        count_runs(n, i + 2, [&](std::uint32_t k) { return mk[n - 1 - k]; }, [&](std::uint32_t k, unsigned v) { run_len[n - 1 - k] = v; });
        for (std::uint32_t k = 0; k < n; ++k) prior_r[k] = std::min(m.caps[i].at(run_len[k]), prior_r[k]);
    }
    if (is_substitution) for (std::uint32_t k = 0; k < n; ++k) if (is_substitution[k]) { prior_f[k] = max_quality; prior_r[k] = max_quality; }
    for (std::uint32_t k = 0; k < n; ++k) {          // the base before / after, cyclically (:174-178)
        mask_f[k] = (char)s[k == 0 ? n - 1 : k - 1];
        mask_r[k] = (char)s[k + 1 == n ? 0 : k + 1];
    }
}

// custom_repeat_based_indel_error_model.cpp:104-158: "MOTIF:p0,p1,...\n" lines ('#' comments), "MOTIF+:" rows are extension penalties
bool parse_custom_model(const std::string& text, phmm_error_model& m, bool& has_open)
{
    has_open = false;
    const std::size_t end = text.size();
    for (std::size_t i = 0; i < end;) {
        if (text[i] == '#') { const std::size_t nl = text.find('\n', i); i = nl == std::string::npos ? end : nl + 1; continue; }
        if (text[i] == '\n') { ++i; continue; }
        const std::size_t colon = text.find(':', i);
        if (colon == std::string::npos || colon == i) return false;
        std::string motif = text.substr(i, colon - i);
        bool extend = false;
        if (motif.back() == '+') { extend = true; m.custom_has_extend = true; motif.pop_back(); if (motif.empty()) return false; }
        else has_open = true;
        std::vector<Penalty> row;
        for (i = colon + 1; i < end && text[i - 1] != '\n'; ++i) {
            std::size_t stop = text.find_first_of(",\n", i);
            if (stop == std::string::npos) stop = end;
            const std::string token = text.substr(i, stop - i);
            // whole-token integer (boost::lexical_cast<int>), then the int8 range (boost::numeric_cast)
            std::size_t k = 0;
            if (k < token.size() && (token[k] == '-' || token[k] == '+')) ++k;
            if (k == token.size()) return false;
            long value = 0;
            for (; k < token.size(); ++k) { if (token[k] < '0' || token[k] > '9' || value > 100000) return false; value = value * 10 + (token[k] - '0'); }
            if (token[0] == '-') value = -value;
            if (value < -128 || value > 127) return false;
            row.push_back((Penalty)value);
            i = stop;
            if (i == end) break;
        }
        if (row.empty()) return false;
        (extend ? m.custom_extend : m.custom_open).emplace(std::move(motif), std::move(row));
    }
    return true;
}

// ---------------------------------------------------------------------------------------------------------
// DeNovoModel's context indel model (IndelMutationModel::evaluate, indel_mutation_model.cpp:67-98)
// ---------------------------------------------------------------------------------------------------------

// find_exact_tandem_repeats(sequence, region, 1, 5) (utils/repeat_finder.hpp:33-55): the finder runs on the sequence with '$'
// appended and every run of N collapsed to one N (tandem::collapse, tandem.hpp:528-554), and its positions are mapped back by
// tandem::rebase (tandem.cpp:138-148). Both are restated as written: collapse's keys count the kept N of earlier runs as removed,
// so a repeat that ends just before an N run can be shifted past its true position.
void mutation_repeats(const unsigned char* s, const std::uint32_t n, std::vector<unsigned char>& buf, std::vector<Run>& runs)
{
    buf.assign(s, s + n);
    buf.push_back('$');
    std::vector<std::pair<std::size_t, std::size_t>> shift;          // collapse's map, keys strictly increasing
    const std::size_t len = buf.size();
    std::size_t first = 0, position = 0, removed = 0;
    while (first < len) {
        std::size_t it1 = first;
        while (it1 + 1 < len && !(buf[it1] == 'N' && buf[it1 + 1] == 'N')) ++it1;
        if (it1 + 1 >= len) break;
        std::size_t it2 = it1;
        while (it2 < len && buf[it2] == 'N') ++it2;
        position += it1 - first;
        removed += it2 - it1 - 1;
        shift.emplace_back(position, removed);
        first = it2;
    }
    if (!shift.empty()) {
        std::size_t w = 0;
        for (std::size_t r = 0; r < len; ++r) if (!(w > 0 && buf[r] == 'N' && buf[w - 1] == 'N')) buf[w++] = buf[r];
        buf.resize(w);
    }
    tandem_repeats(buf.data(), (std::uint32_t)buf.size(), 1, 5, runs);
    if (shift.empty()) return;
    std::size_t k = 0;
    for (Run& r : runs) {
        while (k + 1 < shift.size() && shift[k + 1].first <= r.pos) ++k;
        r.pos += (std::uint32_t)shift[k].second;
    }
}

// Per base the repeat-table cell IndelMutationModel::evaluate copies gap_open / gap_extend from (:78-96): cell [0][0], replaced by a
// later repeat's cell only where that cell's open probability is strictly larger, in the finder's output order.
void mutation_cells(const phmm_mutation_model& m, const unsigned char* s, const std::uint32_t n, std::int32_t* cell,
                    std::vector<unsigned char>& buf, std::vector<Run>& runs)
{
    std::fill(cell, cell + n, 0);
    mutation_repeats(s, n, buf, runs);
    const int width = m.max_periodicity + 1;
    for (const Run& r : runs) {
        const std::uint32_t periods = std::min<std::uint32_t>(r.len / r.period, (std::uint32_t)m.max_periodicity);
        const int c = (int)r.period * width + (int)periods;
        // the reference asserts the repeat lies inside the haplotype; a rebased position past the end is skipped here
        for (std::uint32_t pos = r.pos; pos < r.pos + r.period && pos < n; ++pos) {
            if (m.open[cell[pos]] < m.open[c]) cell[pos] = c;
        }
    }
}

// probability_to_penalty (denovo_model.cpp:23-27)
std::int8_t mutation_penalty(const double probability)
{
    constexpr double ln10_div_10 = 0.230258509299404568401799145468436420760110148862877297603;   // maths::constants::ln10Div10<>
    return (std::int8_t)std::max(std::min(std::round(std::log(probability) / -ln10_div_10), 127.0), 1.0);
}

int fail(const char* what) { g_error = what; return PHMM_ERR_INVALID; }

} // namespace

extern "C" {

const char* phmm_error_model_last_error(void) { return g_error.c_str(); }

int phmm_error_model_create(phmm_error_model** out, const char* label)
{
    if (!out) return PHMM_ERR_INVALID;
    *out = nullptr;
    // parse_model_config (error_model_factory.cpp:531-547): "<library>[.<sequencer>]", missing parts keep the default PCR-free.HiSeq-2500
    int library = 1, sequencer = 1;
    const std::string text = label ? label : "";
    const std::size_t dot = text.find('.');
    const std::string lib_name = text.substr(0, dot);
    if (!lib_name.empty()) { library = library_index(first_token(lib_name)); if (library < 0) return fail("unknown library preparation name"); }
    if (dot != std::string::npos) {
        const std::string seq_name = text.substr(dot + 1);
        if (!seq_name.empty()) { sequencer = sequencer_index(first_token(seq_name)); if (sequencer < 0) return fail("unknown sequencer name"); }
    }
    if (kIndelRows[library][sequencer][0] < 0) return fail("no built-in indel error model for this library / sequencer");
    phmm_error_model* m = new phmm_error_model();
    const short* rows = kIndelRows[library][sequencer];
    m->open_at = row50(rows[0]); m->open_cg = row50(rows[1]); m->open_di = row50(rows[2]); m->open_tri = row50(rows[3]);
    m->ext_homo = row50(kExtendRows[0]); m->ext_di = row50(kExtendRows[1]); m->ext_tri = row50(kExtendRows[2]);
    m->default_open = m->open_di.v[0];           // complex_open_penalty_ (basic_…:32-33)
    m->default_extend = m->ext_di.v[0];
    if (sequencer != 6 && sequencer != 7) set_snv(*m, library);   // no SNV model for PacBio (error_model_factory.cpp:492-495)
    *out = m;
    return PHMM_OK;
}

int phmm_error_model_create_custom(phmm_error_model** out, const char* model_text)
{
    if (!out) return PHMM_ERR_INVALID;
    *out = nullptr;
    if (!model_text) return fail("null model text");
    phmm_error_model* m = new phmm_error_model();
    m->custom = true;
    bool has_open = false;
    if (!parse_custom_model(model_text, *m, has_open)) { delete m; return fail("Bad model"); }
    if (!has_open) { delete m; return fail("malformed model: no gap-open penalties"); }
    // defaults: first entry of the map in ITS iteration order, periodicity 0 (custom_…:30-61); scalar extension 3 without "+" rows
    if (!m->custom_open.empty()) m->default_open = lookup(m->custom_open.cbegin()->second, 0u);
    if (m->custom_has_extend) { if (!m->custom_extend.empty()) m->default_extend = lookup(m->custom_extend.cbegin()->second, 0u); }
    else m->default_extend = 3;
    for (std::size_t i = 0; i <= 10; ++i) m->ns.emplace_back(i, 'N');
    set_snv(*m, 1);                               // make_snv_error_model(default_model_config) (:587)
    *out = m;
    return PHMM_OK;
}

void phmm_error_model_destroy(phmm_error_model* m) { delete m; }

int phmm_reset_haplotypes(const phmm_error_model* m, int32_t n, const int64_t* off, const char* seq, const uint8_t* is_substitution,
                          char* snv_mask_fwd, int8_t* snv_prior_fwd, char* snv_mask_rev, int8_t* snv_prior_rev,
                          int8_t* gap_open, int8_t* gap_extend, int32_t n_threads)
{
    if (!m || n < 0 || (n > 0 && (!off || !seq || !snv_mask_fwd || !snv_prior_fwd || !snv_mask_rev || !snv_prior_rev || !gap_open || !gap_extend)))
        return fail("null argument");
    for (int32_t h = 0; h < n; ++h) if (off[h + 1] < off[h] || off[h + 1] - off[h] > 0x7FFFFFF0LL) return fail("bad haplotype offsets");
    int workers = n_threads > 0 ? n_threads : (int)std::thread::hardware_concurrency();
    workers = std::max(1, std::min(workers, (int)std::min<int32_t>(n, 64)));
    std::atomic<int32_t> next {0};
    auto work = [&] {
        std::vector<Run> runs;
        for (;;) {
            const int32_t h = next.fetch_add(1);
            if (h >= n) break;
            const int64_t o = off[h];
            const std::uint32_t len = (std::uint32_t)(off[h + 1] - o);
            const unsigned char* s = (const unsigned char*)seq + o;
            if (m->has_snv) snv_arrays(*m, s, len, is_substitution ? is_substitution + o : nullptr, snv_mask_fwd + o, snv_prior_fwd + o, snv_mask_rev + o, snv_prior_rev + o, runs);
            else {                                 // haplotype_likelihood_model.cpp:68-74
                std::memset(snv_prior_fwd + o, 100, len); std::memcpy(snv_mask_fwd + o, s, len);
                std::memset(snv_prior_rev + o, 100, len); std::memcpy(snv_mask_rev + o, s, len);
            }
            indel_penalties(*m, s, len, gap_open + o, gap_extend + o, runs);
        }
    };
    if (workers == 1) work();
    else {
        std::vector<std::thread> pool;
        for (int w = 1; w < workers; ++w) pool.emplace_back(work);
        work();
        for (std::thread& t : pool) t.join();
    }
    return PHMM_OK;
}

int phmm_tandem_repeats(const char* seq, int32_t n, int32_t min_period, int32_t max_period, uint32_t* out_triples, int32_t cap)
{
    if (!seq || n < 0 || min_period < 0 || max_period < 0 || (cap > 0 && !out_triples)) return fail("bad argument");
    std::vector<Run> runs;
    if (!tandem_repeats((const unsigned char*)seq, (std::uint32_t)n, (std::uint32_t)min_period, (std::uint32_t)max_period, runs)) return fail("min_period > max_period");
    for (std::size_t i = 0; i < runs.size() && (int32_t)i < cap; ++i) { out_triples[3 * i] = runs[i].pos; out_triples[3 * i + 1] = runs[i].len; out_triples[3 * i + 2] = runs[i].period; }
    return (int)runs.size();
}


int phmm_mutation_model_create(phmm_mutation_model** out, double snv_prior, const float* open, const float* extend,
                               int32_t max_period, int32_t max_periodicity, int32_t max_indel_length)
{
    if (!out) return fail("null output");
    *out = nullptr;
    if (!open || !extend) return fail("null repeat table");
    if (!(snv_prior > 0.0 && snv_prior <= 1.0)) return fail("snv_prior outside (0, 1]");
    if (max_period < 5 || max_period > 1000 || max_periodicity < 1 || max_periodicity > 1000 || max_indel_length < 2 || max_indel_length > 1000)
        return fail("repeat table dimensions out of range (max_period 5..1000, max_periodicity 1..1000, max_indel_length 2..1000)");
    phmm_mutation_model* m = new phmm_mutation_model();
    m->snv_prior = snv_prior;
    m->snv_log_prior = std::log(snv_prior);
    m->snv_penalty = mutation_penalty(snv_prior);
    m->max_period = max_period; m->max_periodicity = max_periodicity; m->max_indel_length = max_indel_length;
    const int cells = m->cells(), X = max_indel_length;
    m->open.assign(open, open + cells);
    m->extend.assign(extend, extend + (std::size_t)cells * X);
    for (const float v : m->open) if (!(v > 0.0f && v <= 1.0f)) { delete m; return fail("repeat table open probability outside (0, 1]"); }
    for (const float v : m->extend) if (!(v > 0.0f && v <= 1.0f)) { delete m; return fail("repeat table extend probability outside (0, 1]"); }
    const std::int32_t dims[3] = {max_period, max_periodicity, max_indel_length};
    m->key.append(reinterpret_cast<const char*>(&snv_prior), sizeof(snv_prior));
    m->key.append(reinterpret_cast<const char*>(dims), sizeof(dims));
    m->key.append(reinterpret_cast<const char*>(m->open.data()), m->open.size() * sizeof(float));
    m->key.append(reinterpret_cast<const char*>(m->extend.data()), m->extend.size() * sizeof(float));
    m->open_penalty.resize(cells); m->extend_penalty.resize(cells); m->logp.resize((std::size_t)cells * X);
    for (int c = 0; c < cells; ++c) {
        const float* ext = m->extend.data() + (std::size_t)c * X;
        m->open_penalty[c] = mutation_penalty(m->open[c]);
        m->extend_penalty[c] = mutation_penalty(ext[1]);
        // calculate_indel_probability: gap_open * gap_extend[1] * ... * gap_extend[length - 1] in float, at most X - 1 factors
        float product = m->open[c];
        for (int k = 0; k < X; ++k) {
            if (k > 0) product = product * ext[k];
            m->logp[(std::size_t)c * X + k] = std::log(product);
        }
    }
    *out = m;
    return PHMM_OK;
}

void phmm_mutation_model_destroy(phmm_mutation_model* m) { delete m; }

int phmm_mutation_context(const phmm_mutation_model* m, int32_t n, const int64_t* off, const char* seq,
                          int32_t* cell, int8_t* open_penalty, int8_t* extend_penalty, int32_t n_threads)
{
    if (!m || n < 0 || (n > 0 && (!off || !seq))) return fail("null argument");
    if (n > 0 && off[0] != 0) return fail("bad haplotype offsets");
    for (int32_t h = 0; h < n; ++h) if (off[h + 1] < off[h] || off[h + 1] - off[h] > 0x7FFFFFF0LL) return fail("bad haplotype offsets");
    int workers = n_threads > 0 ? n_threads : (int)std::thread::hardware_concurrency();
    workers = std::max(1, std::min(workers, (int)std::min<int32_t>(n, 64)));
    std::atomic<int32_t> next {0};
    auto work = [&] {
        std::vector<Run> runs;
        std::vector<unsigned char> buf;
        std::vector<std::int32_t> tmp;
        for (;;) {
            const int32_t h = next.fetch_add(1);
            if (h >= n) break;
            const int64_t o = off[h];
            const std::uint32_t len = (std::uint32_t)(off[h + 1] - o);
            std::int32_t* c = cell ? cell + o : (tmp.resize(len), tmp.data());
            mutation_cells(*m, (const unsigned char*)seq + o, len, c, buf, runs);
            for (std::uint32_t i = 0; i < len; ++i) {
                if (open_penalty) open_penalty[o + i] = m->open_penalty[c[i]];
                if (extend_penalty) extend_penalty[o + i] = m->extend_penalty[c[i]];
            }
        }
    };
    if (workers == 1) work();
    else {
        std::vector<std::thread> pool;
        for (int w = 1; w < workers; ++w) pool.emplace_back(work);
        work();
        for (std::thread& t : pool) t.join();
    }
    return PHMM_OK;
}

} // extern "C"
