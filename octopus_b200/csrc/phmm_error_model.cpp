// HaplotypeLikelihoodModel::reset for the H100 pair-HMM engine: the per-haplotype penalty arrays the kernels consume
// (SNV mask / prior per strand, gap_open[], gap_extend[]) from the haplotype sequence alone. The arithmetic is phmm_reset.cuh's,
// shared with the device (phmm_engine_reset_haplotypes); this file holds the models' construction (built-in labels, custom model
// text), the host entry points that run the shared core on host threads, and DeNovoModel's context indel model.
//
// Reference (paths in the octopus source tree):
//   src/core/models/error/basic_repeat_based_indel_error_model.cpp:51-103   penalty lookup by motif period and repeat count
//   src/core/models/error/custom_repeat_based_indel_error_model.cpp:68-158  motif-keyed custom model + its text format
//   src/core/models/error/error_model_factory.cpp:220-589           built-in parameters (generated table include), label parsing
#include "../../include/phmm_b200.h"
#include "phmm_mutation.h"
#include "phmm_reset.cuh"

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

using phmm_reset::Penalty;
using phmm_reset::Run;

// ---------------------------------------------------------------------------------------------------------
// The models
// ---------------------------------------------------------------------------------------------------------

using MotifMap = std::unordered_map<std::string, std::vector<Penalty>>;   // the reference's container: its iteration order picks the defaults

phmm_reset::PaddedRow<50> row50(const int id) { phmm_reset::PaddedRow<50> r; r.set(kRowData + kRowStart[id][0], kRowStart[id][1]); return r; }
phmm_reset::PaddedRow<51> row51(const int id) { phmm_reset::PaddedRow<51> r; r.set(kRowData + kRowStart[id][0], kRowStart[id][1]); return r; }

Penalty lookup(const std::vector<Penalty>& row, const std::uint32_t i) { return i < row.size() ? row[i] : row.back(); }

// A motif map as the core looks it up: the keys the finder can ask for (1..5 bytes), sorted, with their rows back to back
struct FlatMotifs
{
    std::vector<std::uint64_t> key;
    std::vector<std::uint32_t> row;
    std::vector<Penalty> data;

    void assign(const MotifMap& map)
    {
        std::vector<std::pair<std::uint64_t, const std::vector<Penalty>*>> entries;
        for (const auto& kv : map)
            if (!kv.first.empty() && kv.first.size() <= 5)
                entries.emplace_back(phmm_reset::motif_key((const unsigned char*)kv.first.data(), (std::uint32_t)kv.first.size()), &kv.second);
        std::sort(entries.begin(), entries.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
        key.clear(); row.assign(1, 0u); data.clear();
        for (const auto& e : entries) {
            key.push_back(e.first);
            data.insert(data.end(), e.second->begin(), e.second->end());
            row.push_back((std::uint32_t)data.size());
        }
    }
    phmm_reset::MotifTable view() const { return phmm_reset::MotifTable {key.data(), row.data(), data.data(), (std::int32_t)key.size()}; }
};

} // namespace

struct phmm_error_model {
    phmm_reset::Model core;                      // what the shared core reads; the custom tables point into the vectors below
    MotifMap custom_open, custom_extend;         // a custom model as parsed (their iteration order picks the defaults)
    FlatMotifs flat_open, flat_extend;
    std::string key;                             // phmm_reset::model_key
};

const phmm_reset::Model& phmm_reset::model_of(const phmm_error_model* m) { return m->core; }
const std::string& phmm_reset::model_key(const phmm_error_model* m) { return m->key; }

namespace {

// Everything the core reads, as bytes: the flags, the fixed rows, the defaults and a custom model's flattened motif tables. A model
// that holds a penalty outside [0,127] gets the empty key.
void set_key(phmm_error_model& m)
{
    const phmm_reset::Model& c = m.core;
    std::string& k = m.key;
    k.clear();
    bool in_range = c.default_open >= 0 && c.default_extend >= 0;
    auto bytes = [&](const void* p, std::size_t n) { k.append(static_cast<const char*>(p), n); };
    auto penalties = [&](const Penalty* p, std::size_t n) { for (std::size_t i = 0; i < n; ++i) in_range = in_range && p[i] >= 0; bytes(p, n); };
    const char flags[3] = {(char)c.custom, (char)c.custom_has_extend, (char)c.has_snv};
    bytes(flags, sizeof(flags));
    for (const phmm_reset::PaddedRow<50>* r : {&c.open_at, &c.open_cg, &c.open_di, &c.open_tri, &c.ext_homo, &c.ext_di, &c.ext_tri}) penalties(r->v, 50);
    for (const phmm_reset::PaddedRow<51>& r : c.caps) penalties(r.v, 51);
    penalties(&c.default_open, 1);
    penalties(&c.default_extend, 1);
    for (const FlatMotifs* f : {&m.flat_open, &m.flat_extend}) {
        const std::uint64_t n = f->key.size();
        bytes(&n, sizeof(n));
        bytes(f->key.data(), f->key.size() * sizeof(std::uint64_t));
        bytes(f->row.data(), f->row.size() * sizeof(std::uint32_t));
        penalties(f->data.data(), f->data.size());
    }
    if (!in_range) k.clear();
}

} // namespace

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

void set_snv(phmm_reset::Model& m, const int library)
{
    m.has_snv = true;
    for (int i = 0; i < 3; ++i) m.caps[i] = row51(kSnvRows[library][i]);
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
        if (motif.back() == '+') { extend = true; m.core.custom_has_extend = true; motif.pop_back(); if (motif.empty()) return false; }
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
void mutation_repeats(const unsigned char* s, const std::uint32_t n, std::vector<unsigned char>& buf, phmm_reset::HostScratch& scratch, std::vector<Run>& runs)
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
    phmm_reset::tandem_repeats_host(buf.data(), (std::uint32_t)buf.size(), 1, 5, scratch, runs);
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
                    std::vector<unsigned char>& buf, phmm_reset::HostScratch& scratch, std::vector<Run>& runs)
{
    std::fill(cell, cell + n, 0);
    mutation_repeats(s, n, buf, scratch, runs);
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
    phmm_reset::Model& c = m->core;
    const short* rows = kIndelRows[library][sequencer];
    c.open_at = row50(rows[0]); c.open_cg = row50(rows[1]); c.open_di = row50(rows[2]); c.open_tri = row50(rows[3]);
    c.ext_homo = row50(kExtendRows[0]); c.ext_di = row50(kExtendRows[1]); c.ext_tri = row50(kExtendRows[2]);
    c.default_open = c.open_di.v[0];             // complex_open_penalty_ (basic_…:32-33)
    c.default_extend = c.ext_di.v[0];
    if (sequencer != 6 && sequencer != 7) set_snv(c, library);   // no SNV model for PacBio (error_model_factory.cpp:492-495)
    set_key(*m);
    *out = m;
    return PHMM_OK;
}

int phmm_error_model_create_custom(phmm_error_model** out, const char* model_text)
{
    if (!out) return PHMM_ERR_INVALID;
    *out = nullptr;
    if (!model_text) return fail("null model text");
    phmm_error_model* m = new phmm_error_model();
    phmm_reset::Model& c = m->core;
    c.custom = true;
    bool has_open = false;
    if (!parse_custom_model(model_text, *m, has_open)) { delete m; return fail("Bad model"); }
    if (!has_open) { delete m; return fail("malformed model: no gap-open penalties"); }
    // defaults: first entry of the map in ITS iteration order, periodicity 0 (custom_…:30-61); scalar extension 3 without "+" rows
    if (!m->custom_open.empty()) c.default_open = lookup(m->custom_open.cbegin()->second, 0u);
    if (c.custom_has_extend) { if (!m->custom_extend.empty()) c.default_extend = lookup(m->custom_extend.cbegin()->second, 0u); }
    else c.default_extend = 3;
    m->flat_open.assign(m->custom_open);
    m->flat_extend.assign(m->custom_extend);
    c.custom_open = m->flat_open.view();
    c.custom_extend = m->flat_extend.view();
    set_snv(c, 1);                               // make_snv_error_model(default_model_config) (:587)
    set_key(*m);
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
        phmm_reset::HostScratch scratch;
        for (;;) {
            const int32_t h = next.fetch_add(1);
            if (h >= n) break;
            const int64_t o = off[h];
            phmm_reset::reset_haplotype_host(m->core, (const unsigned char*)seq + o, (std::uint32_t)(off[h + 1] - o), is_substitution ? is_substitution + o : nullptr,
                                             snv_mask_fwd + o, snv_prior_fwd + o, snv_mask_rev + o, snv_prior_rev + o, gap_open + o, gap_extend + o, scratch);
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
    phmm_reset::HostScratch scratch;
    if (phmm_reset::tandem_repeats_host((const unsigned char*)seq, (std::uint32_t)n, (std::uint32_t)min_period, (std::uint32_t)max_period, scratch, runs) != phmm_reset::kOk)
        return fail("min_period > max_period");
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
        phmm_reset::HostScratch scratch;
        for (;;) {
            const int32_t h = next.fetch_add(1);
            if (h >= n) break;
            const int64_t o = off[h];
            const std::uint32_t len = (std::uint32_t)(off[h + 1] - o);
            std::int32_t* c = cell ? cell + o : (tmp.resize(len), tmp.data());
            mutation_cells(*m, (const unsigned char*)seq + o, len, c, buf, scratch, runs);
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
