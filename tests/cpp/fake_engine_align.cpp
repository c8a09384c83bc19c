// A CPU stand-in for the engine's read-assignment and realignment symbols (phmm_assign_reads, phmm_realign_reads), next to
// tests/cpp/fake_engine.cpp's populate and mutation ones, so that the request batcher's assign and realign requests run their whole
// life cycle without a GPU (tests/test_batcher_align_cpu.py).
//
// Every value hashes only its own pair's data (the config, the pair's haplotype and read bytes and the flank state the call uses), so a
// request gets the same values in a merged call as alone exactly when the batcher stages, shifts and slices correctly. Assign: top
// follows find_map_haplotypes' rule over the fake values plus the log priors (haplotypes with identical data tie). Realign: each pair
// has a CIGAR text of its own length (up to a few hundred characters), written as the kernel writes it at the call's stride; an
// exact match (the read equals the haplotype's start) gets a single '=' run. The engine's host checks are kept in its order with
// its messages. Marker reads: a read starting with "MMMM" has more than 4096 mapping positions, which fails a whole assign call
// that maps positions; a read starting with "RRRR" fails a whole realign call that maps positions (a stand-in for a failure only a
// merged call can see, so that the batcher's rerun of a realign batch is exercised); a read longer than its haplotype gets a SHORT_HAP
// status. Each scored pair adds its haplotype length x read length to the call's DP cells. Every call is recorded.
#include "../../include/phmm_b200.h"
#include "../../octopus_b200/csrc/phmm_checks.h"

#include <cmath>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

struct phmm_engine {        // fake_engine.cpp's engine, declared identically
    std::string err;
    int64_t dp_cells = 0;
};

namespace fake_align {

struct Call {
    std::string entry;       // "assign_reads" or "realign_reads"
    int members;             // groups of an assign call, pairs of a realign call
    long long haps;
    int32_t stride;          // realign: the call's CIGAR stride
};

namespace {
std::mutex g_m;
std::vector<Call> g_calls;

void record(Call c)
{
    std::lock_guard<std::mutex> lk(g_m);
    g_calls.push_back(std::move(c));
}

struct Hash {
    unsigned long long h = 1469598103934665603ULL;
    Hash& add(const void* p, size_t n)
    {
        const unsigned char* c = static_cast<const unsigned char*>(p);
        for (size_t i = 0; i < n; ++i) { h ^= c[i]; h *= 1099511628211ULL; }
        return *this;
    }
    template <typename T> Hash& value(const T& v) { return add(&v, sizeof(T)); }
    double finish() const { return -1e-3 - (double)(h >> 11) * (100.0 / 9007199254740992.0); }
};

// the hash of pair (h, r): the haplotype's data, the read's (its mapping quality only where the config reads it), the config and flank
unsigned long long pair_hash(const phmm_config* cfg, const phmm_haplotypes* haps, int h, const phmm_reads* reads, int r, const phmm_flank_state& f)
{
    const long long hb = haps->off[h], hl = haps->off[h + 1] - hb, rb = reads->off[r], rl = reads->off[r + 1] - rb;
    Hash x;
    x.add(cfg, sizeof(phmm_config));
    x.add(haps->seq + hb, (size_t)hl).add(haps->snv_mask_fwd + hb, (size_t)hl).add(haps->snv_prior_fwd + hb, (size_t)hl);
    x.add(haps->snv_mask_rev + hb, (size_t)hl).add(haps->snv_prior_rev + hb, (size_t)hl);
    x.add(haps->gap_open + hb, (size_t)hl).add(haps->gap_extend + hb, (size_t)hl);
    x.value(haps->begin ? haps->begin[h] : (int64_t)0);
    x.add(reads->bases + rb, (size_t)rl).add(reads->quals + rb, (size_t)rl).value(reads->reverse[r]);
    if (cfg->use_mapping_quality) x.value(reads->mapq[r]);
    x.value(reads->begin ? reads->begin[r] : (int64_t)0);
    x.value(f.has_flank).value(f.lhs_flank).value(f.rhs_flank);
    return x.h;
}

int32_t short_status(const phmm_haplotypes* haps, int h, const phmm_reads* reads, int r)
{
    const long long hl = haps->off[h + 1] - haps->off[h], rl = reads->off[r + 1] - reads->off[r];
    return hl < rl ? PHMM_STATUS_SHORT_HAP | (int32_t)((rl - hl) << 16) : PHMM_STATUS_OK;
}

bool marker_read(const phmm_reads* reads, int r, const char* marker = "MMMM")
{
    return reads->off[r + 1] - reads->off[r] >= 4 && std::memcmp(reads->bases + reads->off[r], marker, 4) == 0;
}

long long cells_of(const phmm_haplotypes* haps, int h, const phmm_reads* reads, int r)
{
    return (haps->off[h + 1] - haps->off[h]) * (reads->off[r + 1] - reads->off[r]);
}

// the blocks' host checks of stage_batch: blocks, offsets; *len_max the longest read, *max_hap the longest haplotype
int check_blocks(phmm_engine* e, const phmm_haplotypes* haps, const phmm_reads* reads, long long* len_max, long long* max_hap)
{
    int rc;
    if ((rc = phmm_checks::blocks(haps, reads, e->err)) != PHMM_OK) return rc;
    long long len_min;
    phmm_checks::read_length_range(reads, &len_min, len_max);
    if ((rc = phmm_checks::offsets(haps->off[0], haps->off[haps->n], reads->off[0], reads->off[reads->n], len_min, *len_max, e->err)) != PHMM_OK) return rc;
    *max_hap = 0;
    for (int h = 0; h < haps->n; ++h) *max_hap = std::max<long long>(*max_hap, haps->off[h + 1] - haps->off[h]);
    return PHMM_OK;
}

// maths::almost_equal(l, r, 1)
bool almost_equal(double l, double r) { return l == r || std::fabs(l - r) < 2.220446049250313080847263336181640625e-16 * std::fabs(l + r); }
} // namespace

std::vector<Call> calls()
{
    std::lock_guard<std::mutex> lk(g_m);
    return g_calls;
}

void clear_calls()
{
    std::lock_guard<std::mutex> lk(g_m);
    g_calls.clear();
}

// The CIGAR text of a traceback for a pair hash: runs of '=', 'X', 'I' and 'D' up to a length the hash picks (8 to ~300 characters).
std::string traceback_text(unsigned long long h)
{
    static const char ops[] = "=XID";
    const size_t want = 8 + (size_t)(h % 300);
    std::string t;
    unsigned long long x = h;
    while (t.size() < want) {
        x = x * 6364136223846793005ULL + 1442695040888963407ULL;
        t += std::to_string(1 + (x >> 33) % 120);
        t += ops[(x >> 20) % 4];
    }
    return t;
}

} // namespace fake_align

extern "C" {

int phmm_assign_reads(phmm_engine* e, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                      const phmm_regions* groups, const double* log_priors, uint64_t* top, double* lnl, int32_t* status, int space)
{
    fake_align::record({"assign_reads", groups ? groups->n : 0, haps ? haps->n : 0, 0});
    e->dp_cells = 0;
    e->err.clear();
    int rc;
    if (space != PHMM_SPACE_HOST) { e->err = "bad space"; return PHMM_ERR_INVALID; }
    if ((rc = phmm_checks::regions(haps, reads, groups, e->err)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::config_and_output(cfg, top, reads, e->err)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::assign_groups(groups, e->err)) != PHMM_OK) return rc;
    long long len_max, max_hap;
    if ((rc = fake_align::check_blocks(e, haps, reads, &len_max, &max_hap)) != PHMM_OK) return rc;
    if (cfg->map_positions) {
        if ((rc = phmm_checks::mapper_reads(len_max, e->err)) != PHMM_OK) return rc;
        if ((rc = phmm_checks::mapper_haplotypes(max_hap, haps->off[haps->n], e->err)) != PHMM_OK) return rc;
        for (int r = 0; r < reads->n; ++r) {
            if (fake_align::marker_read(reads, r)) { e->err = "more than 4096 candidate positions for one (haplotype, read) pair"; return PHMM_ERR_INVALID; }
        }
    }
    bool short_hap = false;
    long long slot = 0;
    std::vector<double> v;
    for (int g = 0; g < groups->n; ++g) {
        const int h0 = groups->hap_first[g], nH = groups->hap_first[g + 1] - h0, r0 = groups->read_first[g], nR = groups->read_first[g + 1] - r0;
        const phmm_flank_state none {0, 0, 0};
        const phmm_flank_state f = groups->flank && groups->flank[g].has_flank && cfg->use_flank_state ? groups->flank[g] : none;
        v.assign((size_t)nH * nR, 0.0);
        for (int k = 0; k < nH; ++k) {
            for (int i = 0; i < nR; ++i) {
                fake_align::Hash x;
                x.h = fake_align::pair_hash(cfg, haps, h0 + k, reads, r0 + i, f);
                v[(size_t)k * nR + i] = x.finish();
                e->dp_cells += fake_align::cells_of(haps, h0 + k, reads, r0 + i);
                const int32_t st = fake_align::short_status(haps, h0 + k, reads, r0 + i);
                short_hap |= st != PHMM_STATUS_OK;
                if (lnl) lnl[slot + (long long)k * nR + i] = v[(size_t)k * nR + i];
                if (status) status[slot + (long long)k * nR + i] = st;
            }
        }
        for (int i = 0; i < nR; ++i) {
            double max_value = -1.7976931348623157e308;
            uint64_t set = 0;
            for (int k = 0; k < nH; ++k) {
                const double cur = v[(size_t)k * nR + i] + (log_priors ? log_priors[h0 + k] : 0.0);
                if (fake_align::almost_equal(cur, max_value)) set |= 1ull << k;
                else if (cur > max_value) { set = 1ull << k; max_value = cur; }
            }
            top[r0 + i] = set ? set : (nH == 64 ? ~0ull : (1ull << nH) - 1);
        }
        slot += (long long)nH * nR;
    }
    if ((rc = phmm_checks::penalties(haps, haps->off[haps->n], e->err)) != PHMM_OK) return rc;
    if (short_hap) { e->err = "Haplotype is too short for alignment"; return PHMM_ERR_SHORT_HAPLOTYPE; }
    return PHMM_OK;
}

int phmm_realign_reads(phmm_engine* e, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                       const phmm_pair* pairs, int64_t n_pairs, const phmm_flank_state* flank,
                       int64_t* mapping_position, double* likelihood, char* cigar, int32_t cigar_stride, int32_t* status, int space)
{
    fake_align::record({"realign_reads", (int)n_pairs, haps ? haps->n : 0, cigar_stride});
    e->dp_cells = 0;
    e->err.clear();
    int rc;
    if (space != PHMM_SPACE_HOST) { e->err = "bad space"; return PHMM_ERR_INVALID; }
    if ((rc = phmm_checks::align_arguments(cfg, pairs, n_pairs, mapping_position, likelihood, cigar, cigar_stride, status, e->err)) != PHMM_OK) return rc;
    if (n_pairs == 0) return PHMM_OK;
    if ((rc = phmm_checks::align_reads(cfg, reads, e->err)) != PHMM_OK) return rc;
    long long len_max, max_hap;
    if ((rc = fake_align::check_blocks(e, haps, reads, &len_max, &max_hap)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::penalties(haps, haps->off[haps->n], e->err)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::pair_indices(pairs, n_pairs, haps->n, reads->n, e->err)) != PHMM_OK) return rc;
    if (cfg->map_positions) {
        if ((rc = phmm_checks::mapper_reads(len_max, e->err)) != PHMM_OK) return rc;
        if ((rc = phmm_checks::mapper_haplotypes(max_hap, haps->off[haps->n], e->err)) != PHMM_OK) return rc;
        for (int64_t j = 0; j < n_pairs; ++j) {
            if (fake_align::marker_read(reads, pairs[j].read, "RRRR")) { e->err = "fake: a failure of the whole realign call"; return PHMM_ERR_INVALID; }
        }
    }
    const phmm_flank_state none {0, 0, 0};
    const phmm_flank_state f = flank && flank->has_flank && cfg->use_flank_state ? *flank : none;
    for (int64_t j = 0; j < n_pairs; ++j) {
        const int r = pairs[j].read, h = pairs[j].hap;
        char* cg = cigar + (size_t)j * cigar_stride;
        cg[0] = 0;
        status[j] = fake_align::short_status(haps, h, reads, r);
        const unsigned long long x = fake_align::pair_hash(cfg, haps, h, reads, r, f);
        e->dp_cells += fake_align::cells_of(haps, h, reads, r);
        if (status[j] != PHMM_STATUS_OK) { mapping_position[j] = 0; likelihood[j] = -1.7976931348623157e308; continue; }
        fake_align::Hash hx;
        hx.h = x;
        likelihood[j] = hx.finish();
        const long long rl = reads->off[r + 1] - reads->off[r];
        const bool exact = std::memcmp(reads->bases + reads->off[r], haps->seq + haps->off[h], (size_t)rl) == 0;
        mapping_position[j] = exact ? 0 : (int64_t)(x % 1000);
        const std::string text = exact ? std::to_string(rl) + "=" : fake_align::traceback_text(x);
        // cigar_emit / make_cigar_text: at most stride - 1 characters and a NUL; a traceback's text is reported truncated unless it is
        // shorter than stride - 1, an exact match's single run never
        const size_t keep = std::min(text.size(), (size_t)cigar_stride - 1);
        std::memcpy(cg, text.data(), keep);
        cg[keep] = 0;
        if (!exact && text.size() >= (size_t)cigar_stride - 1) status[j] = PHMM_STATUS_CIGAR_TRUNCATED;
    }
    return PHMM_OK;
}

} // extern "C"
