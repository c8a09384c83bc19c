// Shared engine for many host threads (include/phmm_b200.h, phmm_batcher_*): the populate requests that concurrent threads
// have in flight are merged into one phmm_populate_regions call, their mutation-prime requests into one phmm_mutation_prime_sets
// call, their assign, template assign and realign requests into one phmm_assign_reads / phmm_assign_templates / phmm_realign_reads
// call. Host C++ over the public C ABI; a
// batch runs the engine's existing multi-region / multi-set / pair-list kernel chain. No thread of its own: the first member of a
// batch (its leader) makes the call.
#include "../../include/phmm_b200.h"
#include "phmm_batcher_seam.h"
#include "phmm_checks.h"
#include "phmm_mutation.h"

#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <cstring>
#include <limits>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

namespace {

thread_local std::string t_error;

constexpr long long kMaxBatchHaps = 65535;          // the DP task word's 16-bit haplotype field (phmm_engine.cu, task_word_ok)
constexpr long long kMaxBatchPairs = 4LL << 20;     // (haplotype, read) pairs of one merged call
constexpr long long kMaxBatchCigarBytes = 128LL << 20;   // CIGAR text of one merged realign call: its pairs x its largest stride
constexpr long long kMaxMapperHapBases = 65535LL * 65535LL;   // the k-mer mapper's haplotype block (phmm_checks::mapper_haplotypes)
constexpr int kDefaultMaxWaitUs = 500;

using Clock = std::chrono::steady_clock;

// No count of a batch derived from its others.
struct NoDerived { static void apply(long long*) {} };

// Element counts of a request or a batch; each request kind names its N counts. The first SUMMED add up over a batch's members,
// the others (a size every member's slot shares, such as the CIGAR stride) take the members' largest; then Derive::apply recomputes
// the counts that follow from the others (a realign batch's CIGAR bytes: its pairs x its stride). max() is per count: a high-water
// mark of each.
template <int N, int SUMMED = N, typename Derive = NoDerived>
struct Counts {
    long long n[N] = {};
    long long& operator[](int i) { return n[i]; }
    long long operator[](int i) const { return n[i]; }
    Counts& operator+=(const Counts& o)
    {
        for (int i = 0; i < N; ++i) n[i] = i < SUMMED ? n[i] + o.n[i] : std::max(n[i], o.n[i]);
        Derive::apply(n);
        return *this;
    }
    bool within(const Counts& cap) const { for (int i = 0; i < N; ++i) if (n[i] > cap.n[i]) return false; return true; }
    static Counts max(const Counts& a, const Counts& b)
    {
        Counts s;
        for (int i = 0; i < N; ++i) s.n[i] = std::max(a.n[i], b.n[i]);
        return s;
    }
};

// A page-locked array that only grows. Its contents do not survive a growth; it grows only while no batch uses it.
template <typename T>
struct Pinned {
    T* p = nullptr;
    long long cap = 0;
    Pinned() = default;
    Pinned(const Pinned&) = delete;
    Pinned& operator=(const Pinned&) = delete;
    ~Pinned() { phmm_host_free(p); }
    bool ensure(long long n)
    {
        if (n <= cap) return true;
        const long long want = std::max(n, 2 * cap);
        T* q = static_cast<T*>(phmm_host_alloc((size_t)want * sizeof(T)));
        if (!q) return false;
        phmm_host_free(p);
        p = q; cap = want;
        return true;
    }
};

// What a kind whose merged call is never rerun reports: the DP cells of its call are the engine's count for its last call.
struct KindBase {
    static constexpr bool reran = false;
    static int64_t dp_cells(const phmm_engine* e) { return phmm_last_dp_cells(e); }
};

// The request kinds. Each supplies what differs between them: its counts, its staging, its merge key and limits, its per-member
// bookkeeping (a Kind object lives in each batch), the copy in, the merged engine call and the copy out.

// What the two populate kinds share: their counts, the read side of their staging, a batch's regions (one per member; the batch is
// one multi-region call) and the copy out.
struct PopulateBase : KindBase {
    enum { HAPS, HAP_BASES, READS, READ_BASES, PAIRS, N_COUNTS };
    using Sizes = Counts<N_COUNTS>;

    // One batch's page-locked copy of its members' reads and its results.
    struct ReadStaging {
        Pinned<int64_t> read_off, read_begin;
        Pinned<char> bases;
        Pinned<uint8_t> quals, mapq, reverse;
        Pinned<double> out;
        Pinned<int32_t> status;
        Sizes cap;
        bool busy = false;

        bool grow_reads(const Sizes& s)
        {
            const bool ok = read_off.ensure(s[READS] + 1) && read_begin.ensure(s[READS]) && bases.ensure(s[READ_BASES]) && quals.ensure(s[READ_BASES]) &&
                            mapq.ensure(s[READS]) && reverse.ensure(s[READS]) && out.ensure(s[PAIRS]) && status.ensure(s[PAIRS]);
            if (!ok) return false;
            cap[READS] = std::min({read_off.cap - 1, read_begin.cap, mapq.cap, reverse.cap});
            cap[READ_BASES] = std::min(bases.cap, quals.cap);
            cap[PAIRS] = std::min(out.cap, status.cap);
            return true;
        }

        void copy_in_reads(const Sizes& at, const phmm_reads* reads)
        {
            const int R = reads->n;
            const long long rb = reads->off[R];
            if (at[READS] == 0) read_off.p[0] = 0;
            for (int r = 0; r < R; ++r) read_off.p[at[READS] + r + 1] = at[READ_BASES] + reads->off[r + 1];
            if (reads->begin) std::memcpy(read_begin.p + at[READS], reads->begin, (size_t)R * sizeof(int64_t));
            else std::memset(read_begin.p + at[READS], 0, (size_t)R * sizeof(int64_t));
            std::memcpy(bases.p + at[READ_BASES], reads->bases, (size_t)rb);
            std::memcpy(quals.p + at[READ_BASES], reads->quals, (size_t)rb);
            // a realign request without mapping qualities has a config that does not read them
            if (reads->mapq) std::memcpy(mapq.p + at[READS], reads->mapq, (size_t)R);
            else std::memset(mapq.p + at[READS], 0, (size_t)R);
            std::memcpy(reverse.p + at[READS], reads->reverse, (size_t)R);
        }

        phmm_reads reads(const Sizes& used) const { return {(int32_t)used[READS], read_off.p, bases.p, quals.p, mapq.p, reverse.p, read_begin.p}; }
    };

    // first staging size: some tens of regions of a few hundred reads; it grows to what merged batches ask for
    static Sizes initial_staging() { return {{4096, 1LL << 20, 1LL << 16, 8LL << 20, 1LL << 20}}; }
    static bool within_limits(const Sizes& s) { return s[HAPS] <= kMaxBatchHaps && s[PAIRS] <= kMaxBatchPairs; }

    phmm_config cfg;
    std::vector<int32_t> hap_first {0}, read_first {0};
    std::vector<phmm_flank_state> flanks;

    explicit PopulateBase(const phmm_config* c) : cfg(*c) {}

    // a new member's region, ending at the batch's counts `used`
    template <typename Request>
    void add(const Request& q, const Sizes& used)
    {
        hap_first.push_back((int32_t)used[HAPS]);
        read_first.push_back((int32_t)used[READS]);
        flanks.push_back(q.flank ? *q.flank : phmm_flank_state {0, 0, 0});
    }

    phmm_regions regions() const { return {(int32_t)flanks.size(), hap_first.data(), read_first.data(), flanks.data()}; }

    // this member's slice of the call's result, [H][R] at the pair offset of its region
    template <typename Request>
    static int copy_out(const ReadStaging& st, const Sizes& at, const Request& q, int rc, const std::string& err)
    {
        if (rc != PHMM_OK && rc != PHMM_ERR_SHORT_HAPLOTYPE) { t_error = err; return rc; }
        const long long H = q.need[HAPS], R = q.need[READS];
        const double* res = st.out.p + at[PAIRS];
        const int32_t* res_status = st.status.p + at[PAIRS];
        rc = PHMM_OK;
        for (long long i = 0; i < q.need[PAIRS]; ++i) if ((res_status[i] & 0xFFFF) == PHMM_STATUS_SHORT_HAP) { rc = PHMM_ERR_SHORT_HAPLOTYPE; break; }
        t_error = rc == PHMM_OK ? std::string() : std::string("Haplotype is too short for alignment");
        if (q.status) std::memcpy(q.status, res_status, (size_t)q.need[PAIRS] * sizeof(int32_t));
        if (q.template_off) {
            // k_template_sum's order: each template's reads left to right from 0.0
            for (long long h = 0; h < H; ++h) {
                for (int t = 0; t < q.n_templates; ++t) {
                    double acc = 0.0;
                    for (long long r = q.template_off[t]; r < q.template_off[t + 1]; ++r) acc += res[(size_t)h * R + r];
                    q.out[(size_t)h * q.n_templates + t] = acc;
                }
            }
        } else {
            std::memcpy(q.out, res, (size_t)q.need[PAIRS] * sizeof(double));
        }
        return rc;
    }
};

// Populate requests: a batch is one phmm_populate_regions call and each member one of its regions; equal configs merge.
struct Populate : PopulateBase {
    struct Request {
        const phmm_config* cfg; const phmm_haplotypes* haps; const phmm_reads* reads;
        const int64_t* template_off; int32_t n_templates;     // template_off NULL: a read request
        const phmm_flank_state* flank; double* out; int32_t* status;
        Sizes need;
    };

    // One batch's page-locked copy of its members' blocks and its results.
    struct Staging : ReadStaging {
        Pinned<int64_t> hap_off, hap_begin;
        Pinned<char> seq, mask_f, mask_r;
        Pinned<int8_t> prior_f, prior_r, gap_open, gap_extend;

        bool grow(const Sizes& s)
        {
            const bool ok = hap_off.ensure(s[HAPS] + 1) && hap_begin.ensure(s[HAPS]) && seq.ensure(s[HAP_BASES]) && mask_f.ensure(s[HAP_BASES]) &&
                            mask_r.ensure(s[HAP_BASES]) && prior_f.ensure(s[HAP_BASES]) && prior_r.ensure(s[HAP_BASES]) &&
                            gap_open.ensure(s[HAP_BASES]) && gap_extend.ensure(s[HAP_BASES]) && grow_reads(s);
            if (!ok) return false;
            cap[HAPS] = std::min(hap_off.cap - 1, hap_begin.cap);
            cap[HAP_BASES] = std::min({seq.cap, mask_f.cap, mask_r.cap, prior_f.cap, prior_r.cap, gap_open.cap, gap_extend.cap});
            return true;
        }
    };

    static std::string key(const Request& q) { return std::string(reinterpret_cast<const char*>(q.cfg), sizeof(phmm_config)); }

    explicit Populate(const Request& q) : PopulateBase(q.cfg) {}

    // the request into its slot at `at` (outside the lock: each member writes its own ranges only)
    static void copy_in(Staging& st, const Sizes& at, const Request& q) { copy_in_blocks(st, at, q.haps, q.reads); }

    // a request's two blocks into their slots at `at` (populate, assign and realign requests)
    static void copy_in_blocks(Staging& st, const Sizes& at, const phmm_haplotypes* haps, const phmm_reads* reads)
    {
        const int H = haps->n;
        const long long hb = haps->off[H];
        if (at[HAPS] == 0) st.hap_off.p[0] = 0;
        for (int h = 0; h < H; ++h) st.hap_off.p[at[HAPS] + h + 1] = at[HAP_BASES] + haps->off[h + 1];
        if (haps->begin) std::memcpy(st.hap_begin.p + at[HAPS], haps->begin, (size_t)H * sizeof(int64_t));
        else std::memset(st.hap_begin.p + at[HAPS], 0, (size_t)H * sizeof(int64_t));
        std::memcpy(st.seq.p + at[HAP_BASES], haps->seq, (size_t)hb);
        std::memcpy(st.mask_f.p + at[HAP_BASES], haps->snv_mask_fwd, (size_t)hb);
        std::memcpy(st.prior_f.p + at[HAP_BASES], haps->snv_prior_fwd, (size_t)hb);
        std::memcpy(st.mask_r.p + at[HAP_BASES], haps->snv_mask_rev, (size_t)hb);
        std::memcpy(st.prior_r.p + at[HAP_BASES], haps->snv_prior_rev, (size_t)hb);
        std::memcpy(st.gap_open.p + at[HAP_BASES], haps->gap_open, (size_t)hb);
        std::memcpy(st.gap_extend.p + at[HAP_BASES], haps->gap_extend, (size_t)hb);
        st.copy_in_reads(at, reads);
    }

    // the leader's call: the batch's members as the regions of one phmm_populate_regions call
    int run(phmm_engine* e, Staging& st, const Sizes& used) const
    {
        const phmm_haplotypes hv {(int32_t)used[HAPS], st.hap_off.p, st.seq.p, st.mask_f.p, st.prior_f.p, st.mask_r.p, st.prior_r.p,
                                  st.gap_open.p, st.gap_extend.p, st.hap_begin.p};
        const phmm_reads rv = st.reads(used);
        const phmm_regions rg = regions();
        return phmm_populate_regions(e, &cfg, &hv, &rv, &rg, st.out.p, st.status.p, PHMM_SPACE_HOST);
    }
};

// Populate requests with an error model: a batch is one phmm_populate_regions_reset call. Equal configs under models equal by
// content merge; the staging holds the sequences and their substitution flags instead of the six penalty arrays.
struct PopulateReset : PopulateBase {
    struct Request {
        const phmm_batcher_seam::ResetRequest* r;
        const phmm_config* cfg; const phmm_haplotype_sequences* seqs; const phmm_reads* reads;
        const int64_t* template_off; int32_t n_templates; const phmm_flank_state* flank; double* out; int32_t* status;
        Sizes need;
    };

    struct Staging : ReadStaging {
        Pinned<int64_t> hap_off, hap_begin;
        Pinned<char> seq;
        Pinned<uint8_t> is_substitution;

        bool grow(const Sizes& s)
        {
            if (!(hap_off.ensure(s[HAPS] + 1) && hap_begin.ensure(s[HAPS]) && seq.ensure(s[HAP_BASES]) && is_substitution.ensure(s[HAP_BASES]) &&
                  grow_reads(s)))
                return false;
            cap[HAPS] = std::min(hap_off.cap - 1, hap_begin.cap);
            cap[HAP_BASES] = std::min(seq.cap, is_substitution.cap);
            return true;
        }
    };

    static std::string key(const Request& q) { return std::string(reinterpret_cast<const char*>(q.cfg), sizeof(phmm_config)) + q.r->model_key; }

    const phmm_error_model* model;                       // the leader's model (the members' are equal by content)
    const phmm_batcher_seam::ResetCalls* calls;

    explicit PopulateReset(const Request& q) : PopulateBase(q.cfg), model(q.r->m), calls(q.r->calls) {}

    static void copy_in(Staging& st, const Sizes& at, const Request& q)
    {
        const phmm_haplotype_sequences* seqs = q.seqs;
        const int H = seqs->n;
        const long long hb = seqs->off[H];
        if (at[HAPS] == 0) st.hap_off.p[0] = 0;
        for (int h = 0; h < H; ++h) st.hap_off.p[at[HAPS] + h + 1] = at[HAP_BASES] + seqs->off[h + 1];
        if (seqs->begin) std::memcpy(st.hap_begin.p + at[HAPS], seqs->begin, (size_t)H * sizeof(int64_t));
        else std::memset(st.hap_begin.p + at[HAPS], 0, (size_t)H * sizeof(int64_t));
        std::memcpy(st.seq.p + at[HAP_BASES], seqs->seq, (size_t)hb);
        // no flags and all-zero flags give the same arrays
        if (seqs->is_substitution) std::memcpy(st.is_substitution.p + at[HAP_BASES], seqs->is_substitution, (size_t)hb);
        else std::memset(st.is_substitution.p + at[HAP_BASES], 0, (size_t)hb);
        st.copy_in_reads(at, q.reads);
    }

    int run(phmm_engine* e, Staging& st, const Sizes& used) const
    {
        const phmm_haplotype_sequences sv {(int32_t)used[HAPS], st.hap_off.p, st.seq.p, st.is_substitution.p, st.hap_begin.p};
        const phmm_reads rv = st.reads(used);
        const phmm_regions rg = regions();
        return calls->populate_regions(e, &cfg, model, &sv, &rv, &rg, st.out.p, st.status.p, PHMM_SPACE_HOST);
    }
};

// Mutation-prime requests: a batch is one phmm_mutation_prime_sets call and each member one of its sets; models equal by content
// (phmm_mutation_model::key) merge.
struct MutationPrime : KindBase {
    enum { HAPS, BASES, PAIRS, N_COUNTS };
    using Sizes = Counts<N_COUNTS>;

    struct Request {
        const phmm_mutation_model* m; int32_t n; const int64_t* off; const char* seq; double* out; int32_t* status;
        Sizes need;
    };

    // One batch's page-locked copy of its members' haplotypes and its results.
    struct Staging {
        Pinned<int64_t> off;
        Pinned<char> seq;
        Pinned<double> out;
        Pinned<int32_t> status;
        Sizes cap;
        bool busy = false;

        bool grow(const Sizes& s)
        {
            if (!(off.ensure(s[HAPS] + 1) && seq.ensure(s[BASES]) && out.ensure(s[PAIRS]) && status.ensure(s[PAIRS]))) return false;
            cap[HAPS] = off.cap - 1; cap[BASES] = seq.cap; cap[PAIRS] = std::min(out.cap, status.cap);
            return true;
        }
    };

    // first staging size: some tens of mutation sets of 50 haplotypes
    static Sizes initial_staging() { return {{2048, 1LL << 20, 1LL << 17}}; }
    static bool within_limits(const Sizes& s) { return s[PAIRS] <= PHMM_MUT_MAX_PAIRS; }
    static std::string key(const Request& q) { return q.m->key; }

    const phmm_mutation_model* model;     // the leader's model (the members' are equal by content)
    std::vector<int32_t> set_first {0};

    explicit MutationPrime(const Request& q) : model(q.m) {}

    void add(const Request&, const Sizes& used) { set_first.push_back((int32_t)used[HAPS]); }

    static void copy_in(Staging& st, const Sizes& at, const Request& q)
    {
        if (at[HAPS] == 0) st.off.p[0] = 0;
        for (int h = 0; h < q.n; ++h) st.off.p[at[HAPS] + h + 1] = at[BASES] + q.off[h + 1];
        std::memcpy(st.seq.p + at[BASES], q.seq, (size_t)q.need[BASES]);
    }

    int run(phmm_engine* e, Staging& st, const Sizes&) const
    {
        return phmm_mutation_prime_sets(e, model, (int32_t)set_first.size() - 1, set_first.data(), st.off.p, st.seq.p, st.out.p, st.status.p);
    }

    // this member's n x n matrix at the pair offset of its set
    static int copy_out(const Staging& st, const Sizes& at, const Request& q, int rc, const std::string& err)
    {
        if (rc != PHMM_OK) { t_error = err; return rc; }
        std::memcpy(q.out, st.out.p + at[PAIRS], (size_t)q.need[PAIRS] * sizeof(double));
        std::memcpy(q.status, st.status.p + at[PAIRS], (size_t)q.need[PAIRS] * sizeof(int32_t));
        t_error.clear();
        return PHMM_OK;
    }
};

// What the assign and realign kinds share: their members' requests, and the rerun of a merged call that failed with
// PHMM_ERR_INVALID. That is a failure a member's own call need not see (assign's more than 4096 mapping positions for one pair fail
// the whole call), so the leader then calls the engine once per member, in the same engine turn, straight into the member's own
// outputs, and each member returns its own code and message.
template <typename Request>
struct Members {
    std::vector<const Request*> reqs;                     // alive while their threads wait in the batch
    std::vector<std::pair<int, std::string>> solo;       // after a rerun: each member's code and message
    bool reran = false;
    int64_t cells = 0;                                    // after a rerun: the DP cells of the merged call and of every rerun

    void add(const Request& q) { reqs.push_back(&q); }

    template <typename Solo>
    void rerun_if_invalid(phmm_engine* e, int rc, Solo&& solo_call)
    {
        if (rc != PHMM_ERR_INVALID || reqs.size() < 2) return;
        cells = phmm_last_dp_cells(e);
        for (const Request* q : reqs) {
            const int r = solo_call(e, *q);
            solo.emplace_back(r, r == PHMM_OK ? std::string() : std::string(phmm_last_error(e)));
            cells += phmm_last_dp_cells(e);
        }
        reran = true;
    }

    int64_t dp_cells(const phmm_engine* e) const { return reran ? cells : phmm_last_dp_cells(e); }

    // after a rerun: the member's own code, with its message in t_error
    int own(const Request& q) const
    {
        const size_t i = (size_t)(std::find(reqs.begin(), reqs.end(), &q) - reqs.begin());
        t_error = solo[i].second;
        return solo[i].first;
    }
};

// Assign requests: a batch is one phmm_assign_reads call whose groups are the members' groups one after the other; equal configs
// merge. The staging is populate's plus the log priors (zeros for a member without) and the top sets; lnl and status are always
// staged and copied out to the members that asked for them. Template requests (phmm_batcher_assign_templates) merge only with each
// other: their batch is one phmm_assign_templates call whose templates are the members' one after the other. Their top sets (one per
// template, at most one per read) and template values (at most one per pair) fit the read-sized staging; each member's share of
// them starts where the members before it end, which Assign::add records in the member's request.
struct Assign : Members<struct AssignRequestSized> {
    using Sizes = PopulateBase::Sizes;
    enum { HAPS = PopulateBase::HAPS, HAP_BASES = PopulateBase::HAP_BASES, READS = PopulateBase::READS, PAIRS = PopulateBase::PAIRS };
    using Request = AssignRequestSized;

    struct Staging : Populate::Staging {
        Pinned<double> priors;
        Pinned<uint64_t> top;

        bool grow(const Sizes& s)
        {
            if (!(Populate::Staging::grow(s) && priors.ensure(s[HAPS]) && top.ensure(s[READS]))) return false;
            cap[HAPS] = std::min(cap[HAPS], priors.cap);
            cap[READS] = std::min(cap[READS], top.cap);
            return true;
        }
    };

    static Sizes initial_staging() { return PopulateBase::initial_staging(); }
    static bool within_limits(const Sizes& s) { return PopulateBase::within_limits(s) && s[HAP_BASES] <= kMaxMapperHapBases; }
    static std::string key(const Request& q);

    phmm_config cfg;
    const phmm_batcher_seam::AlignCalls* calls;
    const phmm_batcher_seam::TemplateCalls* template_calls;       // a batch of template requests
    std::vector<int32_t> hap_first {0}, read_first {0};
    std::vector<phmm_flank_state> flanks;
    std::vector<int64_t> template_off {0};
    long long template_values = 0;                               // the template values of the members so far

    explicit Assign(const Request& q);
    void add(const Request& q, const Sizes& used);
    static void copy_in(Staging& st, const Sizes& at, const Request& q);
    int run(phmm_engine* e, Staging& st, const Sizes& used);
    int copy_out(const Staging& st, const Sizes& at, const Request& q, int rc, const std::string& err) const;
};

struct AssignRequestSized {
    const phmm_batcher_seam::AssignRequest* r;
    Assign::Sizes need;
    long long template_values;          // a template request: its groups' [H_g][T_g] values
    // a template request: its first template and first template value in the batch, set by Assign::add under the batcher's lock
    // and read by copy_out after the call
    mutable long long template_first = 0, value_first = 0;
};

std::string Assign::key(const Request& q)
{
    return std::string(reinterpret_cast<const char*>(q.r->cfg), sizeof(phmm_config)) + (q.r->template_calls ? "templates" : "reads");
}

Assign::Assign(const Request& q) : cfg(*q.r->cfg), calls(q.r->calls), template_calls(q.r->template_calls) {}

// a request's own engine call, as the plain entry point makes it
int assign_alone(phmm_engine* e, const phmm_batcher_seam::AssignRequest& r)
{
    if (r.template_calls)
        return r.template_calls->assign(e, r.cfg, r.haps, r.reads, r.groups, r.template_off, r.n_templates, r.log_priors, r.top, r.lnl, r.status,
                                        PHMM_SPACE_HOST);
    return r.calls->assign(e, r.cfg, r.haps, r.reads, r.groups, r.log_priors, r.top, r.lnl, r.status, PHMM_SPACE_HOST);
}

// the [H_g][T_g] values of a template request's checked groups and templates
long long count_template_values(const phmm_batcher_seam::AssignRequest& r)
{
    long long values = 0;
    int t = 0;
    for (int g = 0; g < r.groups->n; ++g) {
        const int t0 = t;
        while (t < r.n_templates && r.template_off[t] < r.groups->read_first[g + 1]) ++t;
        values += (long long)(r.groups->hap_first[g + 1] - r.groups->hap_first[g]) * (t - t0);
    }
    return values;
}

// the member's groups, their bounds shifted to its slot (its slot ends at the batch's counts `used`); no flank is a flank state of 0
void Assign::add(const Request& q, const Sizes& used)
{
    Members::add(q);
    const phmm_regions* g = q.r->groups;
    const long long h0 = used[HAPS] - q.need[HAPS], r0 = used[READS] - q.need[READS];
    for (int i = 0; i < g->n; ++i) {
        hap_first.push_back((int32_t)(h0 + g->hap_first[i + 1]));
        read_first.push_back((int32_t)(r0 + g->read_first[i + 1]));
        flanks.push_back(g->flank ? g->flank[i] : phmm_flank_state {0, 0, 0});
    }
    if (template_calls) {
        q.template_first = (long long)template_off.size() - 1;
        q.value_first = template_values;
        for (int t = 0; t < q.r->n_templates; ++t) template_off.push_back(r0 + q.r->template_off[t + 1]);
        template_values += q.template_values;
    }
}

void Assign::copy_in(Staging& st, const Sizes& at, const Request& q)
{
    const phmm_batcher_seam::AssignRequest& r = *q.r;
    Populate::copy_in_blocks(st, at, r.haps, r.reads);
    // no priors and zero priors choose the same top sets: k_assign_top adds 0.0 for either
    if (r.log_priors) std::memcpy(st.priors.p + at[HAPS], r.log_priors, (size_t)r.haps->n * sizeof(double));
    else std::fill(st.priors.p + at[HAPS], st.priors.p + at[HAPS] + r.haps->n, 0.0);
}

int Assign::run(phmm_engine* e, Staging& st, const Sizes& used)
{
    const phmm_haplotypes hv {(int32_t)used[HAPS], st.hap_off.p, st.seq.p, st.mask_f.p, st.prior_f.p, st.mask_r.p, st.prior_r.p,
                              st.gap_open.p, st.gap_extend.p, st.hap_begin.p};
    const phmm_reads rv = st.reads(used);
    const phmm_regions groups {(int32_t)flanks.size(), hap_first.data(), read_first.data(), flanks.data()};
    const int rc = template_calls ? template_calls->assign(e, &cfg, &hv, &rv, &groups, template_off.data(), (int32_t)template_off.size() - 1,
                                                           st.priors.p, st.top.p, st.out.p, st.status.p, PHMM_SPACE_HOST)
                                  : calls->assign(e, &cfg, &hv, &rv, &groups, st.priors.p, st.top.p, st.out.p, st.status.p, PHMM_SPACE_HOST);
    rerun_if_invalid(e, rc, [](phmm_engine* en, const Request& q) { return assign_alone(en, *q.r); });
    return rc;
}

// this member's reads' (or templates') top sets and its groups' slots (or template values); its code from its own statuses, as the
// call's would be for it alone
int Assign::copy_out(const Staging& st, const Sizes& at, const Request& q, int rc, const std::string& err) const
{
    if (reran) return own(q);
    if (rc != PHMM_OK && rc != PHMM_ERR_SHORT_HAPLOTYPE) { t_error = err; return rc; }
    const phmm_batcher_seam::AssignRequest& r = *q.r;
    const long long P = q.need[PAIRS];
    const int32_t* res_status = st.status.p + at[PAIRS];
    rc = PHMM_OK;
    for (long long i = 0; i < P; ++i) if ((res_status[i] & 0xFFFF) == PHMM_STATUS_SHORT_HAP) { rc = PHMM_ERR_SHORT_HAPLOTYPE; break; }
    t_error = rc == PHMM_OK ? std::string() : std::string("Haplotype is too short for alignment");
    if (template_calls) {
        std::memcpy(r.top, st.top.p + q.template_first, (size_t)r.n_templates * sizeof(uint64_t));
        if (r.lnl) std::memcpy(r.lnl, st.out.p + q.value_first, (size_t)q.template_values * sizeof(double));
    } else {
        std::memcpy(r.top, st.top.p + at[READS], (size_t)q.need[READS] * sizeof(uint64_t));
        if (r.lnl) std::memcpy(r.lnl, st.out.p + at[PAIRS], (size_t)P * sizeof(double));
    }
    if (r.status) std::memcpy(r.status, res_status, (size_t)P * sizeof(int32_t));
    return rc;
}

// The CIGAR text and status a pair gets at its own stride, from its text and status at the batch's stride (not smaller). The kernel
// (cigar_emit / make_cigar_text, phmm_kernels.cuh) writes at most stride - 1 characters and a NUL, and turns status PHMM_STATUS_OK
// into PHMM_STATUS_CIGAR_TRUNCATED unless the whole text is shorter than stride - 1 characters. An exact match's single '=' run is
// the exception: it is cut without that status. Requests whose longest read's run would not fit their stride run alone, so here a
// text too long for its stride is always a traceback's.
int32_t restride_cigar(const char* text, int32_t status, char* out, int32_t stride)
{
    const size_t n = std::strlen(text), room = (size_t)stride - 1;
    const size_t keep = std::min(n, room);
    std::memcpy(out, text, keep);
    out[keep] = 0;
    return status == PHMM_STATUS_OK && n >= room ? PHMM_STATUS_CIGAR_TRUNCATED : status;
}

// whether a stride holds the single '=' run of an exact match of a read of `len` bases with room to spare (see restride_cigar)
bool single_run_fits(long long len, int32_t stride)
{
    int digits = 1;
    for (long long v = len; v >= 10; v /= 10) ++digits;
    return digits + 1 < (long long)stride - 1;
}

// Realign requests: a batch is one phmm_realign_reads call over the members' blocks one after the other, their pair indices shifted
// to their slots. Equal configs under equal effective flank states merge, whatever their strides: the call runs at the largest.
struct Realign : Members<struct RealignRequestSized> {
    enum { HAPS, HAP_BASES, READS, READ_BASES, PAIRS, STRIDE, CIGAR, N_COUNTS };
    // the stride: the members' largest; CIGAR: the text bytes the call writes, its pairs x that stride. The staging's CIGAR buffer and
    // the lane's high-water mark follow this count, never a product of the largest pair count and the largest stride seen apart.
    struct CigarBytes { static void apply(long long* n) { n[CIGAR] = n[PAIRS] * n[STRIDE]; } };
    using Sizes = Counts<N_COUNTS, STRIDE, CigarBytes>;
    using Request = RealignRequestSized;

    struct Staging {
        Populate::Staging blocks;                              // its out / status: the likelihoods and statuses
        Pinned<phmm_pair> pairs;
        Pinned<int64_t> mapping_position;
        Pinned<char> cigar;
        Sizes cap;
        bool busy = false;

        bool grow(const Sizes& s)
        {
            if (!(blocks.grow(head(s)) && pairs.ensure(s[PAIRS]) && mapping_position.ensure(s[PAIRS]) && cigar.ensure(s[CIGAR])))
                return false;
            for (int i = 0; i < PopulateBase::N_COUNTS; ++i) cap[i] = blocks.cap[i];
            cap[PAIRS] = std::min({cap[PAIRS], pairs.cap, mapping_position.cap});
            cap[STRIDE] = std::numeric_limits<long long>::max();      // no room of its own: the CIGAR bytes hold it
            cap[CIGAR] = cigar.cap;
            return true;
        }
    };

    static PopulateBase::Sizes head(const Sizes& s)
    {
        PopulateBase::Sizes h;
        for (int i = 0; i < PopulateBase::N_COUNTS; ++i) h[i] = s[i];
        return h;
    }
    // first staging size: some tens of requests of a few hundred reads of up to a few hundred bases
    static Sizes initial_staging() { return {{1024, 1LL << 20, 1LL << 15, 4LL << 20, 1LL << 15, 0, 4LL << 20}}; }
    static bool within_limits(const Sizes& s)
    {
        return s[PAIRS] <= kMaxBatchPairs && s[CIGAR] <= kMaxBatchCigarBytes && s[HAP_BASES] <= kMaxMapperHapBases;
    }
    static phmm_flank_state effective_flank(const phmm_config* cfg, const phmm_flank_state* f)
    {
        return f && f->has_flank && cfg->use_flank_state ? phmm_flank_state {1, f->lhs_flank, f->rhs_flank} : phmm_flank_state {0, 0, 0};
    }
    static std::string key(const Request& q);

    phmm_config cfg;
    phmm_flank_state flank;
    const phmm_batcher_seam::AlignCalls* calls;
    int32_t stride = 0;                                         // the batch's: its members' largest

    explicit Realign(const Request& q);
    void add(const Request& q, const Sizes& used) { Members::add(q); stride = (int32_t)used[STRIDE]; }
    static void copy_in(Staging& st, const Sizes& at, const Request& q);
    int run(phmm_engine* e, Staging& st, const Sizes& used);
    int copy_out(const Staging& st, const Sizes& at, const Request& q, int rc, const std::string& err) const;
};

struct RealignRequestSized {
    const phmm_batcher_seam::RealignRequest* r;
    Realign::Sizes need;
};

// the config bytes and the flank state the call uses (phmm_realign_reads ignores a flank without has_flank or use_flank_state)
std::string Realign::key(const Request& q)
{
    const phmm_flank_state f = effective_flank(q.r->cfg, q.r->flank);
    std::string k(reinterpret_cast<const char*>(q.r->cfg), sizeof(phmm_config));
    k.append(reinterpret_cast<const char*>(&f.has_flank), sizeof(f.has_flank));
    k.append(reinterpret_cast<const char*>(&f.lhs_flank), sizeof(f.lhs_flank));
    k.append(reinterpret_cast<const char*>(&f.rhs_flank), sizeof(f.rhs_flank));
    return k;
}

Realign::Realign(const Request& q) : cfg(*q.r->cfg), flank(effective_flank(q.r->cfg, q.r->flank)), calls(q.r->calls) {}

void Realign::copy_in(Staging& st, const Sizes& at, const Request& q)
{
    const phmm_batcher_seam::RealignRequest& r = *q.r;
    Populate::copy_in_blocks(st.blocks, head(at), r.haps, r.reads);
    for (int64_t j = 0; j < r.n_pairs; ++j)
        st.pairs.p[at[PAIRS] + j] = phmm_pair {(int32_t)(at[READS] + r.pairs[j].read), (int32_t)(at[HAPS] + r.pairs[j].hap)};
}

int Realign::run(phmm_engine* e, Staging& st, const Sizes& used)
{
    const Populate::Staging& b = st.blocks;
    const phmm_haplotypes hv {(int32_t)used[HAPS], b.hap_off.p, b.seq.p, b.mask_f.p, b.prior_f.p, b.mask_r.p, b.prior_r.p,
                              b.gap_open.p, b.gap_extend.p, b.hap_begin.p};
    const phmm_reads rv = b.reads(head(used));
    const int rc = calls->realign(e, &cfg, &hv, &rv, st.pairs.p, used[PAIRS], &flank, st.mapping_position.p, b.out.p, st.cigar.p, stride,
                                  b.status.p, PHMM_SPACE_HOST);
    rerun_if_invalid(e, rc, [](phmm_engine* en, const Request& q) {
        const phmm_batcher_seam::RealignRequest& r = *q.r;
        return r.calls->realign(en, r.cfg, r.haps, r.reads, r.pairs, r.n_pairs, r.flank, r.mapping_position, r.likelihood, r.cigar,
                                r.cigar_stride, r.status, PHMM_SPACE_HOST);
    });
    return rc;
}

// this member's pairs; each CIGAR text restated at the member's own stride
int Realign::copy_out(const Staging& st, const Sizes& at, const Request& q, int rc, const std::string& err) const
{
    if (reran) return own(q);
    if (rc != PHMM_OK) { t_error = err; return rc; }
    const phmm_batcher_seam::RealignRequest& r = *q.r;
    const long long p0 = at[PAIRS];
    std::memcpy(r.mapping_position, st.mapping_position.p + p0, (size_t)r.n_pairs * sizeof(int64_t));
    std::memcpy(r.likelihood, st.blocks.out.p + p0, (size_t)r.n_pairs * sizeof(double));
    for (int64_t j = 0; j < r.n_pairs; ++j)
        r.status[j] = restride_cigar(st.cigar.p + (size_t)(p0 + j) * stride, st.blocks.status.p[p0 + j], r.cigar + (size_t)j * r.cigar_stride,
                                     r.cigar_stride);
    t_error.clear();
    return PHMM_OK;
}

// A batch of one kind's requests: the kind's own data and the shared life cycle.
template <typename Kind>
struct Batch {
    Batch(const typename Kind::Request& q, std::string k, typename Kind::Staging* s, Clock::time_point d)
        : kind(q), key(std::move(k)), st(s), deadline(d) {}
    Kind kind;
    std::string key;
    typename Kind::Staging* st;
    typename Kind::Sizes used;
    Clock::time_point deadline;
    int members = 0;
    int pending_copies = 0;     // members that reserved space and have not finished copying in
    int readers = 0;            // members that have not finished copying out
    bool open = true;           // accepts members
    bool full = false;          // a request did not fit: send without waiting for company
    bool done = false;          // the call has returned
    int rc = PHMM_OK;
    std::string err;
};

// One kind's open batches (one per merge key), its staging pool and the pool's high-water mark: what merged batches have asked for.
template <typename Kind>
struct Lane {
    std::map<std::string, Batch<Kind>*> open;
    std::vector<std::unique_ptr<typename Kind::Staging>> staging;
    typename Kind::Sizes want = Kind::initial_staging();
};

} // namespace

struct phmm_batcher {
    phmm_engine* engine = nullptr;
    int clients = 0;
    int max_wait_us = kDefaultMaxWaitUs;
    mutable std::mutex m;
    std::condition_variable cv;
    Lane<Populate> populate;
    Lane<PopulateReset> populate_reset;
    Lane<MutationPrime> mutation;
    Lane<Assign> assign;
    Lane<Realign> realign;
    bool engine_busy = false;
    int waiting = 0;                                  // requests in batches not yet sent + requests running alone
    int in_flight = 0;                                // requests inside the batcher
    phmm_batcher_stats stats {};
    int64_t reruns = 0;                               // merged calls rerun one member at a time
};

namespace {

void count_call(phmm_batcher* b, int requests, int64_t dp_cells)
{
    b->stats.requests += requests;
    b->stats.gpu_calls += 1;
    if (requests > 1) b->stats.merged_calls += 1;
    b->stats.max_regions_per_call = std::max<int64_t>(b->stats.max_regions_per_call, requests);
    b->stats.dp_cells += dp_cells;
}

// A request a multi-region call cannot merge: one engine call of its own, call(engine), in turn with the batches.
template <typename Call>
int run_alone(phmm_batcher* b, Call&& call)
{
    std::unique_lock<std::mutex> lk(b->m);
    ++b->waiting;
    b->cv.notify_all();
    b->cv.wait(lk, [&] { return !b->engine_busy; });
    b->engine_busy = true;
    lk.unlock();
    const int rc = call(b->engine);
    t_error = rc == PHMM_OK ? std::string() : std::string(phmm_last_error(b->engine));
    lk.lock();
    count_call(b, 1, phmm_last_dp_cells(b->engine));
    b->engine_busy = false;
    --b->waiting;
    b->cv.notify_all();
    return rc;
}

// A free staging set of the lane's pool, large enough for `need` (grown to the high-water mark) and marked busy; nullptr when out
// of memory.
template <typename Kind>
typename Kind::Staging* free_staging(Lane<Kind>& lane, const typename Kind::Sizes& need)
{
    typename Kind::Staging* st = nullptr;
    for (auto& s : lane.staging) if (!s->busy) { st = s.get(); break; }
    if (!st) { lane.staging.emplace_back(new typename Kind::Staging()); st = lane.staging.back().get(); }
    const typename Kind::Sizes size = Kind::Sizes::max(need, lane.want);
    if (!size.within(st->cap) && !st->grow(size)) return nullptr;
    st->busy = true;
    return st;
}

template <typename Kind>
void close_batch(Lane<Kind>& lane, Batch<Kind>* bt)
{
    if (!bt->open) return;
    bt->open = false;
    const auto it = lane.open.find(bt->key);
    if (it != lane.open.end() && it->second == bt) lane.open.erase(it);
}

// Under the lock: the batch the request joins, with its slot at *at reserved. That is the open batch of the request's merge key if
// the request fits it (the kind's limits and the batch's staging); a batch it does not fit is marked full and closed (when only
// the staging was too small, the high-water mark rises), and a new batch with a free staging set, sent at the latest max_wait_us
// from now, takes the request. nullptr when out of page-locked memory.
template <typename Kind>
Batch<Kind>* join(phmm_batcher* b, Lane<Kind>& lane, const std::string& key, const typename Kind::Request& q, typename Kind::Sizes* at)
{
    Batch<Kind>* bt = nullptr;
    for (;;) {
        const auto it = lane.open.find(key);
        if (it == lane.open.end()) {
            typename Kind::Staging* st = free_staging(lane, q.need);
            if (!st) return nullptr;
            bt = new Batch<Kind>(q, key, st, Clock::now() + std::chrono::microseconds(b->max_wait_us));
            lane.open[key] = bt;
            break;
        }
        bt = it->second;
        typename Kind::Sizes total = bt->used;
        total += q.need;
        const bool limits = Kind::within_limits(total);
        if (limits && total.within(bt->st->cap)) break;
        if (limits) lane.want = Kind::Sizes::max(lane.want, total);   // staging too small
        bt->full = true;
        close_batch(lane, bt);
        b->cv.notify_all();
    }
    *at = bt->used;
    bt->used += q.need;
    bt->kind.add(q, bt->used);
    return bt;
}

// The life of a request in a batch, the same for every kind: it joins a batch under the lock, then copies itself into its slot of
// the staging outside the lock (each member its own ranges). The first member leads: it waits until `clients` requests wait, the
// batch is full or its deadline has passed, and the engine is free, then seals the batch and makes the kind's call; the others
// wait for it. Each member copies its own slice out (outside the lock) and returns its code; the last reader frees the staging
// and the batch. A kind whose merged call can fail for one member's sake reruns its members alone inside run (Members).
template <typename Kind>
int take_part(phmm_batcher* b, Lane<Kind>& lane, const typename Kind::Request& q)
{
    const std::string key = Kind::key(q);
    std::unique_lock<std::mutex> lk(b->m);
    typename Kind::Sizes at;
    Batch<Kind>* bt = join(b, lane, key, q, &at);
    if (!bt) { t_error = "out of page-locked host memory for the batch staging"; return PHMM_ERR_NOMEM; }
    const bool leader = bt->members == 0;
    ++bt->members; ++bt->pending_copies; ++bt->readers; ++b->waiting;
    b->cv.notify_all();
    lk.unlock();

    Kind::copy_in(*bt->st, at, q);

    lk.lock();
    --bt->pending_copies;
    if (leader) {
        for (;;) {
            const bool company = b->clients > 0 && b->waiting >= b->clients;
            const bool go = bt->full || company || Clock::now() >= bt->deadline;
            if (go && !b->engine_busy) break;
            if (go) b->cv.wait(lk);
            else b->cv.wait_until(lk, bt->deadline);
        }
        close_batch(lane, bt);
        b->engine_busy = true;
        b->waiting -= bt->members;
        b->cv.wait(lk, [&] { return bt->pending_copies == 0; });
        lk.unlock();
        bt->rc = bt->kind.run(b->engine, *bt->st, bt->used);
        if (bt->rc != PHMM_OK) bt->err = phmm_last_error(b->engine);
        lk.lock();
        count_call(b, bt->members, bt->kind.dp_cells(b->engine));
        if (bt->kind.reran) { b->reruns += 1; b->stats.gpu_calls += bt->members; }
        b->engine_busy = false;
        bt->done = true;
        b->cv.notify_all();
    } else {
        b->cv.notify_all();                       // the leader may be waiting for this copy
        b->cv.wait(lk, [&] { return bt->done; });
    }
    lk.unlock();

    const int rc = bt->kind.copy_out(*bt->st, at, q, bt->rc, bt->err);

    lk.lock();
    if (--bt->readers == 0) {
        bt->st->busy = false;
        delete bt;
    }
    return rc;
}

// The host-side checks of phmm_populate, in its order, for a request without position lists. Sets *alone when the request has to
// run on its own (pipelined size, too many haplotypes, a haplotype too long for the task word); the remaining checks are then
// phmm_populate's own. `derived`: a request with an error model, whose penalty arrays the engine derives (haps holds n / off / seq).
int check_request(const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads, const double* out, bool* alone, Populate::Sizes* need,
                  bool derived = false)
{
    int rc;
    if ((rc = phmm_checks::config_and_output(cfg, out, reads, t_error)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::blocks(haps, reads, t_error, derived)) != PHMM_OK) return rc;
    const long long pairs = (long long)haps->n * reads->n;
    if (pairs >= 2 * phmm_checks::populate_chunk_pairs(pairs) || haps->n > kMaxBatchHaps) { *alone = true; return PHMM_OK; }
    long long len_min, len_max;
    phmm_checks::read_length_range(reads, &len_min, &len_max);
    const long long hap_bases = haps->off[haps->n], read_bases = reads->off[reads->n];
    if ((rc = phmm_checks::offsets(haps->off[0], hap_bases, reads->off[0], read_bases, len_min, len_max, t_error)) != PHMM_OK) return rc;
    long long max_hap = 0;
    for (int h = 0; h < haps->n; ++h) max_hap = std::max<long long>(max_hap, haps->off[h + 1] - haps->off[h]);
    if (cfg->map_positions && (rc = phmm_checks::mapper_haplotypes(max_hap, hap_bases, t_error)) != PHMM_OK) return rc;
    if (max_hap > 65535) { *alone = true; return PHMM_OK; }
    if (!derived && (rc = phmm_checks::penalties(haps, hap_bases, t_error)) != PHMM_OK) return rc;
    *need = {{haps->n, hap_bases, reads->n, read_bases, pairs}};
    return PHMM_OK;
}

int submit(phmm_batcher* b, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads, const phmm_positions* positions,
           const int64_t* template_off, int32_t n_templates, const phmm_flank_state* flank, double* out, int32_t* status)
{
    bool alone = positions && positions->off && positions->pos;
    Populate::Request q {cfg, haps, reads, template_off, n_templates, flank, out, status, {}};
    if (!alone) {
        const int rc = check_request(cfg, haps, reads, out, &alone, &q.need);
        if (rc != PHMM_OK) return rc;
    }
    if (alone) {
        return run_alone(b, [&](phmm_engine* e) {
            return template_off ? phmm_populate_templates(e, cfg, haps, reads, template_off, n_templates, positions, flank, out, status, PHMM_SPACE_HOST)
                                : phmm_populate(e, cfg, haps, reads, positions, flank, out, status, PHMM_SPACE_HOST);
        });
    }
    return take_part(b, b->populate, q);
}

// Entry and exit of every request: destroy waits until no request is inside.
struct InFlight {
    phmm_batcher* b;
    explicit InFlight(phmm_batcher* batcher) : b(batcher) { std::lock_guard<std::mutex> lk(b->m); ++b->in_flight; }
    ~InFlight() { std::lock_guard<std::mutex> lk(b->m); --b->in_flight; b->cv.notify_all(); }
};

} // namespace

int phmm_batcher_seam::submit_assign(phmm_batcher* b, const AssignRequest& r)
{
    if (!b) { t_error = "null batcher"; return PHMM_ERR_INVALID; }
    // phmm_assign_reads' (phmm_assign_templates') host checks in its order: the groups, the config and top, the group limits, (the
    // templates,) the blocks, the mapper's limits
    int rc;
    if ((rc = phmm_checks::regions(r.haps, r.reads, r.groups, t_error)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::config_and_output(r.cfg, r.top, r.reads, t_error)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::assign_groups(r.groups, t_error)) != PHMM_OK) return rc;
    if (r.template_calls && (rc = phmm_checks::assign_templates(r.template_off, r.n_templates, r.reads, r.groups, t_error)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::blocks(r.haps, r.reads, t_error)) != PHMM_OK) return rc;
    long long len_min, len_max;
    phmm_checks::read_length_range(r.reads, &len_min, &len_max);
    const long long hap_bases = r.haps->off[r.haps->n], read_bases = r.reads->off[r.reads->n];
    if ((rc = phmm_checks::offsets(r.haps->off[0], hap_bases, r.reads->off[0], read_bases, len_min, len_max, t_error)) != PHMM_OK) return rc;
    long long max_hap = 0;
    for (int h = 0; h < r.haps->n; ++h) max_hap = std::max<long long>(max_hap, r.haps->off[h + 1] - r.haps->off[h]);
    if (r.cfg->map_positions) {
        if ((rc = phmm_checks::mapper_reads(len_max, t_error)) != PHMM_OK) return rc;
        if ((rc = phmm_checks::mapper_haplotypes(max_hap, hap_bases, t_error)) != PHMM_OK) return rc;
    }
    long long pairs = 0;
    for (int g = 0; g < r.groups->n; ++g)
        pairs += (long long)(r.groups->hap_first[g + 1] - r.groups->hap_first[g]) * (r.groups->read_first[g + 1] - r.groups->read_first[g]);
    // a penalty outside [0,127] fails the call that holds it (after its mapping), and too large a request would not fit a batch
    std::string penalty_error;
    InFlight guard(b);
    if (r.haps->n > kMaxBatchHaps || pairs > kMaxBatchPairs || max_hap > 65535 || phmm_checks::penalties(r.haps, hap_bases, penalty_error) != PHMM_OK) {
        return run_alone(b, [&](phmm_engine* e) { return assign_alone(e, r); });
    }
    const Assign::Request q {&r, {{r.haps->n, hap_bases, r.reads->n, read_bases, pairs}}, r.template_calls ? count_template_values(r) : 0};
    return take_part(b, b->assign, q);
}

int phmm_batcher_seam::submit_realign(phmm_batcher* b, const RealignRequest& r)
{
    if (!b) { t_error = "null batcher"; return PHMM_ERR_INVALID; }
    // phmm_realign_reads' host checks in its order: the arguments, the reads' arrays, the blocks, the penalties, the pair indices,
    // the mapper's limits
    int rc;
    if ((rc = phmm_checks::align_arguments(r.cfg, r.pairs, r.n_pairs, r.mapping_position, r.likelihood, r.cigar, r.cigar_stride, r.status,
                                           t_error)) != PHMM_OK)
        return rc;
    if (r.n_pairs == 0) { t_error.clear(); return PHMM_OK; }
    if ((rc = phmm_checks::align_reads(r.cfg, r.reads, t_error)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::blocks(r.haps, r.reads, t_error)) != PHMM_OK) return rc;
    long long len_min, len_max;
    phmm_checks::read_length_range(r.reads, &len_min, &len_max);
    const long long hap_bases = r.haps->off[r.haps->n], read_bases = r.reads->off[r.reads->n];
    if ((rc = phmm_checks::offsets(r.haps->off[0], hap_bases, r.reads->off[0], read_bases, len_min, len_max, t_error)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::penalties(r.haps, hap_bases, t_error)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::pair_indices(r.pairs, r.n_pairs, r.haps->n, r.reads->n, t_error)) != PHMM_OK) return rc;
    if (r.cfg->map_positions) {
        long long max_hap = 0;
        for (int h = 0; h < r.haps->n; ++h) max_hap = std::max<long long>(max_hap, r.haps->off[h + 1] - r.haps->off[h]);
        if ((rc = phmm_checks::mapper_reads(len_max, t_error)) != PHMM_OK) return rc;
        if ((rc = phmm_checks::mapper_haplotypes(max_hap, hap_bases, t_error)) != PHMM_OK) return rc;
    }
    InFlight guard(b);
    const Realign::Request q {&r, {{r.haps->n, hap_bases, r.reads->n, read_bases, r.n_pairs, r.cigar_stride, r.n_pairs * r.cigar_stride}}};
    if (!Realign::within_limits(q.need) || !single_run_fits(len_max, r.cigar_stride)) {
        return run_alone(b, [&](phmm_engine* e) {
            return r.calls->realign(e, r.cfg, r.haps, r.reads, r.pairs, r.n_pairs, r.flank, r.mapping_position, r.likelihood, r.cigar,
                                    r.cigar_stride, r.status, PHMM_SPACE_HOST);
        });
    }
    return take_part(b, b->realign, q);
}

int phmm_batcher_seam::submit_reset(phmm_batcher* b, const ResetRequest& r)
{
    if (!b) { t_error = "null batcher"; return PHMM_ERR_INVALID; }
    // phmm_populate(_templates)_reset's checks in their order: the sequences block, the template offsets, the reset, the populate
    if (!r.seqs) { t_error = "null argument"; return PHMM_ERR_INVALID; }
    int rc;
    if (r.template_off && (rc = phmm_checks::template_offsets(r.template_off, r.n_templates, r.reads, true, t_error)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::reset_sequences(r.m, r.seqs, t_error)) != PHMM_OK) return rc;
    InFlight guard(b);
    const phmm_haplotypes shell {r.seqs->n, r.seqs->off, r.seqs->seq, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, r.seqs->begin};
    bool alone = (r.positions && r.positions->off && r.positions->pos) || r.model_key.empty();
    PopulateReset::Request q {&r, r.cfg, r.seqs, r.reads, r.template_off, r.n_templates, r.flank, r.out, r.status, {}};
    if (!alone && (rc = check_request(r.cfg, &shell, r.reads, r.out, &alone, &q.need, true)) != PHMM_OK) return rc;
    if (alone) {
        return run_alone(b, [&](phmm_engine* e) {
            return r.template_off ? r.calls->populate_templates(e, r.cfg, r.m, r.seqs, r.reads, r.template_off, r.n_templates, r.positions, r.flank,
                                                                r.out, r.status, PHMM_SPACE_HOST)
                                  : r.calls->populate(e, r.cfg, r.m, r.seqs, r.reads, r.positions, r.flank, r.out, r.status, PHMM_SPACE_HOST);
        });
    }
    return take_part(b, b->populate_reset, q);
}

extern "C" {

int phmm_batcher_create(phmm_batcher** out, int device, const phmm_batcher_options* opt)
{
    if (!out) { t_error = "null output handle"; return PHMM_ERR_INVALID; }
    *out = nullptr;
    if (opt && (opt->clients < 0 || opt->max_wait_us < 0)) { t_error = "clients and max_wait_us must be >= 0"; return PHMM_ERR_INVALID; }
    phmm_engine* e = nullptr;
    const int rc = phmm_create(&e, device);
    if (rc != PHMM_OK) { t_error = phmm_last_error(nullptr); return rc; }
    phmm_batcher* b = new phmm_batcher();
    b->engine = e;
    if (opt) { b->clients = opt->clients; b->max_wait_us = opt->max_wait_us; }
    *out = b;
    return PHMM_OK;
}

void phmm_batcher_destroy(phmm_batcher* b)
{
    if (!b) return;
    {
        std::unique_lock<std::mutex> lk(b->m);
        b->cv.wait(lk, [&] { return b->in_flight == 0; });
    }
    phmm_destroy(b->engine);
    delete b;
}

const char* phmm_batcher_last_error(void) { return t_error.c_str(); }

int phmm_batcher_populate(phmm_batcher* b, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                          const phmm_positions* positions, const phmm_flank_state* flank, double* out, int32_t* status)
{
    if (!b) { t_error = "null batcher"; return PHMM_ERR_INVALID; }
    InFlight guard(b);
    return submit(b, cfg, haps, reads, positions, nullptr, 0, flank, out, status);
}

int phmm_batcher_populate_templates(phmm_batcher* b, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                                    const int64_t* template_off, int32_t n_templates, const phmm_flank_state* flank,
                                    double* out, int32_t* status)
{
    if (!b) { t_error = "null batcher"; return PHMM_ERR_INVALID; }
    const int rc = phmm_checks::template_offsets(template_off, n_templates, reads, true, t_error);
    if (rc != PHMM_OK) return rc;
    InFlight guard(b);
    return submit(b, cfg, haps, reads, nullptr, template_off, n_templates, flank, out, status);
}

int phmm_batcher_mutation_prime(phmm_batcher* b, const phmm_mutation_model* m, int32_t n, const int64_t* off, const char* seq,
                                double* out, int32_t* status)
{
    if (!b) { t_error = "null batcher"; return PHMM_ERR_INVALID; }
    InFlight guard(b);
    const int rc = phmm_checks::mutation_set(m, n, off, seq, out, status, t_error);
    if (rc != PHMM_OK) return rc;
    const MutationPrime::Request q {m, n, off, seq, out, status, {{n, off[n], (long long)n * n}}};
    return take_part(b, b->mutation, q);
}

int phmm_batcher_stats_get(const phmm_batcher* b, phmm_batcher_stats* out)
{
    if (!b || !out) return PHMM_ERR_INVALID;
    std::lock_guard<std::mutex> lk(b->m);
    *out = b->stats;
    return PHMM_OK;
}

int64_t phmm_batcher_reruns(const phmm_batcher* b)
{
    if (!b) return 0;
    std::lock_guard<std::mutex> lk(b->m);
    return b->reruns;
}

} // extern "C"
