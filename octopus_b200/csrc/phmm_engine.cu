// C ABI of the H100 pair-HMM engine (include/phmm_b200.h): host-side orchestration only. All arithmetic of the
// hot path runs in the kernels of phmm_kernels.cuh; there is no CPU fallback — without a usable GPU every
// computing entry point returns PHMM_ERR_CUDA.
#include "../../include/phmm_b200.h"
#include "phmm_checks.h"
#include "phmm_mutation.h"
#include "phmm_kernels.cuh"
#include "phmm_vb.cuh"
#include "phmm_vb_mm.cuh"

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstdio>
#include <cstring>
#include <condition_variable>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <type_traits>
#include <vector>

using namespace phmm;

namespace {

// A device allocation of the engine: grows on demand and is freed with its owner (phmm_destroy selects the device first).
struct DBuf {
    void* p = nullptr;
    size_t cap = 0;
    DBuf() = default;
    DBuf(const DBuf&) = delete;
    DBuf& operator=(const DBuf&) = delete;
    ~DBuf() { release(); }
    cudaError_t ensure(size_t bytes)
    {
        if (bytes <= cap) return cudaSuccess;
        release();
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) { e = cudaMalloc(&p, bytes); want = bytes; }
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <typename T> T* as() const { return static_cast<T*>(p); }
};

int round_band(int requested)
{
    // simd_pair_hmm_wrapper.hpp:218-241: smallest supported band >= request, from {8,16,32,64,128,256}
    for (int b = 8; b <= 256; b <<= 1) if (requested <= b) return b;
    return -1;
}

} // namespace

struct phmm_engine {
    int device = 0;
    int sm_count = 132;
    int reserved_sms = 0;       // phmm_reserve_sms
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    std::string err;
    int64_t launches_last = 0, launches_total = 0;
    double last_dp_ms = 0.0;
    int64_t last_dp_cells = 0;
    // device copies of caller arrays (host-space calls)
    DBuf h_off, h_seq, h_mf, h_pf, h_mr, h_pr, h_go, h_ge, h_begin;
    DBuf r_off, r_bases, r_quals, r_mapq, r_rev, r_begin;
    DBuf c_off, c_pos;
    // derived / scratch
    DBuf tab_f, tab_r, rowhalf, info, flags, best, status, out, slow, counters, pairs, generic_reads, wide_reads, bp, regs, rregion, rpbase, rpstride;
    DBuf tasks_lane, tasks_generic, works, scores, mapq_tab;
    DBuf rhash, kbins, kitems, kpos, kcnt, ftasks, fcnt, gtasks, atasks, gcnt, sched, sorted, fb_scratch, fb_pairs, npre_f, npre_r;
    DBuf pm_best, pm_cnt, pm_inl, pm_part, pm_misc;   // the pair mapper's first pass (k_kmer_map_pairs) and its offset scan
    DBuf as_pairs, as_prior, as_top;                  // phmm_assign_reads: slot-ordered pair list, log priors, top sets
    DBuf at_groups, at_off, at_lnl;                   // phmm_assign_templates: per-group template layout, template offsets, values
    DBuf mu_in, mu_list, mu_res, mu_cig, mu_out;      // phmm_mutation_prime: staged set, DP pair list, per-tile results, CIGARs, matrix
    DBuf rs_sub, rs_model, rs_words, rs_runs, rs_flags;   // phmm_engine_reset_haplotypes: flags, model tables, scratch slots, overflow
    DBuf vb_lnl, vb_gt, vb_in, vb_idx, vb_ws, vb_seed, vb_out;   // phmm_variational_bayes: staged inputs, genotype index, workspace, results
    DBuf mm_lnl, mm_gt, mm_in, mm_idx, mm_pairs, mm_ws, mm_seed, mm_out;   // phmm_variational_bayes_mixture_mixture: the same, and the slot pairs
    std::vector<cudaEvent_t> tile_events;
    std::vector<int2> info_host;
    // per-kernel launch configuration already applied / queried (the runtime calls are not free and need not be repeated)
    std::map<std::pair<const void*, size_t>, int> occupancy;
    // host-space calls on large batches are pipelined over two sub-engines (own stream + buffers each), driven by two host
    // threads, so that the H2D / D2H copies of one read chunk overlap the kernels of the other
    phmm_engine* sub[2] = {nullptr, nullptr};
    bool is_sub = false;
    // Chunk c's DP kernels wait (on the device) for chunk c-1's, so that the DP kernels run back to back in chunk order —
    // each with the whole GPU — while the other chunk's copies, preparation and classify pass fill in around them.
    // order_ev marks "this sub-engine's DP kernels of its current chunk are done"; the parent's order state tells the other
    // worker thread that the event has been recorded (a wait enqueued before the record would see the previous one).
    phmm_engine* parent = nullptr;
    phmm_engine* peer = nullptr;
    cudaEvent_t order_ev = nullptr;
    long long chunk_index = -1;
    struct OrderState { std::mutex m; std::condition_variable cv; long long recorded = -1; } order;
};

// Sub-engine side of the chunk ordering; no-ops on a plain engine.
struct ChunkOrder {
    phmm_engine* e;
    bool waited = false, recorded = false;
    explicit ChunkOrder(phmm_engine* eng) : e(eng) {}
    cudaError_t wait_for_previous()   // before this chunk's first DP launch
    {
        if (!e->is_sub || !e->parent || waited) return cudaSuccess;
        waited = true;
        if (e->chunk_index <= 0) return cudaSuccess;
        phmm_engine::OrderState& st = e->parent->order;
        {
            std::unique_lock<std::mutex> lk(st.m);
            st.cv.wait(lk, [&] { return st.recorded >= e->chunk_index - 1; });
        }
        return cudaStreamWaitEvent(e->stream, e->peer->order_ev, 0);
    }
    void publish(bool record)         // after this chunk's last DP launch (or on any exit)
    {
        if (!e->is_sub || !e->parent || recorded) return;
        recorded = true;
        if (record) cudaEventRecord(e->order_ev, e->stream);
        phmm_engine::OrderState& st = e->parent->order;
        { std::lock_guard<std::mutex> lk(st.m); st.recorded = std::max(st.recorded, e->chunk_index); }
        st.cv.notify_all();
    }
    ~ChunkOrder() { publish(false); }
};

#define CU(call)                                                                                   \
    do {                                                                                           \
        cudaError_t _e = (call);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            e->err = std::string(#call) + ": " + cudaGetErrorString(_e);                           \
            return _e == cudaErrorMemoryAllocation ? PHMM_ERR_NOMEM : PHMM_ERR_CUDA;               \
        }                                                                                          \
    } while (0)

#define LAUNCHED() do { ++e->launches_last; ++e->launches_total; } while (0)

namespace {

// Bring one caller array into device memory (copy for host space, alias for device space).
template <typename T>
int stage(phmm_engine* e, DBuf& buf, const T* src, size_t count, int space, const T** dev)
{
    if (src == nullptr) { *dev = nullptr; return PHMM_OK; }
    if (space == PHMM_SPACE_DEVICE) { *dev = src; return PHMM_OK; }
    CU(buf.ensure(std::max<size_t>(count, 1) * sizeof(T)));
    if (count) CU(cudaMemcpyAsync(buf.p, src, count * sizeof(T), cudaMemcpyHostToDevice, e->stream));
    *dev = buf.as<T>();
    return PHMM_OK;
}

struct Staged {
    DevHaps hp {};
    DevReads rd {};
    long long hap_bases = 0, read_bases = 0;
    std::vector<long long> hap_off_host;                  // haplotype offsets on the host (sizes, window checks); H + 1 entries
    long long max_hap_len = 0;                            // the longest haplotype (mapper limits and variant, DP task word)
    long long read_len_min = 0, read_len_max = 0;         // all the host needs to know about the (possibly millions of) reads
};

int fetch_offsets(phmm_engine* e, const int64_t* off, int n, int space, std::vector<long long>& out)
{
    out.resize((size_t)n + 1);
    if (space == PHMM_SPACE_HOST) {
        for (int i = 0; i <= n; ++i) out[i] = off[i];
    } else {
        static_assert(sizeof(long long) == sizeof(int64_t), "");
        CU(cudaMemcpyAsync(out.data(), off, ((size_t)n + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, e->stream));
        CU(cudaStreamSynchronize(e->stream));
    }
    return PHMM_OK;
}

// Upload (or alias) the batch and run the preparation kernels: column tables, row half-words, read info. The haplotypes live in
// hap_space (< 0: `space`, the reads'): a populate call with an error model hands over the arrays it derived on the device, and
// the haplotype offsets it already holds on the host (hap_off_host, else they are fetched).
int stage_batch(phmm_engine* e, const phmm_haplotypes* haps, const phmm_reads* reads, int space, Staged& s, bool need_info_host = true,
                bool defer_flag_check = false, int hap_space = -1, const std::vector<long long>* hap_off_host = nullptr)
{
    int rc;
    if (hap_space < 0) hap_space = space;
    if ((rc = phmm_checks::blocks(haps, reads, e->err)) != PHMM_OK) return rc;
    if (hap_off_host) s.hap_off_host = *hap_off_host;
    else if ((rc = fetch_offsets(e, haps->off, haps->n, hap_space, s.hap_off_host)) != PHMM_OK) return rc;
    for (int h = 0; h < haps->n; ++h) s.max_hap_len = std::max(s.max_hap_len, s.hap_off_host[h + 1] - s.hap_off_host[h]);
    OffsetSummary rs {};
    if (space == PHMM_SPACE_HOST) {
        const int64_t* off = reads->off;
        long long lo, hi;
        phmm_checks::read_length_range(reads, &lo, &hi);
        rs.first = off[0]; rs.last = off[reads->n]; rs.len_max = hi; rs.inv_len_min = kOffsetBig - lo;
    } else {
        // device-resident offsets: reduce them where they are instead of copying the array back
        CU(e->scores.ensure(sizeof(OffsetSummary)));
        CU(cudaMemsetAsync(e->scores.p, 0, sizeof(OffsetSummary), e->stream));
        k_offsets_summary<<<(unsigned)std::min<long long>(((long long)reads->n + 255) / 256, 1024), 256, 0, e->stream>>>((const long long*)reads->off, reads->n,
                                                                                                                          e->scores.as<OffsetSummary>());
        LAUNCHED();
        CU(cudaMemcpyAsync(&rs, e->scores.p, sizeof(OffsetSummary), cudaMemcpyDeviceToHost, e->stream));
        CU(cudaStreamSynchronize(e->stream));
    }
    s.hap_bases = s.hap_off_host[haps->n];
    s.read_bases = rs.last;
    s.read_len_min = kOffsetBig - rs.inv_len_min;
    s.read_len_max = rs.len_max;
    if ((rc = phmm_checks::offsets(s.hap_off_host[0], s.hap_bases, rs.first, s.read_bases, s.read_len_min, s.read_len_max, e->err)) != PHMM_OK) return rc;
    DevHaps& hp = s.hp;
    DevReads& rd = s.rd;
    hp.n = haps->n; rd.n = reads->n;
    const long long* tmp_ll;
    if ((rc = stage(e, e->h_off, (const long long*)haps->off, (size_t)haps->n + 1, hap_space, &tmp_ll))) return rc; hp.off = tmp_ll;
    if ((rc = stage(e, e->h_seq, haps->seq, s.hap_bases, hap_space, &hp.seq))) return rc;
    if ((rc = stage(e, e->h_mf, haps->snv_mask_fwd, s.hap_bases, hap_space, &hp.mask_f))) return rc;
    if ((rc = stage(e, e->h_pf, haps->snv_prior_fwd, s.hap_bases, hap_space, &hp.prior_f))) return rc;
    if ((rc = stage(e, e->h_mr, haps->snv_mask_rev, s.hap_bases, hap_space, &hp.mask_r))) return rc;
    if ((rc = stage(e, e->h_pr, haps->snv_prior_rev, s.hap_bases, hap_space, &hp.prior_r))) return rc;
    if ((rc = stage(e, e->h_go, haps->gap_open, s.hap_bases, hap_space, &hp.gap_open))) return rc;
    if ((rc = stage(e, e->h_ge, haps->gap_extend, s.hap_bases, hap_space, &hp.gap_extend))) return rc;
    if ((rc = stage(e, e->h_begin, (const long long*)haps->begin, haps->n, hap_space, &tmp_ll))) return rc; hp.begin = tmp_ll;
    if ((rc = stage(e, e->r_off, (const long long*)reads->off, (size_t)reads->n + 1, space, &tmp_ll))) return rc; rd.off = tmp_ll;
    if ((rc = stage(e, e->r_bases, reads->bases, s.read_bases, space, &rd.bases))) return rc;
    if ((rc = stage(e, e->r_quals, reads->quals, s.read_bases, space, &rd.quals))) return rc;
    if ((rc = stage(e, e->r_mapq, reads->mapq, reads->n, space, &rd.mapq))) return rc;
    if ((rc = stage(e, e->r_rev, reads->reverse, reads->n, space, &rd.reverse))) return rc;
    if ((rc = stage(e, e->r_begin, (const long long*)reads->begin, reads->n, space, &tmp_ll))) return rc; rd.begin = tmp_ll;

    CU(e->tab_f.ensure((size_t)s.hap_bases * sizeof(ColEntry)));
    CU(e->tab_r.ensure((size_t)s.hap_bases * sizeof(ColEntry)));
    CU(e->rowhalf.ensure((size_t)s.read_bases * sizeof(uint16_t)));
    CU(e->info.ensure((size_t)rd.n * sizeof(int2)));
    CU(e->flags.ensure(64));
    CU(cudaMemsetAsync(e->flags.p, 0, 64, e->stream));
    k_build_tables<<<(unsigned)((s.hap_bases + 255) / 256), 256, 0, e->stream>>>(s.hap_bases, hp.seq, hp.mask_f, hp.prior_f, hp.mask_r, hp.prior_r,
                                                                                 hp.gap_open, hp.gap_extend, e->tab_f.as<ColEntry>(),
                                                                                 e->tab_r.as<ColEntry>(), e->flags.as<int>());
    LAUNCHED();
    k_read_info<<<(unsigned)(((long long)rd.n * 32 + 255) / 256), 256, 0, e->stream>>>(rd.n, rd.off, rd.bases, rd.quals, e->rowhalf.as<uint16_t>(),
                                                                                       e->info.as<int2>());
    LAUNCHED();
    CU(cudaGetLastError());
    hp.tab_f = e->tab_f.as<ColEntry>(); hp.tab_r = e->tab_r.as<ColEntry>();
    rd.rowhalf = e->rowhalf.as<uint16_t>(); rd.info = e->info.as<int2>();
    // read info is needed on the host where the host schedules (8 bytes per read); phmm_populate schedules on the device
    if (need_info_host) {
        e->info_host.resize(rd.n);
        CU(cudaMemcpyAsync(e->info_host.data(), e->info.p, (size_t)rd.n * sizeof(int2), cudaMemcpyDeviceToHost, e->stream));
    }
    if (defer_flag_check) return PHMM_OK;   // the caller reads flags bit 0 at its own final synchronisation
    int flags_host[1] = {0};
    CU(cudaMemcpyAsync(flags_host, e->flags.p, sizeof(int), cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    if (flags_host[0] & 1) {
        e->err = "snv prior / gap penalty outside [0,127]";
        return PHMM_ERR_INVALID;
    }
    return PHMM_OK;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize belongs to the (device, kernel) pair, not to an engine: several engines of one process
// (the two pipeline sub-engines, an application's own) share it, and setting it to a smaller value LOWERS the limit another engine's
// next launch relies on. So the high-water mark is kept per process and the attribute is only ever raised.
template <typename F>
int fast_smem_attr(phmm_engine* e, F kernel, size_t bytes)
{
    static std::mutex mu;
    static std::map<std::pair<int, const void*>, size_t> high_water;
    std::lock_guard<std::mutex> lock(mu);
    size_t& have = high_water[std::make_pair(e->device, (const void*)kernel)];
    if (bytes <= have) return PHMM_OK;
    CU(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    have = bytes;
    return PHMM_OK;
}

template <typename F>
int blocks_per_sm_of(phmm_engine* e, F kernel, int threads, size_t smem, int* out)
{
    const auto key = std::make_pair((const void*)kernel, smem);
    const auto it = e->occupancy.find(key);
    if (it != e->occupancy.end()) { *out = it->second; return PHMM_OK; }
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(out, kernel, threads, smem));
    e->occupancy[key] = *out;
    return PHMM_OK;
}

// What a kernel with dynamic shared memory needs before its grid can be sized: the attribute raised, its resident blocks per SM.
template <typename F>
int prepare_kernel(phmm_engine* e, F kernel, int threads, size_t smem, int* blocks_per_sm)
{
    const int rc = fast_smem_attr(e, kernel, smem);
    return rc != PHMM_OK ? rc : blocks_per_sm_of(e, kernel, threads, smem, blocks_per_sm);
}

// Runtime value → template argument. Each helper below hands f one std::integral_constant (or Type) per template parameter and
// returns what f returns; it lists exactly the instantiations its kernels exist for, so a launch site cannot ask for another.
template <int V> using Int = std::integral_constant<int, V>;
template <typename T> struct Type { using type = T; };

// f(Int<B>) for the band among B, Rest...; the last one listed takes every other band
template <int B, int... Rest, typename F>
auto with_band_in(int band, F&& f)
{
    if constexpr (sizeof...(Rest) == 0) return f(Int<B> {});
    else return band == B ? f(Int<B> {}) : with_band_in<Rest...>(band, f);
}
template <typename F> auto with_band(int band, F&& f) { return with_band_in<8, 16, 32, 64, 128, 256>(band, f); }

// the 32-bit multi-lane kernels (k_wide_tasks, k_populate_wide): f(Int<C>, Int<NL>), chunk and lanes by band
template <typename F>
auto with_wide_shape(int band, F&& f)
{
    switch (band) {
        case 8: return f(Int<16> {}, Int<1> {});  case 16: return f(Int<32> {}, Int<1> {});  case 32: return f(Int<32> {}, Int<2> {});
        case 64: return f(Int<32> {}, Int<4> {}); case 128: return f(Int<32> {}, Int<8> {}); default: return f(Int<32> {}, Int<16> {});
    }
}

// k_populate_fast: f(Int<B>, Int<G>) for the band and the lane groups per warp (band 256 has room for two groups at most)
template <typename F>
auto with_fast_shape(int band, int groups, F&& f)
{
    switch (band * 10 + groups) {
        case 81: return f(Int<8> {}, Int<1> {});     case 82: return f(Int<8> {}, Int<2> {});     case 84: return f(Int<8> {}, Int<4> {});
        case 161: return f(Int<16> {}, Int<1> {});   case 162: return f(Int<16> {}, Int<2> {});   case 164: return f(Int<16> {}, Int<4> {});
        case 321: return f(Int<32> {}, Int<1> {});   case 322: return f(Int<32> {}, Int<2> {});   case 324: return f(Int<32> {}, Int<4> {});
        case 641: return f(Int<64> {}, Int<1> {});   case 642: return f(Int<64> {}, Int<2> {});   case 644: return f(Int<64> {}, Int<4> {});
        case 1281: return f(Int<128> {}, Int<1> {}); case 1282: return f(Int<128> {}, Int<2> {}); case 1284: return f(Int<128> {}, Int<4> {});
        case 2561: return f(Int<256> {}, Int<1> {}); default: return f(Int<256> {}, Int<2> {});
    }
}

// the k-mer mappers: f(Int<MAXT>, Type<CountT>), the vote-array capacity by the longest haplotype (longer ones: tiles of 2048
// diagonals) and byte counters when no read can cast more than 255 votes
template <typename F>
auto with_mapper_variant(const Staged& s, F&& f)
{
    const bool bytes = s.read_len_max - kKmer + 1 <= 255;
    if (s.max_hap_len - kKmer + 1 <= 512) return bytes ? f(Int<512> {}, Type<uint8_t> {}) : f(Int<512> {}, Type<uint16_t> {});
    return bytes ? f(Int<2048> {}, Type<uint8_t> {}) : f(Int<2048> {}, Type<uint16_t> {});
}

// First statement of every computing entry point: no stale error, the per-call counters at zero, the engine's device selected.
int begin_call(phmm_engine* e)
{
    if (!e) return PHMM_ERR_INVALID;
    e->err.clear(); e->launches_last = 0; e->last_dp_ms = 0.0; e->last_dp_cells = 0;
    if (cudaSetDevice(e->device) != cudaSuccess) { e->err = "cudaSetDevice failed"; return PHMM_ERR_CUDA; }
    return PHMM_OK;
}

// The (read, haplotype) indices of a host-space pair list: checked where they are cheap to read.
int check_pairs(phmm_engine* e, const phmm_pair* pairs, int n, const Staged& s)
{
    return phmm_checks::pair_indices(pairs, n, s.hp.n, s.rd.n, e->err);
}

// A caller's candidate positions, a CSR over n lists, on the device (copied for host space, aliased for device space); *total = off[n].
int stage_positions(phmm_engine* e, const phmm_positions* positions, long long n, int space, const long long** off, const int32_t** pos, long long* total)
{
    int rc;
    if (space == PHMM_SPACE_HOST) *total = positions->off[n];
    else { CU(cudaMemcpyAsync(total, positions->off + n, sizeof(int64_t), cudaMemcpyDeviceToHost, e->stream)); CU(cudaStreamSynchronize(e->stream)); }
    if ((rc = stage(e, e->c_off, (const long long*)positions->off, (size_t)n + 1, space, off))) return rc;
    return stage(e, e->c_pos, positions->pos, (size_t)std::max<long long>(*total, 1), space, pos);
}

// What both k-mer mappers (the uncapped one over a pair list, populate's capped one) read: their limits checked, the k-mer hashes of
// the reads, the k-mer tables of the haplotypes.
int prepare_mapper(phmm_engine* e, const Staged& s)
{
    const int rc = phmm_checks::mapper_haplotypes(s.max_hap_len, s.hap_bases, e->err);
    if (rc != PHMM_OK) return rc;
    const int R = s.rd.n, H = s.hp.n;
    CU(e->rhash.ensure((size_t)s.read_bases * sizeof(uint16_t)));
    CU(e->kbins.ensure((size_t)H * (kKmerBins + 1) * sizeof(int)));
    CU(e->kitems.ensure((size_t)s.hap_bases * sizeof(uint16_t)));
    k_read_kmers<<<(unsigned)(((long long)R * 32 + 255) / 256), 256, 0, e->stream>>>(s.read_bases, R, s.rd.off, s.rd.bases, e->rhash.as<uint16_t>());
    LAUNCHED();
    k_build_kmer_table<<<H, 256, 0, e->stream>>>(H, s.hp.off, s.hp.seq, e->kbins.as<uint32_t>(), e->kitems.as<uint16_t>());
    LAUNCHED();
    CU(cudaGetLastError());
    return PHMM_OK;
}

// One pass of the uncapped pair mapper. Counting (EMIT false): per pair the maximum and how many mapping begins reach it, *bad set by a
// pair index out of range. Emitting: every mapping begin of pair j into pos_dev[off_dev[j] ..).
template <bool EMIT>
void pair_map_pass(phmm_engine* e, const Staged& s, const int2* d_pairs, int n, int* bad, const long long* off_dev, int32_t* pos_dev)
{
    const unsigned grid = (unsigned)((n + 127) / 128);
    with_mapper_variant(s, [&](auto maxt, auto count) {
        k_kmer_map_pairs<decltype(maxt)::value, typename decltype(count)::type, EMIT><<<grid, 128, 0, e->stream>>>(
            n, d_pairs, s.hp, s.rd, e->rhash.as<uint16_t>(), e->kbins.as<uint32_t>(), e->kitems.as<uint16_t>(), e->pm_best.as<unsigned>(),
            e->pm_cnt.as<int>(), e->pm_inl.as<int32_t>(), bad, off_dev, pos_dev);
    });
    LAUNCHED();
}

} // namespace

extern "C" {

const char* phmm_version(void) { return "octopus_b200 phmm 0.1 (sm_90a)"; }

void phmm_default_config(phmm_config* c)
{
    if (!c) return;
    c->max_indel_error = 8;                 // HaplotypeLikelihoodModel::Config defaults, haplotype_likelihood_model.hpp:36-44
    c->use_int_scores = 0;
    c->use_mapping_quality = 1;
    c->mapping_quality_cap = 120;
    c->mapping_quality_cap_trigger = -1;
    c->use_flank_state = 1;
    c->nuc_prior = 2;
    c->disable_naive_shortcut = 0;
    c->map_positions = 1;
}

static std::string g_create_error;

int phmm_create(phmm_engine** out, int device)
{
    if (!out) return PHMM_ERR_INVALID;
    *out = nullptr;
    int count = 0;
    cudaError_t ce = cudaGetDeviceCount(&count);
    if (ce != cudaSuccess || count == 0) {
        g_create_error = std::string("no CUDA device: ") + (ce != cudaSuccess ? cudaGetErrorString(ce) : "device count 0");
        return PHMM_ERR_CUDA;
    }
    if (device < 0) { if (cudaGetDevice(&device) != cudaSuccess) device = 0; }
    if (device >= count) { g_create_error = "device ordinal out of range"; return PHMM_ERR_INVALID; }
    if (cudaSetDevice(device) != cudaSuccess) { g_create_error = "cudaSetDevice failed"; return PHMM_ERR_CUDA; }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { g_create_error = "cudaGetDeviceProperties failed"; return PHMM_ERR_CUDA; }
    if (prop.major != 9 || prop.minor != 0) {   // sm_90a code loads on compute capability 9.0 only
        g_create_error = "this library is built for sm_90a (H100) only; found compute capability " + std::to_string(prop.major) + "." + std::to_string(prop.minor);
        return PHMM_ERR_CUDA;
    }
    phmm_engine* e = new phmm_engine();
    e->device = device;
    e->sm_count = prop.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreate(&e->ev0) != cudaSuccess || cudaEventCreate(&e->ev1) != cudaSuccess) {
        g_create_error = "stream / event creation failed";
        delete e;
        return PHMM_ERR_CUDA;
    }
    *out = e;
    return PHMM_OK;
}

void phmm_destroy(phmm_engine* e)
{
    if (!e) return;
    for (phmm_engine*& sub : e->sub) { if (sub) phmm_destroy(sub); sub = nullptr; }
    cudaSetDevice(e->device);
    for (cudaEvent_t ev : e->tile_events) cudaEventDestroy(ev);
    if (e->ev0) cudaEventDestroy(e->ev0);
    if (e->ev1) cudaEventDestroy(e->ev1);
    if (e->order_ev) cudaEventDestroy(e->order_ev);
    if (e->stream) cudaStreamDestroy(e->stream);
    delete e;       // frees every DBuf, on the device selected above
}

const char* phmm_last_error(const phmm_engine* e) { return e ? e->err.c_str() : g_create_error.c_str(); }

// Ordering against the caller's streams. Every call runs on the engine's own stream and is complete on return; what a caller
// cannot express that way is "the buffer this call will WRITE is still being read by work I enqueued earlier on another stream"
// (a gather of the previous result). phmm_wait_event makes the engine's stream(s) wait, on the device, for that work.
int phmm_wait_event(phmm_engine* e, void* cuda_event)
{
    if (!e || !cuda_event) return PHMM_ERR_INVALID;
    if (cudaSetDevice(e->device) != cudaSuccess) { e->err = "cudaSetDevice failed"; return PHMM_ERR_CUDA; }
    CU(cudaStreamWaitEvent(e->stream, (cudaEvent_t)cuda_event, 0));
    for (phmm_engine* sub : e->sub) if (sub) CU(cudaStreamWaitEvent(sub->stream, (cudaEvent_t)cuda_event, 0));
    return PHMM_OK;
}
void* phmm_engine_stream(phmm_engine* e) { return e ? (void*)e->stream : nullptr; }

int phmm_reserve_sms(phmm_engine* e, int n_sms)
{
    if (!e || n_sms < 0) return PHMM_ERR_INVALID;
    e->reserved_sms = std::min(n_sms, std::max(0, e->sm_count - 1));
    for (phmm_engine* sub : e->sub) if (sub) sub->reserved_sms = e->reserved_sms;
    return PHMM_OK;
}

// Page-locked host memory for callers without the CUDA headers (the C++ adapter's blocks): a PHMM_SPACE_HOST call copies from /
// to pinned buffers at full PCIe / C2C rate and overlaps with compute; pageable memory is staged by the driver.
void* phmm_host_alloc(size_t bytes)
{
    void* p = nullptr;
    if (bytes == 0) bytes = 1;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
void phmm_host_free(void* p) { if (p) cudaFreeHost(p); }

int64_t phmm_launch_count(const phmm_engine* e, int total) { return e ? (total ? e->launches_total : e->launches_last) : 0; }
double phmm_last_dp_kernel_ms(const phmm_engine* e) { return e ? e->last_dp_ms : 0.0; }
int64_t phmm_last_dp_cells(const phmm_engine* e) { return e ? e->last_dp_cells : 0; }

// -------------------------------------------------------------------------------------------------------------
// phmm_align_scores
// -------------------------------------------------------------------------------------------------------------
int phmm_align_scores(phmm_engine* e, int band, int precision_bits, int nuc_prior,
                      const phmm_haplotypes* haps, const phmm_reads* reads,
                      const phmm_task* tasks, int64_t n_tasks, int32_t* scores, int space)
{
    if (int rc0 = begin_call(e)) return rc0;
    if (band > 256) { e->err = "band > 256"; return PHMM_ERR_BAND; }
    if (band < 8 || (band & (band - 1))) { e->err = "band must be one of 8,16,...,256"; return PHMM_ERR_INVALID; }
    if (precision_bits != 16 && precision_bits != 32) { e->err = "precision_bits must be 16 or 32"; return PHMM_ERR_INVALID; }
    if (nuc_prior < 0 || nuc_prior > 127) { e->err = "nuc_prior outside [0,127]"; return PHMM_ERR_INVALID; }
    if (n_tasks < 0 || n_tasks > 0x7fffffff) { e->err = "task count out of range"; return PHMM_ERR_INVALID; }
    if (n_tasks == 0) return PHMM_OK;
    if (!tasks || !scores) { e->err = "null tasks / scores"; return PHMM_ERR_INVALID; }
    Staged s;
    int rc = stage_batch(e, haps, reads, space, s);
    if (rc != PHMM_OK) return rc;
    // tasks on the host for scheduling
    std::vector<phmm_task> th;
    const phmm_task* tk = tasks;
    if (space == PHMM_SPACE_DEVICE) {
        th.resize(n_tasks);
        CU(cudaMemcpyAsync(th.data(), tasks, (size_t)n_tasks * sizeof(phmm_task), cudaMemcpyDeviceToHost, e->stream));
        CU(cudaStreamSynchronize(e->stream));
        tk = th.data();
    }
    const int n = (int)n_tasks, H = s.hp.n, R = s.rd.n;
    std::vector<int> fast_idx, wide_idx;
    std::vector<GenericTask> gen;
    // packed s16x2 lanes where they are exact (precision 16, ACGT reads whose quality sum fits); 32-bit multi-lane kernel for the
    // rest of the ACGTN reads; thread-per-task generic kernel for foreign bytes / qualities above 127 / reads beyond shared memory
    const int NL = lanes_per_alignment(band), TPR = 32 / NL;
    int64_t cells = 0;
    int Lmax = 1, Lmax_wide = 1;
    for (int j = 0; j < n; ++j) {
        const phmm_task& t = tk[j];
        if (t.read < 0 || t.read >= R || t.hap < 0 || t.hap >= H) { e->err = "task index out of range"; return PHMM_ERR_INVALID; }
        const int L = e->info_host[t.read].x, fl = e->info_host[t.read].y;
        const long long hl = s.hap_off_host[t.hap + 1] - s.hap_off_host[t.hap];
        if (L < 1 || t.win_off < 0 || (long long)t.win_off + L + 2 * band - 1 > hl) { e->err = "task window outside the haplotype"; return PHMM_ERR_INVALID; }
        cells += 2LL * (L + band) * band;
        if (precision_bits == 16 && (fl & (kReadNonACGT | kReadBadQual | kReadUnsafe16 | kReadTooLong | kReadHasN)) == 0) { fast_idx.push_back(j); Lmax = std::max(Lmax, L); }
        else if ((fl & (kReadNonACGT | kReadBadQual)) == 0 && L <= kWideMaxReadLen) { wide_idx.push_back(j); Lmax_wide = std::max(Lmax_wide, L); }
        else gen.push_back(GenericTask {t.read, t.hap, t.win_off, t.reverse ? 1 : 0, j});
    }
    e->last_dp_cells = cells;
    CU(e->scores.ensure((size_t)n * sizeof(int)));
    int* d_scores = space == PHMM_SPACE_DEVICE ? scores : e->scores.as<int>();
    auto by_length_and_read = [&](int a, int b) {
        const int la = e->info_host[tk[a].read].x, lb = e->info_host[tk[b].read].x;
        if (la != lb) return la < lb;
        if (tk[a].read != tk[b].read) return tk[a].read < tk[b].read;
        return a < b;
    };
    struct Chunk { int read, first, n, L; };
    bool have_ev0 = false;

    if (!fast_idx.empty()) {
        // group by (length, read); chunks of 32 / NL tasks of one read; chunks of equal length are paired into one warp
        std::sort(fast_idx.begin(), fast_idx.end(), by_length_and_read);
        std::vector<LaneTask> lane(fast_idx.size());
        std::vector<Chunk> chunks;
        for (size_t i = 0; i < fast_idx.size(); ++i) {
            const phmm_task& t = tk[fast_idx[i]];
            lane[i] = LaneTask {s.hap_off_host[t.hap] + t.win_off, t.reverse ? 1 : 0, fast_idx[i]};
            if (chunks.empty() || chunks.back().read != t.read || chunks.back().n == TPR)
                chunks.push_back(Chunk {t.read, (int)i, 0, e->info_host[t.read].x});
            ++chunks.back().n;
        }
        std::vector<WarpWork> works;
        for (size_t c = 0; c < chunks.size();) {
            WarpWork w {};
            w.read0 = chunks[c].read; w.first0 = chunks[c].first; w.n0 = chunks[c].n; w.L = chunks[c].L;
            w.read1 = -1; w.first1 = chunks[c].first; w.n1 = 0;
            if (c + 1 < chunks.size() && chunks[c + 1].L == w.L) {
                w.read1 = chunks[c + 1].read; w.first1 = chunks[c + 1].first; w.n1 = chunks[c + 1].n;
                c += 2;
            } else c += 1;
            works.push_back(w);
        }
        CU(e->tasks_lane.ensure(lane.size() * sizeof(LaneTask)));
        CU(e->works.ensure(works.size() * sizeof(WarpWork)));
        CU(cudaMemcpyAsync(e->tasks_lane.p, lane.data(), lane.size() * sizeof(LaneTask), cudaMemcpyHostToDevice, e->stream));
        CU(cudaMemcpyAsync(e->works.p, works.data(), works.size() * sizeof(WarpWork), cudaMemcpyHostToDevice, e->stream));
        const int row_stride = (Lmax + 2) & ~1;
        const size_t smem = (size_t)kFastWarpsPerBlock * row_stride * sizeof(RowEntry);
        const int nw = (int)works.size();
        const unsigned grid = (unsigned)((nw + kFastWarpsPerBlock - 1) / kFastWarpsPerBlock);
        const uint32_t nucp = (uint32_t)nuc_prior | ((uint32_t)nuc_prior << 16);
        CU(cudaEventRecord(e->ev0, e->stream)); have_ev0 = true;
        rc = with_band(band, [&](auto b) -> int {
            constexpr int B = decltype(b)::value;
            if (int arc = fast_smem_attr(e, k_packed_tasks<B>, smem)) return arc;
            k_packed_tasks<B><<<grid, kFastWarpsPerBlock * 32, smem, e->stream>>>(e->works.as<WarpWork>(), nw, e->tasks_lane.as<LaneTask>(), s.hp, s.rd, row_stride, nucp, d_scores, e->flags.as<int>(), 1u);
            return PHMM_OK;
        });
        if (rc != PHMM_OK) return rc;
        LAUNCHED();
        CU(cudaEventRecord(e->ev1, e->stream));
        CU(cudaGetLastError());
    }
    if (!wide_idx.empty()) {
        std::sort(wide_idx.begin(), wide_idx.end(), by_length_and_read);
        std::vector<LaneTask> lane(wide_idx.size());
        std::vector<WarpWork> works;
        for (size_t i = 0; i < wide_idx.size(); ++i) {
            const phmm_task& t = tk[wide_idx[i]];
            lane[i] = LaneTask {s.hap_off_host[t.hap] + t.win_off, t.reverse ? 1 : 0, wide_idx[i]};
            if (works.empty() || works.back().read0 != t.read || works.back().n0 == TPR) {
                WarpWork w {};
                w.read0 = t.read; w.read1 = -1; w.first0 = (int)i; w.n0 = 0; w.first1 = (int)i; w.n1 = 0; w.L = e->info_host[t.read].x;
                works.push_back(w);
            }
            ++works.back().n0;
        }
        CU(e->ftasks.ensure(lane.size() * sizeof(LaneTask)));
        CU(e->gtasks.ensure(works.size() * sizeof(WarpWork)));
        CU(cudaMemcpyAsync(e->ftasks.p, lane.data(), lane.size() * sizeof(LaneTask), cudaMemcpyHostToDevice, e->stream));
        CU(cudaMemcpyAsync(e->gtasks.p, works.data(), works.size() * sizeof(WarpWork), cudaMemcpyHostToDevice, e->stream));
        const int row_stride = (Lmax_wide + 2) & ~1;
        const int warps = (int)std::max<long long>(1, std::min<long long>(kFastWarpsPerBlock, (220LL << 10) / ((long long)row_stride * (long long)sizeof(RowEntry))));
        const size_t smem = (size_t)warps * row_stride * sizeof(RowEntry);
        const int nw = (int)works.size();
        const unsigned grid = (unsigned)((nw + warps - 1) / warps);
        if (!have_ev0) { CU(cudaEventRecord(e->ev0, e->stream)); have_ev0 = true; }
        rc = with_wide_shape(band, [&](auto c, auto nl) -> int {
            constexpr int C = decltype(c)::value, N = decltype(nl)::value;
            if (int arc = fast_smem_attr(e, k_wide_tasks<C, N>, smem)) return arc;
            k_wide_tasks<C, N><<<grid, warps * 32, smem, e->stream>>>(e->gtasks.as<WarpWork>(), nw, e->ftasks.as<LaneTask>(), s.hp, s.rd, row_stride, nuc_prior, d_scores, e->flags.as<int>());
            return PHMM_OK;
        });
        if (rc != PHMM_OK) return rc;
        LAUNCHED();
        CU(cudaEventRecord(e->ev1, e->stream));
        CU(cudaGetLastError());
    }
    if (!gen.empty()) {
        CU(e->tasks_generic.ensure(gen.size() * sizeof(GenericTask)));
        CU(cudaMemcpyAsync(e->tasks_generic.p, gen.data(), gen.size() * sizeof(GenericTask), cudaMemcpyHostToDevice, e->stream));
        const int ng = (int)gen.size();
        if (!have_ev0) CU(cudaEventRecord(e->ev0, e->stream));
        if (band <= 32) k_generic_tasks<64><<<(ng + 63) / 64, 64, 0, e->stream>>>(e->tasks_generic.as<GenericTask>(), ng, s.hp, s.rd, band, nuc_prior, d_scores);
        else k_generic_tasks<kGenericMaxDiag><<<(ng + 63) / 64, 64, 0, e->stream>>>(e->tasks_generic.as<GenericTask>(), ng, s.hp, s.rd, band, nuc_prior, d_scores);
        LAUNCHED();
        if (!have_ev0) CU(cudaEventRecord(e->ev1, e->stream));
        CU(cudaGetLastError());
    }
    if (space == PHMM_SPACE_HOST) CU(cudaMemcpyAsync(scores, d_scores, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, e->ev0, e->ev1) == cudaSuccess) e->last_dp_ms = ms;
    return PHMM_OK;
}

// -------------------------------------------------------------------------------------------------------------
// phmm_align_traceback
// -------------------------------------------------------------------------------------------------------------
int phmm_align_traceback(phmm_engine* e, int band,
                         const char* truth, const char* target, const int8_t* quals, int truth_len, int target_len,
                         const char* snv_mask, const int8_t* snv_prior, const int8_t* gap_open,
                         const int8_t* gap_extend, int gap_extend_scalar, int nuc_prior,
                         int* score, int* first_pos, char* align1, char* align2)
{
    if (int rc0 = begin_call(e)) return rc0;
    if (band > 256) { e->err = "band > 256"; return PHMM_ERR_BAND; }
    if (band < 1 || !truth || !target || !quals || !gap_open || !score || !first_pos || !align1 || !align2 ||
        target_len < 1 || truth_len != target_len + 2 * band - 1) {
        e->err = "bad argument (truth_len must be target_len + 2*band - 1)";
        return PHMM_ERR_INVALID;
    }
    if (snv_mask && !snv_prior) { e->err = "snv_mask given without snv_prior"; return PHMM_ERR_INVALID; }
    const int W = truth_len, L = target_len;
    std::vector<char> host((size_t)5 * W + 2 * L);
    std::memcpy(host.data(), truth, W);
    if (snv_mask) { std::memcpy(host.data() + W, snv_mask, W); std::memcpy(host.data() + 2 * W, snv_prior, W); }
    else { std::memset(host.data() + W, 0, W); std::memset(host.data() + 2 * W, 127, W); }   // a mask byte no base equals
    std::memcpy(host.data() + 3 * W, gap_open, W);
    if (gap_extend) std::memcpy(host.data() + 4 * W, gap_extend, W); else std::memset(host.data() + 4 * W, gap_extend_scalar, W);
    std::memcpy(host.data() + 5 * W, target, L);
    std::memcpy(host.data() + 5 * W + L, quals, L);
    const size_t nal = (size_t)2 * (L + band) + 1, nbp = (size_t)(L + 1) * 2 * band;
    CU(e->tasks_generic.ensure(host.size()));
    CU(e->bp.ensure(nbp + 2 * nal + 64));
    CU(e->scores.ensure(2 * sizeof(int)));
    CU(cudaMemcpyAsync(e->tasks_generic.p, host.data(), host.size(), cudaMemcpyHostToDevice, e->stream));
    CU(cudaMemsetAsync(e->bp.p, 0, nbp + 2 * nal, e->stream));
    unsigned char* bp = e->bp.as<unsigned char>();
    k_align_one<<<1, 32, 0, e->stream>>>(band, L, e->tasks_generic.as<char>(), nuc_prior, bp, e->scores.as<int>(), (char*)bp + nbp, (char*)bp + nbp + nal);
    LAUNCHED();
    CU(cudaGetLastError());
    int out[2];
    CU(cudaMemcpyAsync(out, e->scores.p, sizeof(out), cudaMemcpyDeviceToHost, e->stream));
    CU(cudaMemcpyAsync(align1, bp + nbp, nal, cudaMemcpyDeviceToHost, e->stream));
    CU(cudaMemcpyAsync(align2, bp + nbp + nal, nal, cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    *score = out[0]; *first_pos = out[1];
    return PHMM_OK;
}

// -------------------------------------------------------------------------------------------------------------
// phmm_genotype_likelihoods
// -------------------------------------------------------------------------------------------------------------
int phmm_genotype_likelihoods(phmm_engine* e, const double* lnl, int32_t H, int32_t R,
                              const int32_t* genotypes, int32_t G, int32_t ploidy, double* out, int space)
{
    if (int rc0 = begin_call(e)) return rc0;
    if (!lnl || H <= 0 || R <= 0 || G < 0 || ploidy < 0 || ploidy > 64) { e->err = "bad argument"; return PHMM_ERR_INVALID; }
    if (G == 0) return PHMM_OK;       // empty arrays may come as null pointers (an empty torch tensor's data pointer)
    if (!out || (!genotypes && ploidy > 0)) { e->err = "bad argument"; return PHMM_ERR_INVALID; }
    if (ploidy == 0) {   // the empty genotype's likelihood is 0 (ln 1) whatever the reads; nothing is read
        if (space == PHMM_SPACE_HOST) { std::fill(out, out + G, 0.0); return PHMM_OK; }
        CU(cudaMemsetAsync(out, 0, (size_t)G * sizeof(double), e->stream));
        CU(cudaStreamSynchronize(e->stream));
        return PHMM_OK;
    }
    const double* d_lnl; const int32_t* d_gt;
    int rc;
    if (space == PHMM_SPACE_HOST) {   // haplotype indices are checked where they are cheap to read (the kernel checks device ones)
        for (long long i = 0; i < (long long)G * ploidy; ++i) if (genotypes[i] < 0 || genotypes[i] >= H) { e->err = "haplotype index out of range"; return PHMM_ERR_INVALID; }
    }
    if ((rc = stage(e, e->out, lnl, (size_t)H * R, space, &d_lnl))) return rc;
    if ((rc = stage(e, e->pairs, genotypes, (size_t)G * ploidy, space, &d_gt))) return rc;
    CU(e->scores.ensure((size_t)G * sizeof(double)));
    CU(e->counters.ensure(sizeof(int)));
    CU(cudaMemsetAsync(e->counters.p, 0, sizeof(int), e->stream));
    double* d_out = space == PHMM_SPACE_DEVICE ? out : e->scores.as<double>();
    k_genotype_likelihoods<<<G, 256, 0, e->stream>>>(d_lnl, H, R, d_gt, ploidy, d_out, e->counters.as<int>());
    LAUNCHED();
    CU(cudaGetLastError());
    int bad = 0;
    CU(cudaMemcpyAsync(&bad, e->counters.p, sizeof(int), cudaMemcpyDeviceToHost, e->stream));
    if (space == PHMM_SPACE_HOST) CU(cudaMemcpyAsync(out, d_out, (size_t)G * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    if (bad) { e->err = "haplotype index out of range"; return PHMM_ERR_INVALID; }
    return PHMM_OK;
}

// -------------------------------------------------------------------------------------------------------------
// phmm_variational_bayes
// -------------------------------------------------------------------------------------------------------------
// Device memory the seeds' workspaces may take at once: blocks = min(seeds, 2 per SM, this budget / one workspace).
static constexpr size_t kVbWorkspaceBudget = (size_t)2 << 30;
static constexpr int kVbMaxHaplotypes = 50000;   // k_vb_index keeps one int per haplotype in shared memory

int phmm_variational_bayes(phmm_engine* e, const double* lnl, int32_t H, int32_t R, const int64_t* sample_off, int32_t S,
                           const int32_t* genotypes, int32_t G, int32_t K, const double* prior_alphas, const double* genotype_log_priors,
                           const double* seeds, int32_t n_seeds, double epsilon, int32_t max_iterations,
                           double* posteriors, double* log_posteriors, double* alphas, double* weighted_posteriors,
                           double* max_log_evidence, int32_t* max_seed, double* seed_log_evidence, int32_t* seed_iterations, int space)
{
    using namespace phmm::vb;
    if (int rc0 = begin_call(e)) return rc0;
    if (K < 1 || K > kMaxK) { e->err = "K must be in [1, 100]"; return PHMM_ERR_INVALID; }
    if (G < 1 || n_seeds < 1 || S < 1) { e->err = "no genotypes, seeds or samples"; return PHMM_ERR_INVALID; }
    if (max_iterations < 1) { e->err = "max_iterations must be at least 1"; return PHMM_ERR_INVALID; }
    if (H < 1 || H > kVbMaxHaplotypes || R < 0) { e->err = "bad matrix shape (1 <= H <= 50000, R >= 0)"; return PHMM_ERR_INVALID; }
    if ((!lnl && R > 0) || !sample_off || !genotypes || !prior_alphas || !genotype_log_priors || !seeds || !posteriors || !log_posteriors ||
        !alphas || !weighted_posteriors || !max_log_evidence || !max_seed) { e->err = "bad argument"; return PHMM_ERR_INVALID; }
    if (sample_off[0] != 0 || sample_off[S] != R) { e->err = "sample_off must run from 0 to R"; return PHMM_ERR_INVALID; }
    for (int s = 0; s < S; ++s) if (sample_off[s + 1] < sample_off[s]) { e->err = "sample_off decreases"; return PHMM_ERR_INVALID; }
    if (space == PHMM_SPACE_HOST)   // the kernel checks device-space indices
        for (long long i = 0; i < (long long)G * K; ++i) if (genotypes[i] < 0 || genotypes[i] >= H) { e->err = "haplotype index out of range"; return PHMM_ERR_INVALID; }

    const long long KH = (long long)K * H, KG = (long long)K * G, SK = (long long)S * K;
    const double *d_lnl, *d_prior, *d_lp, *d_seeds; const int32_t* d_gt;
    int rc;
    if ((rc = stage(e, e->vb_lnl, lnl, (size_t)H * R, space, &d_lnl))) return rc;
    if ((rc = stage(e, e->vb_gt, genotypes, (size_t)KG, space, &d_gt))) return rc;
    if (space == PHMM_SPACE_HOST) {
        CU(e->vb_in.ensure((SK + G + (size_t)n_seeds * G) * sizeof(double)));
        double* p = e->vb_in.as<double>();
        CU(cudaMemcpyAsync(p, prior_alphas, SK * sizeof(double), cudaMemcpyHostToDevice, e->stream));
        CU(cudaMemcpyAsync(p + SK, genotype_log_priors, G * sizeof(double), cudaMemcpyHostToDevice, e->stream));
        CU(cudaMemcpyAsync(p + SK + G, seeds, (size_t)n_seeds * G * sizeof(double), cudaMemcpyHostToDevice, e->stream));
        d_prior = p; d_lp = p + SK; d_seeds = p + SK + G;
    } else {
        d_prior = prior_alphas; d_lp = genotype_log_priors; d_seeds = seeds;
    }

    // ints: cnt, start, kh [K*H]; nk [K]; L, sid [K*G]; bad; soff [S+1]; first, modes [G]; n_modes, max_seed; map, iters [n_seeds]
    const long long n_int = 3 * KH + K + 2 * KG + 1 + (S + 1) + 2LL * G + 2 + 2LL * n_seeds;
    CU(e->vb_idx.ensure((size_t)n_int * sizeof(int)));
    int* ip = e->vb_idx.as<int>();
    int *cnt = ip, *start = cnt + KH, *kh = start + KH, *nk = kh + KH, *L = nk + K, *sid = L + KG, *bad = sid + KG, *soff = bad + 1,
        *first = soff + S + 1, *modes = first + G, *n_modes = modes + G, *d_max_seed = n_modes + 1, *map = d_max_seed + 1, *iters = map + n_seeds;
    std::vector<int> soff_host(sample_off, sample_off + S + 1);
    CU(cudaMemcpyAsync(soff, soff_host.data(), (S + 1) * sizeof(int), cudaMemcpyHostToDevice, e->stream));
    CU(cudaMemsetAsync(bad, 0, sizeof(int), e->stream));
    CU(cudaMemsetAsync(first, 0x7f, G * sizeof(int), e->stream));   // 0x7f7f7f7f: above every seed index

    // doubles: lpost [n_seeds][G]; ev [n_seeds]; alpha [n_seeds][S][K]; weights [G]; keys [G] (u64)
    const long long n_dbl = (long long)n_seeds * G + n_seeds + n_seeds * SK + 2LL * G;
    CU(e->vb_seed.ensure((size_t)n_dbl * sizeof(double)));
    double* dp = e->vb_seed.as<double>();
    double *lpost = dp, *ev = lpost + (long long)n_seeds * G, *seed_alpha = ev + n_seeds, *weights = seed_alpha + n_seeds * SK,
           *keys = weights + G;
    CU(cudaMemsetAsync(keys, 0, G * sizeof(double), e->stream));

    const long long ws = Workspace::doubles(H, R, S, G, K);
    const long long by_budget = std::max<long long>(1, (long long)(kVbWorkspaceBudget / sizeof(double)) / ws);
    const int blocks = (int)std::min<long long>({(long long)n_seeds, 2LL * std::max(1, e->sm_count), by_budget});
    CU(e->vb_ws.ensure((size_t)blocks * ws * sizeof(double)));

    // The limit covers the kernel's static shared memory too, so the 48 KB default fails already at H = 12 288: it is set for every
    // H, through the per-process high-water mark (only ever raised; another engine may be about to launch with more).
    const size_t smem = (size_t)H * sizeof(int);
    if (int arc = fast_smem_attr(e, k_vb_index, smem)) return arc;
    k_vb_index<<<K, 256, smem, e->stream>>>(d_gt, G, K, H, cnt, start, kh, nk, L, sid, bad);
    LAUNCHED();
    Args a{d_lnl, H, R, S, G, K, n_seeds, soff, d_gt, d_prior, d_lp, d_seeds, epsilon, max_iterations,
           cnt, start, kh, nk, L, sid, bad, e->vb_ws.as<double>(), ws, lpost, ev, iters, map, seed_alpha};
    k_vb_seeds<<<blocks, kThreads, 0, e->stream>>>(a);
    LAUNCHED();
    const unsigned seed_grid = (unsigned)((n_seeds + 255) / 256), g_grid = (unsigned)((G + 255) / 256);
    unsigned long long* ukeys = reinterpret_cast<unsigned long long*>(keys);
    k_vb_mode_max<<<seed_grid, 256, 0, e->stream>>>(bad, ev, map, n_seeds, ukeys);
    k_vb_mode_first<<<seed_grid, 256, 0, e->stream>>>(bad, ev, map, n_seeds, ukeys, first);
    k_vb_modes_compact<<<1, kFinishThreads, 0, e->stream>>>(bad, ev, n_seeds, first, G, modes, weights, n_modes, d_max_seed);
    LAUNCHED(); LAUNCHED(); LAUNCHED();

    double *o_post = posteriors, *o_lpost = log_posteriors, *o_w = weighted_posteriors, *o_alpha = alphas, *o_mev = max_log_evidence;
    int* o_ms = max_seed;
    if (space == PHMM_SPACE_HOST) {
        CU(e->vb_out.ensure((3 * (size_t)G + SK + 2) * sizeof(double)));
        o_post = e->vb_out.as<double>(); o_lpost = o_post + G; o_w = o_lpost + G; o_alpha = o_w + G; o_mev = o_alpha + SK;
        o_ms = reinterpret_cast<int*>(o_mev + 1);
    }
    k_vb_weighted<<<g_grid, 256, 0, e->stream>>>(bad, lpost, G, modes, weights, n_modes, d_max_seed, o_w, o_post, o_lpost);
    k_vb_normalise<<<1, kFinishThreads, 0, e->stream>>>(bad, G, o_w, o_post, ev, seed_alpha, (int)SK, d_max_seed, o_alpha, o_mev, o_ms);
    LAUNCHED(); LAUNCHED();
    CU(cudaGetLastError());
    const cudaMemcpyKind out_kind = space == PHMM_SPACE_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
    if (seed_log_evidence) CU(cudaMemcpyAsync(seed_log_evidence, ev, n_seeds * sizeof(double), out_kind, e->stream));
    if (seed_iterations) CU(cudaMemcpyAsync(seed_iterations, iters, n_seeds * sizeof(int), out_kind, e->stream));
    if (space == PHMM_SPACE_HOST) {
        CU(cudaMemcpyAsync(posteriors, o_post, G * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
        CU(cudaMemcpyAsync(log_posteriors, o_lpost, G * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
        CU(cudaMemcpyAsync(weighted_posteriors, o_w, G * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
        CU(cudaMemcpyAsync(alphas, o_alpha, SK * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
        CU(cudaMemcpyAsync(max_log_evidence, o_mev, sizeof(double), cudaMemcpyDeviceToHost, e->stream));
        CU(cudaMemcpyAsync(max_seed, o_ms, sizeof(int), cudaMemcpyDeviceToHost, e->stream));
    }
    int bad_host = 0;
    CU(cudaMemcpyAsync(&bad_host, bad, sizeof(int), cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    if (bad_host) { e->err = "haplotype index out of range"; return PHMM_ERR_INVALID; }
    return PHMM_OK;
}

// -------------------------------------------------------------------------------------------------------------
// phmm_variational_bayes_mixture_mixture
// -------------------------------------------------------------------------------------------------------------
int phmm_variational_bayes_mixture_mixture(phmm_engine* e, const double* lnl, int32_t H, int32_t R, const int64_t* sample_off, int32_t S,
                                           const int32_t* group_sizes, int32_t T, const int32_t* combinations, int32_t C,
                                           const double* genotype_log_priors, const double* group_priors, const int32_t* group_prior_mask,
                                           const double* group_concentrations, const double* mixture_concentrations, const double* seeds,
                                           int32_t n_seeds, double epsilon, int32_t max_iterations, double* posteriors,
                                           double* log_posteriors, double* group_concentrations_out, double* mixture_concentrations_out,
                                           double* group_responsibilities, double* weighted_posteriors,
                                           double* weighted_group_responsibilities, double* max_log_evidence, int32_t* max_seed,
                                           double* seed_log_evidence, int32_t* seed_iterations, int space)
{
    using namespace phmm::vbmm;
    if (int rc0 = begin_call(e)) return rc0;
    if (T < 1 || T > kMaxGroups || !group_sizes) { e->err = "the number of groups must be in [1, 32]"; return PHMM_ERR_INVALID; }
    int K = 0, maxK = 0;
    std::vector<int> koff_host(T + 1, 0), slot_host;
    for (int t = 0; t < T; ++t) {
        if (group_sizes[t] < 1 || group_sizes[t] > kMaxSlots) { e->err = "group sizes must be in [1, 100]"; return PHMM_ERR_INVALID; }
        koff_host[t] = K;
        K += group_sizes[t];
        maxK = std::max(maxK, (int)group_sizes[t]);
        if (K > kMaxSlots) { e->err = "the group sizes must sum to at most 100"; return PHMM_ERR_INVALID; }
        slot_host.insert(slot_host.end(), group_sizes[t], t);
    }
    koff_host[T] = K;
    if (C < 1 || n_seeds < 1 || S < 1) { e->err = "no combinations, seeds or samples"; return PHMM_ERR_INVALID; }
    if (max_iterations < 1) { e->err = "max_iterations must be at least 1"; return PHMM_ERR_INVALID; }
    if (H < 1 || H > kVbMaxHaplotypes || R < 0) { e->err = "bad matrix shape (1 <= H <= 50000, R >= 0)"; return PHMM_ERR_INVALID; }
    if ((!lnl && R > 0) || !sample_off || !combinations || !genotype_log_priors || !group_concentrations || !mixture_concentrations ||
        !seeds || !posteriors || !log_posteriors || !group_concentrations_out || !mixture_concentrations_out || !group_responsibilities ||
        !weighted_posteriors || !weighted_group_responsibilities || !max_log_evidence || !max_seed) { e->err = "bad argument"; return PHMM_ERR_INVALID; }
    if (sample_off[0] != 0 || sample_off[S] != R) { e->err = "sample_off must run from 0 to R"; return PHMM_ERR_INVALID; }
    for (int s = 0; s < S; ++s) if (sample_off[s + 1] < sample_off[s]) { e->err = "sample_off decreases"; return PHMM_ERR_INVALID; }
    if (space == PHMM_SPACE_HOST)   // the kernel checks device-space indices
        for (long long i = 0; i < (long long)C * K; ++i) if (combinations[i] < 0 || combinations[i] >= H) { e->err = "haplotype index out of range"; return PHMM_ERR_INVALID; }

    // the reads' samples and the per-sample chunks of at most kChunk reads
    std::vector<int> rsamp_host(R), chunk_s, chunk_n0, schunk_host(S + 1), has_prior_host(S, group_priors ? 1 : 0);
    for (int s = 0; s < S; ++s) {
        schunk_host[s] = (int)chunk_s.size();
        for (int64_t n = sample_off[s]; n < sample_off[s + 1]; ++n) rsamp_host[n] = s;
        for (int64_t n = sample_off[s]; n < sample_off[s + 1]; n += kChunk) { chunk_s.push_back(s); chunk_n0.push_back((int)n); }
        if (group_priors && group_prior_mask) has_prior_host[s] = group_prior_mask[s] != 0;
    }
    schunk_host[S] = (int)chunk_s.size();
    const int NC = (int)chunk_s.size();

    const long long KH = (long long)K * H, KC = (long long)K * C, SK = (long long)S * K, ST = (long long)S * T;
    const double *d_lnl, *d_lp, *d_seeds, *d_gprior = nullptr, *d_gc0, *d_mc0; const int32_t* d_gt;
    int rc;
    if ((rc = stage(e, e->mm_lnl, lnl, (size_t)H * R, space, &d_lnl))) return rc;
    if ((rc = stage(e, e->mm_gt, combinations, (size_t)KC, space, &d_gt))) return rc;
    if (space == PHMM_SPACE_HOST) {
        const size_t n_in = C + (size_t)n_seeds * C + (group_priors ? ST : 0) + T + SK;
        CU(e->mm_in.ensure(n_in * sizeof(double)));
        double* p = e->mm_in.as<double>();
        auto put = [&](const double* src, size_t n, const double** dst) -> cudaError_t {
            *dst = p;
            cudaError_t r = cudaMemcpyAsync(p, src, n * sizeof(double), cudaMemcpyHostToDevice, e->stream);
            p += n;
            return r;
        };
        CU(put(genotype_log_priors, C, &d_lp));
        CU(put(seeds, (size_t)n_seeds * C, &d_seeds));
        if (group_priors) CU(put(group_priors, ST, &d_gprior));
        CU(put(group_concentrations, T, &d_gc0));
        CU(put(mixture_concentrations, SK, &d_mc0));
    } else {
        d_lp = genotype_log_priors; d_seeds = seeds; d_gprior = group_priors; d_gc0 = group_concentrations; d_mc0 = mixture_concentrations;
    }

    // ints: cnt, start, kh [K*H]; nk [K]; L, sid [K*C]; bad; soff [S+1]; rsamp [R]; gsz [T]; koff [T+1]; slot_t [K]; has_prior [S];
    // chunk_s, chunk_n0 [NC]; schunk [S+1]; pofs [K+1]; first, modes [C]; n_modes, max_seed; map, iters [n_seeds]
    const long long n_int = 3 * KH + K + 2 * KC + 1 + (S + 1) + R + T + (T + 1) + K + S + 2LL * NC + (S + 1) + (K + 1) + 2LL * C + 2 + 2LL * n_seeds;
    CU(e->mm_idx.ensure((size_t)n_int * sizeof(int)));
    int* ip = e->mm_idx.as<int>();
    int *cnt = ip, *start = cnt + KH, *kh = start + KH, *nk = kh + KH, *L = nk + K, *sid = L + KC, *bad = sid + KC, *soff = bad + 1,
        *rsamp = soff + S + 1, *gsz = rsamp + R, *koff = gsz + T, *slot_t = koff + T + 1, *has_prior = slot_t + K, *d_chunk_s = has_prior + S,
        *d_chunk_n0 = d_chunk_s + NC, *schunk = d_chunk_n0 + NC, *pofs = schunk + S + 1, *first = pofs + K + 1, *modes = first + C,
        *n_modes = modes + C, *d_max_seed = n_modes + 1, *map = d_max_seed + 1, *iters = map + n_seeds;
    {   // one staging copy of the host-built int arrays (soff .. schunk are contiguous)
        std::vector<int> h;
        h.reserve((size_t)(schunk + S + 1 - soff));
        h.insert(h.end(), sample_off, sample_off + S + 1);
        h.insert(h.end(), rsamp_host.begin(), rsamp_host.end());
        h.insert(h.end(), group_sizes, group_sizes + T);
        h.insert(h.end(), koff_host.begin(), koff_host.end());
        h.insert(h.end(), slot_host.begin(), slot_host.end());
        h.insert(h.end(), has_prior_host.begin(), has_prior_host.end());
        h.insert(h.end(), chunk_s.begin(), chunk_s.end());
        h.insert(h.end(), chunk_n0.begin(), chunk_n0.end());
        h.insert(h.end(), schunk_host.begin(), schunk_host.end());
        CU(cudaMemcpyAsync(soff, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice, e->stream));
        CU(cudaMemsetAsync(bad, 0, sizeof(int), e->stream));
        CU(cudaMemsetAsync(first, 0x7f, C * sizeof(int), e->stream));   // 0x7f7f7f7f: above every seed index
        const size_t smem = (size_t)H * sizeof(int);
        if (int arc = fast_smem_attr(e, phmm::vb::k_vb_index, smem)) return arc;   // as in phmm_variational_bayes
        phmm::vb::k_vb_index<<<K, 256, smem, e->stream>>>(d_gt, C, K, H, cnt, start, kh, nk, L, sid, bad);
        LAUNCHED();
        CU(cudaGetLastError());
        // the occurring (slot, haplotype) pairs; their count, at most K min(H, C), stays on the device (pofs[K])
        const long long Pmax = (long long)K * std::min(H, C);
        CU(e->mm_pairs.ensure((size_t)(2 * Pmax) * sizeof(int)));
        int *pj = e->mm_pairs.as<int>(), *ph = pj + Pmax;
        k_vbmm_pairs<<<1, 256, 0, e->stream>>>(bad, nk, kh, K, H, pofs, pj, ph);
        LAUNCHED();

        // doubles: lpost [n_seeds][C]; ev [n_seeds]; gconc [n_seeds][T]; mconc [n_seeds][S][K]; sigma [n_seeds][S][T]; weights [C]; keys [C] (u64)
        const long long n_dbl = (long long)n_seeds * C + n_seeds + (long long)n_seeds * (T + SK + ST) + 2LL * C;
        CU(e->mm_seed.ensure((size_t)n_dbl * sizeof(double)));
        double* dp = e->mm_seed.as<double>();
        double *lpost = dp, *ev = lpost + (long long)n_seeds * C, *seed_gconc = ev + n_seeds, *seed_mconc = seed_gconc + (long long)n_seeds * T,
               *seed_sigma = seed_mconc + n_seeds * SK, *weights = seed_sigma + n_seeds * ST, *keys = weights + C;
        CU(cudaMemsetAsync(keys, 0, C * sizeof(double), e->stream));

        const long long ws = Workspace::doubles(H, R, S, C, K, T, (int)Pmax, NC);
        const long long by_budget = std::max<long long>(1, (long long)(kVbWorkspaceBudget / sizeof(double)) / ws);
        const int blocks = (int)std::min<long long>({(long long)n_seeds, 2LL * std::max(1, e->sm_count), by_budget});
        CU(e->mm_ws.ensure((size_t)blocks * ws * sizeof(double)));
        Args a{d_lnl, H, R, S, C, K, T, maxK, n_seeds, soff, rsamp, gsz, koff, slot_t, d_gt, d_lp, d_seeds, d_gprior, has_prior, d_gc0, d_mc0,
               epsilon, max_iterations, cnt, start, kh, nk, L, sid, bad, pofs, pj, ph, 0, (int)Pmax, d_chunk_s, d_chunk_n0, schunk, NC,
               e->mm_ws.as<double>(), ws, lpost, ev, iters, map, seed_gconc, seed_mconc, seed_sigma};
        k_vbmm_seeds<<<blocks, kThreads, 0, e->stream>>>(a);
        LAUNCHED();
        const unsigned seed_grid = (unsigned)((n_seeds + 255) / 256), c_grid = (unsigned)((C + 255) / 256);
        unsigned long long* ukeys = reinterpret_cast<unsigned long long*>(keys);
        phmm::vb::k_vb_mode_max<<<seed_grid, 256, 0, e->stream>>>(bad, ev, map, n_seeds, ukeys);
        phmm::vb::k_vb_mode_first<<<seed_grid, 256, 0, e->stream>>>(bad, ev, map, n_seeds, ukeys, first);
        phmm::vb::k_vb_modes_compact<<<1, kFinishThreads, 0, e->stream>>>(bad, ev, n_seeds, first, C, modes, weights, n_modes, d_max_seed);
        LAUNCHED(); LAUNCHED(); LAUNCHED();

        double *o_post = posteriors, *o_lpost = log_posteriors, *o_w = weighted_posteriors, *o_gc = group_concentrations_out,
               *o_mc = mixture_concentrations_out, *o_sg = group_responsibilities, *o_wsg = weighted_group_responsibilities, *o_mev = max_log_evidence;
        int* o_ms = max_seed;
        if (space == PHMM_SPACE_HOST) {
            CU(e->mm_out.ensure((3 * (size_t)C + T + SK + 2 * ST + 2) * sizeof(double)));
            o_post = e->mm_out.as<double>(); o_lpost = o_post + C; o_w = o_lpost + C; o_gc = o_w + C; o_mc = o_gc + T; o_sg = o_mc + SK;
            o_wsg = o_sg + ST; o_mev = o_wsg + ST; o_ms = reinterpret_cast<int*>(o_mev + 1);
        }
        phmm::vb::k_vb_weighted<<<c_grid, 256, 0, e->stream>>>(bad, lpost, C, modes, weights, n_modes, d_max_seed, o_w, o_post, o_lpost);
        k_vbmm_finish<<<1, kFinishThreads, 0, e->stream>>>(bad, C, S, T, K, o_w, modes, weights, n_modes, d_max_seed, ev, seed_gconc, seed_mconc,
                                                           seed_sigma, o_gc, o_mc, o_sg, o_wsg, o_mev, o_ms);
        LAUNCHED(); LAUNCHED();
        CU(cudaGetLastError());
        const cudaMemcpyKind out_kind = space == PHMM_SPACE_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
        if (seed_log_evidence) CU(cudaMemcpyAsync(seed_log_evidence, ev, n_seeds * sizeof(double), out_kind, e->stream));
        if (seed_iterations) CU(cudaMemcpyAsync(seed_iterations, iters, n_seeds * sizeof(int), out_kind, e->stream));
        if (space == PHMM_SPACE_HOST) {
            CU(cudaMemcpyAsync(posteriors, o_post, C * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
            CU(cudaMemcpyAsync(log_posteriors, o_lpost, C * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
            CU(cudaMemcpyAsync(weighted_posteriors, o_w, C * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
            CU(cudaMemcpyAsync(group_concentrations_out, o_gc, T * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
            CU(cudaMemcpyAsync(mixture_concentrations_out, o_mc, SK * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
            CU(cudaMemcpyAsync(group_responsibilities, o_sg, ST * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
            CU(cudaMemcpyAsync(weighted_group_responsibilities, o_wsg, ST * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
            CU(cudaMemcpyAsync(max_log_evidence, o_mev, sizeof(double), cudaMemcpyDeviceToHost, e->stream));
            CU(cudaMemcpyAsync(max_seed, o_ms, sizeof(int), cudaMemcpyDeviceToHost, e->stream));
        }
        int bad_host = 0;
        CU(cudaMemcpyAsync(&bad_host, bad, sizeof(int), cudaMemcpyDeviceToHost, e->stream));
        CU(cudaStreamSynchronize(e->stream));
        if (bad_host) { e->err = "haplotype index out of range"; return PHMM_ERR_INVALID; }
    }
    return PHMM_OK;
}

// -------------------------------------------------------------------------------------------------------------
// phmm_engine_reset_haplotypes
// -------------------------------------------------------------------------------------------------------------
// Device memory the scratch slots of one call may take: slots = min(haplotypes, budget / slot size, resident threads). The slots
// are spread over at least kResetWarpsPerSm warps per SM (fewer working lanes per warp) before warps are filled.
static constexpr size_t kResetScratchBudget = (size_t)1 << 30;
static constexpr int kResetWarpsPerSm = 16;

} // extern "C"

// The six per-base arrays of phmm_haplotypes that reset() fills.
struct ResetArrays {
    char* mask_f; int8_t* prior_f; char* mask_r; int8_t* prior_r; int8_t* gap_open; int8_t* gap_extend;
};

// What phmm_engine_reset_haplotypes and the populate calls with an error model share: the checks, the staging of off / seq /
// is_substitution, the model's upload, the scratch slots, k_reset_haplotypes and the host recompute of the haplotypes whose runs
// overflow their slot, after the call's one synchronisation. Inputs in `space`. The arrays are written to `dev` (device memory) or,
// with dev null, to the engine's h_mf .. h_ge; there haplotype h starts at off[h] - base, base = off[0] for host space and 0 for device
// space. With `host` they are then copied to those host arrays (h at off[h]). *staged (optional) receives the device copies of off and
// seq, the device arrays and the offsets on the host. n == 0 returns PHMM_OK without touching the GPU.
struct ResetStaged { const int64_t* off = nullptr; const char* seq = nullptr; ResetArrays a {}; std::vector<long long> hoff; };

// Run capacity of a haplotype's first attempt on the device. The haplotype's runs never come near phmm_reset::first_cap, so
// PHMM_RESET_CAP (read once per process) can force a smaller one: a test hook that makes the host recompute of overflowed
// haplotypes run. PHMM_TRACE reports how many haplotypes that recompute took.
static uint32_t reset_first_cap(uint32_t longest)
{
    static const long long forced = [] {
        const char* v = std::getenv("PHMM_RESET_CAP");
        return v ? std::atoll(v) : 0LL;
    }();
    return forced > 0 ? (uint32_t)forced : phmm_reset::first_cap(longest);
}

static int reset_arrays(phmm_engine* e, const phmm_error_model* m, int32_t n, const int64_t* off, const char* seq, const uint8_t* is_substitution,
                        int space, const ResetArrays* dev, const ResetArrays* host, ResetStaged* staged)
{
    if (!m || n < 0 || (n > 0 && (!off || !seq))) { e->err = "null argument"; return PHMM_ERR_INVALID; }
    if (space != PHMM_SPACE_HOST && space != PHMM_SPACE_DEVICE) { e->err = "bad memory space"; return PHMM_ERR_INVALID; }
    if (n == 0) return PHMM_OK;
    if (int rc0 = begin_call(e)) return rc0;
    int rc;
    std::vector<long long> hoff;
    if ((rc = fetch_offsets(e, off, n, space, hoff)) != PHMM_OK) return rc;
    if (hoff[0] < 0) { e->err = "bad haplotype offsets"; return PHMM_ERR_INVALID; }
    long long L = 0;
    for (int h = 0; h < n; ++h) {
        if (hoff[h + 1] < hoff[h]) { e->err = "bad haplotype offsets"; return PHMM_ERR_INVALID; }
        L = std::max(L, hoff[h + 1] - hoff[h]);
    }
    if (L > 65535) { e->err = "haplotype longer than 65535 bases"; return PHMM_ERR_INVALID; }
    // host space: the bases off[0] .. off[n] are staged and the outputs computed from index 0 = off[0]
    const long long base = space == PHMM_SPACE_HOST ? hoff[0] : 0;
    const size_t B = (size_t)(hoff[n] - base);
    const int64_t* d_off;
    const char* d_seq; const uint8_t* d_sub;
    if ((rc = stage(e, e->h_off, off, (size_t)n + 1, space, &d_off))) return rc;
    if ((rc = stage(e, e->h_seq, space == PHMM_SPACE_HOST ? seq + base : seq, B, space, &d_seq))) return rc;
    if ((rc = stage(e, e->rs_sub, is_substitution && space == PHMM_SPACE_HOST ? is_substitution + base : is_substitution, B, space, &d_sub))) return rc;
    ResetArrays d {};
    if (dev) d = *dev;
    else {
        DBuf* bufs[6] = {&e->h_mf, &e->h_pf, &e->h_mr, &e->h_pr, &e->h_go, &e->h_ge};
        for (DBuf* b : bufs) CU(b->ensure(std::max<size_t>(B, 1)));
        d = {e->h_mf.as<char>(), e->h_pf.as<int8_t>(), e->h_mr.as<char>(), e->h_pr.as<int8_t>(), e->h_go.as<int8_t>(), e->h_ge.as<int8_t>()};
    }
    if (staged) { staged->off = d_off; staged->seq = d_seq; staged->a = d; }
    // the model: fixed rows travel in the kernel argument, a custom model's motif tables in one device block
    phmm_reset::Model dm = phmm_reset::model_of(m);
    if (dm.custom) {
        const phmm_reset::MotifTable* t[2] = {&dm.custom_open, &dm.custom_extend};
        size_t bytes = 0, at[2][3];
        for (int i = 0; i < 2; ++i) {
            at[i][0] = bytes; bytes += ((size_t)t[i]->n * sizeof(uint64_t) + 7) & ~(size_t)7;
            at[i][1] = bytes; bytes += (((size_t)t[i]->n + 1) * sizeof(uint32_t) + 7) & ~(size_t)7;
            at[i][2] = bytes; bytes += ((t[i]->n > 0 ? (size_t)t[i]->row[t[i]->n] : 0) + 7) & ~(size_t)7;
        }
        std::vector<char> blob(std::max<size_t>(bytes, 8), 0);
        CU(e->rs_model.ensure(blob.size()));
        phmm_reset::MotifTable* dt[2] = {&dm.custom_open, &dm.custom_extend};
        for (int i = 0; i < 2; ++i) {
            const phmm_reset::MotifTable src = *t[i];
            if (src.n > 0) {
                std::memcpy(blob.data() + at[i][0], src.key, (size_t)src.n * sizeof(uint64_t));
                std::memcpy(blob.data() + at[i][1], src.row, ((size_t)src.n + 1) * sizeof(uint32_t));
                std::memcpy(blob.data() + at[i][2], src.data, src.row[src.n]);
            }
            dt[i]->key = (const uint64_t*)(e->rs_model.as<char>() + at[i][0]);
            dt[i]->row = (const uint32_t*)(e->rs_model.as<char>() + at[i][1]);
            dt[i]->data = (const int8_t*)(e->rs_model.as<char>() + at[i][2]);
        }
        CU(cudaMemcpyAsync(e->rs_model.p, blob.data(), blob.size(), cudaMemcpyHostToDevice, e->stream));
    }
    // scratch slots sized for the longest haplotype
    const uint32_t cap = reset_first_cap((uint32_t)L);
    const size_t slot_words = phmm_reset::scratch_words((uint32_t)L, cap);
    const size_t slot_bytes = slot_words * sizeof(uint32_t) + 2 * (size_t)cap * sizeof(phmm_reset::Run);
    const int resident = std::max(1, e->sm_count) * 2048;
    const long long wanted = std::max<long long>(1, std::min<long long>({(long long)n, (long long)(kResetScratchBudget / slot_bytes), (long long)resident}));
    const int lanes = (int)std::min<long long>(32, (wanted + (long long)std::max(1, e->sm_count) * kResetWarpsPerSm - 1) / ((long long)std::max(1, e->sm_count) * kResetWarpsPerSm));
    const long long warps = (wanted + lanes - 1) / lanes;
    const int slots = (int)(warps * lanes);
    CU(e->rs_words.ensure((size_t)slots * slot_words * sizeof(uint32_t)));
    CU(e->rs_runs.ensure((size_t)slots * 2 * cap * sizeof(phmm_reset::Run)));
    CU(e->rs_flags.ensure((size_t)n));
    CU(cudaEventRecord(e->ev0, e->stream));
    k_reset_haplotypes<<<(unsigned)((warps + 3) / 4), 128, 0, e->stream>>>(dm, n, (const long long*)d_off, base, (const unsigned char*)d_seq, d_sub,
                                                                        d.mask_f, d.prior_f, d.mask_r, d.prior_r, d.gap_open, d.gap_extend,
                                                                        e->rs_words.as<uint32_t>(), e->rs_runs.as<phmm_reset::Run>(), slot_words,
                                                                        cap, lanes, slots, e->rs_flags.as<uint8_t>());
    LAUNCHED();
    CU(cudaGetLastError());
    CU(cudaEventRecord(e->ev1, e->stream));
    std::vector<uint8_t> overflow((size_t)n);
    CU(cudaMemcpyAsync(overflow.data(), e->rs_flags.p, (size_t)n, cudaMemcpyDeviceToHost, e->stream));
    if (host && B > 0) {
        CU(cudaMemcpyAsync(host->mask_f + base, d.mask_f, B, cudaMemcpyDeviceToHost, e->stream));
        CU(cudaMemcpyAsync(host->prior_f + base, d.prior_f, B, cudaMemcpyDeviceToHost, e->stream));
        CU(cudaMemcpyAsync(host->mask_r + base, d.mask_r, B, cudaMemcpyDeviceToHost, e->stream));
        CU(cudaMemcpyAsync(host->prior_r + base, d.prior_r, B, cudaMemcpyDeviceToHost, e->stream));
        CU(cudaMemcpyAsync(host->gap_open + base, d.gap_open, B, cudaMemcpyDeviceToHost, e->stream));
        CU(cudaMemcpyAsync(host->gap_extend + base, d.gap_extend, B, cudaMemcpyDeviceToHost, e->stream));
    }
    CU(cudaStreamSynchronize(e->stream));
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, e->ev0, e->ev1) == cudaSuccess) e->last_dp_ms = ms;
    // haplotypes whose runs overflowed their slot: the host core with a growing capacity, the same arithmetic
    phmm_reset::HostScratch scratch;
    const phmm_reset::Model& hm = phmm_reset::model_of(m);
    std::vector<unsigned char> s, sub;
    std::vector<int8_t> out;
    if (std::getenv("PHMM_TRACE"))
        std::fprintf(stderr, "[phmm %p] reset: %lld of %d haplotypes recomputed on the host\n", (void*)e,
                     (long long)std::count(overflow.begin(), overflow.end(), (uint8_t)1), n);
    for (int h = 0; h < n; ++h) {
        if (!overflow[h]) continue;
        const long long o = hoff[h];
        const uint32_t len = (uint32_t)(hoff[h + 1] - o);
        const unsigned char* s_in = (const unsigned char*)seq + o;
        const uint8_t* sub_in = is_substitution ? is_substitution + o : nullptr;
        if (space == PHMM_SPACE_DEVICE) {
            s.resize(len); sub.resize(len);
            CU(cudaMemcpyAsync(s.data(), seq + o, len, cudaMemcpyDeviceToHost, e->stream));
            if (is_substitution) CU(cudaMemcpyAsync(sub.data(), is_substitution + o, len, cudaMemcpyDeviceToHost, e->stream));
            CU(cudaStreamSynchronize(e->stream));
            s_in = s.data(); sub_in = is_substitution ? sub.data() : nullptr;
        }
        if (host) {
            phmm_reset::reset_haplotype_host(hm, s_in, len, sub_in, host->mask_f + o, host->prior_f + o, host->mask_r + o, host->prior_r + o,
                                             host->gap_open + o, host->gap_extend + o, scratch);
            continue;
        }
        out.resize(6 * (size_t)len);
        int8_t* a = out.data();
        phmm_reset::reset_haplotype_host(hm, s_in, len, sub_in, (char*)a, a + len, (char*)a + 2 * len, a + 3 * len, a + 4 * len, a + 5 * len, scratch);
        const long long at = o - base;
        void* dst[6] = {d.mask_f + at, d.prior_f + at, d.mask_r + at, d.prior_r + at, d.gap_open + at, d.gap_extend + at};
        for (int k = 0; k < 6; ++k) CU(cudaMemcpyAsync(dst[k], a + (size_t)k * len, len, cudaMemcpyHostToDevice, e->stream));
        CU(cudaStreamSynchronize(e->stream));
    }
    if (staged) staged->hoff = std::move(hoff);
    return PHMM_OK;
}

extern "C" {

int phmm_engine_reset_haplotypes(phmm_engine* e, const phmm_error_model* m, int32_t n, const int64_t* off, const char* seq,
                                 const uint8_t* is_substitution, char* snv_mask_fwd, int8_t* snv_prior_fwd, char* snv_mask_rev,
                                 int8_t* snv_prior_rev, int8_t* gap_open, int8_t* gap_extend, int space)
{
    if (!e) return PHMM_ERR_INVALID;
    e->err.clear(); e->launches_last = 0; e->last_dp_ms = 0.0; e->last_dp_cells = 0;
    if (n > 0 && (!snv_mask_fwd || !snv_prior_fwd || !snv_mask_rev || !snv_prior_rev || !gap_open || !gap_extend)) { e->err = "null argument"; return PHMM_ERR_INVALID; }
    const ResetArrays out {snv_mask_fwd, snv_prior_fwd, snv_mask_rev, snv_prior_rev, gap_open, gap_extend};
    // device space: the kernel writes the caller's arrays; host space: the engine's buffers, copied back
    return reset_arrays(e, m, n, off, seq, is_substitution, space, space == PHMM_SPACE_DEVICE ? &out : nullptr,
                        space == PHMM_SPACE_HOST ? &out : nullptr, nullptr);
}

// -------------------------------------------------------------------------------------------------------------
// Uncapped k-mer mapper over a pair list (phmm_map_pairs, phmm_realign_reads, phmm_assign_reads)
// -------------------------------------------------------------------------------------------------------------
// Pass 1 and the offset scan: k-mer hashes of the reads, tables of the haplotypes, per pair the maximum and how many mapping begins
// reach it, CSR offsets into off_dev[n + 1] (device). One synchronisation brings the total back; a pair index out of range found on
// the device fails the call here.
static int pair_map_count(phmm_engine* e, const Staged& s, const int2* d_pairs, int n, long long* off_dev, long long* total)
{
    int rc;
    static_assert(kKmer == 6, "phmm_checks::mapper_reads assumes 6-mers");
    if ((rc = phmm_checks::mapper_reads(s.read_len_max, e->err)) != PHMM_OK) return rc;
    if ((rc = prepare_mapper(e, s)) != PHMM_OK) return rc;
    CU(e->pm_best.ensure((size_t)n * sizeof(unsigned)));
    CU(e->pm_cnt.ensure((size_t)n * sizeof(int)));
    CU(e->pm_inl.ensure((size_t)n * kPairMapInline * sizeof(int32_t)));
    const int nb = (n + 1023) / 1024;
    CU(e->pm_part.ensure((size_t)nb * sizeof(long long)));
    CU(e->pm_misc.ensure(2 * sizeof(long long)));
    long long* misc = e->pm_misc.as<long long>();             // [0] total, [1] low word: bad pair index
    CU(cudaMemsetAsync(misc, 0, 2 * sizeof(long long), e->stream));
    pair_map_pass<false>(e, s, d_pairs, n, (int*)(misc + 1), nullptr, nullptr);
    k_csr_scan_blocks<<<nb, 1024, 0, e->stream>>>(n, e->pm_cnt.as<int>(), off_dev, e->pm_part.as<long long>());
    LAUNCHED();
    k_csr_scan_parts<<<1, 1024, 0, e->stream>>>(nb, e->pm_part.as<long long>(), misc);
    LAUNCHED();
    k_csr_scan_carry<<<nb, 1024, 0, e->stream>>>(n, e->pm_part.as<long long>(), off_dev);
    LAUNCHED();
    CU(cudaGetLastError());
    long long host_misc[2] = {0, 0};
    CU(cudaMemcpyAsync(host_misc, misc, sizeof(host_misc), cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    if ((int)host_misc[1] != 0) { e->err = "pair index out of range"; return PHMM_ERR_INVALID; }
    *total = host_misc[0];
    return PHMM_OK;
}

// Pass 2: every mapping begin of every pair into pos_dev[off_dev[j] ..) (device, off_dev[n] entries).
static int pair_map_emit(phmm_engine* e, const Staged& s, const int2* d_pairs, int n, const long long* off_dev, int32_t* pos_dev)
{
    pair_map_pass<true>(e, s, d_pairs, n, nullptr, off_dev, pos_dev);
    CU(cudaGetLastError());
    return PHMM_OK;
}

// Both passes into the engine's own CSR (c_off, c_pos), for the calls that consume the positions on the device.
static int pair_map_resident(phmm_engine* e, const Staged& s, const int2* d_pairs, int n, long long* total)
{
    int rc;
    CU(e->c_off.ensure(((size_t)n + 1) * sizeof(long long)));
    if ((rc = pair_map_count(e, s, d_pairs, n, e->c_off.as<long long>(), total))) return rc;
    CU(e->c_pos.ensure((size_t)std::max<long long>(*total, 1) * sizeof(int32_t)));
    return pair_map_emit(e, s, d_pairs, n, e->c_off.as<long long>(), e->c_pos.as<int32_t>());
}

// -------------------------------------------------------------------------------------------------------------
// phmm_align_reads
// -------------------------------------------------------------------------------------------------------------
// Shared by phmm_align_reads (HaplotypeLikelihoodModel::align: candidate positions, in-range rule, fallback), phmm_realign_reads
// (the same with every pair's positions from the uncapped pair mapper, map_on_device) and phmm_align_pairs (hmm::align: one explicit
// offset per pair).
// The entry points have run begin_call: the DP time adds to the call's, so phmm_mutation_prime can align tile after tile.
static int align_impl(phmm_engine* e, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                      const phmm_pair* pairs, int64_t n_pairs, const phmm_positions* positions, const int32_t* raw_offsets,
                      const phmm_flank_state* flank,
                      int64_t* mapping_position, double* likelihood, char* cigar, int32_t cigar_stride, int32_t* status, int space,
                      bool map_on_device = false)
{
    int rc = phmm_checks::align_arguments(cfg, pairs, n_pairs, mapping_position, likelihood, cigar, cigar_stride, status, e->err);
    if (rc != PHMM_OK) return rc;
    if (n_pairs == 0) return PHMM_OK;
    if ((rc = phmm_checks::align_reads(cfg, reads, e->err)) != PHMM_OK) return rc;
    const int band = round_band(std::max(1, cfg->max_indel_error));
    Staged s;
    rc = stage_batch(e, haps, reads, space, s);
    if (rc != PHMM_OK) return rc;
    const int n = (int)n_pairs;
    if (space == PHMM_SPACE_HOST && (rc = check_pairs(e, pairs, n, s))) return rc;
    AlignParams p {};
    p.hp = s.hp; p.rd = s.rd; p.n_pairs = n;
    p.band = band; p.nuc_prior = cfg->nuc_prior;
    p.use_flanks = (flank && flank->has_flank && cfg->use_flank_state) ? 1 : 0;
    p.lhs_flank = p.use_flanks ? (int)flank->lhs_flank : 0;
    p.rhs_flank = p.use_flanks ? (int)flank->rhs_flank : 0;
    p.use_mapq = cfg->use_mapping_quality; p.mapq_cap = cfg->mapping_quality_cap; p.mapq_trigger = cfg->mapping_quality_cap_trigger;
    const int2* d_pairs;
    if ((rc = stage(e, e->pairs, (const int2*)pairs, (size_t)n, space, &d_pairs))) return rc;
    p.pairs = d_pairs;
    if (raw_offsets) {
        const int32_t* pv;
        if ((rc = stage(e, e->c_pos, raw_offsets, (size_t)n, space, &pv))) return rc;
        p.pos = pv; p.raw_offsets = 1;
    } else if (positions && positions->off && positions->pos) {
        long long total = 0;
        if ((rc = stage_positions(e, positions, n, space, &p.pos_off, &p.pos, &total))) return rc;
    } else if (map_on_device) {
        long long total = 0;
        if ((rc = pair_map_resident(e, s, d_pairs, n, &total))) return rc;
        p.pos_off = e->c_off.as<long long>(); p.pos = e->c_pos.as<int32_t>();
    }
    int Lmax = 1;
    for (int r = 0; r < s.rd.n; ++r) Lmax = std::max(Lmax, e->info_host[r].x);
    // Register traceback for bands up to 32 (one thread per pair, its read in shared memory, one back-pointer word per cell);
    // the generic kernel for wider bands and the reads the register kernel cannot take.
    const int K = 2 * band;
    static const bool no_fast_align = std::getenv("PHMM_NO_FAST_ALIGN") != nullptr;      // measurement hook: the generic traceback kernel for everything
    p.fast_band = (band <= 32 && !no_fast_align) ? band : 0;
    const int fast_cap = (int)((200 << 10) / (kAlignFastThreads * (int)sizeof(uint16_t))) - 4;      // one block's rows in shared memory
    p.fast_max_len = std::min(Lmax, fast_cap);
    p.fast_row_stride = 2 * (((p.fast_max_len + 2) / 2) | 1);                                      // in half-words; 2 * odd (bank spread)
    const size_t fsmem = (size_t)kAlignFastThreads * p.fast_row_stride * sizeof(uint16_t);
    int fast_blocks_per_sm = 1;
    if (p.fast_band) {
        rc = with_band_in<8, 16, 32>(band, [&](auto b) -> int {
            return prepare_kernel(e, k_align_reads_fast<decltype(b)::value>, kAlignFastThreads, fsmem, &fast_blocks_per_sm);
        });
        if (rc != PHMM_OK) return rc;
        if (fast_blocks_per_sm < 1) p.fast_band = 0;
    }
    // threads: bounded by the pairs and by the scratch budgets (byte back-pointers of the generic kernel; words of the register kernel)
    const long long words_per_thread = (long long)(p.fast_max_len + K) * K;
    int fast_threads = p.fast_band ? std::min(e->sm_count * fast_blocks_per_sm * kAlignFastThreads, ((n + kAlignFastThreads - 1) / kAlignFastThreads) * kAlignFastThreads) : 0;
    if (p.fast_band) fast_threads = (int)std::max<long long>(kAlignFastThreads, std::min<long long>(fast_threads, ((6LL << 30) / (4 * words_per_thread)) / kAlignFastThreads * kAlignFastThreads));
    const long long bp_per_thread = (long long)(Lmax + 1) * K;
    int slow_threads = std::min(e->sm_count * 256, ((n + 63) / 64) * 64);
    slow_threads = (int)std::max<long long>(64, std::min<long long>(slow_threads, ((4LL << 30) / bp_per_thread) / 64 * 64));
    const int threads_total = std::max(fast_threads, slow_threads);
    p.str_cap = 2 * (Lmax + band) + 2;
    CU(e->bp.ensure((size_t)slow_threads * (size_t)bp_per_thread));
    if (p.fast_band) CU(e->ftasks.ensure((size_t)fast_threads * (size_t)words_per_thread * sizeof(uint32_t)));
    CU(e->slow.ensure((size_t)threads_total * 4 * p.str_cap));
    p.bp = e->bp.as<unsigned char>();
    p.bp32 = e->ftasks.as<uint32_t>();
    p.strings = e->slow.as<char>();
    // outputs
    const bool dev = space == PHMM_SPACE_DEVICE;
    CU(e->best.ensure((size_t)n * sizeof(long long)));
    CU(e->out.ensure((size_t)n * sizeof(double)));
    CU(e->status.ensure((size_t)n * sizeof(int)));
    CU(e->kpos.ensure((size_t)n * cigar_stride));
    p.mapping_position = dev ? (long long*)mapping_position : e->best.as<long long>();
    p.likelihood = dev ? likelihood : e->out.as<double>();
    p.status = dev ? status : e->status.as<int>();
    p.cigar = dev ? cigar : e->kpos.as<char>();
    p.cigar_stride = cigar_stride;
    CU(cudaEventRecord(e->ev0, e->stream));
    if (p.fast_band) {
        const unsigned fgrid = (unsigned)(fast_threads / kAlignFastThreads);
        with_band_in<8, 16, 32>(band, [&](auto b) { k_align_reads_fast<decltype(b)::value><<<fgrid, kAlignFastThreads, fsmem, e->stream>>>(p); });
        LAUNCHED();
    }
    {
        const unsigned grid = (unsigned)(slow_threads / 64);
        if (band <= 32) k_align_reads<64><<<grid, 64, 0, e->stream>>>(p);
        else k_align_reads<kGenericMaxDiag><<<grid, 64, 0, e->stream>>>(p);
        LAUNCHED();
    }
    CU(cudaEventRecord(e->ev1, e->stream));
    CU(cudaGetLastError());
    if (!dev) {
        CU(cudaMemcpyAsync(mapping_position, p.mapping_position, (size_t)n * sizeof(long long), cudaMemcpyDeviceToHost, e->stream));
        CU(cudaMemcpyAsync(likelihood, p.likelihood, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
        CU(cudaMemcpyAsync(status, p.status, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, e->stream));
        CU(cudaMemcpyAsync(cigar, p.cigar, (size_t)n * cigar_stride, cudaMemcpyDeviceToHost, e->stream));
    }
    CU(cudaStreamSynchronize(e->stream));
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, e->ev0, e->ev1) == cudaSuccess) e->last_dp_ms += ms;
    return PHMM_OK;
}

int phmm_align_reads(phmm_engine* e, const phmm_config* cfg,
                     const phmm_haplotypes* haps, const phmm_reads* reads,
                     const phmm_pair* pairs, int64_t n_pairs,
                     const phmm_positions* positions, const phmm_flank_state* flank,
                     int64_t* mapping_position, double* likelihood, char* cigar, int32_t cigar_stride, int32_t* status, int space)
{
    if (int rc = begin_call(e)) return rc;
    return align_impl(e, cfg, haps, reads, pairs, n_pairs, positions, nullptr, flank, mapping_position, likelihood, cigar, cigar_stride, status, space);
}

int phmm_align_pairs(phmm_engine* e, const phmm_config* cfg,
                     const phmm_haplotypes* truths, const phmm_reads* targets,
                     const phmm_pair* pairs, const int32_t* target_offsets, int64_t n_pairs, const phmm_flank_state* flank,
                     int64_t* target_offset_out, double* likelihood, char* cigar, int32_t cigar_stride, int32_t* status, int space)
{
    if (int rc = begin_call(e)) return rc;
    if (!target_offsets) { e->err = "null target offsets"; return PHMM_ERR_INVALID; }
    return align_impl(e, cfg, truths, targets, pairs, n_pairs, nullptr, target_offsets, flank, target_offset_out, likelihood, cigar, cigar_stride, status, space);
}

int phmm_realign_reads(phmm_engine* e, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                       const phmm_pair* pairs, int64_t n_pairs, const phmm_flank_state* flank,
                       int64_t* mapping_position, double* likelihood, char* cigar, int32_t cigar_stride, int32_t* status, int space)
{
    if (int rc = begin_call(e)) return rc;
    const bool map = cfg && cfg->map_positions;
    return align_impl(e, cfg, haps, reads, pairs, n_pairs, nullptr, nullptr, flank, mapping_position, likelihood, cigar, cigar_stride, status, space, map);
}

int phmm_map_pairs(phmm_engine* e, const phmm_haplotypes* haps, const phmm_reads* reads, const phmm_pair* pairs, int64_t n_pairs,
                   int64_t* off, int32_t* pos, int64_t pos_cap, int space)
{
    if (int rc0 = begin_call(e)) return rc0;
    if (!pairs || !off) { e->err = "null pairs / offsets"; return PHMM_ERR_INVALID; }
    if (n_pairs < 0 || n_pairs > 0x7fffffff) { e->err = "pair count out of range"; return PHMM_ERR_INVALID; }
    const bool dev = space == PHMM_SPACE_DEVICE;
    if (n_pairs == 0) {
        if (!dev) off[0] = 0;
        else { CU(cudaMemsetAsync(off, 0, sizeof(int64_t), e->stream)); CU(cudaStreamSynchronize(e->stream)); }
        return PHMM_OK;
    }
    Staged s;
    int rc = stage_batch(e, haps, reads, space, s, false);
    if (rc != PHMM_OK) return rc;
    const int n = (int)n_pairs;
    if (!dev && (rc = check_pairs(e, pairs, n, s))) return rc;
    const int2* d_pairs;
    if ((rc = stage(e, e->pairs, (const int2*)pairs, (size_t)n, space, &d_pairs))) return rc;
    long long* off_dev = (long long*)off;
    if (!dev) { CU(e->c_off.ensure(((size_t)n + 1) * sizeof(long long))); off_dev = e->c_off.as<long long>(); }
    long long total = 0;
    if ((rc = pair_map_count(e, s, d_pairs, n, off_dev, &total))) return rc;
    if (pos && pos_cap >= total && total > 0) {
        int32_t* pos_dev = pos;
        if (!dev) { CU(e->c_pos.ensure((size_t)total * sizeof(int32_t))); pos_dev = e->c_pos.as<int32_t>(); }
        if ((rc = pair_map_emit(e, s, d_pairs, n, off_dev, pos_dev))) return rc;
        if (!dev) CU(cudaMemcpyAsync(pos, pos_dev, (size_t)total * sizeof(int32_t), cudaMemcpyDeviceToHost, e->stream));
    }
    if (!dev) CU(cudaMemcpyAsync(off, off_dev, ((size_t)n + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    return PHMM_OK;
}

// -------------------------------------------------------------------------------------------------------------
// phmm_mutation_prime_sets, phmm_mutation_prime
// -------------------------------------------------------------------------------------------------------------
// Largest tile of the call's ordered-pair index space, and the CIGAR scratch a tile may use.
static constexpr long long kMutTilePairs = 1LL << 19;
static constexpr long long kMutCigarBudget = 1LL << 30;

// phmm_mutation_prime_sets after begin_call; phmm_mutation_prime is its one-set case.
static int mutation_prime_sets(phmm_engine* e, const phmm_mutation_model* m, int32_t n_sets, const int32_t* set_first,
                               const int64_t* off, const char* seq, double* out, int32_t* status)
{
    if (!m || !set_first || !off || !seq || !out || !status) { e->err = "null argument"; return PHMM_ERR_INVALID; }
    if (n_sets < 0) { e->err = "negative set count"; return PHMM_ERR_INVALID; }
    if (n_sets == 0) return PHMM_OK;
    if (set_first[0] != 0) { e->err = "set_first[0] must be 0"; return PHMM_ERR_INVALID; }
    int rc;
    long long all = 0;                                                            // ordered pairs of the call
    for (int s = 0; s < n_sets; ++s) {
        const long long size = (long long)set_first[s + 1] - set_first[s];
        if (size < 0) { e->err = "set_first must be non-decreasing"; return PHMM_ERR_INVALID; }
        if (size > 0 && (rc = phmm_checks::mutation_haplotype_count(size, e->err)) != PHMM_OK) return rc;
        all += size * size;
    }
    const int H = set_first[n_sets];
    if ((rc = phmm_checks::mutation_offsets(H, off, e->err)) != PHMM_OK) return rc;
    if (all > PHMM_MUT_MAX_PAIRS) { e->err = "more than PHMM_MUT_MAX_PAIRS (2^26) ordered pairs in one call"; return PHMM_ERR_INVALID; }
    if (H == 0) return PHMM_OK;
    // per set: its first pair and its longest haplotype; the call's longest haplotype sizes the CIGAR scratch
    std::vector<long long> pair_first((size_t)n_sets + 1, 0), set_len((size_t)n_sets, 0);
    long long Lmax = 0;
    for (int s = 0; s < n_sets; ++s) {
        const long long size = set_first[s + 1] - set_first[s];
        pair_first[s + 1] = pair_first[s] + size * size;
        for (int h = set_first[s]; h < set_first[s + 1]; ++h) set_len[s] = std::max<long long>(set_len[s], off[h + 1] - off[h]);
        Lmax = std::max(Lmax, set_len[s]);
    }
    const int X = m->max_indel_length;
    const long long B = off[H];
    // 1. the context indel model of every haplotype of the call (host; per haplotype, so the sets' concatenation does not change it)
    std::vector<int32_t> cell((size_t)B);
    std::vector<int8_t> gop((size_t)B), gex((size_t)B);
    rc = phmm_mutation_context(m, H, off, seq, cell.data(), gop.data(), gex.data(), 0);
    if (rc != PHMM_OK) { e->err = phmm_error_model_last_error(); return rc; }
    // 2. one padded truth per given haplotype: 32 N's, the haplotype, N's up to its own set's longest haplotype + 64 (pad penalty 60), no
    //    SNV mask — byte for byte the truth a call of that set alone builds; the targets are the haplotypes with every quality = the SNV
    //    penalty (denovo_model.cpp:208-262, pair_hmm.hpp:853-856)
    long long T = 0;                                                              // truth bases
    for (int s = 0; s < n_sets; ++s) T += (long long)(set_first[s + 1] - set_first[s]) * (set_len[s] + 64);
    auto align_up = [](size_t x) { return (x + 255) & ~(size_t)255; };
    size_t at = 0;
    const size_t o_tseq = at; at = align_up(at + (size_t)T);
    const size_t o_tgo = at;  at = align_up(at + (size_t)T);
    const size_t o_tge = at;  at = align_up(at + (size_t)T);
    const size_t o_zero = at; at = align_up(at + (size_t)T);                      // SNV masks / priors, mapq, reverse, begin (T >= 65 H)
    const size_t o_toff = at; at = align_up(at + ((size_t)H + 1) * sizeof(int64_t));
    const size_t o_goff = at; at = align_up(at + ((size_t)H + 1) * sizeof(int64_t));
    const size_t o_bases = at; at = align_up(at + (size_t)B);
    const size_t o_quals = at; at = align_up(at + (size_t)B);
    const size_t o_cell = at; at = align_up(at + (size_t)B * sizeof(int32_t));
    const size_t o_logp = at; at = align_up(at + m->logp.size() * sizeof(float));
    const size_t o_pfirst = at; at = align_up(at + ((size_t)n_sets + 1) * sizeof(int64_t));
    const size_t o_sfirst = at; at = align_up(at + ((size_t)n_sets + 1) * sizeof(int32_t));
    const long long cigar_stride = 4 * Lmax + 160;                                  // >= 2 characters per alignment column
    const long long tile = std::max(1LL, std::min(kMutTilePairs, kMutCigarBudget / cigar_stride));
    const size_t o_offs = at; at = align_up(at + (size_t)tile * sizeof(int32_t));
    std::vector<char> blob(at, 0);
    char* bp = blob.data();
    long long t0 = 0;
    for (int s = 0; s < n_sets; ++s) {
        const long long Lp = set_len[s] + 64;
        for (int h = set_first[s]; h < set_first[s + 1]; ++h, t0 += Lp) {
            const long long o = off[h], len = off[h + 1] - o;
            std::memset(bp + o_tseq + t0, 'N', (size_t)Lp);
            std::memcpy(bp + o_tseq + t0 + 32, seq + o, (size_t)len);
            std::memset(bp + o_tgo + t0, 60, (size_t)Lp);
            std::memset(bp + o_tge + t0, 60, (size_t)Lp);
            std::memcpy(bp + o_tgo + t0 + 32, gop.data() + o, (size_t)len);
            std::memcpy(bp + o_tge + t0 + 32, gex.data() + o, (size_t)len);
            ((int64_t*)(bp + o_toff))[h] = t0;
        }
    }
    ((int64_t*)(bp + o_toff))[H] = t0;
    std::memcpy(bp + o_goff, off, ((size_t)H + 1) * sizeof(int64_t));
    std::memcpy(bp + o_pfirst, pair_first.data(), pair_first.size() * sizeof(int64_t));
    std::memcpy(bp + o_sfirst, set_first, ((size_t)n_sets + 1) * sizeof(int32_t));
    std::memcpy(bp + o_bases, seq, (size_t)B);
    std::memset(bp + o_quals, m->snv_penalty, (size_t)B);
    std::memcpy(bp + o_cell, cell.data(), (size_t)B * sizeof(int32_t));
    std::memcpy(bp + o_logp, m->logp.data(), m->logp.size() * sizeof(float));
    std::fill((int32_t*)(bp + o_offs), (int32_t*)(bp + o_offs) + tile, 32);
    CU(e->mu_in.ensure(at));
    CU(cudaMemcpyAsync(e->mu_in.p, blob.data(), at, cudaMemcpyHostToDevice, e->stream));
    char* d = e->mu_in.as<char>();
    phmm_haplotypes truths {H, (const int64_t*)(d + o_toff), d + o_tseq, d + o_zero, (const int8_t*)(d + o_zero), d + o_zero,
                            (const int8_t*)(d + o_zero), (const int8_t*)(d + o_tgo), (const int8_t*)(d + o_tge), nullptr};
    phmm_reads targets {H, (const int64_t*)(d + o_goff), d + o_bases, (const uint8_t*)(d + o_quals), (const uint8_t*)(d + o_zero),
                        (const uint8_t*)(d + o_zero), (const int64_t*)(d + o_zero)};
    phmm_config cfg;
    phmm_default_config(&cfg);
    cfg.max_indel_error = 32; cfg.use_mapping_quality = 0; cfg.use_flank_state = 0; cfg.map_positions = 0;
    CU(e->mu_out.ensure((size_t)all * (sizeof(double) + sizeof(int32_t))));
    double* d_out = e->mu_out.as<double>();
    int* d_status = (int*)(d_out + all);
    CU(e->mu_list.ensure((size_t)tile * (sizeof(int2) + sizeof(long long)) + 256));
    int2* d_list = e->mu_list.as<int2>();
    long long* d_oidx = (long long*)(d_list + tile);
    int* d_count = (int*)(d_oidx + tile);
    CU(e->mu_res.ensure((size_t)tile * (sizeof(int64_t) + sizeof(double) + sizeof(int32_t))));
    int64_t* d_toff = e->mu_res.as<int64_t>();
    double* d_lk = (double*)(d_toff + tile);
    int32_t* d_ast = (int32_t*)(d_lk + tile);
    CU(e->mu_cig.ensure((size_t)tile * cigar_stride));
    // 3. per tile of the call's pair space (a tile may begin or end inside a set): list the pairs, align the listed ones (band 32, target
    //    offset 32), re-score their CIGARs
    for (long long lo = 0; lo < all; lo += tile) {
        const long long hi = std::min(all, lo + tile);
        CU(cudaMemsetAsync(d_count, 0, sizeof(int), e->stream));
        k_mutation_pairs<<<(unsigned)std::min<long long>((hi - lo + 255) / 256, 4096), 256, 0, e->stream>>>(lo, hi, n_sets, (const long long*)(d + o_pfirst),
                                                                                                          (const int*)(d + o_sfirst), (const long long*)(d + o_goff),
                                                                                                          d_out, d_status, d_list, d_oidx, d_count);
        LAUNCHED();
        CU(cudaGetLastError());
        int count = 0;
        CU(cudaMemcpyAsync(&count, d_count, sizeof(int), cudaMemcpyDeviceToHost, e->stream));
        CU(cudaStreamSynchronize(e->stream));
        if (count == 0) continue;
        rc = align_impl(e, &cfg, &truths, &targets, (const phmm_pair*)d_list, count, nullptr, (const int32_t*)(d + o_offs), nullptr,
                        d_toff, d_lk, e->mu_cig.as<char>(), (int32_t)cigar_stride, d_ast, PHMM_SPACE_DEVICE);
        if (rc != PHMM_OK) return rc;
        k_mutation_rescore<<<(unsigned)((count + 127) / 128), 128, 0, e->stream>>>(count, d_list, d_oidx, (const long long*)d_toff, d_ast,
                                                                                 e->mu_cig.as<char>(), (int)cigar_stride, (const long long*)(d + o_goff),
                                                                                 (const int*)(d + o_cell), (const float*)(d + o_logp), X,
                                                                                 m->snv_log_prior, d_out, d_status);
        LAUNCHED();
        CU(cudaGetLastError());
    }
    CU(cudaMemcpyAsync(out, d_out, (size_t)all * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
    CU(cudaMemcpyAsync(status, d_status, (size_t)all * sizeof(int32_t), cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    for (long long i = 0; i < all; ++i) if (status[i] < 0) { e->err = "internal error: CIGAR scratch too small"; return PHMM_ERR_CUDA; }
    return PHMM_OK;
}

int phmm_mutation_prime_sets(phmm_engine* e, const phmm_mutation_model* m, int32_t n_sets, const int32_t* set_first,
                             const int64_t* off, const char* seq, double* out, int32_t* status)
{
    if (int rc0 = begin_call(e)) return rc0;
    return mutation_prime_sets(e, m, n_sets, set_first, off, seq, out, status);
}

int phmm_mutation_prime(phmm_engine* e, const phmm_mutation_model* m, int32_t n, const int64_t* off, const char* seq,
                        double* out, int32_t* status)
{
    if (int rc0 = begin_call(e)) return rc0;
    if (int rc = phmm_checks::mutation_set(m, n, off, seq, out, status, e->err)) return rc;
    const int32_t set_first[2] = {0, n};
    return mutation_prime_sets(e, m, 1, set_first, off, seq, out, status);
}

// -------------------------------------------------------------------------------------------------------------
// phmm_populate
// -------------------------------------------------------------------------------------------------------------
// One region list for every call: phmm_populate is the one-region case. Host copies of the region arrays (a few KB).
struct RegionSetup {
    std::vector<RegionInfo> regs;
    long long total_out = 0;
    int Hmax = 0;
    bool any_flank = false;
};

// One more region after those laid out so far: its result offset, the widest region, its flank state where the configuration uses one.
static void add_region(RegionSetup& setup, const phmm_config* cfg, int h0, int nH, int r0, int nR, const phmm_flank_state* flank)
{
    RegionInfo r {};
    r.h0 = h0; r.nH = nH; r.r0 = r0; r.nR = nR;
    r.out_off = setup.total_out;
    setup.total_out += (long long)nH * nR;
    setup.Hmax = std::max(setup.Hmax, nH);
    const bool fl = flank && flank->has_flank && cfg && cfg->use_flank_state;
    r.use_flanks = fl ? 1 : 0; r.lhs = fl ? (int)flank->lhs_flank : 0; r.rhs = fl ? (int)flank->rhs_flank : 0;
    setup.any_flank = setup.any_flank || fl;
    setup.regs.push_back(r);
}

// The region list of phmm_populate_regions / phmm_assign_reads, checked and laid out.
static int region_setup(phmm_engine* e, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                        const phmm_regions* regions, RegionSetup& setup)
{
    const int rc = phmm_checks::regions(haps, reads, regions, e->err);
    if (rc != PHMM_OK) return rc;
    for (int g = 0; g < regions->n; ++g) {
        const int nH = regions->hap_first[g + 1] - regions->hap_first[g], nR = regions->read_first[g + 1] - regions->read_first[g];
        add_region(setup, cfg, regions->hap_first[g], nH, regions->read_first[g], nR, regions->flank ? regions->flank + g : nullptr);
    }
    return PHMM_OK;
}

// One populate call as its entry point describes it. Every call has a region list. Candidate position lists and templates need a
// single region; `staged` marks phmm_assign_reads / phmm_assign_templates, whose matrix stays on the device: the call chooses every
// read's (k_assign_top) or every template's (k_assign_template_top) haplotypes there and copies out top and the optional out / status
// only. An assign call with templates has them in any number of regions: out is then the regions' [H_g][T_g] template values.
struct PopulateCall {
    const phmm_config* cfg = nullptr;
    const phmm_haplotypes* haps = nullptr;
    const phmm_reads* reads = nullptr;
    int space = PHMM_SPACE_HOST;
    RegionSetup regions;
    const phmm_positions* positions = nullptr;      // a caller's candidate lists (CSR over the result slots, in `space`), or null
    double* out = nullptr;                          // the regions' [H_g][R_g] matrices back to back, or [H][templates]
    int32_t* status = nullptr;                      // optional; laid out as the regions' matrices
    long long out_pitch = 0;                        // row pitch of out / status in elements (0: dense [H][R]): a read chunk lands in
                                                    // its column block of the caller's [H][R_total] matrix
    const int64_t* template_off = nullptr;          // phmm_populate_templates: [n_templates + 1] read ranges, one value per (haplotype, template)
    int n_templates = 0;
    // phmm_assign_reads: the batch it has staged already (the pair mapper read it), the mapper's CSR over the result slots on the
    // device (null: cfg->map_positions = 0), the log priors on the device (or null), the caller's top sets
    const Staged* staged = nullptr;
    const long long* mapped_off = nullptr;
    const int32_t* mapped_pos = nullptr;
    long long n_mapped = 0;
    const double* log_priors = nullptr;
    uint64_t* top = nullptr;                        // per read, or per template when the call has templates
    std::vector<TemplateGroup> template_groups;     // phmm_assign_templates: each region's templates (template_off in host memory)
    // the _reset entry points: `haps` holds the sequences block's n / off / seq / begin only; pop_reset derives the six arrays from
    // the sequences under `model` on the device, and the call populates from those
    bool reset = false;
    const phmm_error_model* model = nullptr;
    const uint8_t* is_substitution = nullptr;

    bool listed() const { return positions && positions->off && positions->pos; }
    bool assign() const { return staged != nullptr; }
};

// phmm_populate and its variants: one region of all haplotypes x all reads. Null blocks are rejected when the batch is staged.
static PopulateCall one_region_call(const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads, const phmm_positions* positions,
                                    const phmm_flank_state* flank, double* out, int32_t* status, int space)
{
    PopulateCall c;
    c.cfg = cfg; c.haps = haps; c.reads = reads; c.space = space;
    c.positions = positions; c.out = out; c.status = status;
    add_region(c.regions, cfg, 0, haps ? haps->n : 0, 0, reads ? reads->n : 0, flank);
    return c;
}

// What the phases of populate_impl share: the kernels' parameter block and the host-side sizes and decisions behind it.
struct PopState {
    phmm_haplotypes reset_haps {};              // pop_reset: the derived block, device-resident, and its offsets on the host
    std::vector<long long> reset_off_host;
    Staged s;
    PopParams p {};
    int band = 0, G = 0, R = 0;
    int H = 0;                                  // haplotype slots per read (the widest region)
    long long HR = 0;                           // result slots of the whole call
    int Lmax_all = 0, Lmax_fast = 0;
    // pop_candidates: candidates a pair can have, and how many of them can reach a DP
    int max_cand = 2, max_dp_per_pair = 1;
    bool use_mapper = false;
    // pop_decide
    bool role_band = false, direct = false, flank_fb_ok = false, pair_flank_kernels = false, wide_flank_kernels = false;
    SchedMode mode {};
    int NL = 1, groups = 1, fast_row_stride = 0, wide_row_stride = 0, wide_warps = 0;
    size_t pairs_cap = 0;
    long long n_pairs = 0, n_wide = 0, n_generic = 0;       // upper bounds of the work lists (exact counts stay on the device)
    SchedTotals tot {};
    // pop_outputs, pop_tile_scratch
    double* d_out = nullptr;
    int* counters = nullptr;
    long long reads_per_tile = 0, pairs_per_tile = 0;
    int slow_blocks = 1;
    // pop_kernel_attrs
    size_t smem = 0, role_smem = 0, wsmem = 0;
    int blocks_per_sm = 1, role_blocks_per_sm = 0, wide_blocks_per_sm = 1, role_groups = 1;
    bool role_warps = false;
    // the tile loop: DP kernels timed per tile (tile_events) or, for a call of generic tiles only, once (ev0 / ev1)
    size_t n_timed = 0;
    bool timed = false;

    const std::chrono::steady_clock::time_point t_begin = std::chrono::steady_clock::now();
    static bool tracing() { static const bool on = std::getenv("PHMM_TRACE") != nullptr; return on; }
    void lap(const phmm_engine* e, const char* what) const
    {
        if (tracing()) std::fprintf(stderr, "[phmm %p] %-18s %8.3f ms  (abs %.3f)\n", (const void*)e, what, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_begin).count(),
                                    std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count());
    }
};

// Phase 0, calls with an error model only: reset() for every haplotype on the device (reset_arrays, one synchronisation) into the
// engine's buffers, and the device-resident haplotype block over them that the rest of the call stages.
static int pop_reset(phmm_engine* e, const PopulateCall& c, PopState& st)
{
    const phmm_haplotypes* h = c.haps;
    ResetStaged r;
    int rc = reset_arrays(e, c.model, h->n, h->off, h->seq, c.is_substitution, c.space, nullptr, nullptr, &r);
    if (rc != PHMM_OK) return rc;
    e->last_dp_ms = 0.0;                        // the call's DP kernel time is populate's alone
    const long long* d_begin = nullptr;
    if (h->n > 0 && (rc = stage(e, e->h_begin, (const long long*)h->begin, (size_t)h->n, c.space, &d_begin))) return rc;
    st.reset_haps = {h->n, r.off, r.seq, r.a.mask_f, r.a.prior_f, r.a.mask_r, r.a.prior_r, r.a.gap_open, r.a.gap_extend, (const int64_t*)d_begin};
    st.reset_off_host = std::move(r.hoff);
    return PHMM_OK;
}

// Phase 1: the checks a call can fail before any device work, then the batch, the regions and the per-read region / result slot
// on the device.
static int pop_stage(phmm_engine* e, const PopulateCall& c, PopState& st)
{
    int rc = phmm_checks::config_and_output(c.cfg, c.assign() ? (const void*)c.top : (const void*)c.out, c.reads, e->err);
    if (rc != PHMM_OK) return rc;
    const bool several = c.regions.regs.size() > 1;
    if (c.listed() && several) { e->err = "candidate position lists are not supported with several regions"; return PHMM_ERR_INVALID; }
    if (c.template_off && several && !c.assign()) { e->err = "templates are not supported with several regions"; return PHMM_ERR_INVALID; }
    Staged& s = st.s;
    if (c.assign()) s = *c.staged;
    else if (c.reset) rc = stage_batch(e, &st.reset_haps, c.reads, c.space, s, false, true, PHMM_SPACE_DEVICE, &st.reset_off_host);
    else rc = stage_batch(e, c.haps, c.reads, c.space, s, false, true);
    if (rc != PHMM_OK) return rc;
    const int band = st.band = round_band(std::max(1, c.cfg->max_indel_error));
    const int G = st.G = (int)c.regions.regs.size(), R = st.R = s.rd.n;
    st.H = c.regions.Hmax;
    st.HR = c.regions.total_out;
    CU(e->regs.ensure((size_t)G * sizeof(RegionInfo)));
    CU(cudaMemcpyAsync(e->regs.p, c.regions.regs.data(), (size_t)G * sizeof(RegionInfo), cudaMemcpyHostToDevice, e->stream));
    CU(e->rregion.ensure((size_t)R * sizeof(int)));
    CU(e->rpbase.ensure((size_t)R * sizeof(long long)));
    CU(e->rpstride.ensure((size_t)R * sizeof(int)));
    k_read_regions<<<(R + 255) / 256, 256, 0, e->stream>>>(R, G, e->regs.as<RegionInfo>(), e->rregion.as<int>(), e->rpbase.as<long long>(), e->rpstride.as<int>());
    LAUNCHED();
    s.rd.region = e->rregion.as<int>(); s.rd.pbase = e->rpbase.as<long long>(); s.rd.pstride = e->rpstride.as<int>();
    // Everything from here to the final copy-out is enqueued without waiting for the device: sizes come from upper bounds
    // the host can derive from the offsets, the kernels clip them against the scheduler's device-resident totals.
    st.Lmax_all = (int)s.read_len_max;
    st.Lmax_fast = std::min(st.Lmax_all, kFastMaxReadLen);
    PopParams& p = st.p;
    p.hp = s.hp; p.rd = s.rd;
    p.band = band; p.nuc_prior = c.cfg->nuc_prior; p.one = 1;
    p.shortcut = c.cfg->disable_naive_shortcut ? 0 : 1;
    p.regs = e->regs.as<RegionInfo>();
    p.Hmax = st.H;
    p.reserved_sms = e->reserved_sms;
    p.use_mapq = c.cfg->use_mapping_quality; p.mapq_cap = c.cfg->mapping_quality_cap; p.mapq_trigger = c.cfg->mapping_quality_cap_trigger;
    p.use_flanks = c.regions.any_flank ? 1 : 0;
    if (p.use_flanks && band <= kFlankFbMaxBand) {
        // prefix counts of the 'N'-like table columns per haplotype and strand: the flank kernels' replay test in four loads
        CU(e->npre_f.ensure((size_t)s.hap_bases * sizeof(uint32_t)));
        CU(e->npre_r.ensure((size_t)s.hap_bases * sizeof(uint32_t)));
        k_ncol_prefix<<<(unsigned)((2LL * s.hp.n * 32 + 127) / 128), 128, 0, e->stream>>>(s.hp.n, s.hp.off, s.hp.tab_f, s.hp.tab_r, e->npre_f.as<uint32_t>(), e->npre_r.as<uint32_t>());
        LAUNCHED();
        p.hp.npre_f = e->npre_f.as<uint32_t>(); p.hp.npre_r = e->npre_r.as<uint32_t>();
    }
    return PHMM_OK;
}

// Phase 2: where a pair's candidate positions come from: the caller's lists, phmm_assign_reads' mapped lists, populate's own capped
// mapper per tile, or nowhere (the original position only). Candidates a pair can have: listed / mapped positions + the original
// position + the shifted fallback (haplotype_likelihood_model.cpp:211-259); at most (listed + 1) of them reach a DP.
static int pop_candidates(phmm_engine* e, const PopulateCall& c, PopState& st)
{
    PopParams& p = st.p;
    int rc;
    if (c.listed() || c.mapped_off) {
        // Candidate lists: CSR arrays on the device; the host needs the total (to size the copy) and the longest list (to size the
        // per-read task lists: the reference accepts lists of any length) — reduced on the device, 32 bytes back.
        long long total = c.n_mapped;
        p.pos_off = c.mapped_off; p.pos = c.mapped_pos;
        if (!c.mapped_off) {
            if ((rc = stage_positions(e, c.positions, st.HR, c.space, &p.pos_off, &p.pos, &total))) return rc;
            if (total < 0) { e->err = "candidate position offsets must be non-decreasing and start at 0"; return PHMM_ERR_INVALID; }
        }
        OffsetSummary ps {};
        CU(e->scores.ensure(sizeof(OffsetSummary)));
        CU(cudaMemsetAsync(e->scores.p, 0, sizeof(OffsetSummary), e->stream));
        k_offsets_summary<<<(unsigned)std::min<long long>((st.HR + 255) / 256, 2048), 256, 0, e->stream>>>(p.pos_off, st.HR > 0x7fffffffLL ? 0x7fffffff : (int)st.HR, e->scores.as<OffsetSummary>());
        LAUNCHED();
        CU(cudaMemcpyAsync(&ps, e->scores.p, sizeof(OffsetSummary), cudaMemcpyDeviceToHost, e->stream));
        CU(cudaStreamSynchronize(e->stream));
        if (ps.first != 0 || kOffsetBig - ps.inv_len_min < 0 || ps.last != total) { e->err = "candidate position offsets must be non-decreasing and start at 0"; return PHMM_ERR_INVALID; }
        if (ps.len_max > 4096) { e->err = "more than 4096 candidate positions for one (haplotype, read) pair"; return PHMM_ERR_INVALID; }
        st.max_cand = (int)ps.len_max + 2;
        st.max_dp_per_pair = (int)ps.len_max + 1;
    } else if (c.cfg->map_positions && !c.assign()) {
        st.use_mapper = true;
        st.max_cand = kMaxMapped + 2;   // the mapper emits <= 10 (haplotype_likelihood_array.hpp:103-104)
        st.max_dp_per_pair = kMaxMapped + 1;
        if ((rc = prepare_mapper(e, st.s)) != PHMM_OK) return rc;
    }
    p.single_candidate = st.max_dp_per_pair == 1 ? 1 : 0;
    return PHMM_OK;
}

// Phase 3: which kernels serve the call and how its reads are scheduled. Host arithmetic only, no CUDA call.
static void pop_decide(const PopulateCall& c, PopState& st)
{
    PopParams& p = st.p;
    const int band = st.band, H = st.H, R = st.R;
    // bands 32 / 64 with enough tasks per read to fill a warp: one WARP per chunk of the band (k_populate_roles) instead of one lane
    static const bool no_role_warps = std::getenv("PHMM_NO_ROLE_WARPS") != nullptr;       // measurement hook: the lane-per-chunk kernel for every band
    st.role_band = (band == 32 || band == 64) && H >= 17 && !no_role_warps;
    // Direct mode (PopParams::direct): every pair has one candidate position and a plain DP for it, so the pair list needs neither
    // the classify pass nor the epilogue. Reads with 'N' go to the wide list, which keeps both. k_populate_roles keeps the classify
    // path: the task derivation and the FP64 finish would more than double its register spills.
    static const bool no_direct = std::getenv("PHMM_NO_DIRECT") != nullptr;              // measurement hook: the classify path for every list
    st.direct = !no_direct && !p.pos_off && !st.use_mapper && !p.shortcut && !c.regions.any_flank && !c.cfg->use_int_scores && !st.role_band;
    p.direct = st.direct ? 1 : 0;

    // scheduling: equal-length read pairs for the packed kernels, 32-bit multi-lane kernels for what they cannot take, and the
    // thread-per-pair generic kernel for the rest (foreign alphabet, qualities above 127, reads beyond the shared-memory budget)
    // the DP task word packs (haplotype, window offset) into 16 + 16 bits
    const bool task_word_ok = st.s.hp.n <= 65535 && st.s.max_hap_len <= 65535;
    st.NL = lanes_per_alignment(band);
    // wide (32-bit) path: row entries of one read per warp in shared memory; long reads get fewer warps per block
    st.wide_row_stride = (int)((std::min<long long>(st.Lmax_all, kWideMaxReadLen) + 2) & ~1LL);
    st.wide_warps = (int)std::max<long long>(0, std::min<long long>(kFastWarpsPerBlock, (220LL << 10) / ((long long)st.wide_row_stride * (long long)sizeof(RowEntry))));
    SchedMode& mode = st.mode;
    mode.packed_ok = task_word_ok ? 1 : 0;
    mode.wide_ok = (task_word_ok && st.wide_warps >= 1) ? 1 : 0;
    mode.force_wide = c.cfg->use_int_scores ? 1 : 0;
    mode.n_to_wide = (band > 32 || st.direct) ? 1 : 0;
    mode.wide_max_len = kWideMaxReadLen;
    const bool fast_ok = mode.packed_ok && !mode.force_wide;
    // lane groups per warp of the packed kernel: with few haplotypes a read has few DP tasks, so several read pairs share a warp
    const int groups = st.groups = std::max(1, std::min(32 / st.NL, H >= 17 ? 1 : (H >= 9 ? 2 : 4)));
    // device-side scheduling: length buckets → equal-length read pairs (padded to multiples of `groups` per bucket) + wide + generic lists
    st.pairs_cap = (size_t)R / 2 + (size_t)kLenBins * groups + 8;
    // distinct read lengths the fast path can see: bounds the padding of the length-bucketed pair list
    // (a bucket of c reads holds ceil(c / 2) pairs rounded up to a multiple of `groups`)
    const long long len_bins = std::max<long long>(1, std::min<long long>({(long long)R, (long long)st.Lmax_fast - std::min<long long>(st.s.read_len_min, st.Lmax_fast) + 1, (long long)kLenBins}));
    st.n_pairs = fast_ok ? std::min<long long>((long long)st.pairs_cap, R / 2 + len_bins * groups + 1) : 0;
    // reads the packed path cannot take exist only if the host can see a reason (int scores, a long read) or the device finds one
    // (quality sums, foreign bytes): the wide and generic tiles are always enqueued, their kernels clip against the device totals
    st.n_wide = mode.wide_ok ? R : 0;
    st.n_generic = R;

    st.fast_row_stride = (st.Lmax_fast + 2) & ~1;
    // the packed forward / backward flank kernels instead of the lean labelled one
    static const bool no_flank_fb = std::getenv("PHMM_NO_FLANK_FB") != nullptr;           // measurement hook: the labelled one-alignment-per-thread flank kernels only
    st.flank_fb_ok = !no_flank_fb && band <= kFlankFbMaxBand;
    // Whether a tile's flank kernels run: bands above 32 have none, and on the wide list the labelled kernel needs a warp's row
    // entries of the call's longest read in shared memory (reads of 6 400+ bases do not fit). The classify pass reads this decision:
    // near-flank candidates of a tile whose flank kernels do not run take the traceback queue (k_slow_flank) instead.
    st.pair_flank_kernels = band <= 32;
    st.wide_flank_kernels = band <= 32 && (st.wide_row_stride <= st.fast_row_stride + 8 ||
                                           (size_t)kFastWarpsPerBlock * st.wide_row_stride * sizeof(RowEntry) <= (200u << 10));
}

// Phase 4: the scheduling kernels: the reads into the pair, wide and generic lists; the totals stay on the device (p.tot).
static int pop_schedule(phmm_engine* e, PopState& st)
{
    const Staged& s = st.s;
    const int R = st.R;
    const size_t sched_bytes = (size_t)(4 * (kLenBins + 1) + 16) * sizeof(int) + sizeof(SchedTotals) + 16;
    CU(e->sched.ensure(sched_bytes));
    CU(e->sorted.ensure((size_t)R * sizeof(int)));
    CU(e->pairs.ensure(2 * st.pairs_cap * sizeof(int)));
    CU(e->generic_reads.ensure((size_t)R * sizeof(int)));
    CU(e->wide_reads.ensure((size_t)R * sizeof(int)));
    int* base = e->sched.as<int>();
    int* hist = base, *read_start = base + (kLenBins + 1), *pair_start = base + 2 * (kLenBins + 1), *cursors = base + 3 * (kLenBins + 1);
    int* misc = base + 4 * (kLenBins + 1);          // [0] n_generic, [1] lmax_all, [2] bad, [3] packed reads with 'N', [4] n_wide
    SchedTotals* d_tot = (SchedTotals*)(misc + 16);
    unsigned long long* d_cells = (unsigned long long*)((char*)d_tot + ((sizeof(SchedTotals) + 7) & ~size_t(7)));
    CU(cudaMemsetAsync(base, 0, sched_bytes, e->stream));
    k_sched_hist<<<(R + 255) / 256, 256, 0, e->stream>>>(R, s.rd.info, st.mode, hist, e->generic_reads.as<int>(), e->wide_reads.as<int>(), misc,
                                                          s.rd.region, e->regs.as<RegionInfo>(), st.band, d_cells);
    LAUNCHED();
    k_sched_scan<<<1, kLenBins, 0, e->stream>>>(hist, st.groups, read_start, pair_start, cursors, misc, d_cells, d_tot);
    LAUNCHED();
    k_sched_scatter<<<(R + 255) / 256, 256, 0, e->stream>>>(R, s.rd.info, st.mode, read_start, cursors, e->sorted.as<int>());
    LAUNCHED();
    k_sched_pairs<<<(unsigned)((st.pairs_cap + 255) / 256), 256, 0, e->stream>>>(d_tot, read_start, pair_start, e->sorted.as<int>(), e->pairs.as<int>());
    LAUNCHED();
    CU(cudaGetLastError());
    st.p.tot = d_tot;
    return PHMM_OK;
}

// Phase 5a: the result slots (best / status / out) and the per-tile cursors.
static int pop_outputs(phmm_engine* e, const PopulateCall& c, PopState& st)
{
    PopParams& p = st.p;
    const long long HR = st.HR;
    CU(e->best.ensure((size_t)HR * sizeof(int)));
    CU(e->status.ensure((size_t)HR * sizeof(int)));
    CU(e->counters.ensure(256));
    CU(cudaMemsetAsync(e->counters.p, 0, 256, e->stream));
    if (!st.direct) {           // direct mode: k_list_slots sets up the wide / generic tiles' slots, the pair list needs none
        CU(cudaMemsetAsync(e->status.p, 0, (size_t)HR * sizeof(int), e->stream));
        k_fill_int<<<(unsigned)((HR + 255) / 256), 256, 0, e->stream>>>(e->best.as<int>(), HR, kBestInf);
        LAUNCHED();
    }
    p.best = e->best.as<int>();
    p.status = e->status.as<int>();
    CU(e->out.ensure((size_t)HR * sizeof(double)));
    // a device-space matrix is written in place; templates sum from the engine's copy, and phmm_assign_reads may pass no matrix at all
    st.d_out = (c.space == PHMM_SPACE_DEVICE && !c.template_off && c.out) ? c.out : e->out.as<double>();
    p.out = st.d_out;
    p.out_row_extra = st.d_out == c.out && c.space == PHMM_SPACE_DEVICE && c.out_pitch > st.R ? c.out_pitch - st.R : 0LL;
    p.out_status = c.status ? p.status : nullptr;
    if (st.direct && p.use_mapq) {
        CU(e->mapq_tab.ensure(256 * sizeof(MapqTerms)));
        k_mapq_terms<<<1, 256, 0, e->stream>>>(p.mapq_cap, p.mapq_trigger, e->mapq_tab.as<MapqTerms>());
        LAUNCHED();
        p.mapq_tab = e->mapq_tab.as<MapqTerms>();
    }
    p.flags = e->flags.as<int>();
    int* counters = st.counters = e->counters.as<int>();
    p.pair_cursor = counters + 0;
    p.flank_cursor = counters + 1;
    p.any_flank_tasks = counters + 2;
    p.slow_count = counters + 3;
    p.acc_cursor = counters + 4;
    p.any_acc_tasks = counters + 5;
    p.fb_cursor = counters + 6;
    p.fb_rounds = counters + 7;
    return PHMM_OK;
}

// Phase 5b: the tile size, and the per-tile scratch (mapped candidate lists, DP task lists, traceback queue), which must fit fixed budgets.
static int pop_tile_scratch(phmm_engine* e, PopState& st)
{
    PopParams& p = st.p;
    const int band = st.band, H = st.H, R = st.R, groups = st.groups;
    const long long slow_budget = 8LL << 20;   // traceback-queue entries (16 bytes each)
    // DP tasks a pair can queue: listed / mapped positions (any number when the caller lists them) + the original position
    p.fcap = (int)std::min<long long>(0x7fffffff, (long long)H * st.max_dp_per_pair);   // a read's task list: one DP task per (haplotype, candidate position)
    long long reads_per_tile = std::max<long long>(R, 2 * st.n_pairs);   // one tile unless a budget says otherwise
    if (st.use_mapper) reads_per_tile = std::max<long long>(2, std::min<long long>(reads_per_tile, (1LL << 30) / (41LL * H)));   // (10 x int32 + 1 byte) per pair
    reads_per_tile = std::max<long long>(2, std::min<long long>(reads_per_tile, (160LL << 20) / p.fcap));   // two lists of 4-byte entries: <= 1.25 GiB
    if (p.use_flanks) reads_per_tile = std::max<long long>(2, std::min<long long>(reads_per_tile, slow_budget / ((long long)H * st.max_cand)));
    st.reads_per_tile = reads_per_tile;
    st.pairs_per_tile = std::max<long long>((long long)groups, ((reads_per_tile + 1) / 2 + groups - 1) / (long long)groups * (long long)groups);
    // With several tiles per list the exact list sizes are worth one early synchronisation: empty wide / generic tiles cost a
    // handful of launches each.
    if (reads_per_tile < R) {
        CU(cudaMemcpyAsync(&st.tot, p.tot, sizeof(SchedTotals), cudaMemcpyDeviceToHost, e->stream));
        CU(cudaStreamSynchronize(e->stream));
        st.n_pairs = std::min<long long>(st.n_pairs, st.tot.n_pairs);
        st.n_wide = std::min<long long>(st.n_wide, st.tot.n_wide);
        st.n_generic = std::min<long long>(st.n_generic, st.tot.n_generic);
    }
    // work-list entries one tile can hold (pair tiles: two per pair, padding entries included)
    const size_t tile_list_cap = (size_t)std::max<long long>(std::min<long long>(2 * st.pairs_per_tile, 2 * std::max<long long>(st.n_pairs, groups)), std::min<long long>(reads_per_tile, R)) + 2;
    if (st.use_mapper) {
        CU(e->kpos.ensure(tile_list_cap * H * kMaxMapped * sizeof(int32_t)));
        CU(e->kcnt.ensure(tile_list_cap * H));
    }
    CU(e->ftasks.ensure(tile_list_cap * p.fcap * sizeof(uint32_t)));
    CU(e->fcnt.ensure(4 * tile_list_cap * sizeof(int)));
    p.ftasks = e->ftasks.as<uint32_t>();
    p.fcnt = e->fcnt.as<int>();
    // the 32-bit flank kernel's lists (near-flank candidates, reads holding 'N'): whether any exist is only known on the device
    CU(e->gtasks.ensure(tile_list_cap * p.fcap * sizeof(uint32_t)));
    p.gtasks = e->gtasks.as<uint32_t>();
    p.gcnt = p.fcnt + tile_list_cap;
    p.acnt = p.fcnt + 2 * tile_list_cap;
    p.fb_round_base = p.fcnt + 3 * tile_list_cap;
    if (p.use_flanks && band <= 32) {            // the lean flank kernel's lists
        CU(e->atasks.ensure(tile_list_cap * p.fcap * sizeof(uint32_t)));
        p.atasks = e->atasks.as<uint32_t>();
    }
    // traceback scratch: 1 byte per band cell per resident thread; very long reads get fewer threads instead of more memory
    const long long bp_per_thread = (long long)(st.Lmax_all + 1) * (2 * band);
    st.slow_blocks = (int)std::max<long long>(1, std::min<long long>(e->sm_count, (4LL << 30) / (bp_per_thread * 256)));
    if (p.use_flanks) {
        p.slow_cap = (int)std::min<long long>(slow_budget, (long long)H * st.max_cand * (long long)tile_list_cap);
        CU(e->slow.ensure((size_t)p.slow_cap * sizeof(int4)));
        CU(e->bp.ensure((size_t)st.slow_blocks * 256 * (size_t)(st.Lmax_all + 1) * (size_t)(2 * band)));
    } else {
        p.slow_cap = 0;
        CU(e->slow.ensure(sizeof(int4)));
    }
    p.slow = e->slow.as<int4>();
    return PHMM_OK;
}

// Phase 6: shared-memory attributes and resident blocks per SM of the DP kernels the lists will use.
static int pop_kernel_attrs(phmm_engine* e, PopState& st)
{
    const int band = st.band;
    int rc;
    st.smem = (size_t)kFastWarpsPerBlock * st.groups * st.fast_row_stride * sizeof(RowEntry);
    if (st.n_pairs) {
        rc = with_fast_shape(band, st.groups, [&](auto b, auto g) -> int {
            return prepare_kernel(e, k_populate_fast<decltype(b)::value, decltype(g)::value>, kFastWarpsPerBlock * 32, st.smem, &st.blocks_per_sm);
        });
        if (rc != PHMM_OK) return rc;
        if (st.blocks_per_sm < 1) { e->err = "fast kernel does not fit on an SM (read too long?)"; return PHMM_ERR_INVALID; }
    }
    st.role_warps = st.n_pairs && st.role_band;
    st.role_groups = kFastWarpsPerBlock / std::max(1, st.NL);
    st.role_smem = st.role_warps ? (size_t)st.role_groups * st.fast_row_stride * sizeof(RowEntry) + (size_t)st.role_groups * kRoleWordsPerGroup(st.NL) * sizeof(uint32_t) : 0;
    if (st.role_warps) {
        rc = with_band_in<32, 64>(band, [&](auto b) -> int {
            return prepare_kernel(e, k_populate_roles<decltype(b)::value>, kFastWarpsPerBlock * 32, st.role_smem, &st.role_blocks_per_sm);
        });
        if (rc != PHMM_OK) return rc;
        if (st.role_blocks_per_sm < 1) st.role_warps = false;
    }
    st.wsmem = (size_t)std::max(1, st.wide_warps) * st.wide_row_stride * sizeof(RowEntry);
    if (st.n_wide) {
        rc = with_wide_shape(band, [&](auto c, auto nl) -> int {
            return prepare_kernel(e, k_populate_wide<decltype(c)::value, decltype(nl)::value>, st.wide_warps * 32, st.wsmem, &st.wide_blocks_per_sm);
        });
        if (rc != PHMM_OK) return rc;
        if (st.wide_blocks_per_sm < 1) { e->err = "wide kernel does not fit on an SM"; return PHMM_ERR_INVALID; }
    }
    return PHMM_OK;
}

// Phase 7: the tile loop. Every tile starts the same way: the capped mapper over the tile's list where the call maps on the device,
// then the per-tile cursors and any-tasks flags cleared (the traceback queue is empty between tiles) and the task counts of the
// list's entries; a tile says how much of that it needs.
enum TileReset { kKeepCursors, kResetCursors, kResetCursorsAndCounts };

static int begin_tile(phmm_engine* e, PopState& st, TileReset reset)
{
    PopParams& p = st.p;
    if (st.use_mapper) {
        const long long threads = (long long)p.n_list * st.H;
        const unsigned grid = (unsigned)std::max<long long>(1, std::min<long long>((threads + 127) / 128, (long long)e->sm_count * 64));
        with_mapper_variant(st.s, [&](auto maxt, auto count) {
            k_kmer_map<decltype(maxt)::value, typename decltype(count)::type><<<grid, 128, 0, e->stream>>>(
                p.list, p.n_list, p.tot, p.list_base, p.list_kind, st.s.hp, st.s.rd, e->rhash.as<uint16_t>(), e->kbins.as<uint32_t>(), e->kitems.as<uint16_t>(),
                e->kpos.as<int32_t>(), e->kcnt.as<uint8_t>(), e->regs.as<RegionInfo>(), st.H);
        });
        LAUNCHED();
        p.kpos = e->kpos.as<int32_t>(); p.kcnt = e->kcnt.as<uint8_t>();
    }
    if (reset != kKeepCursors) CU(cudaMemsetAsync(st.counters, 0, 8 * sizeof(int), e->stream));
    if (reset == kResetCursorsAndCounts) {
        CU(cudaMemsetAsync(p.fcnt, 0, (size_t)p.n_list * sizeof(int), e->stream));
        CU(cudaMemsetAsync(p.gcnt, 0, (size_t)p.n_list * sizeof(int), e->stream));
        CU(cudaMemsetAsync(p.acnt, 0, (size_t)p.n_list * sizeof(int), e->stream));
    }
    return PHMM_OK;
}

// The flank-aware kernels over the current list's gtasks / atasks lists (near-flank candidates, and every candidate of pair-list reads
// holding 'N').
static int launch_flank(phmm_engine* e, PopState& st, int n_entries, int row_stride)
{
    PopParams& p = st.p;
    const int band = st.band;
    int rc;
    if (band > 32) return PHMM_OK;              // wide bands: near-flank candidates take the traceback queue
    if (p.atasks && p.fb_route) {
        // the packed forward / backward flank kernels over the atasks lists; they run BEFORE k_populate_flank, which also resolves the
        // candidates they report as tied or could not place in the forward scratch (appended to the gtasks lists)
        // lane groups: a read's candidates (about one per haplotype) should fill its group's 2 * LG half-lanes; rows must fit 4 blocks / SM
        const int fb_stride = (row_stride + 2 * band + 1) & ~1;                  // + the backward pass's pad rows
        int lg = 5;
        while (lg > 2 && (1 << lg) >= st.H && (size_t)kFastWarpsPerBlock * (32 >> (lg - 1)) * fb_stride * sizeof(RowEntry) <= (48u << 10)) --lg;
        const int fbG = 32 >> lg;
        const size_t fbsmem = (size_t)kFastWarpsPerBlock * fbG * fb_stride * sizeof(RowEntry);
        // forward scratch: one warp-round (64 candidates) per fb_round_words; worst case = every claim's longest task list, capped at 4 GiB
        const long long rounds_worst = ((long long)n_entries / fbG + 1) * ((p.fcap + (2 << lg) - 1) >> (lg + 1));
        rc = with_band_in<8, 16>(band, [&](auto b) -> int {
            constexpr int B = decltype(b)::value;
            int fb_blocks = 1, arc;
            if ((arc = fast_smem_attr(e, k_flank_fwd<B>, fbsmem)) || (arc = prepare_kernel(e, k_flank_bwd<B>, kFastWarpsPerBlock * 32, fbsmem, &fb_blocks))) return arc;
            if (fb_blocks < 1) { e->err = "flank kernel does not fit on an SM (read too long?)"; return PHMM_ERR_INVALID; }
            const unsigned bgrid = (unsigned)std::max(1, std::min((n_entries / fbG + kFastWarpsPerBlock) / kFastWarpsPerBlock, e->sm_count * fb_blocks));
            const size_t round_bytes = fb_round_words(B) * sizeof(uint32_t);
            const long long cap = std::max<long long>(1, std::min<long long>(rounds_worst, (long long)((4ull << 30) / round_bytes)));
            cudaError_t ce = e->fb_pairs.ensure((size_t)cap * round_bytes);
            if (ce == cudaSuccess) ce = e->fb_scratch.ensure((size_t)bgrid * kFastWarpsPerBlock * 32 * fb_scratch_words(B) * sizeof(uint32_t));
            if (ce != cudaSuccess) { e->err = cudaGetErrorString(ce); return PHMM_ERR_NOMEM; }
            p.fb_round_cap = (int)std::min<long long>(0x7fffffff, (long long)(e->fb_pairs.cap / round_bytes));
            k_flank_fwd<B><<<bgrid, kFastWarpsPerBlock * 32, fbsmem, e->stream>>>(p, e->fb_pairs.as<uint32_t>(), fb_stride, lg);
            LAUNCHED();
            k_flank_bwd<B><<<bgrid, kFastWarpsPerBlock * 32, fbsmem, e->stream>>>(p, e->fb_pairs.as<uint32_t>(), e->fb_scratch.as<uint32_t>(), fb_stride, lg);
            LAUNCHED();
            return PHMM_OK;
        });
        if (rc != PHMM_OK) return rc;
    }
    // the labelled kernel: whole warps per read when its lists are dense, groups of 4 lanes when they only hold what the packed kernels
    // passed on (ties: one or two candidates per read; the rare reads with 'N' or shorter than 2 * band then take more rounds)
    int flg = 5;
    if (p.atasks && p.fb_route) { flg = 2; while (flg < 5 && (size_t)kFastWarpsPerBlock * (32 >> flg) * row_stride * sizeof(RowEntry) > (48u << 10)) ++flg; }
    const int fG = 32 >> flg;
    const unsigned fgrid = (unsigned)std::max(1, std::min((n_entries / fG + kFastWarpsPerBlock) / kFastWarpsPerBlock, e->sm_count * 3));
    const size_t fsmem = (size_t)kFastWarpsPerBlock * fG * row_stride * sizeof(RowEntry);
    rc = with_band_in<8, 16, 32>(band, [&](auto b) -> int {
        constexpr int B = decltype(b)::value;
        if (int arc = fast_smem_attr(e, k_populate_flank<B>, fsmem)) return arc;
        k_populate_flank<B><<<fgrid, kFastWarpsPerBlock * 32, fsmem, e->stream>>>(p, row_stride, flg);
        return PHMM_OK;
    });
    if (rc != PHMM_OK) return rc;
    LAUNCHED();
    if (p.atasks && !p.fb_route) {
        const unsigned agrid = (unsigned)std::max(1, std::min((n_entries + kFastWarpsPerBlock - 1) / kFastWarpsPerBlock, e->sm_count * 4));
        rc = with_band_in<8, 16, 32>(band, [&](auto b) -> int {
            constexpr int B = decltype(b)::value;
            if (int arc = fast_smem_attr(e, k_populate_flank_acc<B>, fsmem)) return arc;
            k_populate_flank_acc<B><<<agrid, kFastWarpsPerBlock * 32, fsmem, e->stream>>>(p);
            return PHMM_OK;
        });
        if (rc != PHMM_OK) return rc;
        LAUNCHED();
    }
    return PHMM_OK;
}

// A tile of the pair list from pair *p0 on: the packed kernels (k_populate_fast, or k_populate_roles with a warp per band chunk).
static int pair_tile(phmm_engine* e, PopState& st, ChunkOrder& order, long long* p0)
{
    PopParams& p = st.p;
    const int band = st.band, groups = st.groups;
    int rc;
    const int np = (int)std::min<long long>(st.pairs_per_tile, st.n_pairs - *p0);
    p.pair_reads = e->pairs.as<int>() + 2 * *p0;
    p.n_pairs = np;
    p.pair_base = (int)*p0;
    p.list = p.pair_reads; p.list_kind = 0; p.n_list = 2 * np; p.list_base = (int)(2 * *p0);
    p.row_stride = st.fast_row_stride;
    p.fb_route = (p.atasks && st.flank_fb_ok) ? 1 : 0;
    p.flank_kernels = st.pair_flank_kernels ? 1 : 0;
    if ((rc = begin_tile(e, st, st.direct ? kResetCursors : kResetCursorsAndCounts))) return rc;
    if (!st.direct) {
        // classify pass: shortcut values → best[], near-flank candidates → slow queue, DP candidates → task lists
        const long long threads = 2LL * np * st.H;
        k_populate_generic<64, true><<<(unsigned)((threads + 127) / 128), 128, 0, e->stream>>>(p);
        LAUNCHED();
    }
    st.lap(e, " classify queued");
    const bool role_warps = st.role_warps;
    const int tasks_per_round = role_warps ? 32 : (32 / groups) / st.NL;
    p.units_per_pair = std::max(1, (p.fcap + tasks_per_round * kRoundsPerUnit - 1) / (tasks_per_round * kRoundsPerUnit));
    const int claimers_per_block = role_warps ? st.role_groups : kFastWarpsPerBlock;      // groups of warps / warps that claim work units
    const int want_blocks = (int)std::min<long long>(1LL << 30, ((long long)(np / groups) * p.units_per_pair + claimers_per_block - 1) / claimers_per_block);
    const unsigned grid = (unsigned)std::max(1, std::min(want_blocks, e->sm_count * (role_warps ? st.role_blocks_per_sm : st.blocks_per_sm)));
    while (e->tile_events.size() < 2 * (st.n_timed + 1)) { cudaEvent_t ev; CU(cudaEventCreate(&ev)); e->tile_events.push_back(ev); }
    CU(order.wait_for_previous());
    CU(cudaEventRecord(e->tile_events[2 * st.n_timed], e->stream));
    if (role_warps) {
        with_band_in<32, 64>(band, [&](auto b) { k_populate_roles<decltype(b)::value><<<grid, kFastWarpsPerBlock * 32, st.role_smem, e->stream>>>(p); });
    } else {
        with_fast_shape(band, groups, [&](auto b, auto g) { k_populate_fast<decltype(b)::value, decltype(g)::value><<<grid, kFastWarpsPerBlock * 32, st.smem, e->stream>>>(p); });
    }
    LAUNCHED();
    // with a flank state the tile's DP work is split between the score-only kernel and the flank-aware kernels: time them together
    if (!p.use_flanks) CU(cudaEventRecord(e->tile_events[2 * st.n_timed + 1], e->stream));
    st.lap(e, " dp queued");
    if (!st.direct && (rc = launch_flank(e, st, 2 * np, st.fast_row_stride))) return rc;
    if (p.use_flanks) CU(cudaEventRecord(e->tile_events[2 * st.n_timed + 1], e->stream));
    ++st.n_timed; st.timed = true;
    *p0 += np;
    return PHMM_OK;
}

// A tile of the wide list from entry *w0 on: the 32-bit multi-lane kernel; it keeps the classify pass in direct mode too.
static int wide_tile(phmm_engine* e, PopState& st, ChunkOrder& order, long long* w0)
{
    PopParams& p = st.p;
    int rc;
    const int nw = (int)std::min<long long>(st.reads_per_tile, st.n_wide - *w0);
    p.list = e->wide_reads.as<int>() + *w0; p.list_kind = 1; p.n_list = nw; p.list_base = (int)*w0;
    p.row_stride = st.wide_row_stride;
    p.fb_route = 0;
    p.flank_kernels = st.wide_flank_kernels ? 1 : 0;
    const long long threads = (long long)nw * st.H;
    const unsigned cgrid = (unsigned)std::max<long long>(1, std::min<long long>((threads + 127) / 128, (long long)e->sm_count * 64));
    if ((rc = begin_tile(e, st, kResetCursorsAndCounts))) return rc;
    if (st.direct) { k_list_slots<<<cgrid, 128, 0, e->stream>>>(p, true); LAUNCHED(); }
    k_populate_generic<64, true><<<cgrid, 128, 0, e->stream>>>(p);          // classify pass over the wide list
    LAUNCHED();
    const unsigned wgrid = (unsigned)std::max(1, std::min((nw + st.wide_warps - 1) / st.wide_warps, e->sm_count * st.wide_blocks_per_sm));
    const bool time_wide = st.n_pairs == 0;
    if (time_wide) { while (e->tile_events.size() < 2 * (st.n_timed + 1)) { cudaEvent_t ev; CU(cudaEventCreate(&ev)); e->tile_events.push_back(ev); } }
    CU(order.wait_for_previous());
    if (time_wide) CU(cudaEventRecord(e->tile_events[2 * st.n_timed], e->stream));
    with_wide_shape(st.band, [&](auto c, auto nl) { k_populate_wide<decltype(c)::value, decltype(nl)::value><<<wgrid, st.wide_warps * 32, st.wsmem, e->stream>>>(p); });
    LAUNCHED();
    if (time_wide) { CU(cudaEventRecord(e->tile_events[2 * st.n_timed + 1], e->stream)); ++st.n_timed; st.timed = true; }
    if (p.flank_kernels && (rc = launch_flank(e, st, nw, st.wide_row_stride))) return rc;
    if (st.direct) { k_list_slots<<<cgrid, 128, 0, e->stream>>>(p, false); LAUNCHED(); }
    *w0 += nw;
    return PHMM_OK;
}

// A tile of the generic list from entry *g0 on: one thread per pair, every candidate aligned where it is found.
static int generic_tile(phmm_engine* e, PopState& st, ChunkOrder& order, long long* g0)
{
    PopParams& p = st.p;
    int rc;
    const int ng = (int)std::min<long long>(st.reads_per_tile, st.n_generic - *g0);
    p.list = e->generic_reads.as<int>() + *g0; p.list_kind = 2; p.n_list = ng; p.list_base = (int)*g0;
    p.fb_route = 0;
    p.flank_kernels = 0;
    // ng is an upper bound (normally there are no generic reads at all): grid-stride kernels on a bounded grid
    const long long threads = (long long)ng * st.H;
    const unsigned ggrid = (unsigned)std::max<long long>(1, std::min<long long>((threads + 63) / 64, (long long)e->sm_count * 32));
    if ((rc = begin_tile(e, st, kKeepCursors))) return rc;
    const bool time_generic = st.n_pairs == 0 && st.n_wide == 0 && st.n_timed == 0;
    if (st.direct) { k_list_slots<<<ggrid, 64, 0, e->stream>>>(p, true); LAUNCHED(); }
    CU(order.wait_for_previous());
    if (time_generic) CU(cudaEventRecord(e->ev0, e->stream));
    if (st.band <= 32) k_populate_generic<64, false><<<ggrid, 64, 0, e->stream>>>(p);
    else k_populate_generic<kGenericMaxDiag, false><<<ggrid, 64, 0, e->stream>>>(p);
    LAUNCHED();
    if (time_generic) { CU(cudaEventRecord(e->ev1, e->stream)); st.timed = true; }
    if (st.direct) { k_list_slots<<<ggrid, 64, 0, e->stream>>>(p, false); LAUNCHED(); }
    *g0 += ng;
    return PHMM_OK;
}

// The lists tile by tile over the same scratch: all pair tiles, then the wide tiles, then the generic ones; after each the
// traceback queue it filled (near-flank candidates no flank kernel took) is drained.
static int pop_tiles(phmm_engine* e, PopState& st, ChunkOrder& order)
{
    PopParams& p = st.p;
    for (long long p0 = 0, w0 = 0, g0 = 0; p0 < st.n_pairs || w0 < st.n_wide || g0 < st.n_generic;) {
        int rc;
        if (p0 < st.n_pairs) rc = pair_tile(e, st, order, &p0);
        else if (w0 < st.n_wide) rc = wide_tile(e, st, order, &w0);
        else rc = generic_tile(e, st, order, &g0);
        if (rc != PHMM_OK) return rc;
        if (p.use_flanks) {
            if (st.band <= 32) k_slow_flank<64><<<st.slow_blocks, 256, 0, e->stream>>>(p, e->bp.as<unsigned char>());
            else k_slow_flank<kGenericMaxDiag><<<st.slow_blocks, 256, 0, e->stream>>>(p, e->bp.as<unsigned char>());
            LAUNCHED();
            CU(cudaMemsetAsync(p.slow_count, 0, sizeof(int), e->stream));
        }
        CU(cudaGetLastError());
    }
    return PHMM_OK;
}

// Phase 8: the FP64 finish, the template sums or the top sets, the copies to the caller, the call's one final synchronisation,
// and what the device flagged.
static int pop_finish(phmm_engine* e, const PopulateCall& c, PopState& st)
{
    PopParams& p = st.p;
    const int H = st.H, R = st.R;
    const long long HR = st.HR;
    const bool host = c.space == PHMM_SPACE_HOST;
    int rc;
    if (!st.direct) {
        const long long threads = (long long)H * R;
        k_epilogue<<<(unsigned)((threads + 255) / 256), 256, 0, e->stream>>>(p.best, p.status, st.s.rd, e->regs.as<RegionInfo>(), H, c.cfg->use_mapping_quality,
                                                                             c.cfg->mapping_quality_cap, c.cfg->mapping_quality_cap_trigger, st.d_out, p.out_row_extra);
        LAUNCHED();
    }
    CU(cudaGetLastError());
    // only a host-space chunk of a larger matrix is copied out row by row: device-space calls wrote their rows in place
    const bool pitched = host && c.out_pitch != 0 && c.out_pitch != R;
    if (c.assign()) {
        // every read's or every template's top set from the finished matrix; then only top and the optional out / status leave the device
        const bool by_template = c.template_off != nullptr;
        const long long n_top = by_template ? c.n_templates : R;
        unsigned long long* d_top = (unsigned long long*)c.top;
        if (host) { CU(e->as_top.ensure((size_t)n_top * sizeof(uint64_t))); d_top = e->as_top.as<unsigned long long>(); }
        double* d_values = st.d_out;
        long long n_values = HR;
        if (by_template) {
            const TemplateGroup& last = c.template_groups.back();
            n_values = last.tout_off + (long long)c.regions.regs.back().nH * last.nT;
            const long long* d_toff;
            const TemplateGroup* d_groups;
            if ((rc = stage(e, e->at_off, (const long long*)c.template_off, (size_t)c.n_templates + 1, PHMM_SPACE_HOST, &d_toff))) return rc;
            if ((rc = stage(e, e->at_groups, c.template_groups.data(), c.template_groups.size(), PHMM_SPACE_HOST, &d_groups))) return rc;
            d_values = c.out;
            if (host && c.out) { CU(e->at_lnl.ensure((size_t)n_values * sizeof(double))); d_values = e->at_lnl.as<double>(); }
            k_assign_template_top<<<(unsigned)((c.n_templates + 127) / 128), 128, 0, e->stream>>>(c.n_templates, st.G, e->regs.as<RegionInfo>(),
                                                                                                   d_groups, d_toff, st.d_out, c.log_priors, d_top, d_values);
        } else {
            k_assign_top<<<(unsigned)((st.G + 3) / 4), 128, 0, e->stream>>>(st.G, e->regs.as<RegionInfo>(), st.d_out, c.log_priors, d_top);
        }
        LAUNCHED();
        CU(cudaGetLastError());
        if (host) {
            CU(cudaMemcpyAsync(c.top, d_top, (size_t)n_top * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->stream));
            if (c.out) CU(cudaMemcpyAsync(c.out, d_values, (size_t)n_values * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
        }
    } else if (c.template_off) {
        // paired / linked reads: one value per (haplotype, template)
        const long long* d_toff;
        if ((rc = stage(e, e->tasks_lane, (const long long*)c.template_off, (size_t)c.n_templates + 1, c.space, &d_toff))) return rc;
        const long long HT = (long long)H * c.n_templates;
        CU(e->tasks_generic.ensure((size_t)HT * sizeof(double)));
        double* d_tout = host ? e->tasks_generic.as<double>() : c.out;
        k_template_sum<<<(unsigned)((HT + 255) / 256), 256, 0, e->stream>>>(st.d_out, H, R, d_toff, c.n_templates, d_tout);
        LAUNCHED();
        CU(cudaGetLastError());
        if (host) CU(cudaMemcpyAsync(c.out, d_tout, (size_t)HT * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
    } else if (pitched) {
        CU(cudaMemcpy2DAsync(c.out, (size_t)c.out_pitch * sizeof(double), st.d_out, (size_t)R * sizeof(double), (size_t)R * sizeof(double), H, cudaMemcpyDeviceToHost, e->stream));
    } else if (host) {
        CU(cudaMemcpyAsync(c.out, st.d_out, (size_t)HR * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
    }
    if (c.status && pitched) CU(cudaMemcpy2DAsync(c.status, (size_t)c.out_pitch * sizeof(int), p.status, (size_t)R * sizeof(int), (size_t)R * sizeof(int), H, cudaMemcpyDeviceToHost, e->stream));
    else if (c.status) CU(cudaMemcpyAsync(c.status, p.status, (size_t)HR * sizeof(int), host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, e->stream));
    int flags_host[1] = {0};
    st.lap(e, "enqueued");
    CU(cudaMemcpyAsync(flags_host, e->flags.p, sizeof(int), cudaMemcpyDeviceToHost, e->stream));
    CU(cudaMemcpyAsync(&st.tot, p.tot, sizeof(SchedTotals), cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    st.lap(e, "done");
    if (flags_host[0] & 1) { e->err = "snv prior / gap penalty outside [0,127]"; return PHMM_ERR_INVALID; }
    const size_t n_timed = st.n_timed;
    if (PopState::tracing() && n_timed) { float ms = 0.f; cudaEventElapsedTime(&ms, e->tile_events[0], e->tile_events[2 * n_timed - 1]); std::fprintf(stderr, "[phmm %p] dp span %.3f ms\n", (void*)e, ms); }
    if (n_timed) {
        double total = 0.0;
        for (size_t t = 0; t < n_timed; ++t) { float ms = 0.f; if (cudaEventElapsedTime(&ms, e->tile_events[2 * t], e->tile_events[2 * t + 1]) == cudaSuccess) total += ms; }
        e->last_dp_ms = total;
    } else if (st.timed) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, e->ev0, e->ev1) == cudaSuccess) e->last_dp_ms = ms;
    }
    // GCUPS numerator when every pair runs exactly one DP (benchmark mode); otherwise an upper bound on DP work
    e->last_dp_cells = st.tot.cells;
    if (flags_host[0] & (4 | 8)) { e->err = "internal task queue overflow"; return PHMM_ERR_NOMEM; }
    if (flags_host[0] & 2) { e->err = "Haplotype is too short for alignment"; return PHMM_ERR_SHORT_HAPLOTYPE; }
    return PHMM_OK;
}

// One synchronous pass over the call's regions: every read against the haplotypes of its region. The entry point has run begin_call
// (phmm_assign_reads before its mapper, whose launches count with the call's).
static int populate_impl(phmm_engine* e, const PopulateCall& c)
{
    PopState st;
    int rc;
    if (c.reset && (rc = pop_reset(e, c, st))) return rc;
    if ((rc = pop_stage(e, c, st))) return rc;
    st.lap(e, "staged");
    if ((rc = pop_candidates(e, c, st))) return rc;
    pop_decide(c, st);
    if ((rc = pop_schedule(e, st))) return rc;
    st.lap(e, "sched enqueued");
    if ((rc = pop_outputs(e, c, st)) || (rc = pop_tile_scratch(e, st))) return rc;
    st.lap(e, "buffers");
    if ((rc = pop_kernel_attrs(e, st))) return rc;
    st.lap(e, "kernel attrs");
    {
        // a sub-engine's DP kernels wait for the previous chunk's; leaving the tile loop early releases the next chunk all the same
        ChunkOrder order(e);
        if ((rc = pop_tiles(e, st, order))) return rc;
        order.publish(true);
    }
    st.lap(e, "tiles enqueued");
    return pop_finish(e, c, st);
}

} // extern "C"

long long phmm_checks::populate_chunk_pairs(long long all_pairs)
{
    static const long long kForcedChunkPairs = [] {
        const char* v = std::getenv("PHMM_CHUNK_PAIRS");          // test hook: force the pipelined path on small batches
        const long long n = v ? std::atoll(v) : 0;
        return n > 0 ? n : 0LL;
    }();
    // chunk size: an eighth of the batch, between 2M pairs (below that the per-chunk launch chain shows) and 8M pairs
    return kForcedChunkPairs ? kForcedChunkPairs : std::max<long long>(2LL << 20, std::min<long long>(8LL << 20, all_pairs / 8));
}

extern "C" {

int phmm_populate_regions(phmm_engine* e, const phmm_config* cfg,
                          const phmm_haplotypes* haps, const phmm_reads* reads, const phmm_regions* regions,
                          double* out, int32_t* status, int space)
{
    int rc;
    if ((rc = begin_call(e))) return rc;
    PopulateCall c;
    c.cfg = cfg; c.haps = haps; c.reads = reads; c.space = space;
    c.out = out; c.status = status;
    if ((rc = region_setup(e, cfg, haps, reads, regions, c.regions)) != PHMM_OK) return rc;
    return populate_impl(e, c);
}

} // extern "C"

// The body of phmm_assign_reads and phmm_assign_templates: the group checks, then (templates: their checks and layout) one staging,
// the uncapped pair mapper over the slot pairs and populate_impl, which chooses the top sets on the device.
static int assign_impl(phmm_engine* e, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads, const phmm_regions* groups,
                       const int64_t* template_off, int32_t n_templates, const double* log_priors, uint64_t* top, double* lnl, int32_t* status,
                       int space, bool by_template)
{
    int rc;
    if ((rc = begin_call(e))) return rc;
    PopulateCall c;
    c.cfg = cfg; c.haps = haps; c.reads = reads; c.space = space;
    c.out = lnl; c.status = status; c.top = top;
    if ((rc = region_setup(e, cfg, haps, reads, groups, c.regions)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::config_and_output(cfg, top, reads, e->err)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::assign_groups(groups, e->err)) != PHMM_OK) return rc;
    if (by_template) {
        if ((rc = phmm_checks::assign_templates(template_off, n_templates, reads, groups, e->err)) != PHMM_OK) return rc;
        c.template_off = template_off; c.n_templates = n_templates;
        long long tout = 0;
        int t = 0;
        for (const RegionInfo& r : c.regions.regs) {
            const int t0 = t;
            while (t < n_templates && template_off[t] < r.r0 + r.nR) ++t;
            c.template_groups.push_back({t0, t - t0, tout});
            tout += (long long)r.nH * (t - t0);
        }
    }
    // the blocks are staged once: the pair mapper and the DP read the same device copies
    Staged s;
    if ((rc = stage_batch(e, haps, reads, space, s, false, true)) != PHMM_OK) return rc;
    c.staged = &s;
    if ((rc = stage(e, e->as_prior, log_priors, (size_t)haps->n, space, &c.log_priors))) return rc;
    if (cfg->map_positions) {
        // every slot's (read, haplotype) pair in slot order, mapped uncapped: a CSR over the result slots (one synchronisation sizes it)
        const int G = (int)c.regions.regs.size(), HR = (int)c.regions.total_out;
        CU(e->regs.ensure((size_t)G * sizeof(RegionInfo)));
        CU(cudaMemcpyAsync(e->regs.p, c.regions.regs.data(), (size_t)G * sizeof(RegionInfo), cudaMemcpyHostToDevice, e->stream));
        CU(e->as_pairs.ensure((size_t)HR * sizeof(int2)));
        k_slot_pairs<<<(unsigned)((HR + 255) / 256), 256, 0, e->stream>>>(HR, G, e->regs.as<RegionInfo>(), e->as_pairs.as<int2>());
        LAUNCHED();
        if ((rc = pair_map_resident(e, s, e->as_pairs.as<int2>(), HR, &c.n_mapped))) return rc;
        c.mapped_off = e->c_off.as<long long>(); c.mapped_pos = e->c_pos.as<int32_t>();
    }
    return populate_impl(e, c);
}

extern "C" {

int phmm_assign_reads(phmm_engine* e, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                      const phmm_regions* groups, const double* log_priors, uint64_t* top, double* lnl, int32_t* status, int space)
{
    return assign_impl(e, cfg, haps, reads, groups, nullptr, 0, log_priors, top, lnl, status, space, false);
}

int phmm_assign_templates(phmm_engine* e, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                          const phmm_regions* groups, const int64_t* template_off, int32_t n_templates,
                          const double* log_priors, uint64_t* top, double* lnl, int32_t* status, int space)
{
    return assign_impl(e, cfg, haps, reads, groups, template_off, n_templates, log_priors, top, lnl, status, space, true);
}

int phmm_populate_ld(phmm_engine* e, const phmm_config* cfg,
                     const phmm_haplotypes* haps, const phmm_reads* reads,
                     const phmm_positions* positions, const phmm_flank_state* flank,
                     double* out, int64_t out_ld, int32_t* status)
{
    if (int rc = begin_call(e)) return rc;
    if (!reads || out_ld < reads->n) { e->err = "out_ld must be at least the number of reads"; return PHMM_ERR_INVALID; }
    PopulateCall c = one_region_call(cfg, haps, reads, positions, flank, out, status, PHMM_SPACE_DEVICE);
    c.out_pitch = (long long)out_ld;
    return populate_impl(e, c);
}

// -------------------------------------------------------------------------------------------------------------
// Peer output: one rank's matrix mapped into the other ranks' address spaces (CUDA IPC over NVLink / NVSwitch)
// -------------------------------------------------------------------------------------------------------------
int phmm_device_alloc(int device, size_t bytes, void** dev_ptr)
{
    if (!dev_ptr || bytes == 0) return PHMM_ERR_INVALID;
    *dev_ptr = nullptr;
    if (cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); return PHMM_ERR_CUDA; }
    if (cudaMalloc(dev_ptr, bytes) != cudaSuccess) { cudaGetLastError(); *dev_ptr = nullptr; return PHMM_ERR_NOMEM; }
    return PHMM_OK;
}

int phmm_device_free(void* dev_ptr)
{
    if (dev_ptr && cudaFree(dev_ptr) != cudaSuccess) { cudaGetLastError(); return PHMM_ERR_CUDA; }
    return PHMM_OK;
}

int phmm_ipc_export(const void* dev_ptr, unsigned char handle[PHMM_IPC_HANDLE_BYTES])
{
    static_assert(sizeof(cudaIpcMemHandle_t) == PHMM_IPC_HANDLE_BYTES, "handle size");
    if (!dev_ptr || !handle) return PHMM_ERR_INVALID;
    cudaIpcMemHandle_t h;
    if (cudaIpcGetMemHandle(&h, const_cast<void*>(dev_ptr)) != cudaSuccess) { cudaGetLastError(); return PHMM_ERR_CUDA; }
    std::memcpy(handle, &h, sizeof(h));
    return PHMM_OK;
}

int phmm_ipc_open(int device, const unsigned char handle[PHMM_IPC_HANDLE_BYTES], void** dev_ptr)
{
    if (!handle || !dev_ptr) return PHMM_ERR_INVALID;
    *dev_ptr = nullptr;
    if (cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); return PHMM_ERR_CUDA; }
    cudaIpcMemHandle_t h;
    std::memcpy(&h, handle, sizeof(h));
    if (cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); *dev_ptr = nullptr; return PHMM_ERR_CUDA; }
    return PHMM_OK;
}

int phmm_ipc_close(void* dev_ptr)
{
    if (dev_ptr && cudaIpcCloseMemHandle(dev_ptr) != cudaSuccess) { cudaGetLastError(); return PHMM_ERR_CUDA; }
    return PHMM_OK;
}

int phmm_populate_templates(phmm_engine* e, const phmm_config* cfg,
                            const phmm_haplotypes* haps, const phmm_reads* reads,
                            const int64_t* template_off, int32_t n_templates,
                            const phmm_positions* positions, const phmm_flank_state* flank,
                            double* out, int32_t* status, int space)
{
    int rc;
    if ((rc = begin_call(e))) return rc;
    if ((rc = phmm_checks::template_offsets(template_off, n_templates, reads, space == PHMM_SPACE_HOST, e->err)) != PHMM_OK) return rc;
    PopulateCall c = one_region_call(cfg, haps, reads, positions, flank, out, status, space);
    c.template_off = template_off; c.n_templates = n_templates;
    return populate_impl(e, c);
}

} // extern "C"

// Whether phmm_populate runs a call as its pipeline: a host-resident batch, no caller-supplied position lists (a [H][R] CSR cannot be
// sliced by columns without a pass over it), enough pairs to amortise the per-chunk overheads.
static bool pipelined(const phmm_engine* e, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                      const phmm_positions* positions, const double* out, int space)
{
    const long long all_pairs = (haps && reads) ? (long long)haps->n * reads->n : 0;
    return !e->is_sub && space == PHMM_SPACE_HOST && haps && reads && cfg && out && haps->n > 0 && reads->n > 1 && reads->off && reads->mapq &&
           reads->reverse && !(positions && positions->off && positions->pos) && all_pairs >= 2 * phmm_checks::populate_chunk_pairs(all_pairs);
}

// A sequences block as the haplotype block of a _reset call before pop_reset has derived its arrays.
static phmm_haplotypes sequences_block(const phmm_haplotype_sequences* seqs)
{
    return phmm_haplotypes {seqs->n, seqs->off, seqs->seq, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, seqs->begin};
}

static PopulateCall& with_model(PopulateCall& c, const phmm_error_model* m, const phmm_haplotype_sequences* seqs)
{
    c.reset = true; c.model = m; c.is_substitution = seqs->is_substitution;
    return c;
}

extern "C" {

int phmm_populate(phmm_engine* e, const phmm_config* cfg,
                  const phmm_haplotypes* haps, const phmm_reads* reads,
                  const phmm_positions* positions, const phmm_flank_state* flank,
                  double* out, int32_t* status, int space)
{
    if (int rc = begin_call(e)) return rc;
    if (!pipelined(e, cfg, haps, reads, positions, out, space)) return populate_impl(e, one_region_call(cfg, haps, reads, positions, flank, out, status, space));
    const long long kChunkPairs = phmm_checks::populate_chunk_pairs((long long)haps->n * reads->n);
    for (phmm_engine*& sub : e->sub) {
        if (!sub) {
            const int rc = phmm_create(&sub, e->device);
            if (rc != PHMM_OK) { e->err = std::string("sub-engine: ") + phmm_last_error(nullptr); return rc; }
            sub->is_sub = true;
            sub->parent = e;
            sub->reserved_sms = e->reserved_sms;
            if (cudaEventCreateWithFlags(&sub->order_ev, cudaEventDisableTiming) != cudaSuccess) {
                phmm_destroy(sub);          // a sub-engine without its ordering event must not survive into the next call
                sub = nullptr;
                e->err = "sub-engine: event creation failed";
                return PHMM_ERR_CUDA;
            }
        }
    }
    e->sub[0]->peer = e->sub[1]; e->sub[1]->peer = e->sub[0];
    e->order.recorded = -1;
    const int R = reads->n, H = haps->n;
    const long long reads_per_chunk = std::max<long long>(64, kChunkPairs / H);
    const int n_chunks = (int)((R + reads_per_chunk - 1) / reads_per_chunk);
    int rcs[2] = {PHMM_OK, PHMM_OK};
    std::string errs[2];
    int64_t cells[2] = {0, 0}, launches[2] = {0, 0};
    auto worker = [&](int k) {
        phmm_engine* se = e->sub[k];
        std::vector<int64_t> off;
        for (int c = k; c < n_chunks; c += 2) {
            const long long lo = (long long)c * reads_per_chunk, hi = std::min<long long>(R, lo + reads_per_chunk);
            const int n = (int)(hi - lo);
            off.resize((size_t)n + 1);
            const int64_t base = reads->off[lo];
            for (int i = 0; i <= n; ++i) off[i] = reads->off[lo + i] - base;
            phmm_reads sub_reads {n, off.data(), reads->bases + base, reads->quals + base, reads->mapq + lo, reads->reverse + lo,
                                  reads->begin ? reads->begin + lo : nullptr};
            se->chunk_index = c;
            PopulateCall chunk = one_region_call(cfg, haps, &sub_reads, nullptr, flank, out + lo, status ? status + lo : nullptr, PHMM_SPACE_HOST);
            chunk.out_pitch = R;
            int rc = begin_call(se);
            if (rc == PHMM_OK) rc = populate_impl(se, chunk);
            {   // a chunk that failed before reaching its DP phase must not leave the other worker waiting for it
                std::lock_guard<std::mutex> lk(e->order.m);
                e->order.recorded = std::max<long long>(e->order.recorded, rc != PHMM_OK && rc != PHMM_ERR_SHORT_HAPLOTYPE ? (long long)n_chunks : (long long)c);
            }
            e->order.cv.notify_all();
            cells[k] += se->last_dp_cells; launches[k] += se->launches_last;
            if (rc != PHMM_OK && rc != PHMM_ERR_SHORT_HAPLOTYPE) { rcs[k] = rc; errs[k] = se->err; return; }
            if (rc == PHMM_ERR_SHORT_HAPLOTYPE) { rcs[k] = rc; errs[k] = se->err; }   // keep going: every pair's status is still written
        }
    };
    std::thread t1(worker, 1);
    worker(0);
    t1.join();
    e->last_dp_cells = cells[0] + cells[1];
    e->launches_last = launches[0] + launches[1];
    e->launches_total += e->launches_last;
    for (int k = 0; k < 2; ++k) if (rcs[k] != PHMM_OK && rcs[k] != PHMM_ERR_SHORT_HAPLOTYPE) { e->err = errs[k]; return rcs[k]; }
    for (int k = 0; k < 2; ++k) if (rcs[k] == PHMM_ERR_SHORT_HAPLOTYPE) { e->err = errs[k]; return rcs[k]; }
    return PHMM_OK;
}

int phmm_populate_reset(phmm_engine* e, const phmm_config* cfg, const phmm_error_model* m, const phmm_haplotype_sequences* seqs,
                        const phmm_reads* reads, const phmm_positions* positions, const phmm_flank_state* flank,
                        double* out, int32_t* status, int space)
{
    if (int rc = begin_call(e)) return rc;
    if (!seqs) { e->err = "null argument"; return PHMM_ERR_INVALID; }
    const phmm_haplotypes shell = sequences_block(seqs);
    if (!pipelined(e, cfg, &shell, reads, positions, out, space)) {
        PopulateCall c = one_region_call(cfg, &shell, reads, positions, flank, out, status, space);
        return populate_impl(e, with_model(c, m, seqs));
    }
    // the pipeline takes a host block: the arrays once, on the device, then phmm_populate's pipeline
    const size_t B = seqs->off ? (size_t)std::max<int64_t>(seqs->off[seqs->n], 0) : 0;
    std::vector<int8_t> arrays(6 * std::max<size_t>(B, 1));
    int8_t* a = arrays.data();
    const size_t k = std::max<size_t>(B, 1);
    const ResetArrays host {(char*)a, a + k, (char*)a + 2 * k, a + 3 * k, a + 4 * k, a + 5 * k};
    const int rc = reset_arrays(e, m, seqs->n, seqs->off, seqs->seq, seqs->is_substitution, space, nullptr, &host, nullptr);
    if (rc != PHMM_OK) return rc;
    const phmm_haplotypes haps {seqs->n, seqs->off, seqs->seq, host.mask_f, host.prior_f, host.mask_r, host.prior_r, host.gap_open, host.gap_extend, seqs->begin};
    return phmm_populate(e, cfg, &haps, reads, positions, flank, out, status, space);
}

int phmm_populate_regions_reset(phmm_engine* e, const phmm_config* cfg, const phmm_error_model* m, const phmm_haplotype_sequences* seqs,
                                const phmm_reads* reads, const phmm_regions* regions, double* out, int32_t* status, int space)
{
    int rc;
    if ((rc = begin_call(e))) return rc;
    if (!seqs) { e->err = "null argument"; return PHMM_ERR_INVALID; }
    const phmm_haplotypes shell = sequences_block(seqs);
    PopulateCall c;
    c.cfg = cfg; c.haps = &shell; c.reads = reads; c.space = space;
    c.out = out; c.status = status;
    if ((rc = region_setup(e, cfg, &shell, reads, regions, c.regions)) != PHMM_OK) return rc;
    return populate_impl(e, with_model(c, m, seqs));
}

int phmm_populate_templates_reset(phmm_engine* e, const phmm_config* cfg, const phmm_error_model* m, const phmm_haplotype_sequences* seqs,
                                  const phmm_reads* reads, const int64_t* template_off, int32_t n_templates,
                                  const phmm_positions* positions, const phmm_flank_state* flank, double* out, int32_t* status, int space)
{
    int rc;
    if ((rc = begin_call(e))) return rc;
    if (!seqs) { e->err = "null argument"; return PHMM_ERR_INVALID; }
    if ((rc = phmm_checks::template_offsets(template_off, n_templates, reads, space == PHMM_SPACE_HOST, e->err)) != PHMM_OK) return rc;
    const phmm_haplotypes shell = sequences_block(seqs);
    PopulateCall c = one_region_call(cfg, &shell, reads, positions, flank, out, status, space);
    c.template_off = template_off; c.n_templates = n_templates;
    return populate_impl(e, with_model(c, m, seqs));
}

} // extern "C"
