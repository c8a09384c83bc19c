// TEST HELPER (not part of the product library): runs the engine's __host__ __device__ DP cores on the CPU, with the
// sm_90a packed-16 (DPX) instructions emulated (octopus_b200/csrc/phmm_device.cuh), so that `pytest -m "not gpu"` can check
// the very code the kernels execute against the oracle without a GPU.
#include <cstdint>
#include <vector>
#include "../../octopus_b200/csrc/phmm_device.cuh"

using namespace phmm;

// Which deletion update the emulated cores use: -1 = as the kernels choose it (the shorter OGE form when no column of the
// windows has gap_open < gap_extend, kFlagOpenBelowExtend), 0 = always the general form, 1 = always the OGE form.
static int g_form = -1;
extern "C" void emul_force_form(int v) { g_form = v; }
static bool use_oge(const int8_t* go0, const int8_t* ge0, const int8_t* go1, const int8_t* ge1, int W)
{
    if (g_form >= 0) return g_form != 0;
    for (int x = 0; x < W; ++x) if (go0[x] < ge0[x] || (go1 && go1[x] < ge1[x])) return false;
    return true;
}

template <int BAND>
static uint32_t run_pair(int L, const std::vector<RowEntry>& rows, const ColEntry* t0, const ColEntry* t1, uint32_t nucp, bool oge)
{
    return oge ? dp_pair<BAND, true>(rows.data(), L, t0, t1, nucp) : dp_pair<BAND, false>(rows.data(), L, t0, t1, nucp);
}

extern "C" {

// Two alignments of equal read length L through dp_pair<band>. Inputs per alignment a in {0,1}: read bases/quals (L),
// window arrays (W = L + 2*band - 1). Returns 0, or -1 if a read base is not ACGT / band unsupported.
int emul_dp_pair(int band, int L, const char* read0, const uint8_t* q0, const char* read1, const uint8_t* q1,
                 const char* truth0, const char* mask0, const int8_t* prior0, const int8_t* go0, const int8_t* ge0,
                 const char* truth1, const char* mask1, const int8_t* prior1, const int8_t* go1, const int8_t* ge1,
                 int nuc_prior, int* score0, int* score1)
{
    const int W = L + 2 * band - 1;
    std::vector<RowEntry> rows(L + 1);
    for (int y = 0; y < L; ++y) {
        const int c0 = base_code(read0[y]), c1 = base_code(read1[y]);
        if (c0 < 0 || c1 < 0) return -1;
        rows[y] = make_row_entry((uint32_t)c0 | ((uint32_t)q0[y] << 8), (uint32_t)c1 | ((uint32_t)q1[y] << 8));
    }
    rows[L] = pad_row_entry();
    std::vector<ColEntry> t0(W), t1(W);
    for (int x = 0; x < W; ++x) {
        t0[x] = make_col_entry(truth0[x], mask0[x], prior0[x], go0[x], ge0[x]);
        t1[x] = make_col_entry(truth1[x], mask1[x], prior1[x], go1[x], ge1[x]);
    }
    const uint32_t nucp = (uint32_t)nuc_prior | ((uint32_t)nuc_prior << 16);
    uint32_t r;
    const bool oge = use_oge(go0, ge0, go1, ge1, W);
    switch (band) {
        case 8:  r = run_pair<8>(L, rows, t0.data(), t1.data(), nucp, oge); break;
        case 16: r = run_pair<16>(L, rows, t0.data(), t1.data(), nucp, oge); break;
        case 32: r = run_pair<32>(L, rows, t0.data(), t1.data(), nucp, oge); break;
        default: return -1;
    }
    *score0 = (int)(r & 0xFFFF);
    *score1 = (int)(r >> 16);
    return 0;
}

// generic_align<TB> on the CPU. tb != 0 additionally returns first_pos / flank score / in-flank read bases.
int emul_generic(int band, int tb, int L, const char* read, const int8_t* q,
                 const char* truth, const char* mask, const int8_t* prior, const int8_t* go, const int8_t* ge,
                 int nuc_prior, int lhs_flank, int rhs_flank, int* first_pos, int* flank_score, int* mask_size)
{
    GenericModel gm {truth, mask, prior, go, ge, nuc_prior};
    if (2 * band > kGenericMaxDiag) return -1000000;
    if (tb) {
        std::vector<unsigned char> bp((size_t)(L + 1) * 2 * band, 0);
        return generic_align<true, kGenericMaxDiag>(band, gm, read, q, L, bp.data(), 1, lhs_flank, rhs_flank, first_pos, flank_score, mask_size);
    }
    return generic_align<false, kGenericMaxDiag>(band, gm, read, q, L, nullptr, 1, 0, 0, nullptr, nullptr, nullptr);
}

// The FP64 finish of every populate path, host-compiled from the same source: mapq_terms (the read's share, tabulated by
// k_mapq_terms), finish_mixed (the pair's share) and finish_likelihood (both in one, as k_epilogue and k_align_reads call it).
// best == INT_MIN stands for kBestInf (lowest()).
static int best_of(int s) { return s == INT32_MIN ? kBestInf : s; }
void emul_mapq_terms(int mapq, int cap, int trigger, double* ln_mapped, double* ln_miss)
{
    const MapqTerms t = mapq_terms(mapq, cap, trigger);
    *ln_mapped = t.ln_mapped; *ln_miss = t.ln_miss;
}
void emul_finish_mixed(int n, const int* s, const int* mapq, int use_mapq, int cap, int trigger, double* out)
{
    for (int i = 0; i < n; ++i) out[i] = finish_mixed(best_of(s[i]), use_mapq != 0, mapq_terms(mapq[i], cap, trigger));
}
void emul_finish_likelihood(int n, const int* s, const int* mapq, int use_mapq, int cap, int trigger, double* out)
{
    for (int i = 0; i < n; ++i) out[i] = finish_likelihood(best_of(s[i]), use_mapq != 0, mapq[i], cap, trigger);
}

} // extern "C"

// The whole per-(haplotype, read) evaluation exactly as the populate kernels perform it, on the CPU:
// candidate slots → classify → DP (generic_align) → flank discount → min → finish_likelihood.
// Mirrors oracle_model_evaluate's signature. Returns 0 ok, 1 ShortHaplotypeError.
extern "C" int emul_pair_evaluate(int band, const char* hap, int hap_len, const char* mask, const int8_t* prior,
                                  const int8_t* go, const int8_t* ge, const char* read, const uint8_t* quals, int read_len,
                                  int use_flanks, int lhs_flank, int rhs_flank, const int32_t* positions, int n_positions,
                                  long long original_pos, int use_mapq, int mapq, int mapq_cap, int mapq_trigger,
                                  int dp_only, int nuc_prior, double* out, int* required_extension)
{
    const HapView hv {hap, mask, prior, go, ge, hap_len};
    const ReadView rv {read, quals, read_len};
    EnumState st {false, false};
    int best = kBestInf;
    for (int c = 0; c < n_positions + 2; ++c) {
        int p;
        const int k = candidate_slot(c, n_positions, positions, original_pos, read_len, hap_len, band, st, &p);
        if (k < 0) { *required_extension = p; return 1; }
        if (k == 0) continue;
        int v;
        const CandKind kind = classify_candidate(hv, rv, band, p, !dp_only, use_flanks != 0, lhs_flank, rhs_flank, &v);
        int val = kBestInf;
        if (kind == CAND_VALUE) val = v;
        else if (kind == CAND_DP || kind == CAND_DP_FLANK) {
            const int a = v, W = read_len + 2 * band - 1;
            GenericModel gm {hap + a, mask + a, prior + a, go + a, ge + a, nuc_prior};
            if (kind == CAND_DP) {
                val = generic_align<false, kGenericMaxDiag>(band, gm, read, (const int8_t*)quals, read_len, nullptr, 1, 0, 0, nullptr, nullptr, nullptr);
            } else {
                int lhs, rhs, fp, fs, ms;
                window_flanks(a, W, hap_len, lhs_flank, rhs_flank, &lhs, &rhs);
                std::vector<unsigned char> bp((size_t)(read_len + 1) * 2 * band, 0);
                const int score = generic_align<true, kGenericMaxDiag>(band, gm, read, (const int8_t*)quals, read_len, bp.data(), 1, lhs, rhs, &fp, &fs, &ms);
                val = discount_flank(score, fs, read_len, ms, fp);
            }
        }
        if (val < best) best = val;
    }
    *out = finish_likelihood(best, use_mapq != 0, mapq, mapq_cap, mapq_trigger);
    return 0;
}

// dp_flank32<band> on the CPU: one alignment, flanks in window coordinates. Returns 0 / -1.
extern "C" int emul_dp_flank32(int band, int L, const char* read, const uint8_t* q, const char* truth, const char* mask, const int8_t* prior,
                               const int8_t* go, const int8_t* ge, int nuc_prior, int lhs_flank, int rhs_flank,
                               int* score, int* flank, int* mask_size)
{
    const int W = L + 2 * band - 1;
    std::vector<RowEntry> rows(L + 1);
    for (int y = 0; y < L; ++y) {
        const int c = base_code(read[y]);
        if (c < 0) return -1;
        rows[y] = make_row_entry32((uint32_t)c | ((uint32_t)q[y] << 8));
    }
    rows[L] = pad_row_entry32();
    std::vector<ColEntry> t(W);
    for (int x = 0; x < W; ++x) t[x] = make_col_entry(truth[x], mask[x], prior[x], go[x], ge[x]);
    int xl = lhs_flank, xr = W - rhs_flank;
    if (xr <= xl) { xl = 0; xr = W + 1; }   // overlapping flanks: every op is in a flank (caller treats the score as the flank score)
    if (xr >= W) xr = W + 1;
    switch (band) {
        case 8:  dp_flank32<8>(rows.data(), L, t.data(), nuc_prior, xl, xr, score, flank, mask_size); break;
        case 16: dp_flank32<16>(rows.data(), L, t.data(), nuc_prior, xl, xr, score, flank, mask_size); break;
        case 32: dp_flank32<32>(rows.data(), L, t.data(), nuc_prior, xl, xr, score, flank, mask_size); break;
        default: return -1;
    }
    if (W - rhs_flank <= lhs_flank) { *flank = *score; *mask_size = L; }
    // 2: the kernel would hand this candidate to the exact traceback path (flank_replay_may_differ)
    bool low_quality = false;
    for (int y = 0; y < L; ++y) low_quality = low_quality || q[y] < 2;
    return flank_replay_may_differ(t.data(), W, lhs_flank, rhs_flank, low_quality) ? 2 : 0;
}

// The multi-lane band core (band_lane_* in phmm_device.cuh) with its NL lanes stepped in lock-step on the CPU: the two
// exchanges dp_band performs with shuffles are done by hand between the phases.
template <class T, int C, int NL, bool OGE>
static typename T::V run_band_form(const RowEntry* rows, int L, const typename T::Tab& tab, typename T::V nucp)
{
    static BandLane<T, C> s[NL];
    const int W = L + NL * C - 1;
    for (int j = 0; j < NL; ++j) band_lane_init<T, C>(s[j], tab, j * C);
    for (int t = 0; t <= W; ++t) {
        typename T::V d_in[NL], i_in[NL];
        for (int j = 0; j < NL; ++j) { const int x = t - (NL - 1 - j); band_lane_top<T, C, OGE>(s[j], rows, L, x - j * C, x, W, tab, nucp, j == NL - 1); }
        for (int j = 0; j < NL; ++j) d_in[j] = j > 0 ? s[j - 1].d_out : T::inf();
        for (int j = 0; j < NL; ++j) { const int x = t - (NL - 1 - j); band_lane_rest<T, C, OGE>(s[j], rows, L, x - j * C, x, d_in[j], j == 0); }
        for (int j = 0; j < NL; ++j) i_in[j] = j < NL - 1 ? s[j + 1].i_run : T::inf();
        for (int j = 0; j < NL; ++j) s[j].i_run = i_in[j];
    }
    typename T::V best = band_lane_result<T, C>(s[0]);
    for (int j = 1; j < NL; ++j) best = T::min2(best, band_lane_result<T, C>(s[j]));
    return best;
}

static bool g_band_oge = false;      // set by emul_dp_band before run_band_any
template <class T, int C, int NL>
static typename T::V run_band(const RowEntry* rows, int L, const typename T::Tab& tab, typename T::V nucp)
{
    return g_band_oge ? run_band_form<T, C, NL, true>(rows, L, tab, nucp) : run_band_form<T, C, NL, false>(rows, L, tab, nucp);
}

template <class T>
static int run_band_any(int band, const RowEntry* rows, int L, const typename T::Tab& tab, typename T::V nucp, typename T::V* out)
{
    switch (band) {
        case 8:   *out = run_band<T, 16, 1>(rows, L, tab, nucp); return 0;
        case 16:  *out = run_band<T, 32, 1>(rows, L, tab, nucp); return 0;
        case 32:  *out = run_band<T, 32, 2>(rows, L, tab, nucp); return 0;
        case 64:  *out = run_band<T, 32, 4>(rows, L, tab, nucp); return 0;
        case 128: *out = run_band<T, 32, 8>(rows, L, tab, nucp); return 0;
        case 256: *out = run_band<T, 32, 16>(rows, L, tab, nucp); return 0;
        default: return -1;
    }
}

// word32 == 0: two alignments of equal read length through the packed s16x2 lanes (read bases ACGT only);
// word32 != 0: alignment 0 alone through the 32-bit lanes (read bases ACGTN). Same argument layout as emul_dp_pair.
extern "C" int emul_dp_band(int word32, int band, int L, const char* read0, const uint8_t* q0, const char* read1, const uint8_t* q1,
                            const char* truth0, const char* mask0, const int8_t* prior0, const int8_t* go0, const int8_t* ge0,
                            const char* truth1, const char* mask1, const int8_t* prior1, const int8_t* go1, const int8_t* ge1,
                            int nuc_prior, int* score0, int* score1)
{
    const int W = L + 2 * band - 1;
    std::vector<RowEntry> rows(L + 1);
    std::vector<ColEntry> t0(W), t1(W);
    for (int x = 0; x < W; ++x) {
        t0[x] = make_col_entry(truth0[x], mask0[x], prior0[x], go0[x], ge0[x]);
        t1[x] = make_col_entry(truth1[x], mask1[x], prior1[x], go1[x], ge1[x]);
    }
    g_band_oge = word32 ? use_oge(go0, ge0, nullptr, nullptr, W) : use_oge(go0, ge0, go1, ge1, W);
    if (word32) {
        for (int y = 0; y < L; ++y) {
            const int c = base_code(read0[y]);
            if (c < 0) return -1;
            rows[y] = make_row_entry32((uint32_t)c | ((uint32_t)q0[y] << 8));
        }
        rows[L] = pad_row_entry32();
        Lanes32::V r;
        const Lanes32::Tab tab {t0.data()};
        if (run_band_any<Lanes32>(band, rows.data(), L, tab, Lanes32::both(nuc_prior), &r)) return -1;
        *score0 = (int)r; *score1 = (int)r;
        return 0;
    }
    for (int y = 0; y < L; ++y) {
        const int c0 = base_code(read0[y]), c1 = base_code(read1[y]);
        if (c0 < 0 || c1 < 0 || c0 > 3 || c1 > 3) return -1;
        rows[y] = make_row_entry((uint32_t)c0 | ((uint32_t)q0[y] << 8), (uint32_t)c1 | ((uint32_t)q1[y] << 8));
    }
    rows[L] = pad_row_entry();
    Lanes16::V r;
    const Lanes16::Tab tab {t0.data(), t1.data()};
    if (run_band_any<Lanes16>(band, rows.data(), L, tab, Lanes16::both(nuc_prior), &r)) return -1;
    *score0 = (int)(r & 0xFFFF); *score1 = (int)(r >> 16);
    return 0;
}

// dp_flank_acc<band> on the CPU (the lean flank-aware DP: the in-flank penalty rides along as an additive payload).
// Returns 0, 1 when the candidate does not qualify (fewer than two read bases certain to lie outside the flanks, or flanks that
// overlap: the kernel keeps those on dp_flank32 / the plain DP), 2 when the replay quirk sends it to the traceback path, -1 on a bad read base.
extern "C" int emul_dp_flank_acc(int band, int L, const char* read, const uint8_t* q, const char* truth, const char* mask, const int8_t* prior,
                                 const int8_t* go, const int8_t* ge, int nuc_prior, int lhs_flank, int rhs_flank, int* score, int* flank)
{
    const int W = L + 2 * band - 1;
    std::vector<RowEntry> rows(L + 1);
    bool low_quality = false;
    for (int y = 0; y < L; ++y) {
        const int c = base_code(read[y]);
        if (c < 0 || c > 3) return -1;
        rows[y] = make_row_entry_facc((uint32_t)c | ((uint32_t)q[y] << 8));
        low_quality = low_quality || q[y] < 2;
    }
    rows[L] = pad_row_entry_facc();
    std::vector<ColEntry> t(W);
    for (int x = 0; x < W; ++x) t[x] = make_col_entry(truth[x], mask[x], prior[x], go[x], ge[x]);
    int xl = lhs_flank, xr = W - rhs_flank;
    if (xr <= xl) return 1;
    if (xr >= W) xr = W + 1;
    if (!flank_mask_cannot_zero(L, band, xl, xr)) return 1;
    if (flank_replay_may_differ(t.data(), W, lhs_flank, rhs_flank, low_quality)) return 2;
    switch (band) {
        case 8:  dp_flank_acc<8>(rows.data(), L, t.data(), nuc_prior, xl, xr, score, flank); break;
        case 16: dp_flank_acc<16>(rows.data(), L, t.data(), nuc_prior, xl, xr, score, flank); break;
        case 32: dp_flank_acc<32>(rows.data(), L, t.data(), nuc_prior, xl, xr, score, flank); break;
        default: return -1;
    }
    return 0;
}

// dp_traceback_forward + traceback_walk on the CPU: score, first_pos, flank score, in-flank read bases and the two alignment strings.
extern "C" int emul_traceback(int band, int L, const char* read, const uint8_t* q, const char* truth, const char* mask, const int8_t* prior,
                              const int8_t* go, const int8_t* ge, int nuc_prior, int lhs_flank, int rhs_flank,
                              int* score, int* first_pos, int* flank, int* mask_size, char* align1, char* align2)
{
    const int W = L + 2 * band - 1;
    std::vector<uint16_t> rows(L + 1);                      // the kernel's staging: the read's row half-words (TbRows2), pad row 0
    for (int y = 0; y < L; ++y) {
        const int c = base_code(read[y]);
        if (c < 0) return -1;
        rows[y] = (uint16_t)((uint32_t)c | ((uint32_t)q[y] << 8));
        const RowEntry a = TbRows2 {rows.data()}.at(y), b = make_row_entry_tb(rows[y]);
        if (a.x != b.x || a.y != b.y) return -2;            // the three row layouts decode to the same entry
        const uint32_t w4 = TbRows4::pack(rows[y]);
        const RowEntry c4 = TbRows4 {&w4}.at(0);
        if (c4.x != b.x || c4.y != b.y) return -2;
    }
    rows[L] = 0;
    std::vector<ColEntry> t(W);
    for (int x = 0; x < W; ++x) t[x] = make_col_entry(truth[x], mask[x], prior[x], go[x], ge[x]);
    // the kernel's back-pointer scratch is reused across calls and never cleared: fill it with words whose every label reads as an
    // insertion, so a walk that reads a cell the forward pass did not write gives a wrong flank score here too
    std::vector<uint32_t> bp((size_t)(W + 1) * 2 * band, 0x55555555u);
    int x_end = -1, state = 0;
    const TbModel gm {truth, mask, prior, go, ge, nuc_prior};
    switch (band) {
        case 8:  dp_traceback_forward<8>(TbRows2 {rows.data()}, L, t.data(), nuc_prior, bp.data(), 1, score, &x_end, &state);
                 traceback_walk<8>(bp.data(), 1, gm, read, q, L, x_end, state, lhs_flank, rhs_flank, first_pos, flank, mask_size, align1, align2); break;
        case 16: dp_traceback_forward<16>(TbRows2 {rows.data()}, L, t.data(), nuc_prior, bp.data(), 1, score, &x_end, &state);
                 traceback_walk<16>(bp.data(), 1, gm, read, q, L, x_end, state, lhs_flank, rhs_flank, first_pos, flank, mask_size, align1, align2); break;
        case 32: dp_traceback_forward<32>(TbRows2 {rows.data()}, L, t.data(), nuc_prior, bp.data(), 1, score, &x_end, &state);
                 traceback_walk<32>(bp.data(), 1, gm, read, q, L, x_end, state, lhs_flank, rhs_flank, first_pos, flank, mask_size, align1, align2); break;
        default: return -1;
    }
    return 0;
}

// dp_flank_fb<band> on the CPU: two alignments of equal read length packed as the kernel packs them (forward pass to the flank
// boundary, backward pass from the window end, crossing cells from F + B). Flanks per alignment in window coordinates.
// out[a] = {score, flank, mask, tie}. Returns 0, 1 when the kernel would not route the pair here (L < 2*band, overlapping flanks,
// no flank at all), -1 on a bad read base.
extern "C" int emul_dp_flank_fb(int band, int L, const char* read0, const uint8_t* q0, const char* read1, const uint8_t* q1,
                                const char* truth0, const char* mask0, const int8_t* prior0, const int8_t* go0, const int8_t* ge0,
                                const char* truth1, const char* mask1, const int8_t* prior1, const int8_t* go1, const int8_t* ge1,
                                int nuc_prior, int lhs0, int rhs0, int lhs1, int rhs1, int* out0, int* out1)
{
    const int W = L + 2 * band - 1;
    if (L < 2 * band) return 1;
    if (W - rhs0 <= lhs0 || W - rhs1 <= lhs1) return 1;
    if ((lhs0 == 0 && rhs0 == 0) || (lhs1 == 0 && rhs1 == 0)) return 1;
    std::vector<RowEntry> rows(L + 2 * band, pad_row_entry());       // the backward pass reads pad rows down to L + 2*band - 1
    for (int y = 0; y < L; ++y) {
        const int c0 = base_code(read0[y]), c1 = base_code(read1[y]);
        if (c0 < 0 || c1 < 0 || c0 > 3 || c1 > 3) return -1;
        rows[y] = make_row_entry((uint32_t)c0 | ((uint32_t)q0[y] << 8), (uint32_t)c1 | ((uint32_t)q1[y] << 8));
    }
    rows[L] = pad_row_entry();
    std::vector<ColEntry> t0(W), t1(W);
    for (int x = 0; x < W; ++x) {
        t0[x] = make_col_entry(truth0[x], mask0[x], prior0[x], go0[x], ge0[x]);
        t1[x] = make_col_entry(truth1[x], mask1[x], prior1[x], go1[x], ge1[x]);
    }
    const uint32_t nucp = (uint32_t)nuc_prior | ((uint32_t)nuc_prior << 16);
    const bool oge = use_oge(go0, ge0, go1, ge1, W);
    std::vector<uint32_t> fscr(fb_scratch_words(band), 0xDEADBEEFu), bscr(fb_scratch_words(band), 0xDEADBEEFu);
    FbResult r0, r1;
    const int b0 = lhs0, b1 = W - rhs0, b2 = lhs1, b3 = W - rhs1;
#define RUN_FB(B) { if (oge) dp_flank_fb<B, true>(rows.data(), L, t0.data(), t1.data(), nucp, b0, b1, b2, b3, fscr.data(), 1, bscr.data(), 1, &r0, &r1); \
                    else dp_flank_fb<B, false>(rows.data(), L, t0.data(), t1.data(), nucp, b0, b1, b2, b3, fscr.data(), 1, bscr.data(), 1, &r0, &r1); }
    switch (band) {
        case 8:  RUN_FB(8) break;
        case 16: RUN_FB(16) break;
        case 32: RUN_FB(32) break;
        default: return -1;
    }
#undef RUN_FB
    out0[0] = r0.score; out0[1] = r0.flank; out0[2] = r0.mask; out0[3] = r0.tie;
    out1[0] = r1.score; out1[1] = r1.flank; out1[2] = r1.mask; out1[3] = r1.tie;
    return 0;
}

// flank_replay_may_differ (loop over the flank columns) against flank_replay_may_differ_pre (per-haplotype prefix counts, as
// k_ncol_prefix builds them) on one haplotype's table: returns the number of disagreements over all window placements tried.
extern "C" int emul_replay_prefix_check(int hap_len, const char* truth, const char* mask, const int8_t* prior, const int8_t* go, const int8_t* ge,
                                        int n_queries, const int* a, const int* W, const int* lhs, const int* rhs, const int* lowq)
{
    std::vector<ColEntry> t(hap_len);
    std::vector<uint32_t> pre(hap_len);
    uint32_t run = 0;
    for (int x = 0; x < hap_len; ++x) {
        t[x] = make_col_entry(truth[x], mask[x], prior[x], go[x], ge[x]);
        run += ncol_class(t[x].x);
        pre[x] = run;
    }
    int bad = 0;
    for (int i = 0; i < n_queries; ++i) {
        const bool want = flank_replay_may_differ(t.data() + a[i], W[i], lhs[i], rhs[i], lowq[i] != 0);
        const bool got = flank_replay_may_differ_pre(pre.data(), a[i], W[i], lhs[i], rhs[i], lowq[i] != 0);
        bad += want != got;
    }
    return bad;
}
