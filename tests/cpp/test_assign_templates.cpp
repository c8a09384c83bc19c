// Plain C++14 client of octopus_b200::compute_haplotype_support over a TemplateBlock (template assignment for many genotypes in one
// GPU call), on an Engine and on a SharedEngine, with the drop, first and all ambiguity actions and the ShortHaplotypeError it throws.
// Built and run by tests/test_gpu_assign_templates.py. Self-checking: both engines give the same supports; every support follows
// from the per-template top sets of Engine::assign_templates (template indices, ambiguous templates with their sets); the shared
// engine's raw call equals the engine's bit for bit; a short haplotype throws the same ShortHaplotypeError on both, for the first
// short (haplotype, read) pair in group, haplotype, read order. Prints "TEMPLATE SUPPORT ok" and exits 0 when everything holds.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>
#include "phmm_b200.hpp"

namespace {

using namespace octopus_b200;

int g_failures = 0;

void expect(bool ok, const char* what)
{
    if (!ok) { ++g_failures; std::printf("FAIL %s\n", what); }
}

const char* name(AmbiguousAction a) { return a == AmbiguousAction::drop ? "drop" : a == AmbiguousAction::first ? "first" : "all"; }

void add_haplotype(HaplotypeBlock& haps, const std::string& s, std::mt19937& rng)
{
    std::vector<std::int8_t> pf(s.size()), pr(s.size()), go(s.size()), ge(s.size());
    for (std::size_t i = 0; i < s.size(); ++i) {
        pf[i] = static_cast<std::int8_t>(1 + rng() % 120); pr[i] = static_cast<std::int8_t>(1 + rng() % 120);
        go[i] = static_cast<std::int8_t>(3 + rng() % 40); ge[i] = static_cast<std::int8_t>(1 + rng() % 10);
    }
    std::string mf = s, mr = s;
    std::rotate(mf.begin(), mf.begin() + 1, mf.end());
    std::rotate(mr.rbegin(), mr.rbegin() + 1, mr.rend());
    haps.add(s, std::vector<char>(mf.begin(), mf.end()), pf, std::vector<char>(mr.begin(), mr.end()), pr, go, ge, 0);
}

void add_copy(HaplotypeBlock& haps, std::size_t h)
{
    const auto b = static_cast<std::size_t>(haps.off[h]), e = static_cast<std::size_t>(haps.off[h + 1]);
    haps.add(std::string(haps.seq.begin() + b, haps.seq.begin() + e), std::vector<char>(haps.snv_mask_fwd.begin() + b, haps.snv_mask_fwd.begin() + e),
             std::vector<std::int8_t>(haps.snv_prior_fwd.begin() + b, haps.snv_prior_fwd.begin() + e),
             std::vector<char>(haps.snv_mask_rev.begin() + b, haps.snv_mask_rev.begin() + e),
             std::vector<std::int8_t>(haps.snv_prior_rev.begin() + b, haps.snv_prior_rev.begin() + e),
             std::vector<std::int8_t>(haps.gap_open.begin() + b, haps.gap_open.begin() + e),
             std::vector<std::int8_t>(haps.gap_extend.begin() + b, haps.gap_extend.begin() + e), 0);
}

std::string mutate(std::string s, std::mt19937& rng, int n)
{
    static const char kAcgt[] = "ACGT";
    for (int i = 0; i < n; ++i) s[rng() % s.size()] = kAcgt[rng() % 4];
    return s;
}

bool same(const std::vector<HaplotypeSupport>& a, const std::vector<HaplotypeSupport>& b)
{
    if (a.size() != b.size()) return false;
    for (std::size_t g = 0; g < a.size(); ++g) if (a[g].reads != b[g].reads || a[g].ambiguous != b[g].ambiguous) return false;
    return true;
}

} // namespace

int main()
{
    try {
        std::mt19937 rng(4711);
        static const char kAcgt[] = "ACGT";
        HaplotypeBlock haps;
        TemplateBlock templates;
        std::vector<std::int32_t> hap_first {0}, template_first {0};
        const int kHaps[] = {2, 3, 2, 3};
        for (int g = 0; g < 4; ++g) {
            std::string base(500, 'A');
            for (auto& c : base) c = kAcgt[rng() % 4];
            const auto h0 = haps.size();
            for (int k = 0; k < kHaps[g]; ++k) {
                if (g == 1 && k > 0) add_copy(haps, h0);                      // group 1: copies, every template ambiguous
                else add_haplotype(haps, k ? mutate(base, rng, 3) : base, rng);
            }
            const int n_templates = 6 + static_cast<int>(rng() % 10);
            for (int t = 0; t < n_templates; ++t) {
                ReadBlock mates;
                const int n = 1 + static_cast<int>(rng() % 3);
                for (int m = 0; m < n; ++m) {
                    const std::size_t hsrc = h0 + rng() % static_cast<std::size_t>(kHaps[g]);
                    const auto hb = static_cast<std::size_t>(haps.off[hsrc]), hl = static_cast<std::size_t>(haps.off[hsrc + 1]) - hb;
                    const std::size_t p = rng() % (hl - 150);
                    const std::string bases = mutate(std::string(haps.seq.begin() + hb + p, haps.seq.begin() + hb + p + 150), rng, 2);
                    std::vector<std::uint8_t> quals(150);
                    for (auto& q : quals) q = static_cast<std::uint8_t>(8 + rng() % 33);
                    mates.add(bases, quals, 60, m % 2 == 1, static_cast<long long>(p));
                }
                templates.add(mates);
            }
            hap_first.push_back(static_cast<std::int32_t>(haps.size()));
            template_first.push_back(static_cast<std::int32_t>(templates.size()));
        }
        std::vector<double> priors(haps.size(), 0.0);
        priors[0] = -0.5;
        auto cfg = HaplotypeLikelihoodArray::default_config();
        cfg.max_indel_error = 16;
        Engine engine;
        SharedEngine shared(-1, 2, 2000);
        const auto T = static_cast<std::int32_t>(templates.size());
        const auto raw = engine.assign_templates(cfg, haps.view(), templates.reads.view(), templates.off.data(), T, hap_first, template_first, &priors, true);
        const auto raw_s = shared.assign_templates(cfg, haps.view(), templates.reads.view(), templates.off.data(), T, hap_first, template_first, &priors, true);
        expect(raw.top == raw_s.top && raw.status == raw_s.status, "shared engine's top / status");
        expect(raw.likelihood.size() == raw_s.likelihood.size() &&
               std::memcmp(raw.likelihood.data(), raw_s.likelihood.data(), raw.likelihood.size() * sizeof(double)) == 0, "shared engine's likelihoods");
        expect(raw.top.size() == templates.size(), "one top set per template");
        int ambiguous = 0;
        for (const auto action : {AmbiguousAction::drop, AmbiguousAction::first, AmbiguousAction::all}) {
            const auto on_engine = compute_haplotype_support(templates, haps, hap_first, template_first, &priors, action, cfg, engine);
            const auto on_shared = compute_haplotype_support(templates, haps, hap_first, template_first, &priors, action, cfg, shared);
            expect(same(on_engine, on_shared), name(action));
            for (std::size_t g = 0; g + 1 < hap_first.size(); ++g) {
                const auto nh = static_cast<unsigned>(hap_first[g + 1] - hap_first[g]);
                std::vector<std::vector<std::size_t>> want(nh);
                std::vector<std::pair<std::size_t, std::vector<unsigned>>> want_amb;
                for (std::size_t t = static_cast<std::size_t>(template_first[g]); t < static_cast<std::size_t>(template_first[g + 1]); ++t) {
                    std::vector<unsigned> set;
                    for (unsigned k = 0; k < nh; ++k) if (raw.top[t] >> k & 1u) set.push_back(k);
                    if (set.size() == 1) { want[set[0]].push_back(t); continue; }
                    if (action == AmbiguousAction::first) want[set[0]].push_back(t);
                    if (action == AmbiguousAction::all) for (unsigned k : set) want[k].push_back(t);
                    want_amb.emplace_back(t, set);
                }
                expect(on_engine[g].reads == want && on_engine[g].ambiguous == want_amb, name(action));
                ambiguous += static_cast<int>(want_amb.size());
            }
        }
        expect(ambiguous >= 3 * (template_first[2] - template_first[1]), "group 1's templates are ambiguous");
        // one more group: haplotype 0's first 60 bases against group 0's templates, too short for them
        HaplotypeBlock more = haps;
        const std::string seq0(haps.seq.begin(), haps.seq.begin() + 60);
        more.add(seq0, std::vector<char>(haps.snv_mask_fwd.begin(), haps.snv_mask_fwd.begin() + 60),
                 std::vector<std::int8_t>(haps.snv_prior_fwd.begin(), haps.snv_prior_fwd.begin() + 60),
                 std::vector<char>(haps.snv_mask_rev.begin(), haps.snv_mask_rev.begin() + 60),
                 std::vector<std::int8_t>(haps.snv_prior_rev.begin(), haps.snv_prior_rev.begin() + 60),
                 std::vector<std::int8_t>(haps.gap_open.begin(), haps.gap_open.begin() + 60),
                 std::vector<std::int8_t>(haps.gap_extend.begin(), haps.gap_extend.begin() + 60), 0);
        TemplateBlock more_templates = templates;
        for (std::int32_t t = template_first[0]; t < template_first[1]; ++t) {
            ReadBlock mates;
            for (std::int64_t r = templates.off[t]; r < templates.off[t + 1]; ++r) {
                const auto b = static_cast<std::size_t>(templates.reads.off[r]), e = static_cast<std::size_t>(templates.reads.off[r + 1]);
                mates.add(std::string(templates.reads.bases.begin() + b, templates.reads.bases.begin() + e),
                          std::vector<std::uint8_t>(templates.reads.quals.begin() + b, templates.reads.quals.begin() + e), templates.reads.mapq[r],
                          templates.reads.reverse[r] != 0, templates.reads.begin[r]);
            }
            more_templates.add(mates);
        }
        auto hf = hap_first, tf = template_first;
        hf.push_back(hf.back() + 1);
        tf.push_back(tf.back() + (template_first[1] - template_first[0]));
        priors.push_back(0.0);
        const auto short_raw = engine.assign_templates(cfg, more.view(), more_templates.reads.view(), more_templates.off.data(),
                                                       static_cast<std::int32_t>(more_templates.size()), hf, tf, &priors);
        expect(short_raw.code == PHMM_ERR_SHORT_HAPLOTYPE, "short haplotype code");
        unsigned want_ext = 0;
        for (auto s : short_raw.status) if ((s & 0xFFFF) == PHMM_STATUS_SHORT_HAP) { want_ext = static_cast<std::uint32_t>(s) >> 16; break; }
        for (int k = 0; k < 2; ++k) {
            try {
                if (k == 0) compute_haplotype_support(more_templates, more, hf, tf, &priors, AmbiguousAction::drop, cfg, engine);
                else compute_haplotype_support(more_templates, more, hf, tf, &priors, AmbiguousAction::drop, cfg, shared);
                expect(false, "no ShortHaplotypeError");
            } catch (const ShortHaplotypeError& e) {
                std::printf("SHORT hap=%zu ext=%u\n", e.haplotype_index(), e.required_extension());
                expect(e.haplotype_index() == haps.size() && e.required_extension() == want_ext && want_ext > 0, "ShortHaplotypeError");
            }
        }
    } catch (const std::exception& e) {
        std::printf("EXCEPTION %s\n", e.what());
        return 1;
    }
    if (g_failures) return 1;
    std::printf("TEMPLATE SUPPORT ok\n");
    return 0;
}
