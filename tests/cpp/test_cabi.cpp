// Plain C++14 client of the C ABI and the C++ adapter (no torch, no Python): built by tests/test_gpu_cpp.py with g++ and
// run on the GPU box. Reads one KAT and one tiny populate problem from stdin-free hardcoded data, prints results.
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include "phmm_b200.hpp"

int main()
{
    using namespace octopus_b200;
    try {
        // reference KAT: sse2_band_size_8_check_alignments test 5 (test/unit/core/models/pair_hmm_tests.cpp:290-313)
        const std::string truth = "CCCCACGTATATATATATATATGGGGACGT", read = "CCCCACGTGGGACGT";
        std::vector<std::int8_t> quals(read.size(), 40), gap_open(truth.size(), 90);
        gap_open[8] = 70;
        GpuPairHMM<8> hmm;
        std::vector<char> a1(2 * truth.size() + 1, 0), a2(2 * truth.size() + 1, 0);
        int first_pos = -7;
        const int s1 = hmm.align(truth.data(), read.data(), quals.data(), (int)truth.size(), (int)read.size(), gap_open.data(), (short)1, (short)4);
        const int s2 = hmm.align(truth.data(), read.data(), quals.data(), (int)truth.size(), (int)read.size(), gap_open.data(), (short)1, (short)4,
                                 first_pos, a1.data(), a2.data());
        std::printf("KAT %d %d %d %s %s\n", s1, s2, first_pos, a1.data(), a2.data());
        // batch seam: 2 haplotypes x 2 reads
        HaplotypeBlock haps;
        ReadBlock reads;
        const std::string h0 = "ACGTTGCAAGCTTAGGCTAACGTTAGCATCGATCGGATCTAGCTAGGATCGATACGATCGATCGTAGCTAGCTAGTCGATCGATTTAGCGCGATATCGCGAT";
        std::string h1 = h0; h1[50] = h1[50] == 'A' ? 'C' : 'A';
        for (const auto& h : {h0, h1}) {
            std::vector<char> mf(h.begin(), h.end()), mr(h.begin(), h.end());
            std::vector<std::int8_t> p(h.size(), 50), go(h.size(), 40), ge(h.size(), 3);
            haps.add(h, mf, p, mr, p, go, ge, 0);
        }
        reads.add(h0.substr(30, 40), std::vector<std::uint8_t>(40, 30), 60, false, 30);
        reads.add(h1.substr(35, 40), std::vector<std::uint8_t>(40, 25), 60, true, 35);
        auto cfg = HaplotypeLikelihoodArray::default_config();
        cfg.max_indel_error = 16;
        cfg.map_positions = 0;   // the check below evaluates the original position only
        HaplotypeLikelihoodArray arr {cfg};
        arr.populate(reads, haps);
        for (std::size_t h = 0; h < 2; ++h) { const auto row = arr[h]; std::printf("ROW %zu %.17g %.17g\n", h, row[0], row[1]); }
        {   // the same without mapping quality: -ln10/10 times the integer penalty, to be matched bit for bit
            auto exact_cfg = cfg;
            exact_cfg.use_mapping_quality = 0;
            HaplotypeLikelihoodArray exact {exact_cfg};
            exact.populate(reads, haps);
            for (std::size_t h = 0; h < 2; ++h) { const auto row = exact[h]; std::printf("EXACT %zu %.17g %.17g\n", h, row[0], row[1]); }
        }
        {   // multi-sample container semantics (haplotype_likelihood_array.cpp:200-409): samples are column ranges of one batch
            ReadBlock r0, r1;
            r0.add(h0.substr(30, 40), std::vector<std::uint8_t>(40, 30), 60, false, 30);
            r1.add(h1.substr(35, 40), std::vector<std::uint8_t>(40, 25), 60, true, 35);
            r1.add(h0.substr(30, 40), std::vector<std::uint8_t>(40, 30), 60, false, 30);
            HaplotypeLikelihoodArray multi {cfg};
            multi.populate(HaplotypeLikelihoodArray::ReadMap {{"S1", r0}, {"S2", r1}}, haps);
            bool ok = multi.samples().size() == 2 && multi.num_likelihoods("S1") == 1 && multi.num_likelihoods("S2") == 2 && !multi.is_primed();
            for (std::size_t h = 0; h < 2; ++h) {
                ok = ok && multi("S1", h)[0] == arr[h][0] && multi("S2", h)[0] == arr[h][1] && multi("S2", h)[1] == arr[h][0];
            }
            multi.prime("S2");
            ok = ok && multi.is_primed() && multi.num_likelihoods() == 2 && multi[1][0] == arr[1][1];
            const auto merged = multi.merge_samples();
            ok = ok && merged.samples().size() == 1 && merged.samples()[0] == "S1S2" && merged.is_primed() && merged.num_likelihoods() == 3 &&
                 merged[0][0] == arr[0][0] && merged[0][1] == arr[0][1] && merged[1][2] == arr[1][0];
            const auto only2 = multi.merge_samples({"S2"});
            ok = ok && only2.num_likelihoods() == 2 && only2[1][0] == arr[1][1];
            ok = ok && multi.extract_sample("S1").size() == 2 && multi.extract_sample("S1")[1][0] == arr[1][0];
            multi.reset({1});
            ok = ok && multi.num_haplotypes() == 1 && multi("S1", 0)[0] == arr[1][0];
            bool threw = false;
            try { multi("nope", 0); } catch (const std::out_of_range&) { threw = true; }
            // TemplateMap: a template's value is the sum of its reads' values (haplotype_likelihood_model.cpp:306-320)
            TemplateBlock tb;
            tb.add(reads);                  // one template holding both reads
            tb.add(r0);                     // and one holding the first read alone
            HaplotypeLikelihoodArray tarr {cfg};
            tarr.populate(HaplotypeLikelihoodArray::TemplateMap {{"S1", tb}}, haps);
            tarr.prime("S1");
            for (std::size_t h = 0; h < 2; ++h) ok = ok && tarr.num_likelihoods() == 2 && tarr[h][0] == arr[h][0] + arr[h][1] && tarr[h][1] == arr[h][0];
            std::printf("SAMPLES %s %s\n", ok ? "ok" : "MISMATCH", threw ? "throws" : "nothrow");
        }
        {   // reset(): penalty arrays from the library's error models, then a populate on them; pinned (adapter blocks) vs pageable host buffers
            ErrorModel model {"PCR-free.HiSeq-2500"};
            HaplotypeBlock hb;
            std::string base;
            unsigned long long x = 88172645463325252ull;
            auto rnd = [&x] { x ^= x << 13; x ^= x >> 7; x ^= x << 17; return x; };
            for (int i = 0; i < 300; ++i) base += "ACGT"[rnd() % 4];
            base.replace(100, 16, "AAAAAAAAAAAAAAAA"); base.replace(180, 16, "CACACACACACACACA");
            const int H = 64, R = 40000, L = 100;
            for (int h = 0; h < H; ++h) { std::string s2 = base; s2[(rnd() % 280) + 10] = "ACGT"[rnd() % 4]; hb.add(s2, 0); }
            hb.reset(model);
            ReadBlock rb;
            for (int r = 0; r < R; ++r) {
                const int p = 16 + (int)(rnd() % (300 - L - 32));
                std::string b = base.substr(p, L);
                if (rnd() % 3 == 0) b[rnd() % L] = "ACGT"[rnd() % 4];
                rb.add(b, std::vector<std::uint8_t>(L, (std::uint8_t)(20 + rnd() % 20)), 60, (rnd() & 1) != 0, p);
            }
            auto c2 = HaplotypeLikelihoodArray::default_config();
            c2.max_indel_error = 16; c2.map_positions = 0;
            HaplotypeLikelihoodArray big {c2};
            big.populate(rb, hb);                                   // warm-up (allocations)
            auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
            double t0 = now();
            for (int it = 0; it < 5; ++it) big.populate(rb, hb);
            const double pinned_ms = (now() - t0) / 5;
            // the same call on ordinary (pageable) std::vector storage
            std::vector<std::int64_t> hoff(hb.off.begin(), hb.off.end()), roff(rb.off.begin(), rb.off.end()), hbeg(hb.begin.begin(), hb.begin.end()), rbeg(rb.begin.begin(), rb.begin.end());
            std::vector<char> hseq(hb.seq.begin(), hb.seq.end()), mf(hb.snv_mask_fwd.begin(), hb.snv_mask_fwd.end()), mr(hb.snv_mask_rev.begin(), hb.snv_mask_rev.end()), bases(rb.bases.begin(), rb.bases.end());
            std::vector<std::int8_t> pf(hb.snv_prior_fwd.begin(), hb.snv_prior_fwd.end()), pr(hb.snv_prior_rev.begin(), hb.snv_prior_rev.end()), go(hb.gap_open.begin(), hb.gap_open.end()), ge(hb.gap_extend.begin(), hb.gap_extend.end());
            std::vector<std::uint8_t> quals(rb.quals.begin(), rb.quals.end()), mapq(rb.mapq.begin(), rb.mapq.end()), rev(rb.reverse.begin(), rb.reverse.end());
            std::vector<double> out((std::size_t)H * R);
            const phmm_haplotypes hv {H, hoff.data(), hseq.data(), mf.data(), pf.data(), mr.data(), pr.data(), go.data(), ge.data(), hbeg.data()};
            const phmm_reads rv {R, roff.data(), bases.data(), quals.data(), mapq.data(), rev.data(), rbeg.data()};
            Engine eng;
            phmm_populate(eng.get(), &c2, &hv, &rv, nullptr, nullptr, out.data(), nullptr, PHMM_SPACE_HOST);
            t0 = now();
            for (int it = 0; it < 5; ++it) phmm_populate(eng.get(), &c2, &hv, &rv, nullptr, nullptr, out.data(), nullptr, PHMM_SPACE_HOST);
            const double pageable_ms = (now() - t0) / 5;
            bool same = true;
            for (std::size_t h = 0; h < (std::size_t)H && same; ++h) for (std::size_t r = 0; r < (std::size_t)R; r += 997) same = same && big[h][r] == out[h * R + r];
            int go_min = 127, go_max = 0;
            for (const auto v : hb.gap_open) { go_min = std::min<int>(go_min, v); go_max = std::max<int>(go_max, v); }
            std::printf("E2E pinned_ms=%.3f pageable_ms=%.3f same=%d gap_open_range=%d..%d pairs=%d\n", pinned_ms, pageable_ms, same ? 1 : 0, go_min, go_max, H * R);
        }
        // ShortHaplotypeError must surface as the reference's exception type
        ReadBlock longread;
        longread.add(h0.substr(0, 95), std::vector<std::uint8_t>(95, 30), 60, false, 0);
        try { arr.populate(longread, haps); std::printf("SHORT none\n"); }
        catch (const ShortHaplotypeError& e) { std::printf("SHORT hap=%zu ext=%u\n", e.haplotype_index(), e.required_extension()); }
    } catch (const std::exception& e) {
        std::printf("EXCEPTION %s\n", e.what());
        return 1;
    }
    return 0;
}
