// HaplotypeBlock::reset(model, engine) — the GPU reset through the C++ adapter — against reset(model) on host threads.
#include "phmm_b200.hpp"

#include <cstdio>
#include <random>
#include <string>

int main()
{
    using namespace octopus_b200;
    std::mt19937 rng(4242);
    const char* acgt = "ACGT";
    HaplotypeBlock host, device;
    for (int h = 0; h < 3000; ++h) {
        std::string s;
        const int n = (int)(rng() % 600);
        while ((int)s.size() < n) {
            if (rng() % 4 == 0) { const int p = 1 + (int)(rng() % 5), k = 2 + (int)(rng() % 12); std::string motif; for (int i = 0; i < p; ++i) motif += acgt[rng() % 4]; for (int i = 0; i < k; ++i) s += motif; }
            else s += acgt[rng() % 4];
        }
        s.resize(n);
        std::vector<bool> subs(s.size());
        for (std::size_t i = 0; i < s.size(); ++i) subs[i] = rng() % 20 == 0;
        host.add(s, 0, &subs);
        device.add(s, 0, &subs);
    }
    for (const char* label : {"PCR-free.HiSeq-2500", "PCR.NovaSeq", "PCR.PacBio"}) {
        const ErrorModel model {label};
        Engine engine {0};
        host.reset(model, 4);
        device.reset(model, engine);
        const bool same = host.snv_mask_fwd == device.snv_mask_fwd && host.snv_mask_rev == device.snv_mask_rev &&
                          host.snv_prior_fwd == device.snv_prior_fwd && host.snv_prior_rev == device.snv_prior_rev &&
                          host.gap_open == device.gap_open && host.gap_extend == device.gap_extend;
        std::printf("%s same=%d\n", label, same ? 1 : 0);
        if (!same) return 1;
    }
    return 0;
}
