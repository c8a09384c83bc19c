// The shared reset core (octopus_b200/csrc/phmm_reset.cuh) on the CPU:
//   SORT  its introsort gives std::sort's permutation (libstdc++, as the reference build uses it) on random tie-heavy arrays of
//         0..5000 elements and on adversarial inputs that drive the partitioning to the depth limit (heap-sort fallback);
//   CAP   with a deliberately small run capacity the finder and reset report overflow without writing past their buffers, and
//         the growing retry equals a one-shot call with room to spare.
#include "phmm_reset.cuh"

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

namespace {

struct Item { int key, id; };
bool by_key(const Item& a, const Item& b) { return a.key < b.key; }

bool same_permutation(std::vector<Item> v, int* exhausted)
{
    std::vector<Item> want = v;
    std::sort(want.begin(), want.end(), by_key);
    phmm_reset::introsort(v.data(), v.data() + v.size(), by_key, exhausted);
    for (std::size_t i = 0; i < v.size(); ++i) if (v[i].id != want[i].id || v[i].key != want[i].key) return false;
    return true;
}

// McIlroy's adversary ("A killer adversary for quicksort", 1999): keys are decided lazily during one sort so that every
// partition is as bad as it can be; the keys it settles on are a fixed input that drives a median-of-three quicksort quadratic.
std::vector<int> adversary(const int n)
{
    std::vector<int> val((std::size_t)n, n);        // n = "gas": not decided yet
    int solid = 0, candidate = 0;
    std::vector<int> idx((std::size_t)n);
    for (int i = 0; i < n; ++i) idx[(std::size_t)i] = i;
    auto less = [&](const int x, const int y) {
        if (val[(std::size_t)x] == n && val[(std::size_t)y] == n) val[(std::size_t)(x == candidate ? x : y)] = solid++;
        if (val[(std::size_t)x] == n) candidate = x;
        else if (val[(std::size_t)y] == n) candidate = y;
        return val[(std::size_t)x] < val[(std::size_t)y];
    };
    phmm_reset::introsort(idx.data(), idx.data() + n, less);
    for (int& v : val) if (v == n) v = solid++;
    return val;
}

std::vector<unsigned char> repeat_rich(std::mt19937& rng, const int n)
{
    const char* acgt = "ACGT";
    std::vector<unsigned char> s;
    while ((int)s.size() < n) {
        if (rng() % 3 == 0) {
            const int p = 1 + (int)(rng() % 5), k = 2 + (int)(rng() % 20);
            unsigned char motif[5];
            for (int i = 0; i < p; ++i) motif[i] = (unsigned char)acgt[rng() % 4];
            for (int j = 0; j < k; ++j) s.insert(s.end(), motif, motif + p);
        } else s.push_back((unsigned char)acgt[rng() % (1 + rng() % 4)]);
    }
    s.resize((std::size_t)n);
    return s;
}

constexpr std::uint32_t kGuard = 0xA5A5A5A5u;

// The finder / reset in buffers of exactly the given capacity, each followed by guard words; false when a guard was overwritten.
struct Guarded
{
    std::vector<std::uint32_t> w;
    std::vector<phmm_reset::Run> runs, main;
    std::uint32_t n, cap;
    Guarded(std::uint32_t n_, std::uint32_t cap_) : n(n_), cap(cap_)
    {
        w.assign(phmm_reset::scratch_words(n, cap) + 64, kGuard);
        runs.assign(cap + 16, phmm_reset::Run {kGuard, kGuard, kGuard});
        main.assign(cap + 16, phmm_reset::Run {kGuard, kGuard, kGuard});
    }
    phmm_reset::Scratch scratch() { return phmm_reset::Scratch {w.data(), runs.data(), main.data(), cap}; }
    bool intact() const
    {
        for (std::size_t i = phmm_reset::scratch_words(n, cap); i < w.size(); ++i) if (w[i] != kGuard) return false;
        for (std::size_t i = cap; i < runs.size(); ++i) if (runs[i].pos != kGuard || main[i].pos != kGuard || runs[i].len != kGuard || main[i].len != kGuard) return false;
        return true;
    }
};

bool same_runs(const phmm_reset::Run* a, const std::vector<phmm_reset::Run>& b, const std::size_t n)
{
    if (n != b.size()) return false;
    for (std::size_t i = 0; i < n; ++i) if (a[i].pos != b[i].pos || a[i].len != b[i].len || a[i].period != b[i].period) return false;
    return true;
}

} // namespace

int main()
{
    std::mt19937 rng(20261017);
    // SORT: random tie-heavy arrays
    int exhausted = 0, checked = 0;
    for (int n = 0; n <= 5000; n += (n < 100 ? 1 : 37)) {
        for (int rep = 0; rep < 3; ++rep) {
            const int distinct = 1 + (int)(rng() % (1 + n / (1 + (int)(rng() % 8))));
            std::vector<Item> v((std::size_t)n);
            for (int i = 0; i < n; ++i) v[(std::size_t)i] = Item {(int)(rng() % (unsigned)distinct), i};
            if (!same_permutation(v, &exhausted)) { std::printf("SORT fail random n=%d\n", n); return 1; }
            ++checked;
        }
    }
    // SORT: adversarial inputs, plain and with ties (keys halved), at sizes that reach the depth limit
    int adversarial_exhausted = 0;
    for (const int n : {64, 100, 257, 1000, 2048, 5000}) {
        const std::vector<int> keys = adversary(n);
        for (const int shift : {0, 1, 3}) {
            std::vector<Item> v((std::size_t)n);
            for (int i = 0; i < n; ++i) v[(std::size_t)i] = Item {keys[(std::size_t)i] >> shift, i};
            int e = 0;
            if (!same_permutation(v, &e)) { std::printf("SORT fail adversary n=%d shift=%d\n", n, shift); return 1; }
            adversarial_exhausted += e;
            ++checked;
        }
    }
    std::printf("SORT ok arrays=%d depth_limit_hits=%d\n", checked, adversarial_exhausted + exhausted);
    if (adversarial_exhausted == 0) { std::printf("SORT no input reached the depth limit\n"); return 1; }

    // CAP: small capacities report overflow and stay inside their buffers; the retry equals the one-shot result
    const phmm_reset::Model* model = nullptr;
    phmm_reset::Model m;                               // a model with an SNV part and flat rows is enough for the capacity logic
    for (int i = 0; i < 50; ++i) { m.open_at.v[i] = m.open_cg.v[i] = m.open_di.v[i] = m.open_tri.v[i] = (std::int8_t)(40 - i / 2); m.ext_homo.v[i] = m.ext_di.v[i] = m.ext_tri.v[i] = (std::int8_t)(3 + i % 4); }
    for (int k = 0; k < 3; ++k) for (int i = 0; i < 51; ++i) m.caps[k].v[i] = (std::int8_t)(40 - i / 3);
    m.has_snv = true; m.default_open = 40; m.default_extend = 3;
    model = &m;
    int overflows = 0;
    phmm_reset::HostScratch hs;
    for (int t = 0; t < 400; ++t) {
        const int n = 1 + (int)(rng() % 700);
        const std::vector<unsigned char> s = repeat_rich(rng, n);
        for (const std::uint32_t max_period : {3u, 5u}) {
            Guarded big((std::uint32_t)n, 4 * (std::uint32_t)n + 64);
            const int count = phmm_reset::tandem_repeats(s.data(), (std::uint32_t)n, 1, max_period, big.scratch());
            if (count < 0 || !big.intact()) { std::printf("CAP fail one-shot n=%d\n", n); return 1; }
            std::vector<phmm_reset::Run> retried;
            if (phmm_reset::tandem_repeats_host(s.data(), (std::uint32_t)n, 1, max_period, hs, retried) != phmm_reset::kOk ||
                !same_runs(big.runs.data(), retried, (std::size_t)count)) { std::printf("CAP fail retry n=%d\n", n); return 1; }
            for (std::uint32_t cap = 0; cap < (std::uint32_t)count; cap += 1 + (std::uint32_t)count / 7) {
                Guarded small((std::uint32_t)n, cap);
                if (phmm_reset::tandem_repeats(s.data(), (std::uint32_t)n, 1, max_period, small.scratch()) != phmm_reset::kOverflow || !small.intact()) {
                    std::printf("CAP fail overflow n=%d cap=%u count=%d\n", n, cap, count); return 1;
                }
                ++overflows;
            }
        }
        // the whole reset: small capacity overflows inside its buffers; the host retry equals a roomy one-shot call
        std::vector<std::int8_t> a(6 * (std::size_t)n), b(6 * (std::size_t)n);
        auto outs = [&](std::vector<std::int8_t>& o, const int k) { return o.data() + (std::size_t)k * n; };
        Guarded big((std::uint32_t)n, 4 * (std::uint32_t)n + 64);
        if (phmm_reset::reset_haplotype(*model, s.data(), (std::uint32_t)n, nullptr, (char*)outs(a, 0), outs(a, 1), (char*)outs(a, 2), outs(a, 3), outs(a, 4), outs(a, 5), big.scratch()) != phmm_reset::kOk)
            { std::printf("CAP fail reset one-shot\n"); return 1; }
        Guarded small((std::uint32_t)n, 1);
        const int rc = phmm_reset::reset_haplotype(*model, s.data(), (std::uint32_t)n, nullptr, (char*)outs(b, 0), outs(b, 1), (char*)outs(b, 2), outs(b, 3), outs(b, 4), outs(b, 5), small.scratch());
        if (!small.intact() || (rc != phmm_reset::kOk && rc != phmm_reset::kOverflow)) { std::printf("CAP fail reset small\n"); return 1; }
        phmm_reset::reset_haplotype_host(*model, s.data(), (std::uint32_t)n, nullptr, (char*)outs(b, 0), outs(b, 1), (char*)outs(b, 2), outs(b, 3), outs(b, 4), outs(b, 5), hs);
        if (a != b) { std::printf("CAP fail reset retry n=%d\n", n); return 1; }
    }
    std::printf("CAP ok overflows=%d\n", overflows);
    return overflows > 0 ? 0 : 1;
}
