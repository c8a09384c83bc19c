// The request batcher's populate requests with an error model (phmm_batcher_populate*_reset) without a GPU: the batcher, its
// reset requests' translation unit and the real error models, against the CPU fakes of the engine (fake_engine.cpp and
// fake_engine_reset.cpp). Built by tests/test_batcher_reset_cpu.py under ThreadSanitizer and under AddressSanitizer + UBSan.
#include "../../include/phmm_b200.h"

#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <thread>
#include <vector>

namespace fake {
struct Call { std::string entry; int members; long long haps; std::string key; };
std::vector<Call> calls();
std::vector<std::string> violations();
void clear_calls();
void set_call_delay_us(int us);
}
namespace fake_reset {
struct Call { std::string entry; int members; long long haps; std::string model_key; };
std::vector<Call> calls();
void clear_calls();
}

namespace {

int g_failures = 0;
#define CHECK(cond, ...)                                                                       \
    do {                                                                                       \
        if (!(cond)) { ++g_failures; std::printf("FAIL %s:%d: %s ", __FILE__, __LINE__, #cond); std::printf(__VA_ARGS__); std::printf("\n"); } \
    } while (0)

// One request's inputs and outputs.
struct Req {
    phmm_config cfg {};
    const phmm_error_model* m = nullptr;         // null: a plain request (its arrays from the host reset under `plain_model`)
    const phmm_error_model* plain_model = nullptr;
    std::vector<int64_t> hoff {0}, roff {0}, hbegin, rbegin, toff;
    std::string seq, bases;
    std::vector<uint8_t> sub, quals, mapq, rev;
    std::vector<char> mf, mr;
    std::vector<int8_t> pf, pr, go, ge;
    phmm_flank_state flank {1, 3, 5};
    std::vector<double> out;
    std::vector<int32_t> status;
    int rc = 12345;
    std::string err;

    phmm_haplotype_sequences seqs() const { return {(int32_t)(hoff.size() - 1), hoff.data(), seq.data(), sub.data(), hbegin.data()}; }
    phmm_haplotypes haps() const
    {
        return {(int32_t)(hoff.size() - 1), hoff.data(), seq.data(), mf.data(), pf.data(), mr.data(), pr.data(), go.data(), ge.data(), hbegin.data()};
    }
    phmm_reads reads() const { return {(int32_t)(roff.size() - 1), roff.data(), bases.data(), quals.data(), mapq.data(), rev.data(), rbegin.data()}; }
    long long H() const { return (long long)hoff.size() - 1; }
    long long R() const { return (long long)roff.size() - 1; }
    long long cols() const { return toff.empty() ? R() : (long long)toff.size() - 1; }
};

Req make(std::mt19937& g, const phmm_error_model* m, bool plain, int n_haps, int n_reads, int hap_len = 150)
{
    Req q;
    q.cfg = {16, 0, 1, 120, -1, 1, 2, 0, 1};     // phmm_default_config with band 16 (the fakes do not define it)
    q.m = plain ? nullptr : m;
    q.plain_model = m;
    const char* acgt = "ACGT";
    std::string base;
    for (int i = 0; i < hap_len; ++i) base += (i % 37 < 12) ? "CA"[i % 2] : acgt[g() % 4];     // repeats for the indel model
    for (int h = 0; h < n_haps; ++h) {
        std::string s = base;
        s[g() % s.size()] = acgt[g() % 4];
        q.seq += s;
        q.hoff.push_back((int64_t)q.seq.size());
        q.hbegin.push_back(100);
        for (size_t i = 0; i < s.size(); ++i) q.sub.push_back(g() % 20 == 0);
    }
    for (int r = 0; r < n_reads; ++r) {
        const int L = 30 + (int)(g() % 40);
        const int p = hap_len > L ? (int)(g() % (hap_len - L)) : 0;
        std::string read = base.substr(p, L);
        read.resize(L, 'A');
        q.bases += read;
        q.roff.push_back((int64_t)q.bases.size());
        for (int i = 0; i < L; ++i) q.quals.push_back(10 + g() % 30);
        q.mapq.push_back(g() % 61); q.rev.push_back(g() % 2); q.rbegin.push_back(100 + p);
    }
    const size_t B = q.seq.size();
    q.mf.assign(B, 0); q.mr.assign(B, 0); q.pf.assign(B, 0); q.pr.assign(B, 0); q.go.assign(B, 0); q.ge.assign(B, 0);
    phmm_reset_haplotypes(m, (int32_t)q.H(), q.hoff.data(), q.seq.data(), q.sub.data(), q.mf.data(), q.pf.data(), q.mr.data(), q.pr.data(),
                          q.go.data(), q.ge.data(), 1);
    return q;
}

void as_templates(Req& q)
{
    q.toff = {0};
    for (long long r = 3; r < q.R(); r += 3) q.toff.push_back(r);
    q.toff.push_back(q.R());
}

// The request through the batcher (on the calling thread).
void submit(phmm_batcher* b, Req& q)
{
    q.out.assign((size_t)(q.H() * q.cols()), 0.0);
    q.status.assign((size_t)(q.H() * q.R()), -7);
    const phmm_haplotype_sequences s = q.seqs();
    const phmm_haplotypes h = q.haps();
    const phmm_reads r = q.reads();
    if (q.m && !q.toff.empty())
        q.rc = phmm_batcher_populate_templates_reset(b, &q.cfg, q.m, &s, &r, q.toff.data(), (int32_t)q.toff.size() - 1, &q.flank, q.out.data(), q.status.data());
    else if (q.m)
        q.rc = phmm_batcher_populate_reset(b, &q.cfg, q.m, &s, &r, nullptr, &q.flank, q.out.data(), q.status.data());
    else
        q.rc = phmm_batcher_populate(b, &q.cfg, &h, &r, nullptr, &q.flank, q.out.data(), q.status.data());
    q.err = q.rc ? phmm_batcher_last_error() : "";
}

// What the request gets alone: the fake engine's _reset call (host reset + plain populate), or the plain call.
void solo(Req& q)
{
    phmm_engine* e = nullptr;
    phmm_create(&e, 0);
    q.out.assign((size_t)(q.H() * q.cols()), 0.0);
    q.status.assign((size_t)(q.H() * q.R()), -7);
    const phmm_haplotype_sequences s = q.seqs();
    const phmm_haplotypes h = q.haps();
    const phmm_reads r = q.reads();
    if (q.m && !q.toff.empty())
        q.rc = phmm_populate_templates_reset(e, &q.cfg, q.m, &s, &r, q.toff.data(), (int32_t)q.toff.size() - 1, nullptr, &q.flank, q.out.data(), q.status.data(), 0);
    else if (q.m)
        q.rc = phmm_populate_reset(e, &q.cfg, q.m, &s, &r, nullptr, &q.flank, q.out.data(), q.status.data(), 0);
    else
        q.rc = phmm_populate(e, &q.cfg, &h, &r, nullptr, &q.flank, q.out.data(), q.status.data(), 0);
    q.err = q.rc ? phmm_last_error(e) : "";
    phmm_destroy(e);
}

bool same(const Req& a, const Req& b)
{
    return a.rc == b.rc && a.err == b.err && a.status == b.status && std::memcmp(a.out.data(), b.out.data(), a.out.size() * sizeof(double)) == 0;
}

// Runs every request on a thread of its own through one batcher that waits for all of them, then compares each with its solo result.
void run_all(std::vector<Req>& reqs, const char* what)
{
    std::vector<Req> want = reqs;
    for (Req& q : want) solo(q);
    fake::clear_calls(); fake_reset::clear_calls();
    phmm_batcher* b = nullptr;
    const phmm_batcher_options opt {(int32_t)reqs.size(), 5000000};
    CHECK(phmm_batcher_create(&b, 0, &opt) == PHMM_OK, "%s", what);
    std::vector<std::thread> ts;
    for (Req& q : reqs) ts.emplace_back(submit, b, std::ref(q));
    for (std::thread& t : ts) t.join();
    phmm_batcher_destroy(b);
    for (size_t i = 0; i < reqs.size(); ++i) CHECK(same(reqs[i], want[i]), "%s: request %zu rc %d / %d (%s / %s)", what, i, reqs[i].rc, want[i].rc, reqs[i].err.c_str(), want[i].err.c_str());
}

phmm_error_model* model(const char* label)
{
    phmm_error_model* m = nullptr;
    CHECK(phmm_error_model_create(&m, label) == PHMM_OK, "%s", label);
    return m;
}

phmm_error_model* custom(const char* text)
{
    phmm_error_model* m = nullptr;
    CHECK(phmm_error_model_create_custom(&m, text) == PHMM_OK, "%s", text);
    return m;
}

} // namespace

int main()
{
    std::mt19937 g(7);
    phmm_error_model* a1 = model("PCR.NovaSeq");
    phmm_error_model* a2 = model("pcr.novaseq");              // the same model, created separately from another spelling
    phmm_error_model* c1 = custom("A:30,25,20\nCA:26,20,14\nNN:24,18\n");
    phmm_error_model* c2 = custom("A:30,25,20\nCA:26,20,14\nNN:24,18\n");
    phmm_error_model* other = model("PCR-free.HiSeq-2500");
    phmm_error_model* negative = custom("A:-2,-2,-2\nCA:-3,-3\n");

    {   // models equal by content merge, others never share a call
        std::vector<Req> reqs;
        for (int i = 0; i < 12; ++i) reqs.push_back(make(g, (const phmm_error_model*[]) {a1, a2, c1, c2, other, a1}[i % 6], false, 2 + i % 4, 5 + i));
        run_all(reqs, "merge by content");
        const std::vector<fake_reset::Call> calls = fake_reset::calls();
        CHECK(calls.size() == 3, "%zu calls", calls.size());
        int members[3] = {0, 0, 0};
        for (const fake_reset::Call& c : calls) {
            CHECK(c.entry == "populate_regions_reset", "%s", c.entry.c_str());
            const int k = c.members == 6 ? 0 : c.members == 4 ? 1 : c.members == 2 ? 2 : -1;
            CHECK(k >= 0, "a call of %d members", c.members);
            if (k >= 0) ++members[k];
        }
        CHECK(members[0] == 1 && members[1] == 1 && members[2] == 1, "%d %d %d", members[0], members[1], members[2]);
    }
    {   // plain and reset requests never share a call
        std::vector<Req> reqs;
        for (int i = 0; i < 10; ++i) reqs.push_back(make(g, a1, i % 2 == 0, 3, 8));
        run_all(reqs, "plain and reset");
        const std::vector<fake_reset::Call> rcalls = fake_reset::calls();
        const std::vector<fake::Call> pcalls = fake::calls();
        CHECK(rcalls.size() == 1 && rcalls[0].members == 5, "%zu reset calls", rcalls.size());
        CHECK(pcalls.size() == 2 && pcalls[0].members == 5 && pcalls[1].members == 5, "%zu plain calls", pcalls.size());
    }
    {   // templates merge as read requests; positions, a model with a negative penalty and a short haplotype
        std::vector<Req> reqs;
        for (int i = 0; i < 4; ++i) { reqs.push_back(make(g, c1, false, 3, 12)); if (i % 2) as_templates(reqs.back()); }
        reqs.push_back(make(g, negative, false, 2, 6));
        reqs.push_back(make(g, c1, false, 2, 6, 50));               // reads up to 69 bases over 50-base haplotypes
        run_all(reqs, "templates and run-alone");
        CHECK(reqs[4].rc == PHMM_ERR_INVALID && reqs[4].err == "snv prior / gap penalty outside [0,127]", "%d %s", reqs[4].rc, reqs[4].err.c_str());
        CHECK(reqs[5].rc == PHMM_ERR_SHORT_HAPLOTYPE, "%d", reqs[5].rc);
        for (int i = 0; i < 4; ++i) CHECK(reqs[i].rc == PHMM_OK, "%d: %d", i, reqs[i].rc);
        int alone = 0;
        for (const fake_reset::Call& c : fake_reset::calls()) alone += c.entry == "populate_reset";
        CHECK(alone == 1, "%d requests ran alone", alone);

        Req p = make(g, c1, false, 2, 4);
        std::vector<int64_t> poff(9);
        std::vector<int32_t> pos(8, 0);
        for (int i = 0; i <= 8; ++i) poff[i] = i;
        const phmm_positions ps {poff.data(), pos.data()};
        phmm_batcher* b = nullptr;
        phmm_batcher_create(&b, 0, nullptr);
        std::vector<double> out(8), out2(8);
        std::vector<int32_t> st(8), st2(8);
        const phmm_haplotype_sequences s = p.seqs();
        const phmm_reads r = p.reads();
        fake_reset::clear_calls();
        CHECK(phmm_batcher_populate_reset(b, &p.cfg, c1, &s, &r, &ps, nullptr, out.data(), st.data()) == PHMM_OK, "positions");
        CHECK(fake_reset::calls().size() == 1 && fake_reset::calls()[0].entry == "populate_reset", "positions run alone");
        phmm_engine* e = nullptr;
        phmm_create(&e, 0);
        phmm_populate_reset(e, &p.cfg, c1, &s, &r, &ps, nullptr, out2.data(), st2.data(), 0);
        phmm_destroy(e);
        CHECK(out == out2 && st == st2, "positions result");
        phmm_batcher_destroy(b);
    }
    {   // argument errors: checked on the request's own thread, before any engine call, with the engine's messages
        phmm_batcher* b = nullptr;
        phmm_batcher_create(&b, 0, nullptr);
        fake::clear_calls(); fake_reset::clear_calls();
        Req q = make(g, a1, false, 2, 4);
        std::vector<double> out(8);
        phmm_haplotype_sequences s = q.seqs();
        const phmm_reads r = q.reads();
        auto expect = [&](const phmm_error_model* m, const phmm_haplotype_sequences* sp, int rc, const char* msg) {
            const int got = phmm_batcher_populate_reset(b, &q.cfg, m, sp, &r, nullptr, nullptr, out.data(), nullptr);
            CHECK(got == rc && std::string(phmm_batcher_last_error()) == msg, "%d %s (want %d %s)", got, phmm_batcher_last_error(), rc, msg);
        };
        expect(nullptr, &s, PHMM_ERR_INVALID, "null argument");
        expect(a1, nullptr, PHMM_ERR_INVALID, "null argument");
        phmm_haplotype_sequences bad = s; bad.seq = nullptr;
        expect(a1, &bad, PHMM_ERR_INVALID, "null argument");
        std::vector<int64_t> dec {0, 10, 5};
        bad = s; bad.off = dec.data();
        expect(a1, &bad, PHMM_ERR_INVALID, "bad haplotype offsets");
        std::string longseq(70000, 'A');
        std::vector<int64_t> loff {0, 70000};
        const phmm_haplotype_sequences ls {1, loff.data(), longseq.data(), nullptr, nullptr};
        expect(a1, &ls, PHMM_ERR_INVALID, "haplotype longer than 65535 bases");
        bad = s; bad.n = 0;
        expect(a1, &bad, PHMM_ERR_INVALID, "empty or null haplotype / read block");
        std::vector<int64_t> toff {0, 9};
        CHECK(phmm_batcher_populate_templates_reset(b, &q.cfg, a1, &s, &r, toff.data(), 1, nullptr, out.data(), nullptr) == PHMM_ERR_INVALID &&
              std::string(phmm_batcher_last_error()) == "template offsets must cover the reads exactly", "%s", phmm_batcher_last_error());
        CHECK(phmm_batcher_populate_reset(nullptr, &q.cfg, a1, &s, &r, nullptr, nullptr, out.data(), nullptr) == PHMM_ERR_INVALID &&
              std::string(phmm_batcher_last_error()) == "null batcher", "null batcher");
        CHECK(fake::calls().empty() && fake_reset::calls().empty(), "an argument error reached the engine");
        phmm_batcher_destroy(b);
    }
    {   // destroy waits for the requests in flight
        phmm_batcher* b = nullptr;
        phmm_batcher_create(&b, 0, nullptr);
        fake::set_call_delay_us(200000);
        Req q = make(g, a1, false, 2, 4);
        std::atomic<bool> done {false};
        std::thread t([&] { submit(b, q); done = true; });
        std::this_thread::sleep_for(std::chrono::milliseconds(50));
        phmm_batcher_destroy(b);
        CHECK(done.load(), "destroy returned before the request");
        t.join();
        fake::set_call_delay_us(0);
        CHECK(q.rc == PHMM_OK, "%d", q.rc);
    }
    for (const std::string& v : fake::violations()) { ++g_failures; std::printf("VIOLATION %s\n", v.c_str()); }
    for (phmm_error_model* m : {a1, a2, c1, c2, other, negative}) phmm_error_model_destroy(m);
    if (g_failures) { std::printf("%d failures\n", g_failures); return 1; }
    std::printf("BATCHER RESET CPU ok\n");
    return 0;
}
