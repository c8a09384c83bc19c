// Plain C++14 client of octopus_b200::DeNovoModel (DeNovoModel::prime + evaluate in one GPU call) with an approx function that records
// the pairs it is asked for. Built and run by tests/test_gpu_mutation_prime.py, which writes the model and the haplotypes to a file
// (argv[1]) and checks the printed values against the reference DeNovoModel.
//   line 1: snv_prior max_period max_periodicity max_indel_length H; line 2: the open table; line 3: the extend table (space-separated
//   floats as %.9g); then H haplotype lines.
// Output: "V t g <value as %a>" for every pair, "A t g" for every approx call, and "PRIMED 1" / "PRIMED 0" around unprime.
#include <cstdio>
#include <fstream>
#include <string>
#include <vector>
#include "phmm_b200.hpp"

int main(int argc, char** argv)
{
    using namespace octopus_b200;
    if (argc < 2) return 2;
    try {
        std::ifstream in {argv[1]};
        double snv_prior;
        MutationRepeatTable table;
        std::size_t H;
        in >> snv_prior >> table.max_period >> table.max_periodicity >> table.max_indel_length >> H;
        table.open.resize(static_cast<std::size_t>((table.max_period + 1) * (table.max_periodicity + 1)));
        table.extend.resize(table.open.size() * static_cast<std::size_t>(table.max_indel_length));
        for (auto& x : table.open) in >> x;
        for (auto& x : table.extend) in >> x;
        std::vector<std::string> haplotypes(H);
        for (auto& h : haplotypes) in >> h;
        Engine engine {0};
        std::vector<std::pair<std::size_t, std::size_t>> asked;
        SomaticMutationModel model {{snv_prior, 0.0}, table, engine, [&] (std::size_t t, std::size_t g) {
            asked.emplace_back(t, g);
            return -1000.0 - static_cast<double>(t * H + g);
        }};
        model.prime(haplotypes);
        bool threw = false;
        try { model.prime(haplotypes); } catch (const std::runtime_error&) { threw = true; }
        if (!threw) { std::printf("ERROR prime twice did not throw\n"); return 1; }
        for (std::size_t t = 0; t < H; ++t)
            for (std::size_t g = 0; g < H; ++g) std::printf("V %zu %zu %a %d\n", t, g, model.evaluate(t, g), model.status(t, g));
        const std::size_t calls = asked.size();
        for (std::size_t t = 0; t < H; ++t)             // a second pass is served from the kept values
            for (std::size_t g = 0; g < H; ++g) model.evaluate(t, g);
        if (asked.size() != calls) { std::printf("ERROR approx asked twice\n"); return 1; }
        for (const auto& p : asked) std::printf("A %zu %zu\n", p.first, p.second);
        std::printf("PRIMED %d\n", model.is_primed() ? 1 : 0);
        model.unprime();
        std::printf("PRIMED %d\n", model.is_primed() ? 1 : 0);
    } catch (const std::exception& ex) {
        std::printf("ERROR %s\n", ex.what());
        return 1;
    }
    return 0;
}
