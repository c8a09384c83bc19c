// Column-table layout microbenchmark for the packed band-16 DP on sm_90a: the real dp_pair<16, true, CS> of phmm_device.cuh over
// shared-memory rows, 4 blocks x 4 warps per SM as in k_populate_fast<16, 1>, L = 150, lanes of a warp aligning one read pair against
// 32 consecutive haplotypes of 300 bases (the C3 shape). Three layouts of the column tables:
//   (a) hap-major, as tab_f / tab_r: lane l reads tab + (h0 + l) * 300 + a + x      -> 32 distinct 128-B lines per warp load
//   (b) hap-major, every lane the same haplotype                                    -> 1 line per warp load (the floor)
//   (c) tiled, [column][haplotype] per 32 haplotypes: tabT + tile * 300 * 32 + (a + x) * 32 + l (CS = 32) -> 2 lines per warp load
// (a) and (c) run the same alignments and must give the same checksum. Prints cell pairs (L x 2B per thread and call) per SM clock,
// counted by clock64() inside the kernel (every block is resident for the whole run), and the SM clock under load that this implies
// (cycles over event time): a power-capped card runs the three layouts at different clocks, so their times also differ by clock.
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -I/usr/local/cuda/include -o ubench_colgather ubench_colgather.cu \
//        -L/usr/local/cuda/lib64/stubs -lnvidia-ml && ./ubench_colgather
#include <cstdio>
#include <cstdint>
#include <vector>
#include <cuda_runtime.h>
#include <nvml.h>
#include "../octopus_b200/csrc/phmm_device.cuh"

using namespace phmm;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e_), __LINE__); return 1; } } while (0)

constexpr int kBand = 16, kL = 150, kHapLen = 300, kH = 128, kWin = 60, kWarps = 4, kReads = 64;

// LAYOUT 0 = (a), 1 = (b), 2 = (c)
template <int LAYOUT>
__global__ void __launch_bounds__(kWarps * 32, 4)
k_gather(const ColEntry* __restrict__ tf, const ColEntry* __restrict__ tr, const RowEntry* __restrict__ grows, const int rounds,
         const uint32_t nucp, const uint32_t one, uint32_t* __restrict__ out, long long* __restrict__ cycles)
{
    __shared__ RowEntry smem[kWarps][kL + 1];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wid = blockIdx.x * kWarps + warp;
    RowEntry* rows = smem[warp];
    const RowEntry* src = grows + (size_t)(wid % kReads) * (kL + 1);
    for (int y = lane; y <= kL; y += 32) rows[y] = src[y];
    __syncthreads();
    const long long c0 = clock64();
    uint32_t acc = 0u;
    for (int r = 0; r < rounds; ++r) {
        const int h0 = ((wid + r) * 32) % kH;              // the warp's 32 haplotypes of this round (one tile)
        const ColEntry *p0, *p1;
        if (LAYOUT == 0) { p0 = tf + (size_t)(h0 + lane) * kHapLen + kWin; p1 = tr + (size_t)(h0 + lane) * kHapLen + kWin; }
        else if (LAYOUT == 1) { p0 = tf + (size_t)h0 * kHapLen + kWin; p1 = tr + (size_t)h0 * kHapLen + kWin; }
        else { p0 = tf + (size_t)h0 * kHapLen + kWin * 32 + lane; p1 = tr + (size_t)h0 * kHapLen + kWin * 32 + lane; }
        acc += LAYOUT == 2 ? dp_pair<kBand, true, 32>(rows, kL, p0, p1, nucp, one) : dp_pair<kBand, true, 1>(rows, kL, p0, p1, nucp, one);
    }
    const long long c1 = clock64();
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
    if (threadIdx.x == 0) cycles[blockIdx.x] = c1 - c0;
}

static uint32_t rng_state = 12345u;
static uint32_t rnd() { rng_state = rng_state * 1664525u + 1013904223u; return rng_state >> 8; }

int main(int argc, char** argv)
{
    const int rounds = argc > 1 ? atoi(argv[1]) : 6000;
    const int reps = argc > 2 ? atoi(argv[2]) : 3;
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
    const int sms = prop.multiProcessorCount;
    nvmlDevice_t dev; unsigned plimit_mw = 0, clk_max = 0;
    const bool nvml = nvmlInit() == NVML_SUCCESS && nvmlDeviceGetHandleByIndex(0, &dev) == NVML_SUCCESS;
    if (nvml) { nvmlDeviceGetPowerManagementLimit(dev, &plimit_mw); nvmlDeviceGetMaxClockInfo(dev, NVML_CLOCK_SM, &clk_max); }
    printf("device %s, %d SMs, power limit %.0f W, max SM clock %u MHz\n", prop.name, sms, plimit_mw / 1e3, clk_max);

    // column tables: hap-major (tf / tr) and the tiled copies of the same entries (tiles of 32 haplotypes, [column][haplotype])
    const char* acgt = "ACGT";
    std::vector<ColEntry> hf((size_t)kH * kHapLen), hr(hf.size()), tf(hf.size()), tr(hf.size());
    for (int h = 0; h < kH; ++h)
        for (int x = 0; x < kHapLen; ++x) {
            const char t = acgt[rnd() & 3];
            const int go = 20 + rnd() % 30, ge = 1 + rnd() % 10;
            const ColEntry ef = make_col_entry(t, acgt[rnd() & 3], (int)(rnd() % 40), go, ge);
            const ColEntry er = make_col_entry(t, acgt[rnd() & 3], (int)(rnd() % 40), go, ge);
            hf[(size_t)h * kHapLen + x] = ef; hr[(size_t)h * kHapLen + x] = er;
            const size_t ti = (size_t)(h / 32) * 32 * kHapLen + (size_t)x * 32 + h % 32;
            tf[ti] = ef; tr[ti] = er;
        }
    std::vector<RowEntry> rows((size_t)kReads * (kL + 1));
    for (int i = 0; i < kReads; ++i) {
        for (int y = 0; y < kL; ++y) {
            const uint32_t h0 = (rnd() & 3) | (uint32_t)(10 + rnd() % 31) << 8, h1 = (rnd() & 3) | (uint32_t)(10 + rnd() % 31) << 8;
            rows[(size_t)i * (kL + 1) + y] = make_row_entry(h0, h1);
        }
        rows[(size_t)i * (kL + 1) + kL] = pad_row_entry();
    }
    ColEntry *d_hf, *d_hr, *d_tf, *d_tr; RowEntry* d_rows; uint32_t* d_out; long long* d_cyc;
    const size_t tb = hf.size() * sizeof(ColEntry);
    CK(cudaMalloc(&d_hf, tb)); CK(cudaMalloc(&d_hr, tb)); CK(cudaMalloc(&d_tf, tb)); CK(cudaMalloc(&d_tr, tb));
    CK(cudaMemcpy(d_hf, hf.data(), tb, cudaMemcpyHostToDevice)); CK(cudaMemcpy(d_hr, hr.data(), tb, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_tf, tf.data(), tb, cudaMemcpyHostToDevice)); CK(cudaMemcpy(d_tr, tr.data(), tb, cudaMemcpyHostToDevice));
    CK(cudaMalloc(&d_rows, rows.size() * sizeof(RowEntry)));
    CK(cudaMemcpy(d_rows, rows.data(), rows.size() * sizeof(RowEntry), cudaMemcpyHostToDevice));
    int bps = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k_gather<0>, kWarps * 32, 0));
    const int grid = sms * 4;
    printf("resident blocks per SM: %d (grid %d x %d threads), rounds %d, L %d, band %d\n", bps, grid, kWarps * 32, rounds, kL, kBand);
    CK(cudaMalloc(&d_out, (size_t)grid * kWarps * 32 * sizeof(uint32_t))); CK(cudaMalloc(&d_cyc, grid * sizeof(long long)));
    const uint32_t nucp = 3u | (3u << 16), one = (uint32_t)(argc > 3 ? atoi(argv[3]) : 1);
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    const char* names[] = {"(a) hap-major, 2400-B lane stride", "(b) one haplotype per warp", "(c) tiled, CS = 32"};
    const double cellpairs_per_sm = (double)4 * kWarps * 32 * rounds * kL * 2 * kBand;
    std::vector<uint32_t> hout((size_t)grid * kWarps * 32);
    for (int rep = -1; rep < reps; ++rep) {   // rep -1: warm-up
        for (int lay = 0; lay < 3; ++lay) {
            const ColEntry* a = lay == 2 ? d_tf : d_hf;
            const ColEntry* b = lay == 2 ? d_tr : d_hr;
            CK(cudaEventRecord(e0));
            if (lay == 0) k_gather<0><<<grid, kWarps * 32>>>(a, b, d_rows, rep < 0 ? rounds / 10 : rounds, nucp, one, d_out, d_cyc);
            else if (lay == 1) k_gather<1><<<grid, kWarps * 32>>>(a, b, d_rows, rep < 0 ? rounds / 10 : rounds, nucp, one, d_out, d_cyc);
            else k_gather<2><<<grid, kWarps * 32>>>(a, b, d_rows, rep < 0 ? rounds / 10 : rounds, nucp, one, d_out, d_cyc);
            CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1)); CK(cudaGetLastError());
            if (rep < 0) continue;
            float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
            std::vector<long long> cyc(grid);
            CK(cudaMemcpy(cyc.data(), d_cyc, grid * sizeof(long long), cudaMemcpyDeviceToHost));
            CK(cudaMemcpy(hout.data(), d_out, hout.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
            double mc = 0; for (long long c : cyc) mc += (double)c; mc /= grid;
            uint64_t sum = 0; for (uint32_t v : hout) sum = sum * 31u + v;
            printf("rep %d %-36s %9.2f ms  %6.2f cell pairs/clk/SM  (mean block %.4g cycles, SM clock under load %4.0f MHz)  checksum %016llx\n",
                   rep, names[lay], ms, cellpairs_per_sm / mc, mc, mc / (ms * 1e3), (unsigned long long)sum);
        }
    }
    if (nvml) nvmlShutdown();
    return 0;
}
