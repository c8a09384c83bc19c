// Integer-issue roofline microbenchmark for sm_90a: per-SM throughput of the instructions the packed pair-HMM cell is
// made of (VIMNMX.S16x2, VIMNMX3.S16x2, VIADDMNMX.S16x2, PRMT, IMAD.IADD / IADD3, LDS broadcast), each as 8 independent
// dependency chains per thread so that latency is hidden, and of the exact 10-instruction cell mix.
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o ubench_int ubench_int.cu && ./ubench_int
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); return 1; } } while (0)

__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t s) { uint32_t d; asm volatile("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(s)); return d; }

constexpr int CH = 8;      // independent chains per thread
constexpr int UNR = 32;    // ops per chain per loop iteration

template <int OP>
__global__ void __launch_bounds__(256) k_op(uint32_t* out, const uint32_t* in, int iters)
{
    __shared__ uint32_t sm[256];
    sm[threadIdx.x] = in[threadIdx.x] & 0x00ff00ffu;
    __syncthreads();
    uint32_t v[CH], b = in[1] | 0x00010001u, c = in[2] | 0x70007000u;
#pragma unroll
    for (int i = 0; i < CH; ++i) v[i] = in[i] + threadIdx.x;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
#pragma unroll
            for (int i = 0; i < CH; ++i) {
                if (OP == 0) v[i] = __vmins2(v[i], b + u);                       // VIMNMX.S16x2
                else if (OP == 1) v[i] = __vimin3_s16x2(v[i], b, c + u);         // VIMNMX3.S16x2
                else if (OP == 2) v[i] = __viaddmin_s16x2(v[i], b, c);           // VIADDMNMX.S16x2
                else if (OP == 3) v[i] = prmt(v[i], b, c + u);                   // PRMT
                else if (OP == 4) asm volatile("add.u32 %0, %0, %1;" : "+r"(v[i]) : "r"(b));   // IADD3 / IMAD.IADD (compiler's choice)
                else if (OP == 5) v[i] = min((int)v[i], (int)(b + u));            // IMNMX (32-bit)
                else if (OP == 6) v[i] ^= sm[(it + u + i) & 255];               // LDS broadcast (same address for all lanes)
                else if (OP == 7) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(v[i]) : "r"(b), "r"(c));   // IMAD
            }
        }
    }
    uint32_t s = 0;
#pragma unroll
    for (int i = 0; i < CH; ++i) s ^= v[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// the packed pair-HMM cell, 8 independent "diagonals" per thread, rows from shared memory (broadcast)
__global__ void __launch_bounds__(256) k_cell(uint32_t* out, const uint32_t* in, int iters)
{
    __shared__ uint32_t rows[512];
    for (int i = threadIdx.x; i < 512; i += 256) rows[i] = 0x8480u | (in[i & 63] & 0x1f1f0303u);
    __syncthreads();
    uint32_t M[CH], D[CH + 1], i_run = 0x70007000u;
    const uint32_t caps0 = in[3] & 0x7f7f7f7fu, caps1 = in[4] & 0x7f7f7f7fu, go = 0x00050005u, ge = 0x00010001u, gop = 0x00070007u, gep = 0x00030003u;
#pragma unroll
    for (int i = 0; i < CH; ++i) { M[i] = in[i] & 0x00ff00ffu; D[i] = 0x70007000u; }
    D[CH] = 0;
    for (int it = 0; it < iters; ++it) {
        const uint32_t* rp = rows + (it & 255) + 16;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
#pragma unroll
            for (int k = CH - 1; k >= 0; --k) {
                const uint32_t w = rp[u - k];
                const uint32_t cap = prmt(caps0, caps1, w);
                const uint32_t q = prmt(w, 0u, 0x4342u);
                const uint32_t sub = __vmins2(q, cap);
                const uint32_t m = M[k], d = D[k];
                M[k] = __vimin3_s16x2(m, i_run, d) + sub;
                D[k + 1] = __viaddmin_s16x2(d, ge, __vmins2(m, i_run) + go);
                i_run = __viaddmin_s16x2(i_run, gep, m + gop);
            }
            i_run = 0x70007000u;
        }
    }
    uint32_t s = i_run;
#pragma unroll
    for (int i = 0; i < CH; ++i) s ^= M[i] ^ D[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

int main()
{
    cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
    int clk_khz = 0; CK(cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0));
    const int sms = p.multiProcessorCount;
    printf("device %s, %d SMs, max clock %.0f MHz\n", p.name, sms, clk_khz / 1e3);
    uint32_t *in, *out; CK(cudaMalloc(&in, 4096)); CK(cudaMalloc(&out, (size_t)sms * 8 * 256 * 4));
    CK(cudaMemset(in, 0x11, 4096));
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    const char* names[] = {"VIMNMX.S16x2", "VIMNMX3.S16x2", "VIADDMNMX.S16x2", "PRMT", "IADD", "IMNMX.S32", "LDS.bcast+LOP", "IMAD"};
    const int iters = 2000;
    const int grid = sms * 8;
    for (int op = 0; op < 8; ++op) {
        float best = 1e30f;
        for (int rep = 0; rep < 4; ++rep) {
            CK(cudaEventRecord(e0));
            switch (op) {
                case 0: k_op<0><<<grid, 256>>>(out, in, iters); break;
                case 1: k_op<1><<<grid, 256>>>(out, in, iters); break;
                case 2: k_op<2><<<grid, 256>>>(out, in, iters); break;
                case 3: k_op<3><<<grid, 256>>>(out, in, iters); break;
                case 4: k_op<4><<<grid, 256>>>(out, in, iters); break;
                case 5: k_op<5><<<grid, 256>>>(out, in, iters); break;
                case 6: k_op<6><<<grid, 256>>>(out, in, iters); break;
                case 7: k_op<7><<<grid, 256>>>(out, in, iters); break;
            }
            CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
            float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (ms < best) best = ms;
        }
        const double ops = (double)grid * 256 * iters * UNR * CH;    // thread-level ops of the measured kind (loop overhead excluded)
        printf("%-16s %8.3f ms  %8.1f Gop/s  %6.1f thread-ops/clk/SM (at max clock)\n", names[op], best, ops / best / 1e6,
               ops / (best / 1e3) / (clk_khz * 1e3) / sms);
    }
    {
        float best = 1e30f;
        const int it2 = 8000;
        for (int rep = 0; rep < 4; ++rep) {
            CK(cudaEventRecord(e0));
            k_cell<<<grid, 256>>>(out, in, it2);
            CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
            float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (ms < best) best = ms;
        }
        const double cellpairs = (double)grid * 256 * it2 * 4 * CH;
        printf("%-16s %8.3f ms  %8.1f G cell-pairs/s = %8.1f GCUPS-equivalent  (%5.2f thread cell-pairs/clk/SM; 11 instr each)\n", "pair-HMM cell", best,
               cellpairs / best / 1e6, 2 * cellpairs / best / 1e6, cellpairs / (best / 1e3) / (clk_khz * 1e3) / sms);
    }
    return 0;
}
