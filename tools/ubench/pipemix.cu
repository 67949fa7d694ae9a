// Single-warp issue cost of ALU-pipe vs FMA-pipe integer instructions, alone and mixed (ILP 2-4).
#include <cstdio>
#include <cuda_runtime.h>
template <int MODE>
__global__ void chain(unsigned *out, int iters, unsigned one)
{
    const unsigned lane = threadIdx.x & 31;
    unsigned a = lane * 2654435761u + 1, b = a ^ 0x9e3779b9u, c = a + 7, d = b + 11;
#pragma unroll 1
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int k = 0; k < 32; ++k) {
            if (MODE == 0) {            // 4 ALU: 2 SHF+LOP3... (SHF, SHF, LOP3, LOP3)
                a = __funnelshift_r(a, a, 7); b = __funnelshift_r(b, b, 13); c ^= a; d ^= b;
            } else if (MODE == 1) {     // 4 FMA-pipe IMAD (runtime multiplier so it stays IMAD)
                asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(a) : "r"(a), "r"(one), "r"(c));
                asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(b) : "r"(b), "r"(one), "r"(d));
                asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(c) : "r"(c), "r"(one), "r"(a));
                asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(d), "r"(one), "r"(b));
            } else if (MODE == 2) {     // 2 ALU + 2 IMAD, independent pairs
                a = __funnelshift_r(a, a, 7); b = __funnelshift_r(b, b, 13);
                asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(c) : "r"(c), "r"(one), "r"(a));
                asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(d), "r"(one), "r"(b));
            } else {                    // 3 ALU + 1 IMAD
                a = __funnelshift_r(a, a, 7); b = __funnelshift_r(b, b, 13); c ^= a;
                asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(d), "r"(one), "r"(b));
            }
        }
    }
    out[blockIdx.x * 32 + lane] = a ^ b ^ c ^ d;
}
template <int MODE> void run(const char *name, unsigned *out)
{
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    const int iters = 20000;
    for (int wps : {1, 2, 4}) {                 // warps per sub-partition (4 sub-partitions per SM)
        const int blocks = 132 * 4 * wps;        // H100 SXM: 132 SMs
        chain<MODE><<<blocks, 32>>>(out, 100, 1u);
        cudaDeviceSynchronize();
        cudaEventRecord(e0);
        chain<MODE><<<blocks, 32>>>(out, iters, 1u);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        printf("%-22s warps/sub-partition=%d  %.2f cycles per 4-instruction group per warp\n", name, wps,
               ms * 1e-3 * 1.98e9 / ((double)iters * 32));
    }
}
int main()
{
    unsigned *out;
    cudaMalloc(&out, 4 * 32 * 132 * 16);
    run<0>("4 ALU (SHF,SHF,LOP3,LOP3)", out);
    run<1>("4 IMAD", out);
    run<2>("2 ALU + 2 IMAD", out);
    run<3>("3 ALU + 1 IMAD", out);
    return 0;
}
