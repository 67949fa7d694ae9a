// Does an ALU-pipe instruction issue faster when only part of the warp is active?
// One warp per block, one block per SM sub-partition-ish; a long chain of SHF/LOP3/IADD3 with ILP 2.
#include <cstdio>
#include <cuda_runtime.h>
__global__ void chain(unsigned *out, int iters, int active)
{
    const unsigned lane = threadIdx.x & 31;
    unsigned a = lane * 2654435761u + 1, b = a ^ 0x9e3779b9u, c = a + 7, d = b + 11;
    if ((int)lane < active) {
#pragma unroll 1
        for (int i = 0; i < iters; ++i) {
#pragma unroll
            for (int k = 0; k < 32; ++k) {
                a = __funnelshift_r(a, a, 7) ^ c;      // SHF + LOP3
                b = __funnelshift_r(b, b, 13) ^ d;
                c = c + a + 0x428a2f98u;               // IADD3
                d = d + b + 0x71374491u;
            }
        }
    }
    out[blockIdx.x * 32 + lane] = a ^ b ^ c ^ d;
}
int main()
{
    unsigned *out;
    cudaMalloc(&out, 4 * 32 * 1024);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    const int iters = 20000;
    for (int warps_per_sm : {1, 4, 8}) {
        for (int active : {32, 16, 8, 1}) {
            const int blocks = 132 * warps_per_sm;   // H100 SXM: 132 SMs
            chain<<<blocks, 32>>>(out, 100, active);
            cudaDeviceSynchronize();
            cudaEventRecord(e0);
            chain<<<blocks, 32>>>(out, iters, active);
            cudaEventRecord(e1);
            cudaEventSynchronize(e1);
            float ms; cudaEventElapsedTime(&ms, e0, e1);
            const double instr = (double)iters * 32 * 6;      // per warp: 2 SHF + 2 LOP3 + 2 IADD3 per k
            printf("blocks/SM=%d active_lanes=%2d  %.3f ms  -> %.2f cycles per warp-instruction (at 1.98 GHz)\n",
                   warps_per_sm, active, ms, ms * 1e-3 * 1.98e9 / instr);
        }
    }
    return 0;
}
