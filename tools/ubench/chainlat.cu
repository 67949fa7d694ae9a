// Single-warp latency / issue-rate probes that calibrate tools/sass_sched.py (cycles via clock64 inside
// the kernel, one warp per CTA, one CTA per sub-partition at most).
//   dependent chains:  SHF->SHF, IMAD->IMAD, SHF->IMAD->SHF (cross-pipe), IMAD.WIDE, IMAD.HI
//   independent x4:    IMAD with an immediate multiplier (is the imm form 1/cycle like FFMA-imm?),
//                      IMAD.WIDE, IMAD.HI   (are they full rate on the FMA pipe?)
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o chainlat chainlat.cu && ./chainlat
#include <cstdio>
#include <cuda_runtime.h>

template <int MODE>
__global__ void probe(unsigned long long *cycles, unsigned *sink, int iters, unsigned one, unsigned p19)
{
    unsigned a = threadIdx.x * 2654435761u + 1, b = a ^ 0x9e3779b9u, c = a + 7, d = b + 11;
    unsigned long long w = a;
    const long long t0 = clock64();
#pragma unroll 1
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int k = 0; k < 64; ++k) {
            if (MODE == 0) a = __funnelshift_r(a, a, 7);                                           // ALU -> ALU
            else if (MODE == 1) asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(a) : "r"(a), "r"(one), "r"(b));   // FMA -> FMA
            else if (MODE == 2) {                                                                  // ALU -> FMA -> ALU
                a = __funnelshift_r(a, a, 7);
                asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(a) : "r"(a), "r"(one), "r"(b));
            } else if (MODE == 3) {                                                                // IMAD.WIDE chain
                asm("mul.wide.u32 %0, %1, %2;" : "=l"(w) : "r"((unsigned)w), "r"(p19));
                w ^= w >> 32;
            } else if (MODE == 4) asm("mul.hi.u32 %0, %1, %2;" : "=r"(a) : "r"(a | 0x80000000u), "r"(p19));   // IMAD.HI chain
            else if (MODE == 5) {                                                                  // 4 independent IMAD imm
                a = a * 3u + b; b = b * 5u + c; c = c * 7u + d; d = d * 9u + a;
            } else if (MODE == 6) {                                                                // 4 independent IMAD.WIDE
                unsigned long long x, y, z, u;
                asm("mul.wide.u32 %0, %1, %2;" : "=l"(x) : "r"(a), "r"(p19));
                asm("mul.wide.u32 %0, %1, %2;" : "=l"(y) : "r"(b), "r"(p19));
                asm("mul.wide.u32 %0, %1, %2;" : "=l"(z) : "r"(c), "r"(p19));
                asm("mul.wide.u32 %0, %1, %2;" : "=l"(u) : "r"(d), "r"(p19));
                a ^= (unsigned)(x >> 32); b ^= (unsigned)(y >> 32); c ^= (unsigned)(z >> 32); d ^= (unsigned)(u >> 32);
            } else if (MODE == 7) {                                                                // 4 independent IMAD.HI
                unsigned x, y, z, u;
                asm("mul.hi.u32 %0, %1, %2;" : "=r"(x) : "r"(a), "r"(p19));
                asm("mul.hi.u32 %0, %1, %2;" : "=r"(y) : "r"(b), "r"(p19));
                asm("mul.hi.u32 %0, %1, %2;" : "=r"(z) : "r"(c), "r"(p19));
                asm("mul.hi.u32 %0, %1, %2;" : "=r"(u) : "r"(d), "r"(p19));
                a += x; b += y; c += z; d += u;
            } else if (MODE == 8) {                                                                // SHF -> LOP3 -> IADD3 (the short chain)
                const unsigned r = __funnelshift_r(a, a, 6), s = __funnelshift_r(a, a, 11), t = __funnelshift_r(a, a, 25);
                unsigned x;
                asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(x) : "r"(r), "r"(s), "r"(t));
                asm("{ .reg .u32 q; add.u32 q, %1, %2; add.u32 %0, q, %3; }" : "=r"(a) : "r"(x), "r"(b), "r"(c));
            } else if (MODE == 9) asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(a) : "r"(a), "r"(b), "r"(c));          // LOP3 -> LOP3
            else if (MODE == 10) asm("{ .reg .u32 q; add.u32 q, %1, %2; add.u32 %0, q, %3; }" : "=r"(a) : "r"(a), "r"(b), "r"(c));   // IADD3 -> IADD3
            else if (MODE == 11) {                                                                 // SHF -> LOP3 (per pair)
                a = __funnelshift_r(a, a, 7);
                asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(a) : "r"(a), "r"(b), "r"(c));
            } else if (MODE == 12) {                                                               // SHF -> IADD3 (per pair)
                a = __funnelshift_r(a, a, 7);
                asm("{ .reg .u32 q; add.u32 q, %1, %2; add.u32 %0, q, %3; }" : "=r"(a) : "r"(a), "r"(b), "r"(c));
            } else if (MODE == 13) {                                                               // LOP3 -> IADD3 (per pair)
                asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(a) : "r"(a), "r"(b), "r"(c));
                asm("{ .reg .u32 q; add.u32 q, %1, %2; add.u32 %0, q, %3; }" : "=r"(a) : "r"(a), "r"(b), "r"(d));
            } else if (MODE == 14) {                                                               // 3 SHF -> LOP3 (per step)
                const unsigned r = __funnelshift_r(a, a, 6), s = __funnelshift_r(a, a, 11), t = __funnelshift_r(a, a, 25);
                asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(a) : "r"(r), "r"(s), "r"(t));
            } else if (MODE == 15) {                                                               // 3 SHF -> LOP3 -> IMAD (per step)
                const unsigned r = __funnelshift_r(a, a, 6), s = __funnelshift_r(a, a, 11), t = __funnelshift_r(a, a, 25);
                unsigned x;
                asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(x) : "r"(r), "r"(s), "r"(t));
                asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(a) : "r"(x), "r"(one), "r"(b));
            } else if (MODE == 16) {                                                               // LOP3 -> IMAD (per pair)
                asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(a) : "r"(a), "r"(b), "r"(c));
                asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(a) : "r"(a), "r"(one), "r"(d));
            } else if (MODE == 17) {                                                               // ALU x2 + IMAD x2 interleaved, IMADs cross-dependent
                a = __funnelshift_r(a, a, 7);
                asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(b) : "r"(b), "r"(one), "r"(d));
                c = __funnelshift_r(c, c, 9);
                asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(d), "r"(one), "r"(b));
            } else if (MODE == 18) {                                                               // 4 independent chains, alternating pipes
                a = __funnelshift_r(a, a, 7);
                asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(b) : "r"(b), "r"(one), "r"(p19));
                c = __funnelshift_r(c, c, 9);
                asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(d), "r"(one), "r"(p19));
            }
        }
    }
    const long long t1 = clock64();
    if (threadIdx.x == 0) cycles[blockIdx.x] = (unsigned long long)(t1 - t0);
    sink[blockIdx.x * 32 + threadIdx.x] = a ^ b ^ c ^ d ^ (unsigned)w;
}

template <int MODE> void run(const char *name, double per, unsigned long long *cyc, unsigned *sink)
{
    const int iters = 2000;
    probe<MODE><<<1, 32>>>(cyc, sink, 10, 1u, 1u << 19);
    probe<MODE><<<1, 32>>>(cyc, sink, iters, 1u, 1u << 19);
    unsigned long long c = 0;
    cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
    printf("%-44s %.2f cycles per %s\n", name, (double)c / ((double)iters * 64.0) / per, per == 1.0 ? "step" : "instruction");
}

int main()
{
    unsigned long long *cyc; unsigned *sink;
    cudaMalloc(&cyc, 8 * 64); cudaMalloc(&sink, 4 * 32 * 64);
    run<0>("SHF -> SHF (dependent)", 1, cyc, sink);
    run<1>("IMAD -> IMAD (dependent)", 1, cyc, sink);
    run<2>("SHF -> IMAD -> SHF (per pair)", 1, cyc, sink);
    run<3>("IMAD.WIDE -> LOP3 -> IMAD.WIDE (per pair)", 1, cyc, sink);
    run<4>("LOP3 -> IMAD.HI (per pair)", 1, cyc, sink);
    run<5>("4 x IMAD, immediate multiplier", 4, cyc, sink);
    run<6>("4 x IMAD.WIDE (+ 4 LOP3)", 4, cyc, sink);
    run<7>("4 x IMAD.HI (+ 4 IADD)", 4, cyc, sink);
    run<8>("3 SHF -> LOP3 -> IADD3 (short chain step)", 1, cyc, sink);
    run<9>("LOP3 -> LOP3 (dependent)", 1, cyc, sink);
    run<10>("IADD3 -> IADD3 (dependent)", 1, cyc, sink);
    run<11>("SHF -> LOP3 (per pair)", 1, cyc, sink);
    run<12>("SHF -> IADD3 (per pair)", 1, cyc, sink);
    run<13>("LOP3 -> IADD3 (per pair)", 1, cyc, sink);
    run<14>("3 SHF -> LOP3 (per step)", 1, cyc, sink);
    run<15>("3 SHF -> LOP3 -> IMAD (per step)", 1, cyc, sink);
    run<16>("LOP3 -> IMAD (per pair)", 1, cyc, sink);
    run<17>("SHF, IMAD, SHF, IMAD (IMADs cross-dependent)", 4, cyc, sink);
    run<18>("SHF, IMAD, SHF, IMAD (4 independent chains)", 4, cyc, sink);
    return cudaDeviceSynchronize() == cudaSuccess ? 0 : 1;
}
