// Multi-buffer SHA-256 for sm_90a (H100): the hot path of the blob hash-and-cache
// engine.  Pure 32-bit integer work (SHF / LOP3 / IADD3 / IMAD) — no tensor
// cores, no floating point.  Two kernels share the round function; the
// engine picks a shape per launch from the number of co-resident streams
// (streams_per_warp_for, kernel_shape):
//
//   sha256_wide_kernel   one 32-bit lane per live stream (the multi-buffer
//                        form north_star describes): W[16] and the eight
//                        state words live in registers, each lane pulls one
//                        whole 128-byte line (two blocks) per iteration.  The
//                        shipped variant rolls the rounds 16 at a time (round
//                        constants from the constant bank; the fully unrolled
//                        form stalled on the instruction cache), issues the
//                        additions on the FMA pipe and loads each line into
//                        registers (style 2; style 5 stages it in shared memory
//                        with cp.async, slower on H100).  Bound by the ALU
//                        pipe (one warp-instruction per 2 cycles per
//                        sub-partition): <= ~1.0 TB/s on 132 SMs at 1.98 GHz;
//                        needs > ~10^4 streams to fill the chip.
//   sha256_warp_kernel   S = 1/2/4/8/16 streams per warp, for fewer live
//                        streams.  SHA-256's serial chain is only the 64
//                        rounds; the message schedule is state-independent.
//                        The 32 lanes expand the schedules of 32 blocks in
//                        parallel (lane = block_slot * S + stream, coalesced
//                        loads) and stage W[t]+K[t] in shared memory; then the
//                        warp runs 32/S block-steps of 64 dependent rounds, S
//                        round chains per instruction, reading one broadcast
//                        LDS.128 per 4 rounds.  As a warp pair, a second warp
//                        does the loads and schedules one group ahead.
//
// All optionally write every byte they read to `dst` (the blob's CAS
// extent), so hash-and-cache moves 1 B read + 1 B written per blob byte;
// all pad the final block on the device (FIPS 180-4 §5.1.1).
//
// The digest definition is FIPS 180-4 (what Go crypto/sha256 implements —
// the reference names it in BASELINE.json north_star but holds no call site:
// the reference's cmd/demodel/start.go:201-204 returns resp unchanged).
#include "sha256_kernels.cuh"
#include "blobgen.h"
#include "sha256_round.cuh"

namespace dm {
namespace {

template <int kFma, int t0>
__device__ __forceinline__ void sha_rounds4(uint32_t (&v)[8], const uint4 &k4, const FmaK &k)
{
    sha_round<kFma, t0>(v, k4.x, k);
    sha_round<kFma, t0 + 1>(v, k4.y, k);
    sha_round<kFma, t0 + 2>(v, k4.z, k);
    sha_round<kFma, t0 + 3>(v, k4.w, k);
}

template <int kFma, int t>
struct RoundsFrom {   // compile-time unrolled t..63, W in registers, K as immediates
    static __device__ __forceinline__ void run(uint32_t (&v)[8], uint32_t (&w)[16], const FmaK &k)
    {
        constexpr uint32_t K[64] = {DM_K256_TABLE};
        if constexpr (t >= 16) {
            const uint32_t s = addf<kFma>(addf<kFma>(small_sigma1(w[(t - 2) & 15]), w[(t - 7) & 15], k),
                                          small_sigma0(w[(t - 15) & 15]), k);
            w[t & 15] = addf<kFma>(w[t & 15], s, k);
        }
        sha_round<kFma, t>(v, addf<kFma>(w[t & 15], K[t], k), k);
        if constexpr (t < 63) RoundsFrom<kFma, t + 1>::run(v, w, k);
    }
};

// Whole-block compression with everything in registers.  w[] holds the 16
// big-endian message words and is clobbered (rolling 16-word schedule).
template <int kFma>
__device__ __forceinline__ void compress_regs(uint32_t (&s)[8], uint32_t (&w)[16], const FmaK &k)
{
    uint32_t v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = s[i];
    RoundsFrom<kFma, 0>::run(v, w, k);
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i] += v[i];
}

// Round constants for the rolled form below (uniform index -> constant-bank operand).
__constant__ uint32_t c_K256[64] = {DM_K256_TABLE};

template <int kFma, int j>
struct Rounds16 {   // 16 rounds starting at a multiple of 16 (t0 >= 16: with message schedule)
    template <bool kSched>
    static __device__ __forceinline__ void run(uint32_t (&v)[8], uint32_t (&w)[16], int t0, const FmaK &k)
    {
        if constexpr (kSched) {
            const uint32_t s = addf<kFma>(addf<kFma>(small_sigma1(w[(j - 2) & 15]), w[(j - 7) & 15], k),
                                          small_sigma0(w[(j - 15) & 15]), k);
            w[j] = addf<kFma>(w[j], s, k);
        }
        sha_round<kFma, j>(v, addf<kFma>(w[j], c_K256[t0 + j], k), k);
        if constexpr (j < 15) Rounds16<kFma, j + 1>::template run<kSched>(v, w, t0, k);
    }
};

// Same function as compress_regs with the rounds rolled 16 at a time: ~6 KB
// of code instead of ~22 KB, so two of them plus the loads stay resident in
// the instruction cache (ncu on the fully unrolled form: `no_instruction`
// was the second-largest stall after the ALU pipe itself).
template <int kFma>
__device__ __forceinline__ void compress_rolled(uint32_t (&s)[8], uint32_t (&w)[16], const FmaK &k)
{
    uint32_t v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = s[i];
    Rounds16<kFma, 0>::template run<false>(v, w, 0, k);
#pragma unroll 1
    for (int t0 = 16; t0 < 64; t0 += 16) Rounds16<kFma, 0>::template run<true>(v, w, t0, k);
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i] += v[i];
}

__device__ __forceinline__ void unpack_be(uint32_t (&w)[16], const uint4 &a, const uint4 &b,
                                          const uint4 &c, const uint4 &d)
{
    w[0] = bswap32(a.x);  w[1] = bswap32(a.y);  w[2] = bswap32(a.z);  w[3] = bswap32(a.w);
    w[4] = bswap32(b.x);  w[5] = bswap32(b.y);  w[6] = bswap32(b.z);  w[7] = bswap32(b.w);
    w[8] = bswap32(c.x);  w[9] = bswap32(c.y);  w[10] = bswap32(c.z); w[11] = bswap32(c.w);
    w[12] = bswap32(d.x); w[13] = bswap32(d.y); w[14] = bswap32(d.z); w[15] = bswap32(d.w);
}

// Blob bytes are read exactly once: bypass L1 allocation, keep L2 default.
__device__ __forceinline__ uint4 ld_stream(const uint4 *p)
{
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ void st_stream(uint4 *p, const uint4 &v)
{
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// The last < 128 bytes of a run, as up to three "virtual" blocks: whole
// blocks, then (FINAL only) the FIPS 180-4 §5.1.1 padding — a 0x80 byte
// right after the message, zeros, and the 64-bit big-endian bit length in
// the last two words of the last block.  Loads touch only 16-byte pieces
// that hold at least one message byte.
template <int kFma>
__device__ __forceinline__ void hash_tail(uint32_t (&s)[8], const uint8_t *src, uint8_t *dst,
                                          uint32_t rem, bool final, uint64_t total_len, bool do_store,
                                          const FmaK &k)
{
    const uint32_t nvb = final ? ((rem + 72u) >> 6) : (rem >> 6);
    const uint64_t bits = total_len << 3;
#pragma unroll 1
    for (uint32_t vb = 0; vb < nvb; ++vb) {
        const uint32_t base = vb << 6;
        uint32_t w[16];
        uint4 q[4];
#pragma unroll
        for (int g = 0; g < 4; ++g) {
            q[g] = make_uint4(0u, 0u, 0u, 0u);
            if (base + 16u * g < rem) {
                q[g] = ld_stream(reinterpret_cast<const uint4 *>(src + base) + g);
                if (dst != nullptr && do_store) st_stream(reinterpret_cast<uint4 *>(dst + base) + g, q[g]);
            }
        }
        unpack_be(w, q[0], q[1], q[2], q[3]);
        if (final) {
#pragma unroll
            for (int t = 0; t < 16; ++t) {
                const int left = (int)rem - (int)(base + 4u * t);   // message bytes from this word on
                if (left <= 0) w[t] = 0u;
                else if (left < 4) w[t] &= 0xFFFFFFFFu << (32 - 8 * left);
                if (left >= 0 && left < 4) w[t] |= 0x80u << (24 - 8 * left);
            }
            if (vb == nvb - 1) { w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits; }
        }
        compress_rolled<kFma>(s, w, k);
    }
}

__device__ __forceinline__ void load_state(uint32_t (&s)[8], const uint32_t *states, uint32_t slot, uint32_t flags)
{
    if (flags & JOB_INIT) {   // FIPS 180-4 §5.3.3
        s[0] = 0x6a09e667u; s[1] = 0xbb67ae85u; s[2] = 0x3c6ef372u; s[3] = 0xa54ff53au;
        s[4] = 0x510e527fu; s[5] = 0x9b05688cu; s[6] = 0x1f83d9abu; s[7] = 0x5be0cd19u;
    } else {
        const uint4 lo = *reinterpret_cast<const uint4 *>(states + 8ull * slot);
        const uint4 hi = *reinterpret_cast<const uint4 *>(states + 8ull * slot + 4);
        s[0] = lo.x; s[1] = lo.y; s[2] = lo.z; s[3] = lo.w;
        s[4] = hi.x; s[5] = hi.y; s[6] = hi.z; s[7] = hi.w;
    }
}

__device__ __forceinline__ void store_state(const uint32_t (&s)[8], uint32_t *states, uint32_t *digests,
                                            uint32_t slot, uint32_t flags)
{
    const uint4 lo = make_uint4(s[0], s[1], s[2], s[3]);
    const uint4 hi = make_uint4(s[4], s[5], s[6], s[7]);
    *reinterpret_cast<uint4 *>(states + 8ull * slot) = lo;
    *reinterpret_cast<uint4 *>(states + 8ull * slot + 4) = hi;
    if (flags & JOB_FINAL) {
        *reinterpret_cast<uint4 *>(digests + 8ull * slot) = lo;
        *reinterpret_cast<uint4 *>(digests + 8ull * slot + 4) = hi;
    }
}

__device__ __forceinline__ HashJob load_job(const HashJob *jobs, uint32_t j)
{
    const uint4 *p = reinterpret_cast<const uint4 *>(jobs + j);
    const uint4 a = __ldg(p), b = __ldg(p + 1);
    HashJob jb;
    jb.src = reinterpret_cast<const uint8_t *>(((uint64_t)a.y << 32) | a.x);
    jb.dst = reinterpret_cast<uint8_t *>(((uint64_t)a.w << 32) | a.z);
    jb.nbytes = ((uint64_t)b.y << 32) | b.x;
    jb.total_len = ((uint64_t)b.w << 32) | b.z;
    const uint4 c = __ldg(p + 2);
    jb.slot = c.x; jb.flags = c.y; jb.one = c.z; jb.pad_ = 0;
    return jb;
}

// ---------------------------------------------------------------------------
// wide: one lane per stream
// ---------------------------------------------------------------------------
constexpr int kWideThreads = 128;

// kStyle selects the shape of the main loop (all bit-identical):
//   0  one 128-byte line (two blocks) per iteration, rounds fully unrolled  (~44 KB of code)
//   1  one 64-byte block per iteration, rounds fully unrolled               (~22 KB)
//   2  one 128-byte line per iteration, rounds rolled 16 at a time          (~20 KB)
//   3  one 64-byte block per iteration, rolled                              (~10 KB)
//   4  as 2, with the loads software-pipelined half a line ahead
//   5  as 2, with every lane's next 128-byte line fetched by cp.async into its own row of shared memory (two
//      stages) while the current line is hashed: the line load leaves the register file and its ~600-cycle
//      latency off the scoreboard (ncu on style 2: long_scoreboard 0.53 per issue on the first use of the line)
constexpr int kWideRow = 144;                 // bytes per lane row in shared memory: 128 + 16 pad -> conflict-free LDS.128
template <int kFma, int kStyle>
__global__ void __launch_bounds__(kWideThreads, kStyle == 4 ? 5 : 1)
sha256_wide_kernel(const HashJob *__restrict__ jobs, uint32_t njobs, uint32_t *__restrict__ states,
                   uint32_t *__restrict__ digests, FmaK k)
{
    const uint32_t j = blockIdx.x * kWideThreads + threadIdx.x;
    if (j >= njobs) return;
    const HashJob jb = load_job(jobs, j);
    uint32_t s[8];
    load_state(s, states, jb.slot, jb.flags);

    if constexpr (kFma == 2) k.one = jb.one;        // register operand instead of c[0][..]
    const uint4 *p = reinterpret_cast<const uint4 *>(jb.src);
    uint4 *q = reinterpret_cast<uint4 *>(jb.dst);
    const bool copy = q != nullptr;
    uint32_t rem;
    if constexpr (kStyle == 5) {
        __shared__ __align__(16) uint8_t rows[2][kWideThreads * kWideRow];
        const uint32_t my = threadIdx.x * kWideRow;
        auto fetch = [&](int stage, const uint4 *from) {      // this lane's next line -> its row of `stage`, asynchronously
            const uint32_t dst = (uint32_t)__cvta_generic_to_shared(&rows[stage][my]);
#pragma unroll
            for (int i = 0; i < 8; ++i)
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(dst + 16u * i), "l"(from + i) : "memory");
            asm volatile("cp.async.commit_group;" ::: "memory");
        };
        uint64_t npair = jb.nbytes >> 7;
        if (npair) fetch(0, p);
        int stage = 0;
#pragma unroll 1
        for (; npair != 0; --npair) {
            if (npair > 1) { fetch(stage ^ 1, p + 8); asm volatile("cp.async.wait_group 1;" ::: "memory"); }
            else asm volatile("cp.async.wait_group 0;" ::: "memory");
            const uint4 *row = reinterpret_cast<const uint4 *>(&rows[stage][my]);     // only this lane ever touches its row
            uint32_t w[16];
            {
                const uint4 a = row[0], b = row[1], c = row[2], d = row[3];
                if (copy) { st_stream(q, a); st_stream(q + 1, b); st_stream(q + 2, c); st_stream(q + 3, d); }
                unpack_be(w, a, b, c, d);
            }
            compress_rolled<kFma>(s, w, k);
            {
                const uint4 a = row[4], b = row[5], c = row[6], d = row[7];
                if (copy) { st_stream(q + 4, a); st_stream(q + 5, b); st_stream(q + 6, c); st_stream(q + 7, d); q += 8; }
                unpack_be(w, a, b, c, d);
            }
            compress_rolled<kFma>(s, w, k);
            // (running the two blocks through ONE copy of the compression code - half the loop body, 78 registers - was
            //  measured too: 17.12 ms against 17.05 ms, no gain)
            p += 8;
            stage ^= 1;
        }
        rem = (uint32_t)(jb.nbytes & 127u);
    } else if constexpr (kStyle == 4) {
        // rolled rounds, loads software-pipelined half a line ahead: the second half of the
        // current line and the first half of the next one are in flight during a compression
        uint64_t npair = jb.nbytes >> 7;
        uint4 x[8];
        if (npair) {
#pragma unroll
            for (int i = 0; i < 4; ++i) x[i] = ld_stream(p + i);
        }
#pragma unroll 1
        for (; npair != 0; --npair) {
#pragma unroll
            for (int i = 4; i < 8; ++i) x[i] = ld_stream(p + i);
            if (copy) {
#pragma unroll
                for (int i = 0; i < 4; ++i) st_stream(q + i, x[i]);
            }
            uint32_t w[16];
            unpack_be(w, x[0], x[1], x[2], x[3]);
            p += 8;
            if (npair > 1) {
#pragma unroll
                for (int i = 0; i < 4; ++i) x[i] = ld_stream(p + i);
            }
            compress_rolled<kFma>(s, w, k);
            if (copy) {
#pragma unroll
                for (int i = 4; i < 8; ++i) st_stream(q + i, x[i]);
                q += 8;
            }
            unpack_be(w, x[4], x[5], x[6], x[7]);
            compress_rolled<kFma>(s, w, k);
        }
        rem = (uint32_t)(jb.nbytes & 127u);
    } else if constexpr (kStyle == 0 || kStyle == 2) {
        uint64_t npair = jb.nbytes >> 7;               // 128-byte lines
#pragma unroll 1
        for (; npair != 0; --npair) {
            uint4 x[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) x[i] = ld_stream(p + i);
            if (copy) {
#pragma unroll
                for (int i = 0; i < 8; ++i) st_stream(q + i, x[i]);
                q += 8;
            }
            p += 8;
            uint32_t w[16];
            unpack_be(w, x[0], x[1], x[2], x[3]);
            if constexpr (kStyle == 0) compress_regs<kFma>(s, w, k); else compress_rolled<kFma>(s, w, k);
            unpack_be(w, x[4], x[5], x[6], x[7]);
            if constexpr (kStyle == 0) compress_regs<kFma>(s, w, k); else compress_rolled<kFma>(s, w, k);
        }
        rem = (uint32_t)(jb.nbytes & 127u);
    } else {
        uint64_t nblk = jb.nbytes >> 6;
#pragma unroll 1
        for (; nblk != 0; --nblk) {
            uint4 x[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) x[i] = ld_stream(p + i);
            if (copy) {
#pragma unroll
                for (int i = 0; i < 4; ++i) st_stream(q + i, x[i]);
                q += 4;
            }
            p += 4;
            uint32_t w[16];
            unpack_be(w, x[0], x[1], x[2], x[3]);
            if constexpr (kStyle == 1) compress_regs<kFma>(s, w, k); else compress_rolled<kFma>(s, w, k);
        }
        rem = (uint32_t)(jb.nbytes & 63u);
    }
    hash_tail<kFma>(s, reinterpret_cast<const uint8_t *>(p), reinterpret_cast<uint8_t *>(q), rem,
                    (jb.flags & JOB_FINAL) != 0, jb.total_len, true, k);
    store_state(s, states, digests, jb.slot, jb.flags);
}

// ---------------------------------------------------------------------------
// warp: S = 1, 2, 4, 8 or 16 streams per warp, optionally as a warp pair
// ---------------------------------------------------------------------------
// Two phases per group of 32 blocks.  Phase 1: the warp's 32 lanes, lane = b * S + j (stream j, block slot b, B = 32 / S
// blocks per stream), each load one block, write its CAS copy and stage that block's 64-entry schedule, K folded in, as
// a row of shared memory.  Phase 2: B dependent block-steps of 64 rounds, every lane following stream j and reading one
// broadcast LDS.128 per 4 rounds, so S round chains advance per instruction.  Lanes with the same j compute identical
// values (no divergence); a row read is S distinct 16-byte words per LDS.128 (conflict-free for S <= 8, two-way for
// S = 16).  Streams in a warp may differ in length: a lane stops updating its state when its stream has no block in
// a step.  S = 1 (one warp per stream) is ~1.9x the per-stream rate of the lane-per-stream form.
constexpr int kKwStride = 68;                 // words per staged block: 64 + 4 pad -> conflict-free STS.128
constexpr int kWarpsPerCta = 1;               // one-warp form; 1 lets the block scheduler spread few streams over
                                              // all 528 sub-partitions

// One lane expands the 64-entry schedule of its block and stages W[t] + K[t] as 16 uint4 (FIPS 180-4 §6.2.2 step 1,
// K folded in).  Additions are left to ptxas: forcing them onto the FMA pipe lengthens the w[t-2] -> w[t] chain and
// the timing model shows no gain.
__device__ __forceinline__ void expand_schedule(uint32_t (&w)[16], uint4 *out)
{
    constexpr uint32_t K[64] = {DM_K256_TABLE};
#pragma unroll
    for (int t = 0; t < 16; t += 4)
        out[t >> 2] = make_uint4(w[t] + K[t], w[t + 1] + K[t + 1], w[t + 2] + K[t + 2], w[t + 3] + K[t + 3]);
#pragma unroll
    for (int t = 16; t < 64; t += 4) {
#pragma unroll
        for (int u = t; u < t + 4; ++u)
            w[u & 15] += small_sigma1(w[(u - 2) & 15]) + w[(u - 7) & 15] + small_sigma0(w[(u - 15) & 15]);
        out[t >> 2] = make_uint4(w[t & 15] + K[t], w[(t + 1) & 15] + K[t + 1],
                                 w[(t + 2) & 15] + K[t + 2], w[(t + 3) & 15] + K[t + 3]);
    }
}

// Phase 1 of group g for one lane (block slot b = lane / S): if its stream has that block (held in x), copy it out and
// stage its schedule in `row`; then load the lane's block of the next group.  kSync: this warp reads the rows itself,
// so they are published (__syncwarp) first.  The order of the steps and the 32-bit in-group tests at S = 1 are what
// ptxas schedules the rounds best after (tools/sass_sched.py); at S > 1 a stream may have run out before group g.
template <int S, bool kSync>
__device__ __forceinline__ void stage_block(uint4 (&x)[4], const uint4 *&p, uint4 *&q, bool copy, uint32_t lane,
                                            uint64_t g, uint64_t ngroups, uint64_t nblk, uint4 *row)
{
    constexpr uint32_t B = 32 / S;
    const uint32_t b = lane / S;
    const uint64_t blk0 = g * B, left = nblk - blk0;
    if (S == 1 ? lane < (left < 32 ? (uint32_t)left : 32u) : blk0 + b < nblk) {
        if (copy) {
#pragma unroll
            for (int i = 0; i < 4; ++i) st_stream(q + i, x[i]);
        }
        uint32_t w[16];
        unpack_be(w, x[0], x[1], x[2], x[3]);
        expand_schedule(w, row);
    }
    if constexpr (kSync) __syncwarp();
    p += 4 * B; q += 4 * B;
    if (S == 1 ? g + 1 < ngroups && lane < left - 32 : blk0 + B + b < nblk) {
#pragma unroll
        for (int i = 0; i < 4; ++i) x[i] = ld_stream(p + i);
    }
}

// Phase 2, one block-step: the 64 dependent rounds on one staged row, then the feed-forward, kept only where the
// lane's stream has a block in this step (`valid`, always true for one stream per warp).
template <int kFma>
__device__ __forceinline__ void block_step(uint32_t (&s)[8], const uint4 *kp, bool valid, const FmaK &k)
{
    uint32_t v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = s[i];
    sha_rounds4<kFma, 0>(v, kp[0], k);   sha_rounds4<kFma, 4>(v, kp[1], k);
    sha_rounds4<kFma, 8>(v, kp[2], k);   sha_rounds4<kFma, 12>(v, kp[3], k);
    sha_rounds4<kFma, 16>(v, kp[4], k);  sha_rounds4<kFma, 20>(v, kp[5], k);
    sha_rounds4<kFma, 24>(v, kp[6], k);  sha_rounds4<kFma, 28>(v, kp[7], k);
    sha_rounds4<kFma, 32>(v, kp[8], k);  sha_rounds4<kFma, 36>(v, kp[9], k);
    sha_rounds4<kFma, 40>(v, kp[10], k); sha_rounds4<kFma, 44>(v, kp[11], k);
    sha_rounds4<kFma, 48>(v, kp[12], k); sha_rounds4<kFma, 52>(v, kp[13], k);
    sha_rounds4<kFma, 56>(v, kp[14], k); sha_rounds4<kFma, 60>(v, kp[15], k);
    if (valid) {
#pragma unroll
        for (int i = 0; i < 8; ++i) s[i] += v[i];
    }
}

// kPair: two warps per group of S streams, for launches where every group can have two sub-partitions.  The serial
// chain stays on one warp (warp 0), but everything else leaves it: warp 1 loads the next group's blocks, stores the
// fused CAS copy and expands the schedules into the other half of a double-buffered stage while warp 0 still runs the
// rounds of the current group.  Hand-over by named barriers (FULL / EMPTY per buffer: one side arrives, the other
// waits); the round warp never touches global memory inside the loop.  What it buys is phase 1's share of the
// one-warp form: ~1 cycle per round of 25.9 at S = 1, but per group of 32 blocks phase 1 costs ~1500 cycles against
// (32 / S) x ~1600 for the rounds - 19 % of the time at S = 8, 32 % at S = 16.
// (barrier ids as immediates: with a register id ptxas reserves all 16 named barriers for the CTA, and the SM's
//  barrier pool then limits how many CTAs can be resident)
template <int kId> __device__ __forceinline__ void named_bar_sync() { asm volatile("barrier.sync %0, 64;" :: "n"(kId) : "memory"); }
template <int kId> __device__ __forceinline__ void named_bar_arrive() { asm volatile("barrier.arrive %0, 64;" :: "n"(kId) : "memory"); }
__device__ __forceinline__ void full_sync(uint32_t b) { if (b) named_bar_sync<2>(); else named_bar_sync<1>(); }
__device__ __forceinline__ void full_arrive(uint32_t b) { if (b) named_bar_arrive<2>(); else named_bar_arrive<1>(); }
__device__ __forceinline__ void empty_sync(uint32_t b) { if (b) named_bar_sync<4>(); else named_bar_sync<3>(); }
__device__ __forceinline__ void empty_arrive(uint32_t b) { if (b) named_bar_arrive<4>(); else named_bar_arrive<3>(); }

template <int kFma, int S, bool kPair>
__global__ void __launch_bounds__(kPair ? 64 : 32 * kWarpsPerCta)
sha256_warp_kernel(const HashJob *__restrict__ jobs, uint32_t njobs, uint32_t *__restrict__ states,
                   uint32_t *__restrict__ digests, FmaK k)
{
    constexpr uint32_t B = 32 / S;
    __shared__ __align__(16) uint32_t kw_smem[kPair ? 2 : kWarpsPerCta][32 * kKwStride];   // pairs: double-buffered
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t warp = threadIdx.x >> 5;                     // pairs: 0 = rounds, 1 = loads + schedules
    const uint32_t j = lane % S, b = lane / S;
    const uint32_t job = (kPair ? blockIdx.x : blockIdx.x * kWarpsPerCta + warp) * S + j;
    const bool live = job < njobs;
    if constexpr (S == 1) {
        if (!live) return;
    }
    HashJob jb;
    if (live) jb = load_job(jobs, job);
    else { jb.src = nullptr; jb.dst = nullptr; jb.nbytes = 0; jb.total_len = 0; jb.slot = 0; jb.flags = JOB_INIT; jb.one = 1; jb.pad_ = 0; }
    const uint64_t nblk = jb.nbytes >> 6;                       // this lane's stream
    uint64_t ngroups = (nblk + B - 1) / B;
    if constexpr (S > 1) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {                      // warp-wide max: everyone loops together
            const uint64_t other = __shfl_xor_sync(0xffffffffu, ngroups, o);
            ngroups = other > ngroups ? other : ngroups;
        }
    }
    const bool copy = jb.dst != nullptr;
    const uint4 *p = reinterpret_cast<const uint4 *>(jb.src) + 4ull * b;   // block b of group 0
    uint4 *q = reinterpret_cast<uint4 *>(jb.dst) + 4ull * b;
    uint4 x[4];

    if constexpr (kPair) {
        if (warp == 1) {
            if (b < nblk) {
#pragma unroll
                for (int i = 0; i < 4; ++i) x[i] = ld_stream(p + i);
            }
#pragma unroll 1
            for (uint64_t g = 0; g < ngroups; ++g) {
                const uint32_t buf = (uint32_t)g & 1u;
                empty_sync(buf);                                // the round warp is done with this buffer
                stage_block<S, false>(x, p, q, copy, lane, g, ngroups, nblk,
                                      reinterpret_cast<uint4 *>(kw_smem[buf] + lane * kKwStride));
                __threadfence_block();                          // the stage is written before it is announced
                full_arrive(buf);
            }
            return;
        }
    }

    if constexpr (kFma == 2) k.one = jb.one;
    uint32_t s[8];
    load_state(s, states, jb.slot, jb.flags);
    if constexpr (kPair) {
        empty_arrive(0);                                        // both buffers start empty
        empty_arrive(1);
    } else if (b < nblk) {
#pragma unroll
        for (int i = 0; i < 4; ++i) x[i] = ld_stream(p + i);
    }
#pragma unroll 1
    for (uint64_t g = 0; g < ngroups; ++g) {
        const uint64_t blk0 = g * B;
        const uint32_t buf = (uint32_t)g & 1u;
        if constexpr (kPair) {
            full_sync(buf);
        } else {
            // the next group's block is loaded while the serial rounds run
            stage_block<S, true>(x, p, q, copy, lane, g, ngroups, nblk,
                                 reinterpret_cast<uint4 *>(kw_smem[warp] + lane * kKwStride));
        }
        const uint32_t *kw = kw_smem[kPair ? buf : warp];
        if constexpr (S == 1) {
            const uint64_t left = nblk - blk0;
            const uint32_t nv = left < 32 ? (uint32_t)left : 32u;
#pragma unroll 1
            for (uint32_t st = 0; st < nv; ++st) block_step<kFma>(s, reinterpret_cast<const uint4 *>(kw + st * kKwStride), true, k);
        } else {
#pragma unroll 1
            for (uint32_t st = 0; st < B; ++st) {              // row = step * S + j
                const bool valid = blk0 + st < nblk;
                if (__ballot_sync(0xffffffffu, valid) == 0u) break;          // no stream has this step
                block_step<kFma>(s, reinterpret_cast<const uint4 *>(kw + (st * S + j) * kKwStride), valid, k);
            }
        }
        if constexpr (kPair) {
            if (g + 2 < ngroups) empty_arrive(buf);             // (nobody waits for the last two)
        } else {
            __syncwarp();
        }
    }
    if (live) {
        const uint64_t done = nblk << 6;
        hash_tail<kFma>(s, jb.src + done, copy ? jb.dst + done : nullptr, (uint32_t)(jb.nbytes & 63u),
                        (jb.flags & JOB_FINAL) != 0, jb.total_len, b == 0, k);
        if (b == 0) store_state(s, states, digests, jb.slot, jb.flags);
    }
}

// ---------------------------------------------------------------------------
// synthetic blob bytes
// ---------------------------------------------------------------------------
__global__ void synth_fill_kernel(uint64_t key, uint64_t byte_off, uint8_t *dst, size_t len)
{
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    // fast path: generator words (8 B) and 16-byte stores line up
    const bool fast = ((byte_off & 7) == 0) && (((uintptr_t)dst & 15) == 0);
    const size_t nvec = fast ? (len >> 4) : 0;
    const uint64_t w0 = byte_off >> 3;
    ulonglong2 *v = reinterpret_cast<ulonglong2 *>(dst);
    for (size_t i = tid; i < nvec; i += stride)
        v[i] = make_ulonglong2(dm_blob_word_k(key, w0 + 2 * i), dm_blob_word_k(key, w0 + 2 * i + 1));
    for (size_t i = (nvec << 4) + tid; i < len; i += stride) {
        const uint64_t jx = byte_off + i;
        dst[i] = (uint8_t)(dm_blob_word_k(key, jx >> 3) >> (8 * (jx & 7)));
    }
}

// n blobs at ascending 16-byte-aligned offsets[] with lengths[]: one 16-byte
// piece per thread iteration over the whole span, owner found by binary search.
__global__ void synth_fill_many_kernel(uint64_t seed, uint64_t first_blob, uint8_t *base,
                                       const uint64_t *__restrict__ offsets,
                                       const uint64_t *__restrict__ lengths, uint32_t n,
                                       uint64_t first_off, uint64_t span)
{
    const uint64_t nvec = (span + 15) >> 4;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec;
         i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t pos = first_off + (i << 4);
        uint32_t lo = 0, hi = n;                       // offsets[lo] <= pos < offsets[hi]
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (offsets[mid] <= pos) lo = mid; else hi = mid;
        }
        const uint64_t in = pos - offsets[lo], len = lengths[lo];
        if (in >= len) continue;                       // gap between blobs
        const uint64_t key = dm_blob_key(seed, first_blob + lo);
        const uint64_t a = dm_blob_word_k(key, in >> 3), b = dm_blob_word_k(key, (in >> 3) + 1);
        if (in + 16 <= len) {
            *reinterpret_cast<ulonglong2 *>(base + pos) = make_ulonglong2(a, b);
        } else {
            for (uint64_t k = 0; in + k < len; ++k)
                base[pos + k] = (uint8_t)((k < 8 ? a : b) >> (8 * (k & 7)));
        }
    }
}

}  // namespace

static const FmaK kFmaK = {1u, 0xffffffffu, {0u, 0u}};

// The launchers end in `return cudaGetLastError()`.  The runtime's per-thread last-error slot also holds
// cudaErrorNotReady after a cudaEventQuery / cudaStreamQuery that was merely "not yet" (the pump polls events; a host
// application such as PyTorch does too), so it is cleared first: what a launcher returns is about its own launch.
static inline void clear_stale_error() { (void)cudaGetLastError(); }

template <int kFma, int kStyle>
static void launch_wide_t(const HashJob *jobs, uint32_t njobs, uint32_t *states, uint32_t *digests, cudaStream_t stream)
{
    const uint32_t grid = (njobs + kWideThreads - 1) / kWideThreads;
    sha256_wide_kernel<kFma, kStyle><<<grid, kWideThreads, 0, stream>>>(jobs, njobs, states, digests, kFmaK);
}

template <int kFma, int S, bool kPair>
static void launch_warp_t(const HashJob *jobs, uint32_t njobs, uint32_t *states, uint32_t *digests, cudaStream_t stream)
{
    constexpr uint32_t per_cta = kPair ? S : S * kWarpsPerCta;
    sha256_warp_kernel<kFma, S, kPair><<<(njobs + per_cta - 1) / per_cta, kPair ? 64 : 32 * kWarpsPerCta, 0, stream>>>(
        jobs, njobs, states, digests, kFmaK);
}

// One case label per built kernel; -1 for fields no kernel has.
static constexpr int shape_key(int spw, bool pairs, int form)
{
    return spw >= 1 && spw <= 32 && form >= 0 && form < 32 ? (spw * 2 + (pairs ? 1 : 0)) * 32 + form : -1;
}

cudaError_t launch_sha256(const HashJob *jobs, uint32_t njobs, uint32_t *states, uint32_t *digests,
                          cudaStream_t stream, const KernelShape &shape)
{
    if (njobs == 0) return cudaSuccess;
    clear_stale_error();
    switch (shape_key(shape.spw, shape.pairs, shape.form)) {
#define DM_W(f, st) case shape_key(32, false, (f) + 4 * (st)): launch_wide_t<f, st>(jobs, njobs, states, digests, stream); break;
    DM_W(0, 0) DM_W(1, 0) DM_W(2, 0) DM_W(0, 1) DM_W(1, 1) DM_W(2, 1)
    DM_W(0, 2) DM_W(1, 2) DM_W(2, 2) DM_W(0, 3) DM_W(1, 3) DM_W(2, 3)
    DM_W(0, 4) DM_W(1, 4) DM_W(2, 4)
    DM_W(1, 5)
#undef DM_W
#define DM_S(f, s, pr) case shape_key(s, pr, f): launch_warp_t<f, s, pr>(jobs, njobs, states, digests, stream); break;
#define DM_S_ALL(f, pr) DM_S(f, 1, pr) DM_S(f, 2, pr) DM_S(f, 4, pr) DM_S(f, 8, pr) DM_S(f, 16, pr)
    DM_S_ALL(0, false) DM_S(1, 1, false) DM_S(2, 1, false) DM_S_ALL(4, false) DM_S_ALL(5, false) DM_S_ALL(6, false)
    DM_S_ALL(7, false) DM_S_ALL(7, true)
#undef DM_S_ALL
#undef DM_S
    default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

cudaError_t launch_synth_fill(uint64_t seed, uint64_t blob, uint64_t byte_off, void *dst, size_t len,
                              cudaStream_t stream)
{
    if (len == 0) return cudaSuccess;
    size_t blocks = (len / 16 + 255) / 256;
    clear_stale_error();
    if (blocks < 1) blocks = 1;
    if (blocks > kSms * 16) blocks = kSms * 16;
    synth_fill_kernel<<<(unsigned)blocks, 256, 0, stream>>>(dm_blob_key(seed, blob), byte_off,
                                                            static_cast<uint8_t *>(dst), len);
    return cudaGetLastError();
}

cudaError_t launch_synth_fill_many(uint64_t seed, uint64_t first_blob, void *base, const uint64_t *dev_offsets,
                                   const uint64_t *dev_lengths, uint32_t n, uint64_t first_off, uint64_t span,
                                   cudaStream_t stream)
{
    if (n == 0 || span == 0) return cudaSuccess;
    uint64_t blocks = (span / 16 + 255) / 256;
    clear_stale_error();
    if (blocks < 1) blocks = 1;
    if (blocks > kSms * 16) blocks = kSms * 16;
    synth_fill_many_kernel<<<(unsigned)blocks, 256, 0, stream>>>(seed, first_blob, static_cast<uint8_t *>(base),
                                                                 dev_offsets, dev_lengths, n, first_off, span);
    return cudaGetLastError();
}

}  // namespace dm
