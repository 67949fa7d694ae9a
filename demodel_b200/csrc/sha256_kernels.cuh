// Internal interface between the engine (host C++) and the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dm {

// One unit of hashing work: advance one blob's SHA-256 state over a
// contiguous run of bytes in HBM.  Non-final jobs cover whole 64-byte blocks;
// a final job may end in a partial block, which the kernel pads on device
// (FIPS 180-4 §5.1.1) using total_len.
struct alignas(16) HashJob {
    const uint8_t *src;    // 16-byte aligned
    uint8_t *dst;          // CAS extent to copy into while hashing, or nullptr
    uint64_t nbytes;       // bytes of this run
    uint64_t total_len;    // whole-blob length (used when FINAL)
    uint32_t slot;         // index into the state table
    uint32_t flags;        // JOB_*
    uint32_t one;          // always 1: a multiplier the compiler cannot see (FMA-pipe adds)
    uint32_t pad_;
};
static_assert(sizeof(HashJob) == 48, "HashJob layout is shared with the kernels");

enum : uint32_t {
    JOB_INIT  = 1u,   // start from the FIPS 180-4 §5.3.3 initial hash value
    JOB_FINAL = 2u,   // apply padding and emit the digest words
};

// The kernel one launch runs; every shape computes the same digests.
struct KernelShape {
    int spw;      // streams per warp: 1, 2, 4, 8, 16 = sha256_warp_kernel; 32 = sha256_wide_kernel (a lane per stream)
    bool pairs;   // spw <= 16: two warps per group of spw streams, a schedule warp running ahead of the round warp
    int form;     // spw <= 16: the round form (sha256_round.cuh); spw = 32: the wide variant, fma + 4 * style, where
                  // fma = how round additions are issued (0 = ptxas' choice, 1 = all on the FMA pipe, 2 = same with the
                  // multiplier in a register) and style = main-loop shape (see sha256_wide_kernel)
};

// states/digests: uint32[slot][8], native word order (host serialises big-endian).
// `digests` may live in mapped pinned host memory.
// Launches `shape` over njobs jobs; decides nothing.  Built: round forms 0, 1, 2, 4..7 at spw 1 and 0, 4..7 at
// spw 2..16; pairs in form 7 at every spw <= 16; wide variants fma 0..2 x style 0..4, and 21.  Any other shape
// returns cudaErrorInvalidValue.
cudaError_t launch_sha256(const HashJob *jobs, uint32_t njobs, uint32_t *states, uint32_t *digests,
                          cudaStream_t stream, const KernelShape &shape);
// fma 1 + style 2: rolled rounds, additions on the FMA pipe, each lane's 128-byte line loaded into registers.  Measured
// on H100 SXM, 135 168 streams x 112 KiB per launch: variant 9 25.2 ms, variant 21 (style 5: the next line staged in
// shared memory by cp.async) 40.4 ms.
constexpr int kDefaultWideVariant = 9;

// Kernel choice by live-stream count (DESIGN.md §5): aim for one to two warps on
// each of the 528 sub-partitions.  Returns streams per warp: 32 = a lane per stream.
constexpr uint32_t kSms = 132;                       // H100 SXM
constexpr uint32_t kSubPartitions = kSms * 4;
constexpr uint32_t kMaxWarpPairs = kSubPartitions / 2;

inline int streams_per_warp_for(uint32_t njobs)
{
    // A warp must never share its sub-partition with another round warp (the round chain is issue-bound on one
    // sub-partition's ALU pipe), and while there are sub-partitions to spare a SECOND warp per group - loading and
    // expanding the next blocks' schedules ahead of the round warp - is worth more than a smaller S (DESIGN.md §5).
    // So: the smallest S in {1, 2, 4, 8, 16} whose njobs / S groups can each have a warp PAIR (<= 264 groups, up to
    // 4224 streams); then 16 per warp, one warp per sub-partition (<= 8448 streams); then a lane per stream.
    for (int s = 1; s <= 16; s *= 2)
        if ((njobs + s - 1) / s <= kMaxWarpPairs) return s;
    if ((njobs + 15) / 16 <= kSubPartitions) return 16;
    return 32;
}
// One warp per group, no pairs: the smallest S that still leaves every warp a sub-partition (the rule for a launch
// that shares the chip with another one, engine_cache.cu's split batches).
inline int streams_per_warp_unpaired(uint32_t njobs)
{
    for (int s = 1; s <= 16; s *= 2)
        if ((njobs + s - 1) / s <= kSubPartitions) return s;
    return 32;
}
// Can a launch of njobs jobs at S streams per warp run as warp pairs, given that `resident` jobs (this launch and the
// ones still running, all at S per warp) share the chip?
inline bool warp_pairs_fit(uint32_t resident, int s) { return s <= 16 && (resident + (uint32_t)s - 1) / (uint32_t)s <= kMaxWarpPairs; }

// Deep variant (the engine's tuning knob for spw <= 16) -> round form: 0 = ptxas' ordering; 1 and 3 = additions on the
// FMA pipe, 2 = same with the multiplier in a register (one warp per stream only: 0 elsewhere); 4..7 = the short-chain
// rounds (sha256_round.cuh); 8..10 = form 7 as warp pairs.  Form 7 = short-chain round with e' on the FMA pipe and a'
// as one IADD3.  8 pairs one warp per stream, 9 also S streams per warp, both while every group of pair_jobs gets two
// sub-partitions (warp_pairs_fit); 10 pairs one warp per stream whatever the count (A/B of that rule).
constexpr int kDefaultDeepVariant = 9;

// The kernel for a launch at spw streams per warp.  pair_jobs: the jobs that share the chip at spw per warp, this
// launch's included; 0 = never pair.  Other variant numbers run deep form 0 and wide variant 9.
inline KernelShape kernel_shape(int spw, uint32_t pair_jobs, int variant_wide, int variant_deep)
{
    if (spw == 32) {
        const int w = variant_wide;
        const bool built = (w >= 0 && w < 20 && w % 4 != 3) || w == 21;
        return {32, false, built ? w : kDefaultWideVariant};
    }
    const int d = variant_deep;
    const bool fit = pair_jobs != 0 && warp_pairs_fit(pair_jobs, spw);
    const bool pairs = spw == 1 ? (d == 10 && pair_jobs != 0) || ((d == 8 || d == 9) && fit) : d == 9 && fit;
    const int form = d >= 8 && d <= 10 ? 7
                   : d >= 4 && d <= 7 ? d
                   : spw == 1 && (d == 1 || d == 3) ? 1
                   : spw == 1 && d == 2 ? 2
                   : 0;
    return {spw, pairs, form};
}

cudaError_t launch_synth_fill(uint64_t seed, uint64_t blob, uint64_t byte_off, void *dst,
                              size_t len, cudaStream_t stream);
// dev_offsets / dev_lengths: n entries each, offsets ascending and 16-byte aligned;
// span = offsets[n-1] + lengths[n-1] - offsets[0].
cudaError_t launch_synth_fill_many(uint64_t seed, uint64_t first_blob, void *base,
                                   const uint64_t *dev_offsets, const uint64_t *dev_lengths, uint32_t n,
                                   uint64_t first_off, uint64_t span, cudaStream_t stream);

}  // namespace dm
