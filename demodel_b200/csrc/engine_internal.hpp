// engine_internal.hpp - types, constants and internal entry points shared by the engine's translation units:
//   engine_core.cu    extents, ring slabs, CAS commit / eviction, the pump (launch decisions), the disk tier
//   engine_api.cu     C-ABI: engine lifecycle, streams (ingest, ranges, checkpoint / resume, zero-copy windows),
//                     loads of disk-tier blobs back into HBM (promotion, verified opens), checks of disk-tier files and
//                     imports of files from outside the cache and exports of cached blobs to files (internal
//                     streams), the listing of the disk tier
//   engine_cache.cu   C-ABI: hit serving (readers, followers, verified opens), device-resident ingest, the synthetic
//                     generator
// Not installed, not part of the boundary (that is include/demodel_b200.h).
#pragma once
#include "../../include/demodel_b200.h"
#include "sha256_kernels.cuh"
#include "blobgen.h"
#include "host_util.hpp"

#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include <errno.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <sys/types.h>
#include <unistd.h>


namespace dmi {


using dm::Arena;
using dm::add_interval;

extern thread_local std::string g_last_error;      // what dm_last_error() returns (engine_core.cu)
int fail(int code, const char *what);
// Record the calling thread's detail text under a stream / reader id (0 = engine-level call) when rc is an
// error, so that dm_error_detail() can return it from ANY thread (cgo: a goroutine may change OS threads
// between the failing call and the call that asks for the text).  Returns rc.
int note_err(dm_engine *e, uint64_t id, int rc);
cudaError_t poll_event(cudaEvent_t ev);
int fail_cuda(cudaError_t err, const char *where);
#define CU_TRY(expr)                                                   \
    do {                                                               \
        cudaError_t cu_err_ = (expr);                                  \
        if (cu_err_ != cudaSuccess) return fail_cuda(cu_err_, #expr);  \
    } while (0)

constexpr uint64_t kAlign = 256;           // CAS extent granularity
constexpr uint64_t kMaxGrow = 256ull << 20;
constexpr int kCycles = 8;                 // concurrent hash launches, each on its own CUDA stream
constexpr uint32_t kTinyMax = 64u << 10;    // bodies up to this size that arrive in one piece travel in shared "pack" slabs
constexpr int kPackDevBufs = 64;           // device staging buffers for packs (slab_bytes each)
constexpr uint32_t kMaxJobSlabs = 8;       // a job covers 1..8 slabs of backlog (run_cycle): fewer, longer launches when the hash is behind
constexpr int kSlabBatches = 64;           // groups of DMA'd slabs waiting for their copy events
constexpr int kStripes = 64;               // stream-table lock stripes
constexpr int kCopyStreams = 2;
constexpr size_t kBounceBytes = 4u << 20;
constexpr int kBounces = 48;               // 4 MiB each; readers borrow two as read-ahead windows
constexpr int kSpillThreads = 4;           // disk-tier writers (each double-buffers two bounce buffers)
constexpr int kIngestMaxChunks = 8;
constexpr uint32_t kIngestChunkMin = 16384;  // jobs per chunk at least: 512 warps of the lane-per-stream kernel
constexpr int kCompleters = 2;             // threads that compare / publish finished bodies, so the pump only launches and reaps
constexpr int kBounceReserve = 2 * kSpillThreads + 2;          // never lent to windows: the spill thread and one-shot reads need some
constexpr int kDiskThreads = 4;            // file writes, read-backs and publications of disk-backed streams and checks

inline uint64_t round_up(uint64_t x, uint64_t a) { return (x + a - 1) / a * a; }

struct Digest {
    uint8_t b[32];
    bool operator==(const Digest &o) const { return memcmp(b, o.b, 32) == 0; }
};
struct DigestHash {
    size_t operator()(const Digest &d) const
    {
        uint64_t v;
        memcpy(&v, d.b, 8);   // SHA-256 output is already uniform
        return (size_t)v;
    }
};

inline void words_to_digest(const uint32_t *w, uint8_t out[32])
{
    for (int i = 0; i < 8; ++i) {                // big-endian words, FIPS 180-4 section 6.2.2
        const uint32_t be = __builtin_bswap32(w[i]);
        memcpy(out + 4 * i, &be, 4);
    }
}

inline std::string hex_of(const uint8_t *d, size_t n)
{
    static const char *hx = "0123456789abcdef";
    std::string s(2 * n, '0');
    for (size_t i = 0; i < n; ++i) { s[2 * i] = hx[d[i] >> 4]; s[2 * i + 1] = hx[d[i] & 15]; }
    return s;
}

struct Extent { uint64_t off, len; };      // byte range of the HBM arena

struct Blob {
    Digest digest;
    uint64_t size = 0;
    std::vector<Extent> extents;          // empty once evicted from HBM
    uint32_t readers = 0;
    Blob *lru_prev = nullptr, *lru_next = nullptr;   // intrusive LRU links while in_hbm (guarded by e->mu): no node allocation
    bool in_lru = false;
    bool in_hbm = false;
    bool on_disk = false;
    bool spill_done = false;
    // dm_cache_remove took it out of the index while readers had it open: the last dm_cache_close frees its extents
    bool removed = false;
    bool parked = false;                  // DM_ING_REPLACE is rewriting its extent (dm_cache_remove: DM_ESTATE)
    bool renaming = false;                // a spill is moving its file into place: dm_cache_remove waits (remove_cv)
    std::vector<std::pair<std::string, std::string>> meta;   // response headers to replay on a hit
    std::string sidecar;                  // promoted from the disk tier (dm_cache_promote): its .meta text, replayed as is
};

struct Slab { uint8_t *host; uint8_t *dev; };   // dev: same slab of the device-side mirror (verify-only streams)

// Many tiny bodies, ONE H2D DMA.  A body of at most kTinyMax bytes that is still entirely in its first ring slab when it
// finishes is copied into the engine's open pack (a ring slab shared by many such bodies) and gives its own slab
// straight back; the pump DMAs the whole pack to a device staging buffer with one cudaMemcpyAsync, and each member's
// final job hashes its piece from the staging buffer while copying it into the member's own CAS extent (the kernels'
// fused copy).  Without this a 4 KiB manifest / config / tokenizer file costs a cudaMemcpyAsync of its own - the
// driver call, not the bytes, was what capped small-body throughput.
struct Pack {
    Slab *slab = nullptr;            // host side, handed to the ordinary slab-return path once the DMA is enqueued
    uint8_t *dev = nullptr;          // device staging buffer, back to the pool when the last member's job is reaped
    uint32_t fill = 0;               // bytes used; members sit at 256-byte aligned offsets
    uint32_t bytes = 0;              // the members' own bytes (h2d_bytes counts these, not the alignment padding)
    std::atomic<uint32_t> refs{0};   // members whose job has not been reaped (or that have not been aborted)
    std::atomic<bool> dma_issued{false};
    std::atomic<bool> failed{false};
};

enum class St { Open, Finishing, Done, Aborted };

using Clock = std::chrono::steady_clock;
struct Stream;

// One reader attached to a ring load (Reader::part).  Guarded by the mutex of the load's stream.  The reader needs the
// bytes [need, end) once `started`, and every byte before that.
struct RingPart {
    uint64_t need = 0;            // the reader needs no byte below this (reads are forward only)
    uint64_t next = 0;            // the end of the previous read: the next one may not start below it
    uint64_t end = UINT64_MAX;    // the end of its range (dm_cache_open_verified_range: off + len)
    bool started = false;         // the first read has been made, or the range was given at open
    bool inside = false;          // in dm_cache_read
    Clock::time_point left = Clock::now();   // when it last left dm_cache_read (or opened)
    // Taken off a shared load it held back (ring_detach): the load no longer lists it, and its next read starts a
    // shared load of its own with the budget reserved here (`reserved`, until that load takes it over or the reader closes).
    bool detached = false, reserved = false;
    // The loads this reader was detached from (the reader's own, under its mutex).  It got bytes from them, so its last
    // byte and its EOF wait for their verdicts too, and each keeps running until this reader closes (RingLoad::dependents).
    std::vector<std::shared_ptr<Stream>> from;
    int failed = DM_OK;           // ... and one of them failed: every read of the reader returns this (the reader's own)
    bool needs(uint64_t off, uint64_t n) const { return !started || (off + n > need && off < end); }
};

// A check of a tier file (Stream::check_only, disk-backed) whose read-back slabs also serve readers, so the bytes
// handed out are the bytes the H2D copy took to the kernel and the file is read once for all of them.
//   dm_cache_open_verified_ring: one reader, no other open joins it, and it stops when that reader closes.
//   dm_cache_open_verified_range: a shared load.  e->ring_shared lists it while it runs; range opens whose range it can
//   still serve attach to it, and it stops when its last reader closes.
// A slab of the load goes back to the ring only when its job has been reaped AND no attached reader needs it
// (RingPart::needs).  Guarded by the stream's mutex.
struct RingLoad {
    struct Held { Slab *slab; uint64_t off; uint32_t n; bool reaped; Clock::time_point reaped_at; };
    std::deque<Held> held;        // read back, in file order (staged, hashing, or waiting for readers)
    std::vector<std::shared_ptr<RingPart>> parts;   // the attached, open readers
    uint32_t dependents = 0;      // open readers detached from it (RingPart::from): it stops only when these are gone too
    uint32_t cap = 0;             // at most this many slabs out of the ring at once (disk_feed stops issuing reads)
    bool shared = false;          // dm_cache_open_verified_range's
    // The low-water mark: the end of the last slab given back to the ring (0 before any).  Every byte the load read at
    // or past it is still held, so a reader whose range starts there or later can attach.
    uint64_t low = 0;
    uint64_t size = 0;            // the file's, at open
    std::string side;             // the sidecar text read at open (dm_cache_meta of every reader)
    bool closed = false;          // the last reader closed: everything reaped goes back, no further reads are issued
    bool slot_reserved = true;    // one of the tier calls' stream slots (slots_reserved), until the load ends
    bool settled = false;         // the verdict has been acted on (drop_corrupt, recency): `status` is final
    int status = DM_OK;
    struct stat seen{};           // the file that was read (drop_corrupt)
};

struct Stream {
    std::mutex mu;
    std::condition_variable cv;
    uint64_t id = 0;
    uint32_t slot = 0;
    bool has_expect = false;
    Digest expect{};
    std::vector<Extent> extents;
    uint64_t capacity = 0;     // sum of extents
    uint64_t received = 0;     // bytes accepted (count, any order)
    uint64_t dma_issued = 0;   // end of the contiguous run, starting at resume_base, whose H2D is enqueued
    uint64_t hash_issued = 0;  // bytes covered by launched jobs
    // End of the contiguous run whose H2D copies have COMPLETED (the pump learns it from the copy events that return the
    // slabs).  Jobs over landed bytes need no ordering against the copy streams, so a launch does not queue behind
    // hundreds of MiB of other streams' DMAs that merely happen to sit ahead of its event in the copy FIFO (with a
    // 1 GiB ring that was up to ~20 ms per launch while writers ran ahead of the hash).  Not maintained for streams
    // that use range parts, verify-only staging or packs: those launches still wait on the copy events.
    uint64_t landed = 0;
    bool range_mode = false;   // dm_stream_write_at parts were used: `landed` is not the whole story
    Slab *cur = nullptr;       // sequential cursor: stages [dma_issued, dma_issued + cur_fill)
    uint32_t cur_fill = 0;
    // Range parts (dm_stream_write_at): out-of-order pieces staged per part, DMA'd to their place in
    // the extent, and remembered as islands until the contiguous frontier reaches them.
    struct Part { uint64_t base; Slab *slab; uint32_t fill; };
    std::vector<Part> parts;
    std::map<uint64_t, uint64_t> islands;        // [start, end) DMA-enqueued beyond the frontier
    uint64_t resume_base = 0;                    // bytes hashed before this stream existed (checkpoint)
    std::map<uint64_t, uint64_t> prefix_cover;   // what of [0, resume_base) was re-supplied for caching
    bool ckpt_waiter = false;
    // Verify-only streams (DM_F_NO_HBM_CAS, or a blob that could never fit the arena): nothing is
    // retained.  Slabs are DMA'd to the device mirror of the ring and hashed from there, one slab per
    // job in arrival order; a slab returns to the ring when its job has run.
    bool verify_only = false;
    // A verify-only stream whose partly filled slab is recalled by ring back-pressure keeps the bytes past
    // the last whole block here (jobs hash whole blocks); they lead the stream's next slab.  carry_fill > 0
    // implies cur == nullptr.
    uint8_t carry[64];
    uint32_t carry_fill = 0;
    std::deque<std::pair<Slab *, uint32_t>> staged;
    // Disk-backed streams (DM_F_DISK_DIRECT): a verify-only stream whose bytes are kept in a file of their own,
    // <cas_dir>/incoming/<pid>-<device>-<id>.part.  Every slab and range part is written there by a disk thread
    // and goes back to the ring when the write completes; the hash reads the bytes back from the file, in order,
    // into `staged` (whole blocks, at most two slabs ahead).  The verified file is renamed into the disk tier.
    bool disk = false;
    int fd = -1;
    std::string path;
    std::map<uint64_t, uint64_t> written;        // [start, end) whose pwrite has completed
    uint64_t staged_to = 0;                      // bytes read back for hashing (from resume_base on)
    uint32_t disk_writes = 0, disk_reads = 0;    // in flight on the disk threads (at most one read)
    bool publishing = false;                     // the final rename / sidecar is running on a disk thread
    bool suspending = false;                     // dm_stream_suspend: no further read-back or launch
    uint32_t cuts = 0;                           // dm_stream_suspend cut the file at C: followers' bytes past C are gone
    std::string sidecar;                         // the sidecar text of the verified body (followers' dm_cache_meta)
    // dm_cache_verify / dm_cache_import: a check of a stored file, never a download.  A disk-backed check reads the
    // file itself (fd / path, every byte already written: a blob file, or an import's staged copy); a tiny one travels
    // in a pack as a hash-only member.  It holds no arena extent, and its verdict is all it produces: nothing is
    // published, renamed, truncated or unlinked by the stream (an import publishes its copy itself afterwards).
    bool check_only = false;
    std::unique_ptr<RingLoad> ring;   // a check that serves a reader (dm_cache_open_verified_ring); set before it is shared
    // A body announced (Content-Length) as at most tiny_max bytes never takes a ring slab: its bytes gather in this
    // private buffer and go straight into a pack when it finishes.  Anything that needs a real slab (more bytes than
    // announced, range parts, zero-copy windows, checkpoints) moves them into one first (take_slab).
    std::unique_ptr<uint8_t[]> small;
    uint32_t small_fill = 0, small_cap = 0;
    std::shared_ptr<Pack> pack;      // tiny body travelling in a shared pack: [pack_off, pack_off + pack_len) of pack->dev
    uint32_t pack_off = 0, pack_len = 0;
    std::vector<std::pair<std::string, std::string>> meta;   // dm_stream_set_meta
    bool load = false;         // the stream of a Load run by the loader threads: its completion wakes them (load_wake)
    bool held = false;         // counted in e->holds under `expect` until drop_stream (dm_cache_remove: DM_ESTATE)
    uint32_t followers = 0;    // readers attached while the body is still arriving (request coalescing)
    uint32_t follow_reads = 0; // followers' copy-outs in flight: the extents must not be freed or handed over meanwhile
    bool completing = false;   // digest known, extents being handed to the index: followers wait for Done
    uint64_t size_hint = 0;
    bool window_out = false;   // acquire() window outstanding
    bool queued = false;       // in the pump's inbox / ready list (guarded by mu)
    bool final_issued = false;
    uint32_t jobs_inflight = 0;
    St st = St::Open;
    Digest digest{};
    int matched = 0;
    bool cuda_failed = false;  // a copy or launch for this stream failed: whatever digest comes back is not trusted
    int lost = DM_OK;          // sticky: bytes this stream had accepted were dropped by a pump-side submit (arena full while
                               // recalling a partial slab ...).  write / finish / checkpoint return it; never published.
    std::shared_ptr<Blob> blob;   // set at commit
};

// A disk-tier blob being loaded into a fresh HBM extent and hashed there as an internal stream whose expected digest is
// its name (dm_cache_promote, dm_cache_open_verified).  e->loads indexes the running ones by digest, so that a digest is
// never loaded twice at once: a verified open attaches its reader to the running load, a promotion waits for its verdict.
struct Load {
    Digest d;
    // the thread that runs the load: set before `opened`, not touched by anybody else
    int fd = -1;                          // the tier file, open from load_open until load_fill has read it
    struct stat seen{};                   // the file that was read (st_dev / st_ino)
    std::shared_ptr<Blob> mine;           // the disk-only entry this load registered (none if one existed)
    uint64_t stream = 0;
    bool tiny = false;                    // at most tiny_max bytes: read into the stream's private buffer
    bool reserved = false;                // holds one of the tier calls' stream slots (a verified open's load)
    // published under mu: readers wait here for the stream to open and for the verdict
    std::mutex mu;
    std::condition_variable cv;
    std::shared_ptr<Stream> sp;           // the load's stream (readers follow it)
    uint64_t size = 0;
    std::string side;                     // the sidecar text read at open
    bool opened = false, done = false;
    int status = DM_OK;                   // once done: DM_OK (the blob is in HBM) or why the load failed
    std::string why;
};

struct Bounce;
struct Window { Bounce *b = nullptr; uint64_t off = 0, len = 0; bool pending = false; };

struct Reader {
    std::shared_ptr<Blob> blob;
    std::string disk_meta;        // sidecar text, disk-tier readers (and verified readers until the verdict)
    std::shared_ptr<Stream> follow;   // in-flight body this reader is coalesced onto (until it completes)
    std::shared_ptr<Load> load;       // dm_cache_open_verified of a disk-tier blob: the load `follow` belongs to
    std::shared_ptr<Stream> ring;     // dm_cache_open_verified_ring / _range of a disk-tier blob: its load (Stream::ring)
    std::shared_ptr<RingPart> part;   // ... and this reader's place in it
    bool ranged = false;          // dm_cache_open_verified_range: reads stay within [lo, hi)
    uint64_t lo = 0, hi = 0;
    int fd = -1;                  // disk tier; a follower of a disk-backed body: its own descriptor of the body's file
    Digest disk_digest{};         // ... the blob it reads
    bool disk_pin = false;        // ... pinned against disk-tier eviction until dm_cache_close
    uint32_t follow_cut = 0;      // Stream::cuts when a disk-backed body was followed
    uint64_t size = 0;
    std::mutex mu;                // a reader is normally one goroutine; this keeps misuse safe
    Window win[2];                // double-buffered read-ahead in pinned memory (HBM tier)
    bool tried_windows = false;
};

struct Cycle {
    bool busy = false;
    cudaEvent_t copy_ev[kCopyStreams]{};
    cudaEvent_t k_start{}, k_end{};
    cudaStream_t stream{};           // launches on different streams overlap on the GPU
    dm::HashJob *h_jobs = nullptr;   // pinned
    dm::HashJob *d_jobs = nullptr;
    uint32_t njobs = 0;
    bool deep = false;
    bool needs_copy_wait = false;    // some job reads bytes whose DMA may still be in flight
    uint64_t bytes = 0;
    std::vector<std::shared_ptr<Stream>> streams;   // one entry per job
    std::vector<Slab *> job_slabs;                  // verify-only jobs: the ring slab to release at reap
    std::vector<std::shared_ptr<Pack>> job_packs;   // tiny-body jobs: the pack whose staging buffer they read
    std::vector<uint8_t> is_final;
    cudaError_t err = cudaSuccess;                  // first failure while building or running this launch
};

// A slab whose DMA has been enqueued, on its way back to the ring.  For a stream's sequential slabs it also says how
// far the stream's bytes will have LANDED in HBM once the copy event behind it fires (Stream::landed).
struct SentSlab { Slab *slab; std::shared_ptr<Stream> sp; uint64_t end; };

struct SlabBatch {
    bool busy = false;
    cudaEvent_t ev[kCopyStreams]{};
    std::vector<SentSlab> slabs;
};

struct Bounce { uint8_t *host = nullptr; cudaStream_t stream{}; };

// Work for the disk threads of DM_F_DISK_DIRECT.  Write: `slab` holds `n` bytes for blob offset `off`.
// Read: `slab` receives [off, off + n) of the file and is staged for hashing.  Publish: the final job has been
// reaped, the verdict is in the stream.
struct DiskTask {
    enum Kind { Write, Read, Publish } kind = Write;
    std::shared_ptr<Stream> sp;
    Slab *slab = nullptr;
    int fd = -1;
    uint64_t off = 0;
    uint32_t n = 0;
};

// The disk tier under a size limit (dm_cache_set_disk_limit).  Built by the first call with a non-zero limit (one walk
// of blobs/, incoming/ and partial/) and dropped again by a limit of 0.  Every entry is a blob (file + sidecar) or a
// saved download (.ckpt + .part); `order` ranks them least recently used first.  On disk the last use is the blob
// file's mtime, written explicitly (content-addressed files are never rewritten, and reads never move it), except for
// files with more than one link, whose recency lives in memory only.  Bytes are apparent sizes (st_size).
struct TierEntry {
    uint64_t bytes = 0;
    uint64_t seq = 0;                     // key in DiskTier::order
    bool linked = false;                  // st_nlink > 1 (a hard-linked import): its mtime is the source's, not ours
};
struct TierKey { Digest d; bool saved; };
// Bytes set aside for a file that is about to be written (a spill, a saved download).  `gen` says which index they
// were counted in: a reservation taken before the index was dropped and rebuilt is not returned to the new one.
struct TierRes { uint64_t bytes = 0, gen = 0; bool partial = false; };
struct DiskTier {
    bool on = false;                      // a limit is set and the index below is built
    uint64_t limit = 0, gen = 0, seq = 0;
    int64_t last_stamp = 0;               // mtimes written are strictly increasing, so the order survives a restart
    std::unordered_map<Digest, TierEntry, DigestHash> blobs, saved;
    std::map<uint64_t, TierKey> order;
    uint64_t blob_bytes = 0, partial_bytes = 0, staging_bytes = 0, reserved_blob = 0, reserved_partial = 0;
    std::unordered_map<std::string, std::pair<uint64_t, uint64_t>> staging;   // incoming/ file -> (reserved, written)
    // Pins: kept with or without a limit, so that a limit set later sees them.  Never evicted while counted.
    std::unordered_map<Digest, uint32_t, DigestHash> pins, saved_pins;
    std::unordered_map<Digest, uint32_t, DigestHash> spills;   // digests a spill is writing (<hex>.part under blobs/)
    uint64_t evicted_files = 0, evicted_bytes = 0, refused = 0;
    uint64_t used() const { return blob_bytes + reserved_blob + staging_bytes + partial_bytes + reserved_partial; }
};

}  // namespace dmi

using namespace dmi;       // internal header: the engine's own translation units only

struct dm_engine {
    dm_config cfg{};
    std::string cas_dir;
    int device = 0;
    int sm_count = 132;
    int numa_node = -1;              // DM_F_NUMA_LOCAL: the node the engine bound itself to, -1 = not bound
    int force_spw = 0;               // DM_FORCE_SPW: 1/2/4/8/16/32 streams per warp for every launch (tuning only)
    int variant_wide = dm::kDefaultWideVariant, variant_deep = dm::kDefaultDeepVariant;   // DM_KERNEL_VARIANT overrides (tuning only)

    cudaStream_t copy_stream[kCopyStreams]{};
    cudaStream_t ingest_stream{}, util_stream{};

    uint8_t *arena_base = nullptr;
    std::mutex arena_mu;
    Arena arena;

    uint8_t *ring = nullptr;
    uint8_t *dev_ring = nullptr;     // device mirror of the ring, allocated on first verify-only use
    std::vector<Slab> slab_store;
    std::mutex slab_mu;
    std::condition_variable slab_cv;
    std::vector<Slab *> slab_free;

    uint32_t *d_states = nullptr;
    uint32_t *h_digests = nullptr;   // mapped pinned, [max_streams][8]
    uint32_t *d_digests = nullptr;   // device alias of h_digests

    std::mutex mu;                   // blobs / readers / slots
    std::mutex stripe_mu[kStripes];  // stream table, striped by id: dm_stream_write never takes `mu`
    std::unordered_map<uint64_t, std::shared_ptr<Stream>> streams[kStripes];
    std::atomic<uint64_t> n_streams{0};
    std::atomic<bool> ring_starved{false};
    std::mutex slot_mu;              // state / digest slots: a lock of their own, so that opening and closing tiny bodies from
    std::vector<uint32_t> free_slots;                // many threads does not queue on the index lock `mu`
    size_t slots_reserved = 0;       // slots the running tier calls may take: promote, verify, import, export calls,
                                     // verified opens' loads and ring loads (slots_reserve, slot_mu)
    size_t ring_load_slabs = 0;      // ring slabs the open ring loads may hold (RingLoad::cap each, slot_mu)
    // The running shared ring loads by digest (dm_cache_open_verified_range), more than one per digest after a late
    // joiner or a detach.  A range open looks up, attaches and starts under ring_mu, so two opens never both start a
    // load that one could serve.  Lock order: reader.mu → ring_mu → stream.mu; settle and the last close take it
    // with no stream mutex held.
    std::mutex ring_mu;
    std::unordered_multimap<Digest, std::shared_ptr<Stream>, DigestHash> ring_shared;
    std::atomic<uint64_t> next_id{1};
    dm::FlatIndex<Digest, std::shared_ptr<Blob>, DigestHash> blobs;      // guarded by mu; see host_util.hpp
    std::unordered_map<Digest, std::weak_ptr<Stream>, DigestHash> inflight;   // open streams by expected digest
    // Digests something is placing or loading outside e->loads: open streams that expect them, and running
    // dm_cache_promote / verify / import / dm_stream_resume_saved calls.  dm_cache_remove refuses them (DM_ESTATE).
    struct Hold { uint32_t n = 0; const char *what = ""; };
    std::unordered_map<Digest, Hold, DigestHash> holds;
    std::condition_variable remove_cv;  // (with mu) a spill finished moving a blob's file into place (Blob::renaming)
    std::mutex reader_mu[kStripes];
    std::unordered_map<uint64_t, std::shared_ptr<Reader>> readers[kStripes];
    Blob *lru_head = nullptr, *lru_tail = nullptr;   // HBM-resident blobs, least recently used first (guarded by mu):
                                                     // eviction walks from the head instead of scanning the whole index

    std::mutex work_mu;              // pump inbox
    std::condition_variable work_cv;
    std::vector<std::shared_ptr<Stream>> dirty;
    std::vector<SentSlab> pending_slabs;
    std::atomic<bool> stop{false};   // set under work_mu; the spill threads read it under spill_mu
    std::atomic<int> ring_waiters{0};   // writers blocked in slab_get()
    // Slabs that are out of the ring but come back WITHOUT any writer doing anything: handed to the pump
    // with their DMA enqueued (returned when the copy event fires) or staged by a verify-only stream
    // (returned when their job has run).  While this is non-zero a blocked writer only has to wait; the pump
    // recalls partly filled slabs from other streams only when it is zero, i.e. when every slab is being
    // filled by somebody and nothing would otherwise move (more live streams than slabs).
    std::atomic<int> slabs_returning{0};
    uint64_t split_min = 8u << 20;      // dm_ingest_device splits a skewed batch only if its longest blob is at least this long
    uint32_t nt_copy_min = 0;           // dm_stream_write pieces >= this many bytes use streaming stores (0 = never)
    std::thread pump;
    Cycle cycles[kCycles];
    SlabBatch batches[kSlabBatches];
    uint32_t max_jobs = 0;

    // Finished bodies (final job reaped, digest words copied out) waiting to be compared with their expected
    // digest and published: index and arena work that would otherwise sit on the single pump thread and cap
    // small-body throughput.
    struct DoneItem { std::shared_ptr<Stream> sp; uint32_t words[8]; };
    std::mutex done_mu;
    std::condition_variable done_cv;
    std::deque<DoneItem> done_q;
    bool done_stop = false;
    std::vector<std::thread> completers;

    std::mutex spill_mu;
    std::condition_variable spill_cv, spill_done_cv;
    std::deque<std::shared_ptr<Blob>> spill_q;
    std::vector<std::thread> spillers;   // kSpillThreads writers of the disk tier

    std::mutex disk_mu;                  // disk threads (any engine with a cas_dir, or one that exported): their queue (taken after a stream mutex, never before)
    std::condition_variable disk_cv;
    std::deque<DiskTask> disk_q;
    std::vector<std::weak_ptr<Stream>> disk_starved;   // read-backs that found the ring empty: retried by the disk threads
    std::atomic<bool> feed_starved{false};             // ... and the pump recalls partly filled slabs for them
    bool feed_kick = false;                            // a slab was put back while read-backs were starved (disk_mu)
    bool disk_stop = false;
    std::vector<std::thread> disk_threads;

    // Loads of disk-tier blobs (struct Load).  `loads` is guarded by mu.  The loader threads (started by the first
    // dm_cache_open_verified that needs one) read opened loads' files into their streams (load_q) and collect the verdicts
    // of those being hashed (load_wait) when a load stream completes (load_kick).
    std::unordered_map<Digest, std::shared_ptr<Load>, DigestHash> loads;
    std::mutex load_mu;
    std::condition_variable load_cv;
    std::deque<std::shared_ptr<Load>> load_q;
    std::vector<std::shared_ptr<Load>> load_wait;
    bool load_kick = false, load_scanning = false;
    std::atomic<bool> load_stop{false};
    std::vector<std::thread> loaders;

    std::mutex bounce_mu;
    std::condition_variable bounce_cv;
    std::vector<Bounce *> bounce_free;
    std::vector<Bounce> bounce_store;

    std::mutex ckpt_mu;              // checkpoint state transfers: pinned staging + own stream, fully synchronous
    uint32_t *ckpt_pinned = nullptr;
    cudaStream_t ckpt_stream{};

    std::mutex ingest_mu;            // dm_ingest_device scratch
    uint32_t *ing_states = nullptr;
    uint32_t *ing_digests = nullptr;       // device
    dm::HashJob *ing_jobs_h = nullptr;     // pinned
    dm::HashJob *ing_jobs_d = nullptr;
    uint32_t *ing_digests_h = nullptr;     // pinned
    uint32_t ing_cap = 0;
    cudaEvent_t ing_ev0{}, ing_ev1{}, ing_ev2{};
    // dm_ingest_device over >= 2 * kIngestChunkMin lane-per-stream jobs runs as up to kIngestMaxChunks launches on
    // streams of their own, so that the host work of chunk c + 1 (extents, job table) and of chunk c - 1 (verdicts,
    // publication) overlaps the kernel of chunk c
    cudaStream_t ing_streams[kIngestMaxChunks]{};
    cudaEvent_t ing_cev_k[kIngestMaxChunks]{}, ing_cev_done[kIngestMaxChunks]{};
    uint32_t ingest_chunks = 0;            // 0 = by the rule above; DM_INGEST_CHUNKS forces a count (tuning / tests)

    std::mutex pack_mu;              // tiny-body packs (see struct Pack)
    std::shared_ptr<Pack> open_pack;
    std::vector<std::shared_ptr<Pack>> sealed_packs;     // full ones waiting for the pump
    std::vector<uint8_t *> pack_dev_free;                // pool of kPackDevBufs device staging buffers
    uint8_t *pack_dev_base = nullptr;
    uint32_t tiny_max = 0;                               // min(kTinyMax, slab_bytes / 4); 0 = packs disabled
    std::atomic<uint64_t> st_packed{0}, st_packs{0};

    std::mutex alias_mu;             // URL / ETag -> digest (dm_cache_alias_put/get); log = <cas_dir>/aliases.log
    // ordered by key: dm_cache_alias_list pages from a prefix or a key in O(log n) instead of sorting every page
    std::map<std::string, Digest> aliases;
    FILE *alias_log = nullptr;
    std::atomic<uint64_t> n_suspended{0};   // *.ckpt under <cas_dir>/partial

    // Disk-tier limit (struct DiskTier).  Lock order: tier_mu before e->mu (eviction updates the index under it), and
    // never taken while e->mu is held.  A stream mutex may be held when it is taken; tier_mu never takes one.
    std::mutex tier_mu;
    DiskTier tier;
    std::atomic<bool> tier_on{false};       // tier.on, readable without the lock: with no limit the hooks return at once

    std::mutex err_mu;               // dm_error_detail(): last error text by stream / reader id (bounded)
    std::unordered_map<uint64_t, std::string> err_text;
    std::deque<uint64_t> err_order;

    // stats
    // the two counters bumped from caller threads sit on cache lines of their own (many writers / readers at once)
    alignas(64) std::atomic<uint64_t> st_ingested{0};
    alignas(64) std::atomic<uint64_t> st_served{0};
    alignas(64) std::atomic<uint64_t> st_hashed{0};
    std::atomic<uint64_t> st_committed{0}, st_mismatch{0};
    std::atomic<uint64_t> st_group{0};
    std::atomic<uint64_t> st_launches{0}, st_wide{0}, st_deep{0}, st_h2d{0}, st_d2h{0}, st_ring_waits{0};
    std::mutex stat_mu;
    double st_kernel_ms = 0.0;
};

namespace dmi {

// Visit the device segments covering [off, off+len) of a blob laid out over `ext`.
template <class F>
void for_segments(dm_engine *e, const std::vector<Extent> &ext, uint64_t off, uint64_t len, F &&fn)
{
    uint64_t base = 0;
    for (const Extent &x : ext) {
        if (len == 0) break;
        if (off < base + x.len) {
            const uint64_t in = off - base;
            const uint64_t n = std::min(len, x.len - in);
            fn(e->arena_base + x.off + in, n);
            off += n; len -= n;
        }
        base += x.len;
    }
}


uint8_t *seg_at(dm_engine *e, const std::vector<Extent> &ext, uint64_t off, uint64_t *contig);
void free_extents(dm_engine *e, std::vector<Extent> &ext);
bool evict_for(dm_engine *e, uint64_t need);
void lru_touch(dm_engine *e, Blob *b);        // e->mu held: (re)insert as most recently used
void lru_drop(dm_engine *e, Blob *b);         // e->mu held: the blob left HBM
bool arena_alloc(dm_engine *e, uint64_t len, Extent *out);
int ensure_capacity(dm_engine *e, Stream *s, uint64_t need);
Slab *slab_get(dm_engine *e);
Slab *slab_try_get(dm_engine *e);             // non-blocking: nullptr when the ring is empty
bool pack_tiny_body(dm_engine *e, Stream *s);  // stream mutex held: move a finished tiny body into the open pack
void pack_release_member(dm_engine *e, Stream *s);   // stream mutex held: this member no longer needs its pack
void slab_put(dm_engine *e, Slab *s);
void slab_return(dm_engine *e, Slab *s);      // slab_put for a slab that was counted in slabs_returning
void ring_copy(dm_engine *e, void *dst, const void *src, size_t n);   // socket buffer -> ring slab
int take_slab(dm_engine *e, Stream *s, std::unique_lock<std::mutex> &g);
void mark_dirty(dm_engine *e, const std::shared_ptr<Stream> &sp, Slab *submitted, uint64_t landed_end = 0);
int dma_range(dm_engine *e, const std::shared_ptr<Stream> &sp, Slab *slab, uint64_t base, uint32_t n);
void absorb_islands(Stream *s);
int submit_slab(dm_engine *e, const std::shared_ptr<Stream> &sp);
int submit_part(dm_engine *e, const std::shared_ptr<Stream> &sp, size_t idx);
bool range_taken(const Stream *s, uint64_t off, uint64_t len, const Stream::Part *self);
std::string json_quote(const std::string &v);
std::string sidecar_json(const Blob &b);
bool write_sidecar(const std::string &path, const Blob &b);   // false: the sidecar could not be written whole
std::string blob_path(const dm_engine *e, const uint8_t d[32]);
std::shared_ptr<Blob> publish(dm_engine *e, const Digest &d, uint64_t size, std::vector<Extent> &ext,
                              std::vector<std::pair<std::string, std::string>> *meta = nullptr);
struct Verified { Digest d; uint64_t size; Extent x; };      // one blob of a device-resident batch, hashed and matched
struct Parked { std::shared_ptr<Blob> b; Extent x; };        // a cached blob taken out of sight while its extent is rewritten
void publish_many(dm_engine *e, const std::vector<Verified> &items);
void unpark_many(dm_engine *e, std::vector<Parked> &verified, std::vector<Parked> &failed);
void wait_follow_reads(Stream *s, std::unique_lock<std::mutex> &g);
void complete_stream(dm_engine *e, const std::shared_ptr<Stream> &sp, const uint32_t *words);
void completer_main(dm_engine *e);
void reap_cycle(dm_engine *e, Cycle &c);
bool run_cycle(dm_engine *e, Cycle &c, std::vector<std::shared_ptr<Stream>> &ready);
void flush_partial_slabs(dm_engine *e);
void pump_main(dm_engine *e);
Bounce *bounce_get(dm_engine *e);
Bounce *bounce_try_get(dm_engine *e);     // for long-lived borrowers: leaves a reserve
void bounce_put(dm_engine *e, Bounce *b);
void mkdirs(const std::string &path);
bool d2h_to_fd(dm_engine *e, const std::vector<Extent> &ext, uint64_t size, int fd, bool *cuda_failed = nullptr);
bool spill_one(dm_engine *e, Blob *b);
void spill_main(dm_engine *e);
int ensure_dev_ring(dm_engine *e);
std::string incoming_path(const dm_engine *e, uint64_t id);
void disk_enqueue(dm_engine *e, DiskTask t);
void disk_write(dm_engine *e, const std::shared_ptr<Stream> &sp, Slab *slab, uint64_t off, uint32_t n);   // stream mutex held
void disk_feed(dm_engine *e, const std::shared_ptr<Stream> &sp);   // stream mutex held: start the next read-back if one is due
bool disk_fed(const Stream *s);               // stream mutex held: every byte is written and staged (or never will be)
void disk_main(dm_engine *e);
// Engines with a cas_dir start their disk threads at create; one without starts them the first time a check of a file
// needs them (dm_cache_export).
void ensure_disk_threads(dm_engine *e);
std::shared_ptr<Stream> find_stream(dm_engine *e, uint64_t id);
void drop_stream(dm_engine *e, const std::shared_ptr<Stream> &sp, bool release_slot);
int ensure_ingest_scratch(dm_engine *e, uint32_t n);
void alias_load(dm_engine *e);                // dm_engine_create: replay <cas_dir>/aliases.log
// e->holds (dm_cache_remove refuses a held digest).  `what` is a string literal: it names the holder in the refusal.
void hold_digest(dm_engine *e, const Digest &d, const char *what);
void release_digest(dm_engine *e, const Digest &d);
struct DigestHold {                           // hold_digest for the lifetime of a call
    dm_engine *e; Digest d;
    DigestHold(dm_engine *e_, const Digest &d_, const char *what) : e(e_), d(d_) { hold_digest(e, d, what); }
    ~DigestHold() { release_digest(e, d); }
};
// e->mu held: one reader fewer on a blob; returns the extents to free (outside the lock) when it was the last reader of
// a blob dm_cache_remove took out of the index
std::vector<Extent> reader_gone(Blob *b);
bool digest_from_hex(const char *hex, uint8_t out[32]);
bool alias_key_ok(const char *key);           // 1..4096 bytes without control characters: one line of aliases.log
void sweep_incoming(const std::string &dir);  // remove files under incoming/ of processes that are gone

// Loads of disk-tier blobs (engine_api.cu).
// e->mu held: DM_OK when `d` is in HBM, 1 when *L is a new load the caller runs (every outcome must reach load_end),
// 2 when *L is a load of `d` that is already running.
int load_claim(dm_engine *e, const Digest &d, std::shared_ptr<Load> *L);
// dm_cache_open_verified: run a claimed load.  Its stream is opened on the calling thread, the file is read in and the
// verdict collected by the loader threads.  1: running; otherwise the load's final status (it has ended).
int load_begin(dm_engine *e, const std::shared_ptr<Load> &L);
void load_wake(dm_engine *e);                 // a load's stream completed (complete_stream)
void load_stop_all(dm_engine *e);             // dm_engine_destroy, while the pump still runs

// Ring loads (dm_cache_open_verified_ring and _range; struct RingLoad).
// engine_api.cu: start the ring load of a disk-only blob (its check stream finishing, the tier file read in by the disk
// threads) with `part` as its first reader: DM_OK with *sp (R->size and R->side set), or the open's error with nothing
// held.  `shared`: a range open's, with ring_mu held; it enters e->ring_shared, and the range [off, off + len) (len 0:
// to the end) is checked against the file's size (DM_ERANGE).  `reserved`: the slot and ring share were taken by
// ring_load_reserve (given back here on failure).
int ring_load_open(dm_engine *e, const Digest &d, const std::shared_ptr<RingPart> &part, bool shared, uint64_t off,
                   uint64_t len, bool reserved, std::shared_ptr<Stream> *sp);
void ring_load_settle(dm_engine *e, const std::shared_ptr<Stream> &sp);   // the verdict is in (disk_task_publish)
// A reader closed: it leaves the load; the last one stops it and gives everything back
void ring_load_close(dm_engine *e, const std::shared_ptr<Stream> &sp, const std::shared_ptr<RingPart> &part);
// slot_mu held: the stream slots and ring shares of n new ring loads, all or none: 0, or 1 (no slot) / 2 (no share)
int ring_load_reserve(dm_engine *e, size_t n);
void ring_load_unreserve(dm_engine *e, size_t n);                        // slot_mu held
// engine_core.cu, stream mutex held: slabs no reader needs any more and whose jobs are reaped go back to the ring
void ring_release(dm_engine *e, const std::shared_ptr<Stream> &sp);

// Disk-tier limit (engine_core.cu).  None takes a stream mutex or may be called with e->mu held.  With no limit set
// they only count pins; reservations always succeed and nothing is stat'ed, touched or written.
void tier_pin(dm_engine *e, const Digest &d, bool saved = false, bool spill = false);   // spill: a running spill's pin
void tier_unpin(dm_engine *e, const Digest &d, bool saved = false, bool spill = false);
bool tier_reserve(dm_engine *e, uint64_t bytes, bool partial, TierRes *r);   // false: no room could be made (refused)
void tier_release(dm_engine *e, TierRes &r);
// The file(s) of `d` are in place (blobs/ or, saved, partial/): release `r`, enter them at their st_size; `use`: as
// the most recently used entry.
void tier_placed(dm_engine *e, const Digest &d, bool saved, TierRes *r, bool use);
void tier_touch(dm_engine *e, const Digest &d);   // a use of blob d (no-op for blobs not in the tier)
void tier_forget(dm_engine *e, const Digest &d, bool saved = false);   // its files were removed: count what is left
// A file under incoming/ that will hold `reserve` bytes, `counted` of which the tier already counts elsewhere (a saved
// download being resumed, whose entry goes when the resume takes it over); false: refused.
bool tier_stage(dm_engine *e, const std::string &path, uint64_t reserve, uint64_t counted = 0);
void tier_stage_grow(dm_engine *e, const std::string &path, uint64_t written);   // never refuses, never evicts
void tier_unstage(dm_engine *e, const std::string &path);
// The staged file at `path` is about to become a blob of `size` bytes with a `side`-byte sidecar: false (refused) when no
// room can be made and none was reserved for the body when it was staged.
bool tier_stage_to_blob(dm_engine *e, const std::string &path, uint64_t size, uint64_t side, TierRes *r);
void tier_build(dm_engine *e);                         // tier_mu held: the walk that builds the index
bool tier_make_room(dm_engine *e, uint64_t need, bool partial);   // tier_mu held: evict until `need` more bytes fit
void tier_enter(dm_engine *e, const Digest &d, bool saved, bool use);   // tier_mu held, limit on: count the files of d as they are now

}  // namespace dmi
