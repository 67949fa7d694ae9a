/*
 * demodel_b200.h — C-ABI of the H100 blob hash-and-cache engine.
 *
 * This is the drop-in boundary for demodel's cache path.  The reference
 * (moeru-ai/demodel @ fb8342aa) has no FFI, plugin or C interface of its own
 * (SURVEY.md §8b; demodel/pkg/utils/fs.go:1-8 is all of pkg/), so
 * each entry point below cites the reference *hook* whose body it serves:
 *
 *   OnResponse hook  cmd/demodel/start.go:201-204   (today: Println, return resp)
 *       -> a Go io.ReadCloser wrapped around resp.Body calls
 *          dm_stream_open / dm_stream_write (or acquire+commit) /
 *          dm_stream_finish / dm_stream_abort        — "hash while copying
 *          into the cache".
 *   OnRequest hook   cmd/demodel/start.go:197-200   (today: Println, return req,nil)
 *       -> dm_cache_open / dm_cache_read / dm_cache_close build the
 *          *http.Response that short-circuits upstream — "serve a cache hit".
 *   start()          cmd/demodel/start.go:167-216
 *       -> dm_engine_create once per GPU before net.Listen (start.go:206),
 *          dm_engine_destroy on shutdown; dm_shard_of picks the engine.
 *
 * The cgo binding a maintainer would add is in INTEGRATION.md and go/.
 *
 * Conventions: plain C types only (no CUDA / torch types).  Every function is
 * thread-safe: net/http runs one goroutine per connection (start.go:210-215)
 * and cgo enters from many OS threads.  Functions return DM_OK (0) or a
 * negative dm_err; they never abort, throw or call exit.  There is NO CPU
 * fallback: without a usable CUDA device dm_engine_create fails with
 * DM_ENODEV / DM_ECUDA and nothing else can be called.
 */
#ifndef DEMODEL_B200_H
#define DEMODEL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DM_ABI_VERSION 2u   /* 2: dm_error_detail, URL aliases, saved checkpoints, dm_gunzip, DM_F_NUMA_LOCAL; dm_stats grew */

typedef enum dm_err {
    DM_OK        = 0,
    DM_EINVAL    = -1,   /* bad argument / unknown id */
    DM_ENOMEM    = -2,   /* HBM arena, pinned ring or stream table exhausted; or no room under the disk-tier limit
                          * (dm_cache_import, dm_stream_suspend: see dm_cache_set_disk_limit) */
    DM_ENOENT    = -3,   /* digest not in the content-addressed store */
    DM_ECUDA     = -4,   /* CUDA runtime error; dm_last_error() has the text */
    DM_ESTATE    = -5,   /* call not valid in the stream's current state */
    DM_EIO       = -6,   /* on-disk CAS tier I/O error */
    DM_ENODEV    = -7,   /* no CUDA device / device ordinal out of range */
    DM_ERANGE    = -8,   /* offset beyond blob end */
    DM_ECORRUPT  = -9    /* a disk tier copy does not hash to its name (dm_cache_promote, dm_cache_verify,
                          * dm_cache_open_verified and its reads), or a file
                          * to import does not hash to its expected digest (dm_cache_import), or the copy of a blob
                          * to export does not (dm_cache_export) */
} dm_err;

typedef struct dm_engine dm_engine;   /* opaque; owned by caller between create/destroy */

/* dm_config.flags */
#define DM_F_NO_HBM_CAS   0x1u  /* verify only: streams are hashed from a device mirror of the ring and
                                  * nothing is retained or published (also what a blob whose size_hint
                                  * exceeds hbm_cas_bytes gets automatically) */
#define DM_F_DISK_SYNC    0x2u  /* dm_stream_finish returns only after the disk tier holds the blob */
#define DM_F_NUMA_LOCAL   0x4u  /* pin the ring / bounce buffers and start the engine's threads on the NUMA node the
                                  * GPU hangs off (sysfs); silently skipped when the topology is not visible */
#define DM_F_DISK_DIRECT  0x8u  /* needs cas_dir (else dm_engine_create: DM_EINVAL).  A stream that would be verify-only
                                  * (size_hint > hbm_cas_bytes, or every stream under DM_F_NO_HBM_CAS) is DISK-BACKED
                                  * instead: its bytes are written to <cas_dir>/incoming/ as they arrive, each ring slab
                                  * returns as soon as its write completes, the GPU hashes the bytes read back from that
                                  * file, and the verified file is renamed into the disk tier.  Range parts, suspend and
                                  * resume work as on HBM streams, and followers (dm_cache_follow) attach to them: they
                                  * read the body from its file as its writes complete (see dm_cache_follow). */

typedef struct dm_config {
    uint32_t struct_size;     /* = sizeof(dm_config); ABI guard */
    int32_t  device;          /* CUDA ordinal; one engine per GPU */
    uint64_t hbm_cas_bytes;   /* HBM arena for the content-addressed store; 0 = 1/2 of free HBM */
    uint64_t ring_bytes;      /* pinned host ring; 0 = 256 MiB */
    uint32_t slab_bytes;      /* ring slab = one H2D DMA; multiple of 256; 0 = 1 MiB */
    uint32_t max_streams;     /* concurrently open streams; 0 = 65536 */
    const char *cas_dir;      /* on-disk tier root, NULL = HBM tier only */
    uint32_t flags;
    uint32_t reserved;
} dm_config;

typedef struct dm_stats {
    uint64_t bytes_ingested;      /* through dm_stream_write/write_at/commit, counted per slab as it goes to the device */
    uint64_t bytes_hashed;        /* by the SHA-256 kernels */
    uint64_t bytes_served;        /* through dm_cache_read */
    uint64_t blobs_committed;
    uint64_t blobs_mismatched;
    uint64_t kernel_launches;     /* SHA-256 kernel launches (wide + deep) */
    uint64_t launches_wide;
    uint64_t launches_deep;
    double   kernel_ms;           /* CUDA-event time summed over those launches */
    uint64_t h2d_bytes;
    uint64_t d2h_bytes;
    uint64_t hbm_cas_used;
    uint64_t hbm_cas_capacity;
    uint64_t open_streams;
    uint64_t ring_waits;          /* times a writer had to wait for a free ring slab (back-pressure) */
    uint64_t launches_group;      /* launches of the S-streams-per-warp kernel (counted in kernel_launches) */
    uint64_t ring_slabs_total;    /* leak accounting: every slab is either free, being filled, or in flight */
    uint64_t ring_slabs_free;
    uint64_t open_readers;
    uint64_t free_stream_slots;   /* == max_streams when no stream is open or draining */
    int64_t  numa_node;           /* DM_F_NUMA_LOCAL: the node the engine bound itself to; -1 = not bound */
    uint64_t aliases;             /* URL / ETag -> digest entries (dm_cache_alias_put) */
    uint64_t suspended;           /* interrupted downloads saved under <cas_dir>/partial (dm_stream_suspend) */
    uint64_t packed_bodies;       /* tiny bodies (<= 64 KiB, one piece) that shared a pack slab and its one H2D DMA */
    uint64_t packs;               /* ... and how many such packs went to the device */
} dm_stats;

/* ---- engine lifetime (start.go:167-216) -------------------------------- */
uint32_t    dm_abi_version(void);
int         dm_device_count(void);                       /* <0: dm_err */
int         dm_engine_create(const dm_config *cfg, dm_engine **out);
void        dm_engine_destroy(dm_engine *e);
int         dm_engine_stats(dm_engine *e, dm_stats *out);
const char *dm_strerror(int err);
const char *dm_last_error(void);                         /* thread-local detail text */
/* Detail text of the last failing call on stream / reader `id` (0: calls that take no id, such as
 * dm_stream_open, dm_cache_open, dm_ingest_device), retrievable from ANY thread - what a cgo caller
 * uses instead of dm_last_error(): a goroutine can change OS threads between the call that failed and
 * the one that asks why.  e == NULL: the last dm_engine_create failure in this process.  *len receives
 * the full length; up to cap-1 bytes + NUL are copied.  The engine remembers the last 4096 ids. */
int         dm_error_detail(dm_engine *e, uint64_t id, char *buf, size_t cap, size_t *len);

/* Kernel shape the engine picks for `n_resident` co-resident streams: streams per
 * warp, 1 = warp-per-stream (deep), 2..16 = group, 32 = lane-per-stream (wide).  Pure function. */
uint32_t    dm_streams_per_warp(uint32_t n_resident);

/* The kernel variant an engine uses unless DM_KERNEL_VARIANT overrides it: which = 0 the lane-per-stream (wide)
 * kernel's `fma + 4*style`, which = 1 the round form of the warp-per-stream / group kernels.  Reported next to
 * measurements (a profile taken with one variant says nothing about another).  Pure function. */
uint32_t    dm_default_kernel_variant(int which);

/* Digest-prefix sharding (SURVEY.md §8e): which of n_shards engines owns a
 * blob.  Uses the leading 16 bits so any n_shards (not only powers of two)
 * splits the digest space evenly; for n = 2,4,8 it equals digest[0] >> (8-log2 n). */
uint32_t    dm_shard_of(const uint8_t digest[32], uint32_t n_shards);

/* ---- ingest: OnResponse body tee (start.go:201-204) -------------------- */
/* expect: the LFS oid / OCI layer digest known from the URL, or NULL.
 * size_hint: Content-Length, or 0 when unknown (chunked). */
int dm_stream_open(dm_engine *e, const uint8_t expect[32], uint64_t size_hint, uint64_t *id);
/* Copies buf before returning (the Go caller reuses its 32 KiB io.Copy
 * buffer on the next Read).  Blocks only for ring back-pressure. */
int dm_stream_write(dm_engine *e, uint64_t id, const void *buf, size_t len);
/* Range parts: bytes for blob offset `offset`, in any order (HF clients and
 * Ollama fetch one large blob as parallel `Range` requests).  The bytes land
 * at their place in the blob's HBM extent at once; the digest advances over the
 * contiguous prefix as it grows.  Ranges must not overlap; up to 64 parts may
 * be open on one stream.  dm_stream_finish fails with DM_ESTATE while holes remain.
 * Disk-backed streams (DM_F_DISK_DIRECT) accept parts too: they are written at their offset in the stream's
 * file, and the hash reads the contiguous prefix back from there.  A failed file write (disk full, file size
 * limit, I/O error) makes every later call on the stream return DM_EIO; nothing is published. */
int dm_stream_write_at(dm_engine *e, uint64_t id, uint64_t offset, const void *buf, size_t len);

/* Mid-state checkpoint / resume of an interrupted download (SURVEY.md §8f-3).
 * dm_stream_checkpoint waits until every whole block received in order is
 * hashed and returns (state words, byte count).  dm_stream_resume opens a new
 * stream that continues from such a checkpoint: bytes from `ck->bytes` on are
 * hashed; the prefix may be re-supplied with dm_stream_write_at purely for
 * caching — if it is not, the blob is verified but not published in the CAS.
 * On a disk-backed stream (DM_F_DISK_DIRECT) the hash trails the client by the hash rate (one stream: tens of
 * MB/s), so dm_stream_checkpoint, which waits for every in-order block, can take minutes on a large body. */
typedef struct dm_checkpoint {
    uint32_t h[8];      /* SHA-256 chaining value after `bytes` bytes */
    uint64_t bytes;     /* multiple of 64 */
    uint32_t abi;
    uint32_t reserved;
} dm_checkpoint;
int dm_stream_checkpoint(dm_engine *e, uint64_t id, dm_checkpoint *out);
int dm_stream_resume(dm_engine *e, const dm_checkpoint *ck, const uint8_t expect[32], uint64_t size_hint, uint64_t *id);

/* Interrupted downloads that survive a proxy restart (SURVEY.md §8f-3; needs cas_dir).
 * dm_stream_suspend closes a stream opened WITH an expected digest and saves what it has: the SHA-256
 * mid-state after the last whole block received in order, and those bytes, under
 * <cas_dir>/partial/<hex>.ckpt / <hex>.part.  *resume_from = the byte count saved (multiple of 64): the
 * proxy re-requests upstream with `Range: bytes=<resume_from>-`.  The id is released.
 * dm_stream_resume_saved - in this process or after dm_engine_create over the same cas_dir - opens a stream
 * that continues from the saved state: the saved prefix is loaded back into the blob's HBM extent (so the
 * finished blob is cached whole) and only the bytes from *resume_from on are hashed.  DM_ENOENT when
 * nothing is saved for `expect`.  The saved files are removed once a resumed stream has taken them over.
 * Disk-backed streams (DM_F_DISK_DIRECT): suspend does not wait for the hash and copies nothing.  It saves the
 * mid-state at the hashed position H, cuts the stream's file to the contiguous written prefix rounded down to 64
 * (C >= H) and renames it to <hex>.part; *resume_from = C.  dm_stream_resume_saved hashes [H, C) from the saved
 * file - a disk-backed stream adopts the file by renaming it back, an engine that can now hold the blob in HBM
 * loads it - and the client continues at C. */
int dm_stream_suspend(dm_engine *e, uint64_t id, uint64_t *resume_from);
int dm_stream_resume_saved(dm_engine *e, const uint8_t expect[32], uint64_t size_hint, uint64_t *id, uint64_t *resume_from);

/* Response headers worth replaying on a hit (Content-Type, ETag, Last-Modified,
 * the request URL ...).  Stored with the blob — in the `.meta` sidecar on the
 * disk tier — and returned by dm_cache_meta.  At most 64 entries per stream. */
int dm_stream_set_meta(dm_engine *e, uint64_t id, const char *key, const char *value);

/* Zero-copy variant: borrow a window of the pinned ring, Read() into it,
 * then commit the bytes actually read.  At most one outstanding window per
 * stream; *cap >= 1 on success.
 * Lifetime: [ptr, ptr+cap) belongs to the caller from dm_stream_acquire until
 * dm_stream_commit RETURNS.  After the commit the engine may DMA the slab and
 * hand it to another stream at any moment, so anything else that reads the
 * window (the client-side write of the same bytes) must finish BEFORE the
 * commit: acquire, Read, Write to the client, commit. */
int dm_stream_acquire(dm_engine *e, uint64_t id, void **ptr, size_t *cap);
int dm_stream_commit(dm_engine *e, uint64_t id, size_t len);
/* Optional, non-blocking: upstream hit EOF, no more bytes will be written.
 * Starts the final hash so a later dm_stream_finish returns at once; lets one
 * OS thread multiplex many connections (goroutines on GOMAXPROCS threads). */
int dm_stream_flush(dm_engine *e, uint64_t id);
/* Blocks until every byte is hashed.  digest_out receives the SHA-256 of
 * the bytes written.  *matched = 1 if expect was NULL or equals the digest
 * (the blob is then published in the CAS under digest_out), 0 otherwise (the
 * bytes are discarded).  The id is released either way.
 * Errors: DM_ESTATE (holes left by range parts), DM_ENOMEM, DM_ECUDA before the
 * final hash was started leave the stream open - call dm_stream_abort.  DM_ECUDA
 * after it (a copy or launch failed while the body was being hashed): *matched = 0,
 * nothing was cached, the id is released. */
int dm_stream_finish(dm_engine *e, uint64_t id, uint8_t digest_out[32], int *matched);
/* Upstream error / client went away: drop the partial blob, release the id. */
int dm_stream_abort(dm_engine *e, uint64_t id);

/* ---- hit serving: OnRequest short-circuit (start.go:197-200) ----------- */
int dm_cache_contains(dm_engine *e, const uint8_t digest[32], uint64_t *size);  /* DM_ENOENT on miss */
int dm_cache_open(dm_engine *e, const uint8_t digest[32], uint64_t *reader, uint64_t *size);
/* dm_cache_open that never serves a disk-tier blob it has not verified.  Returns at once, without waiting for a load.
 *   in HBM       exactly dm_cache_open (those bytes were verified when they entered HBM), LRU touch included
 *   disk only    the file is loaded into a fresh HBM extent and hashed there, as dm_cache_promote loads it, and the
 *                reader is served from that extent as the bytes land: the same bytes the kernel hashes, never a second
 *                read of the file.  *size is the file's size, checked against its sidecar.  The stream and its extent
 *                (evicting HBM LRU blobs) are set up on the calling thread; the file is read in and the verdict is
 *                collected by engine threads.  A load of the digest that is already running (another verified open, a
 *                dm_cache_promote) is followed instead: a digest is never loaded twice at once.
 * dm_cache_read on a reader whose load has no verdict yet blocks until bytes past `off` have landed in the extent, and
 * NO read returns byte size - 1, nor the EOF at off == size, before the verdict: a caller that sent Content-Length from
 * *size never completes a body that does not hash to its name (on an error it closes the connection, and the client
 * sees a short body).  A blob of at most 64 KiB travels in a pack and lands in HBM together with its verdict: every
 * read of it waits for the verdict.  Then:
 *   verified     the reader is an ordinary HBM reader (it pins the blob; dm_cache_device_extents works, dm_cache_meta
 *                returns the sidecar's text unchanged).  The blob stays in HBM, as if promoted, also when every reader
 *                closed before the verdict.  Before it, dm_cache_meta returns the sidecar read at open and
 *                dm_cache_device_extents DM_ESTATE
 *   mismatch     that read and every later one return DM_ECORRUPT (dm_error_detail(reader) says why); file and sidecar
 *                are removed if the path still names the file that was read, and the digest is a miss
 *   DM_EIO       the file could not be read or shrank; DM_ECUDA: a copy or launch failed.  The file is left untouched
 *                and the blob is not in HBM
 * Every outcome wakes blocked readers; dm_cache_close never aborts a load.  The load pins the digest against disk-tier
 * eviction until its verdict, and a verified load is a use of the blob.  bytes_hashed and h2d_bytes grow by the blob
 * once however many readers follow it; bytes_served by what they read.  dm_cache_follow does not see loads.
 * A load holds ring slabs only while it fills them: a reader that stops reading holds none, and no stream slot once the
 * verdict is in.
 * Errors (nothing is opened, the file is left untouched unless DM_ECORRUPT):
 *   DM_ENOENT    on neither tier (a body still being ingested too: dm_cache_follow attaches to those)
 *   DM_ECORRUPT  the file is not the size its sidecar states: file and sidecar removed
 *   DM_EIO       the file could not be opened
 *   DM_ENOMEM    larger than hbm_cas_bytes, no room even after LRU eviction, or no stream slot to spare (the budget
 *                dm_cache_promote, dm_cache_verify and dm_cache_import share): dm_cache_open still serves it, unverified
 *   DM_ESTATE    the engine has no HBM tier (DM_F_NO_HBM_CAS); DM_EINVAL: bad arguments
 * Verified serving finishes at one SHA-256 chain's rate per blob (DESIGN.md section 7), where dm_cache_open reads the
 * file at memory speed. */
int dm_cache_open_verified(dm_engine *e, const uint8_t digest[32], uint64_t *reader, uint64_t *size);
/* A verified hit that takes no HBM extent: for blobs larger than the arena, an arena with no room, and engines without
 * an HBM tier (DM_F_NO_HBM_CAS, with or without DM_F_DISK_DIRECT).  Returns at once, without waiting for a load.
 *   in HBM       exactly dm_cache_open (those bytes were verified when they entered HBM), LRU touch included
 *   disk only    a ring load starts: the file is read into pinned ring slabs by engine threads, copied from each slab
 *                to the device and hashed there as a check whose expected digest is the blob's name, as dm_cache_verify
 *                hashes it, at any size.  The reader copies its bytes straight out of those slabs: the bytes the kernel
 *                hashes, and the file is read once.  hbm_cas_used, the HBM LRU order and HBM contents do not change.
 *                *size is the file's size, checked against its sidecar.
 * Reads of a ring load's reader:
 *   - forward only.  The first dm_cache_read may start at any offset (a Range: request); after it, each read starts at
 *     or after the end of the previous one.  A read below that point returns DM_ESTATE (dm_error_detail(reader) says
 *     why).  The load always hashes from byte 0; slabs below the first read's offset go back as soon as they are hashed.
 *   - a read blocks until the slab holding `off` has been read back, and returns what is there (possibly less than
 *     `len`).  NO read returns byte size - 1, nor the EOF at off == size, before the verdict.
 *   verified     the remaining reads and EOF succeed.  Nothing is published or placed in HBM and the file stays as it
 *                is; the load counts as a use of the blob for disk-tier recency
 *   mismatch     that read and every later one return DM_ECORRUPT; file and sidecar are removed if the path still names
 *                the file that was read, and the digest is a miss
 *   DM_EIO       the file could not be read or shrank; DM_ECUDA: a copy or launch failed.  The file is left untouched
 * dm_cache_meta returns the sidecar text read at open; dm_cache_device_extents returns DM_ESTATE (there are no extents).
 * Each load holds at most 4 ring slabs (two being hashed, two the reader may still need): when the reader falls behind,
 * its load stops reading the file, and a stalled client slows its own load only, never the pump or other streams.  A
 * slab goes back to the ring once its job has been reaped and the reader has read past it, started beyond it, or closed.
 * dm_cache_close before the verdict stops the load: no further reads are issued, its slabs go back as their jobs are
 * reaped, and its stream slot is released.  Each ring open is a load of its own, not coalesced with other ring opens
 * or with HBM loads, and dm_cache_follow does not see it: bytes_hashed and h2d_bytes grow by the blob for every ring
 * open.  The load pins the digest against disk-tier eviction until its verdict and the reader keeps the pin until
 * dm_cache_close; dm_cache_remove of the digest returns DM_ESTATE while the load runs.
 * Errors (nothing is opened, the file is left untouched unless DM_ECORRUPT):
 *   DM_ENOENT    on neither tier
 *   DM_ECORRUPT  the file is not the size its sidecar states: file and sidecar removed
 *   DM_EIO       the file could not be opened
 *   DM_ENOMEM    ring loads already hold their share of the ring (a quarter of its slabs), or no stream slot to spare
 *                (the budget dm_cache_promote, dm_cache_verify and dm_cache_import share)
 *   DM_EINVAL    bad arguments
 * Like dm_cache_open_verified, the last byte arrives at one SHA-256 chain's rate per blob. */
int dm_cache_open_verified_ring(dm_engine *e, const uint8_t digest[32], uint64_t *reader, uint64_t *size);
/* dm_cache_open_verified_range: a verified hit on the byte range [off, off + len) of a blob (len = 0: to the end, as
 * Range: bytes=off- asks), for the parallel Range: requests in which clients fetch large blobs.  Every reader of a
 * disk-only blob is served by one SHA-256 check of the tier file shared with every other range reader it can serve,
 * instead of a ring load of its own.  *size is the whole blob's size.  Errors at open are dm_cache_open_verified_ring's,
 * plus DM_ERANGE when off > size or off + len > size (nothing is opened).
 *   in HBM       exactly dm_cache_open (LRU touch included), with reads kept within the range, in any order
 *   disk only    the reader is served by a shared ring load of the digest: a ring load (as above) whose read-back slabs
 *                serve every reader attached to it.  The open attaches to a shared load of the digest that has not
 *                failed and whose low-water mark is at most `off`: the end of the last slab the load gave back to the
 *                ring (0 before it gave any back), below which it no longer holds what it read (a load whose verdict
 *                is in only while the slabs it still holds cover the range).  When none can serve it, the open starts
 *                a new shared load, which hashes the file from byte 0 and which later opens may attach to.
 * Reads of a range reader:
 *   - within the range: a read below `off` or past off + len returns DM_ERANGE.  A read at off + len returns 0 bytes:
 *     the end of the range, and when off + len == size the blob's EOF, which waits for the verdict.
 *   - of a shared load's reader: forward only, as a ring load's reader's (DM_ESTATE), and blocking until the slab
 *     holding `off` has been read back.  NO read returns byte size - 1, nor the EOF at off == size, before the verdict.
 *     Verdicts are a ring load's, for every attached reader at once: on a match the remaining reads succeed and the
 *     load counts once as a use of the blob; on a mismatch every attached reader gets DM_ECORRUPT on that read and
 *     every later one, and file and sidecar are removed once; DM_EIO and DM_ECUDA as above.  Every outcome wakes every
 *     blocked reader.
 * Pacing: a slab of a shared load goes back to the ring once its job has been reaped and no attached, open reader
 * still needs it.  A reader needs the slabs that overlap the unread part of its range, [max(off, end of its previous
 * read), off + len): a reader whose range lies ahead of the load holds nothing and does not slow it.  The load as a
 * whole holds at most the 4 slabs of a ring load.
 * Detach: when the slab at a load's low-water mark has been held for a grace time (DESIGN.md §4) only by readers that
 * are not inside dm_cache_read, while another reader of the load waits for bytes, those stalled readers are detached,
 * provided a stream slot and ring share can be reserved for each of them at that moment (otherwise they keep pacing the
 * load).  A detached reader holds nothing of the old load, and its next read is served by a shared load started for it;
 * its last byte and EOF also wait for the verdict of the load it left, which keeps running until the reader closes.
 * dm_cache_close of one reader detaches it only; the load stops before its verdict only when its last reader closes.
 * dm_cache_meta returns the sidecar text read by the open that started the load; dm_cache_device_extents returns
 * DM_ESTATE.
 * Budget: each shared load takes one stream slot and a ring load's share of the ring, as a ring load does; a reader
 * that attaches takes neither, so DM_ENOMEM is returned only when a new load is needed and none can be reserved.
 * The digest is pinned against disk-tier eviction while a shared load of it runs, and each reader keeps its pin until
 * dm_cache_close; dm_cache_remove returns DM_ESTATE while a shared load runs.  bytes_hashed and h2d_bytes grow by the
 * blob once per shared load, bytes_served by what the readers read.  Shared loads and dm_cache_open_verified_ring loads
 * never attach to each other, and dm_cache_follow sees neither. */
int dm_cache_open_verified_range(dm_engine *e, const uint8_t digest[32], uint64_t off, uint64_t len,
                                 uint64_t *reader, uint64_t *size);
int dm_cache_read(dm_engine *e, uint64_t reader, uint64_t off, void *buf, size_t len, size_t *nread);
/* The blob's sidecar as JSON text: {"digest":"sha256:..","size":N,"encoding":"identity",
 * ..,"headers":{..}}.  *len receives the full length; up to cap-1 bytes + NUL are copied. */
int dm_cache_meta(dm_engine *e, uint64_t reader, char *buf, size_t cap, size_t *len);
int dm_cache_close(dm_engine *e, uint64_t reader);
int dm_cache_evict(dm_engine *e, const uint8_t digest[32]);   /* HBM tier only; disk copy stays */
/* dm_cache_remove flags */
#define DM_RM_ALIASES 0x1u   /* also delete every alias whose digest is removed (logged as tombstones, see the aliases) */
#define DM_RM_PARTIAL 0x2u   /* also delete a download of the digest saved by dm_stream_suspend */
/* Remove blobs from the cache on request: the operator's delete (a model nobody uses, a superseded revision, a
 * repository that must stop being served, a bad upload).  Blocks until every status is known; duplicates in digests[]
 * are handled once.  status_out[i]:
 *   DM_OK        removed from every tier that held it (rules below)
 *   DM_ENOENT    on neither tier, and no saved download under DM_RM_PARTIAL (its aliases still go under DM_RM_ALIASES)
 *   DM_ESTATE    something is placing or loading the digest right now, and nothing of it is removed: retry later.
 *                dm_error_detail(e, 0) names the first such digest and what holds it: a stream opened with it as its
 *                expected digest (HBM, verify-only or disk-backed, until dm_stream_finish / dm_stream_abort returns), a
 *                running load (dm_cache_open_verified, dm_cache_promote), a running dm_cache_verify or dm_cache_import
 *                that holds it, a DM_ING_REPLACE re-ingest of it in a running dm_ingest_device, or a
 *                dm_stream_resume_saved taking its saved download over
 *   DM_EIO       an unlink failed with something other than ENOENT: what was already removed stays removed, and the
 *                engine's indexes (HBM, disk-tier limit) match what is left on disk; dm_error_detail(e, 0) says which
 * HBM copy: leaves the index and the LRU order at once, so dm_cache_contains, dm_cache_open, dm_cache_open_verified,
 * dm_cache_follow and dm_cache_promote miss from then on.  Readers that have it open keep reading the same extent until
 * dm_cache_close (dm_cache_device_extents on them stays valid); the extent is freed, and hbm_cas_used drops, when the
 * last of them closes.  (dm_cache_evict instead refuses while readers are open.)  A queued spill of the blob is
 * dropped; a running one finishes its .part and unlinks it instead of renaming it into place: no file of the digest
 * appears under blobs/ after DM_OK.
 * Disk copy: the blob file is unlinked, then its sidecar.  Readers that hold a descriptor (dm_cache_open, a follower of
 * a completed disk-backed body) keep reading it.  With a disk-tier limit, used_bytes falls by the file and its sidecar;
 * evicted_files, evicted_bytes and refused do not move (a removal is not an eviction).
 * DM_RM_PARTIAL: <hex>.ckpt, then <hex>.part under partial/ are unlinked; dm_stream_resume_saved is DM_ENOENT for the
 * digest afterwards and dm_stats.suspended drops.
 * Not a ban: a new download, an import, a promotion of a re-imported file or dm_ingest_device may cache the digest
 * again, as may a stream opened without an expected digest whose bytes hash to it.  blobs_committed,
 * blobs_mismatched and the byte counters do not move.
 * Returns DM_OK once every status is filled; DM_EINVAL on bad arguments or unknown flags.  Without cas_dir only the
 * HBM tier is looked at (DM_RM_PARTIAL finds nothing).  One digest at a time holds the disk tier's lock (see
 * dm_cache_set_disk_limit) for its unlinks. */
int dm_cache_remove(dm_engine *e, const uint8_t *digests, uint32_t n, uint32_t flags, int32_t *status_out);
/* Bring cached blobs back into HBM, verifying each disk copy on the GPU as it loads.  A blob leaves HBM when it is
 * evicted or the engine restarts, and dm_cache_open serves it from <cas_dir>/blobs/ from then on, unverified and
 * without dm_cache_device_extents (dm_cache_open_verified loads it the same way on a hit).  This reads each file into the pinned ring, DMAs it into a fresh HBM extent and
 * hashes it there as an ordinary stream with the digest as its expected value; many files load at once, so their
 * hash chains share launches.  Blocks until every status is known.  status_out[i]:
 *   DM_OK        it was in HBM when the call looked, or its disk copy was loaded and hashed to digests[i].  HBM is
 *                an LRU cache: a call over more bytes than hbm_cas_bytes evicts blobs it promoted earlier to make
 *                room for later ones (they stay DM_OK, and stay on disk), as any other ingest may evict them later
 *   DM_ENOENT    on neither tier
 *   DM_ENOMEM    larger than hbm_cas_bytes, no room even after LRU eviction, or no stream slot to spare (see
 *                below): left on disk, untouched
 *   DM_EIO       the file could not be read: left untouched
 *   DM_ECUDA     a copy or launch failed while it loaded: left untouched, not in HBM
 *   DM_ECORRUPT  the disk copy does NOT hash to its name (or is shorter / longer than its sidecar says):
 *                file and sidecar removed, the digest is now a miss
 * A file is removed only if its path still names the file that was read (one a stream published meanwhile stays).
 * A disk reader that opened a corrupt file before keeps its descriptor and reads what the file holds.  The file and
 * sidecar of a verified blob stay as they are (nothing is written back), and dm_cache_meta returns the sidecar's text
 * unchanged; a blob without a sidecar is promoted with no headers.  Duplicates in digests[] are loaded once, and a
 * digest whose load is already running (dm_cache_open_verified, another promotion) is not loaded again: its status is
 * that load's verdict, waited for.  The
 * call opens at most half of the stream slots that are free when it starts and not reserved by other running calls,
 * so it never takes the last one from dm_stream_open; with fewer than two such slots it loads nothing, and each blob
 * it would have loaded is DM_ENOMEM.
 * Returns DM_OK once every status is filled; DM_EINVAL on bad arguments; DM_ESTATE on a DM_F_NO_HBM_CAS engine
 * (there is no HBM tier).  Without cas_dir every blob not already in HBM is DM_ENOENT. */
int dm_cache_promote(dm_engine *e, const uint8_t *digests, uint32_t n, int32_t *status_out);
/* Check disk-tier copies in place: hash each file <cas_dir>/blobs/sha256/<aa>/<hex> on the GPU and compare the result
 * with its name, at any size, with or without an HBM tier (DM_F_NO_HBM_CAS) or DM_F_DISK_DIRECT.  Nothing goes into
 * the HBM arena: hbm_cas_used, the LRU order and what is cached in HBM stay as they are.  Each file is read back
 * through the pinned ring by the engine's disk threads, as a disk-backed stream reads its own file; files of at most
 * 64 KiB share pack DMAs and launches.  Blocks until every status is known.  status_out[i]:
 *   DM_OK        the file exists, has the size its sidecar states and hashes to digests[i]; or there is no file but
 *                the blob is in HBM (its spill is pending, or there is no cas_dir): that copy was verified at ingest
 *   DM_ENOENT    on neither tier
 *   DM_ECORRUPT  the file does NOT hash to its name, or its size is not its sidecar's "size": file and sidecar removed
 *                (only if the path still names the file that was read).  A blob that is also in HBM is written to the
 *                disk tier again from its verified HBM copy; otherwise the digest is now a miss
 *   DM_EIO       the file could not be opened or read: left untouched
 *   DM_ECUDA     a copy or launch failed: left untouched
 *   DM_ENOMEM    no stream slot to spare (the same budget as dm_cache_promote, shared with it): left untouched
 * A file is checked even when the blob is also in HBM.  Nothing is published, renamed, rewritten or logged;
 * blobs_committed and blobs_mismatched do not move, bytes_hashed and h2d_bytes grow by the bytes checked.
 * Duplicates in digests[] are checked once.  At most a quarter of the ring's slabs' worth of files are in flight at
 * once (each holds at most two slabs), so live streams keep the rest of the ring.
 * Returns DM_OK once every status is filled; DM_EINVAL on bad arguments. */
int dm_cache_verify(dm_engine *e, const uint8_t *digests, uint32_t n, int32_t *status_out);
/* Blobs in the disk tier in ascending digest order, strictly after `after` (NULL: from the start).  Up to cap
 * entries; *n_out < cap means the listing is complete.  sizes_out may be NULL.  Stateless: page by passing the last
 * digest returned.  Only files named by 64 lowercase hex digits in their own <aa>/ directory are listed (no sidecars,
 * no partial files); a file removed between the directory read and its stat is skipped.  Without cas_dir: *n_out = 0.
 * Host code only: "check the whole tier" is dm_cache_list, then dm_cache_verify on each page. */
int dm_cache_list(dm_engine *e, const uint8_t after[32], uint8_t *digests_out, uint64_t *sizes_out,
                  uint32_t cap, uint32_t *n_out);
/* dm_cache_import flags */
#define DM_IMP_LINK 0x1u   /* hard-link instead of copy when the source is on cas_dir's filesystem */
/* Seed the disk tier from files already on the host (a HuggingFace hub cache, an Ollama models directory, a copy of
 * another node's cache): each file is hashed on the GPU and placed at <cas_dir>/blobs/sha256/<aa>/<hex>.
 *   paths[i]     a regular file; symlinks are followed (HuggingFace snapshots are symlinks into blobs/)
 *   expect       NULL, or n x 32 bytes: row i is the SHA-256 paths[i] must hash to, all zero when it is not known
 *   keys         NULL, or n nullable strings: when entry i ends DM_OK, keys[i] is entered in the alias index under its
 *                digest exactly as dm_cache_alias_put does, on this engine (the one that now holds the blob)
 *   flags        DM_IMP_LINK: hard-link the source into the cache instead of copying it (falls back to a copy when
 *                the link fails with EXDEV or EPERM, or when the source was renamed over after it was opened).  The
 *                tier file then shares the source's inode: a later in-place
 *                change of the source changes the cached bytes, which only dm_cache_verify would notice
 * Each source is first staged as a private file <cas_dir>/incoming/<pid>-<device>-<id>.part (copy_file_range, a
 * reflink on XFS and btrfs, with a pread / pwrite fall-back), and that file is what the GPU hashes, through the ring as
 * dm_cache_verify reads a tier file (files of at most 64 KiB share pack DMAs and launches), and what is renamed into
 * the tier: a source that changes while it is copied cannot put bytes in the tier that were never hashed.  The blob is
 * given a sidecar with its digest and size and no response headers, and registered as on the disk tier only.
 * Nothing goes into HBM: hbm_cas_used and the LRU order stay as they are (dm_cache_promote loads blobs later).
 * Blocks until every status is known.  status_out[i] (digests_out[i] is 32 zero bytes unless stated):
 *   DM_OK        in the disk tier now, imported or already there; digests_out[i] is its SHA-256.  An entry whose
 *                digest is known and already on either tier is DM_OK at once: nothing is read, copied or hashed
 *   DM_ECORRUPT  it does not hash to expect[i]; nothing is cached, digests_out[i] is what it hashed to
 *   DM_ENOENT    no such file
 *   DM_EINVAL    not a regular file
 *   DM_EIO       the source could not be read, or the copy could not be written, renamed or given its sidecar
 *   DM_ECUDA     a copy or launch failed
 *   DM_ENOMEM    no stream slot to spare (the budget of dm_cache_promote and dm_cache_verify, shared with them), or
 *                no room for it under the disk-tier limit (dm_cache_set_disk_limit)
 * After any of these the source is untouched, bytes and inode, and <cas_dir>/incoming/ holds nothing of the call.
 * Duplicate entries (same path and expect row) are imported once; each gets the status, digest and its own alias.
 * Threads, slot budget and ring share are dm_cache_verify's.  bytes_hashed and h2d_bytes grow by the bytes hashed,
 * blobs_committed by the blobs newly placed; bytes_ingested and blobs_mismatched do not move.
 * Each call first removes the files under <cas_dir>/incoming/ of processes that are gone, as dm_engine_create does
 * under DM_F_DISK_DIRECT: engines that import must not share a cas_dir across PID namespaces either.
 * Returns DM_OK once every status is filled; DM_EINVAL on bad arguments (a null path, a key that dm_cache_alias_put
 * would refuse, an unknown flag); DM_ESTATE without cas_dir. */
int dm_cache_import(dm_engine *e, const char *const *paths, const uint8_t *expect, const char *const *keys,
                    uint32_t n, uint32_t flags, uint8_t *digests_out, int32_t *status_out);
/* Write cached blobs to files the caller names, each checked on the GPU on its way out: the other half of
 * dm_cache_import (an air-gapped copy, a client's Ollama models directory or HuggingFace hub cache, a second node's
 * cache, a backup).  Works with or without cas_dir and with DM_F_NO_HBM_CAS.
 *   digests      n x 32 bytes
 *   dest_paths   n file names; missing parent directories are created
 * Entry i is copied from its HBM extent (verified at ingest; a reader reference holds it while it is copied out) or,
 * when not in HBM, from its disk-tier file (copy_file_range, a reflink on XFS and btrfs; the digest is pinned against
 * disk-tier eviction meanwhile) into a private file next to the destination, <dir>/.<basename>.dm-export-<pid>-<id>.part,
 * created with O_EXCL.  That file is hashed on the GPU as dm_cache_import hashes its staged copy, through the ring
 * (files of at most 64 KiB share pack DMAs and launches), and renamed over dest_paths[i] only when it hashed to
 * digests[i]: a destination that already exists is replaced atomically (a reader that had it open keeps the old bytes).
 * On a DM_F_DISK_SYNC engine the file is fsynced before the rename and its directory after it.  On any other outcome
 * the staged file is unlinked and dest_paths[i] is left as it was.  Blocks until every status is known.  status_out[i]:
 *   DM_OK        dest_paths[i] holds the blob, and those bytes hashed to digests[i] on the GPU
 *   DM_ENOENT    on neither tier (a body still being ingested is not cached yet)
 *   DM_ECORRUPT  the copy did not hash to its name, or the tier file is not its sidecar's size.  Nothing is written at
 *                dest_paths[i], and the cache is NOT touched: dm_cache_verify decides about the tier file
 *                (dm_error_detail(e, 0) says so)
 *   DM_EIO       the source could not be read, or the staged file could not be created, written, synced or renamed
 *                (a destination that names a directory is one)
 *   DM_ECUDA     a copy or launch failed
 *   DM_ENOMEM    no stream slot to spare (the budget dm_cache_promote, dm_cache_verify and dm_cache_import share)
 * Duplicate (digest, destination) pairs are exported once; each copy gets the status.
 * The cache is only read: HBM contents, hbm_cas_used, the LRU order, disk-tier recency (the tier file's mtime), the
 * disk-tier limit's accounting, blobs_committed, blobs_mismatched and bytes_ingested stay as they are.  bytes_hashed
 * and h2d_bytes grow by the bytes checked, d2h_bytes by the bytes copied out of HBM.
 * While a call holds a digest (from its source copy until its verdict) dm_cache_remove of it returns DM_ESTATE.
 * Threads, slot budget and ring share (a quarter of the ring) are dm_cache_verify's, so live streams keep the rest.
 * Each call first removes, from the directories it writes to, the staged files of processes that are gone.
 * Returns DM_OK once every status is filled; DM_EINVAL for a null argument or path, or for one destination named with
 * two different digests (nothing is done then). */
int dm_cache_export(dm_engine *e, const uint8_t *digests, const char *const *dest_paths, uint32_t n,
                    int32_t *status_out);
/* Keep the disk tier under a size limit.  Opt-in: an engine that never sets one touches, scans and reserves nothing.
 * Bytes are apparent sizes (st_size) of the regular files under <cas_dir>/blobs/, incoming/ and partial/
 * (aliases.log is not counted).  A hard-linked import (DM_IMP_LINK) counts at its full size although its inode is
 * shared with the source.  With a limit set, a cas_dir belongs to ONE engine (the Go pool gives each GPU <dir>/gpu<N>).
 * The limit is not a free-space guard: other writers on the filesystem are not seen.
 *
 * dm_cache_set_disk_limit: limit_bytes = 0 turns the limit off again (the index is dropped).  The first call with a
 * non-zero limit builds the disk index synchronously: one walk of blobs/, incoming/ and partial/ with one stat per name
 * (the walk dm_cache_list does), which also removes spill leftovers (<hex>.part under blobs/ with no spill of this engine
 * running), sidecars whose blob file is missing and incoming/ files of processes that are gone.  Every call then evicts
 * until used_bytes <= limit_bytes or only pinned entries are left, and returns DM_OK either way (dm_cache_disk_usage
 * shows which).  DM_ESTATE without cas_dir.  The walk and each eviction's unlinks run under the tier's lock, which
 * disk-tier opens (dm_cache_open of a blob not in HBM) and spills also take for their pins, with or without a limit:
 * they wait for the first walk (about 4 s per 100 000 files on tmpfs) and for the evictions of a placement.
 *
 * Recency.  Entries - blobs (file + sidecar) and saved downloads (.ckpt + .part) - are evicted least recently used
 * first.  A use is a placement (spill, disk-backed publish, import), dm_cache_open served from disk, dm_cache_promote
 * returning DM_OK, and a blob leaving HBM.  dm_cache_verify, dm_cache_list, dm_cache_contains and an import that finds
 * the digest already cached are not uses.  The last use is stored as the blob file's mtime (written explicitly; reads
 * never move it), so the order survives a restart; files with more than one link keep their recency in memory only,
 * since writing their mtime would modify an import's source.  HBM-resident blobs rank above every disk-only entry: their
 * disk copies go only after every evictable disk-only entry, in HBM LRU order, and such a blob stays servable from HBM
 * and is dropped when it leaves HBM (it is not written to disk again).
 *
 * Room.  Each placement reserves its bytes before they reach the disk, evicting as needed.  When no room can be made:
 *   spill of an HBM blob (size + sidecar)     skipped, as after a failed spill (DM_F_DISK_SYNC finish: DM_EIO); refused++
 *   disk-backed stream with size_hint         opens verify-only: verified, not cached, no file in incoming/; refused++.
 *                                             Once open its room is kept: it is placed at publish even if unknown-size
 *                                             bodies have run the tier over the limit meanwhile (not if the limit has
 *                                             been lowered below its size)
 *   disk-backed stream of unknown size        never failed by the limit: charged as it is written and may run over the
 *                                             limit while live (the overshoot is bounded by the unknown-size disk-backed
 *                                             bodies in flight).  At publish its final size must fit: if not, the file is
 *                                             removed, dm_stream_finish returns DM_OK with *matched as the digest says,
 *                                             nothing is cached; refused++
 *   dm_cache_import staging copy (its size)   DM_ENOMEM for that entry: the source is untouched, nothing in incoming/
 *   dm_stream_suspend of an HBM stream        DM_ENOMEM, the stream stays open
 *   suspend / resume of a disk-backed stream  nothing new: its bytes move between incoming/ and partial/ (a resumed
 *                                             stream makes room for its size_hint less the bytes saved)
 *
 * Pins: never evicted while a disk reader has the blob open (until dm_cache_close), while a dm_cache_promote,
 * dm_cache_verify or dm_cache_import call holds the digest, while a disk-backed stream publishes it or a spill writes
 * it, and while dm_stream_resume_saved takes a saved download over.  Evicting a blob removes its file, then its sidecar;
 * its aliases stay (dm_cache_open then misses).  Evicting a saved download removes .ckpt, then .part; a later
 * dm_stream_resume_saved for it is DM_ENOENT.  A reader that opened a file just before its eviction keeps reading its
 * descriptor.  A follower of a disk-backed body (dm_cache_follow) pins the blob as a disk reader from its EOF read on. */
typedef struct dm_disk_usage {
    uint32_t struct_size;      /* = sizeof(dm_disk_usage); ABI guard */
    uint32_t reserved;
    uint64_t limit_bytes;      /* 0 = no limit (the default) */
    uint64_t used_bytes;       /* blob_bytes + staging_bytes + partial_bytes */
    uint64_t blob_files;       /* blobs in blobs/sha256/ */
    uint64_t blob_bytes;       /* their files + sidecars, plus spills being written (at their reservation) */
    uint64_t staging_bytes;    /* incoming/: disk-backed streams and import copies, at max(reservation, written) */
    uint64_t partial_bytes;    /* partial/: downloads saved by dm_stream_suspend (.ckpt + .part) */
    uint64_t evicted_files;    /* blobs and saved downloads removed to stay under the limit, since create */
    uint64_t evicted_bytes;
    uint64_t refused;          /* placements skipped because no room could be made (see above) */
} dm_disk_usage;
int dm_cache_set_disk_limit(dm_engine *e, uint64_t limit_bytes);
/* DM_EINVAL on a wrong struct_size.  Without a limit set: limit_bytes = 0, the three counters, zero for the rest (it
 * never walks the directory by itself). */
int dm_cache_disk_usage(dm_engine *e, dm_disk_usage *out);
/* Request coalescing: the blob is not cached yet but another connection is
 * ingesting it right now (a stream opened with this expected digest; the first
 * one opened is followed).  The reader follows that body out of HBM:
 * dm_cache_read blocks until bytes past `off` have arrived, and once the body
 * completes and verifies the reader becomes an ordinary cache reader.  If the
 * body is aborted or fails verification, reads fail with DM_ESTATE.
 * DM_ENOENT: nothing in flight, or a stream that retains nothing to serve (a
 * verify-only stream: DM_F_NO_HBM_CAS or over-arena without DM_F_DISK_DIRECT,
 * or a disk-backed open the disk-tier limit refused).
 * *size_hint = the Content-Length the ingesting stream was opened with (0 = unknown).
 * A body the GPU hashes once is read by any number of followers.
 *
 * Disk-backed bodies (DM_F_DISK_DIRECT), from dm_stream_open on, and from byte 0 again once dm_stream_resume_saved
 * has taken a saved download over (its file holds the saved prefix):
 *   - the follower keeps a descriptor of the body's file of its own (a body whose file is being renamed into the tier
 *     at that moment is opened as dm_cache_open opens it), and dm_cache_read blocks until `off` lies in a
 *     range whose file write has completed, then reads from the file straight into buf, up to the end of that range.
 *     Range parts are served as they land: a reader inside a later part does not wait for the prefix.
 *   - the read at EOF (off = the size, known or final) returns once the verdict is in: after the GPU has hashed the
 *     whole file, which for one body runs at one hash chain's rate (tens of MB/s).  Verified, the reader is an
 *     ordinary disk-tier reader of its descriptor: dm_cache_meta returns the published sidecar and, when the blob was
 *     placed in the tier, the blob is pinned against disk-tier eviction until dm_cache_close, as a dm_cache_open
 *     reader's is.  A verified body that was not placed (no room under the limit, or the tier already had it) is still
 *     read to the end from the descriptor.
 *   - an abort, a mismatch, a failed file write (DM_EIO), a failed copy or launch and dm_stream_suspend wake blocked
 *     followers; their reads return DM_ESTATE, and dm_error_detail(reader) says which it was.  A read that would
 *     return bytes past a suspend's cut returns DM_ESTATE too, never short data.  Follow again after
 *     dm_stream_resume_saved.
 *   - nothing a follower holds delays an abort, a publication or a suspend.  Its descriptor of a file that is
 *     unlinked or evicted later keeps the bytes readable and is not counted by the disk-tier limit, as an open disk
 *     reader's is not.
 *   - bytes_served grows by what followers read; bytes_hashed and h2d_bytes by the body once.  open_readers counts
 *     followers. */
int dm_cache_follow(dm_engine *e, const uint8_t digest[32], uint64_t *reader, uint64_t *size_hint);

/* URL -> digest index for the OnRequest hit check (start.go:197-200 hands the hook a request, not a
 * digest).  OCI blob URLs carry `sha256:<hex>`; HuggingFace `resolve/<rev>/<file>` URLs (the first clients
 * demodel/README.md:16-21 lists) do not.  The tee records URL (or ETag / LFS oid string) -> digest
 * when a body verifies; a later request for the same key is answered from the CAS.  `key` is any
 * NUL-terminated string up to 4096 bytes.  With cas_dir the index is an append-only log
 * (<cas_dir>/aliases.log) replayed by dm_engine_create; a put for an existing key replaces it.
 * dm_cache_alias_get: DM_ENOENT when the key is unknown (the digest may since have been evicted from both
 * tiers: dm_cache_open decides).
 * dm_cache_alias_del: DM_OK, or DM_ENOENT when the key is unknown.  A deletion (and each alias DM_RM_ALIASES deletes)
 * is appended to the log as a tombstone line "-\t<key>", and replay applies the lines in order.  Tombstones and the
 * lines they deleted count as dead when the log is compacted at start.  An engine of an older build skips tombstone
 * lines as unreadable, so a deleted alias comes back if the cache is downgraded.
 * dm_cache_alias_list: keys starting with `prefix` ("" or NULL = all), in ascending byte order, strictly after `after`
 * (NULL = from the start).  Keys are copied NUL-terminated back to back into keys[keys_cap]; digests_out[i] is key i's
 * digest.  Stops at cap entries or when the next key does not fit; *more = 1 if anything was left out.  Stateless,
 * like dm_cache_list: page by passing the last key returned.  The index is ordered by key, so a page costs
 * O(log n + page) at any number of aliases. */
int dm_cache_alias_put(dm_engine *e, const char *key, const uint8_t digest[32]);
int dm_cache_alias_get(dm_engine *e, const char *key, uint8_t digest_out[32]);
int dm_cache_alias_del(dm_engine *e, const char *key);
int dm_cache_alias_list(dm_engine *e, const char *prefix, const char *after, char *keys, size_t keys_cap,
                        uint8_t *digests_out, uint32_t cap, uint32_t *n_out, int *more);

/* ---- device-resident ingest -------------------------------------------- */
/* Hash-and-cache n blobs whose bytes are ALREADY in this GPU's HBM (landed
 * by GPUDirect, produced on device, or the bench's "inputs resident" leg).
 * Blob i occupies [dev_base + offsets[i], dev_base + offsets[i] + lengths[i]);
 * every offsets[i] must be a multiple of 16 and the blobs must not overlap.
 * expect (n*32 bytes) may be NULL.
 * One fused kernel pass reads each byte once, advances its blob's SHA-256
 * state and writes the byte into the blob's CAS extent.  digests_out gets
 * n*32 bytes; matched_out (n bytes, optional) the per-blob verdicts.
 * kernel_ms (optional) = CUDA-event time of the hash launches on the
 * engine's own stream(s): a batch of 32 768 or more small blobs goes out as
 * up to 8 launches on as many streams, so that extents, verdicts and index
 * updates of one part overlap the kernel of another; kernel_ms then runs
 * from the first launch to the end of the last.  flags: DM_ING_* below. */
#define DM_ING_HASH_ONLY   0x1u   /* do not copy into the CAS (1 B/B of traffic instead of 2) */
#define DM_ING_REPLACE     0x2u   /* re-ingest: a cached blob with an expected digest is taken out of sight for the
                                   * call and - when it has no reader - its extent is rewritten in place */
#define DM_ING_FORCE_WIDE  0x4u   /* kernel selection override: lane-per-stream */
#define DM_ING_FORCE_DEEP  0x8u   /* kernel selection override: warp-per-stream */
#define DM_ING_SPW_SHIFT   8      /* kernel selection override: (log2(streams per warp) + 1) << 8, */
#define DM_ING_SPW_MASK    0x700u /*   i.e. 1..6 for 1, 2, 4, 8, 16, 32 streams per warp          */
int dm_ingest_device(dm_engine *e, const void *dev_base, const uint64_t *offsets,
                     const uint64_t *lengths, uint32_t n, const uint8_t *expect, uint8_t *digests_out, uint8_t *matched_out,
                     uint32_t flags, double *kernel_ms);

/* Device pointer + extent walk of a cached blob, for consumers that want the
 * bytes in HBM (e.g. a weight loader on the same GPU).  Returns the number
 * of extents; fills up to max_ext (dev_ptr, len) pairs. */
int dm_cache_device_extents(dm_engine *e, uint64_t reader, void **dev_ptrs, uint64_t *lens, uint32_t max_ext);

/* ---- manifest-aware prefetch (SURVEY.md §8f-4) --------------------------- */
/* An OCI / Ollama image manifest (shape: the reference's cached fixture,
 * CONTRIBUTING.md:128-153) lists every blob with digest and size before the
 * bodies are requested. */
typedef struct dm_layer {
    uint8_t  digest[32];
    uint64_t size;
    char     media_type[96];   /* NUL-terminated, truncated if longer */
} dm_layer;
/* Collects every descriptor (object with a "sha256:" digest and an integer
 * size) in document order: config first, then layers.  *n_layers receives the
 * total found even if it exceeds max_layers.  DM_EINVAL on malformed JSON. */
int dm_manifest_parse(const char *json, size_t len, dm_layer *out, uint32_t max_layers, uint32_t *n_layers);
/* Pre-open one stream per layer that is not already cached, carrying its
 * expected digest and size (so its extent is reserved and the body is verified
 * as it arrives).  ids[i] = 0 for layers that are cache hits or duplicates. */
int dm_manifest_prefetch(dm_engine *e, const dm_layer *layers, uint32_t n, uint64_t *ids);
/* Registries answer manifest requests with `Content-Encoding: gzip` when the client allows it - the one
 * cached body the reference documents is such a response (CONTRIBUTING.md:76-99,116).  Inflates a gzip
 * (RFC 1952) or raw-deflate-in-zlib (RFC 1950) body of `len` bytes into dst[cap]; *out_len = inflated size.
 * DM_EINVAL: malformed stream or CRC / length mismatch; DM_ENOMEM: cap too small (*out_len = needed size
 * when the trailer states it).  Pure host code; manifests are a few KiB. */
int dm_gunzip(const void *src, size_t len, void *dst, size_t cap, size_t *out_len);

/* ---- synthetic blob bytes (SURVEY.md §8d) ------------------------------ */
/* Counter-based generator: byte j of blob `blob` under `seed` is a pure
 * function of (seed, blob, j); host and device versions agree bit for bit. */
void dm_synth_fill_host(uint64_t seed, uint64_t blob, uint64_t byte_off, void *dst, size_t len);
int  dm_synth_fill_device(dm_engine *e, uint64_t seed, uint64_t blob, uint64_t byte_off,
                          void *dev_dst, size_t len);
/* Fill n blobs laid out by offsets[]/lengths[] (as in dm_ingest_device, offsets
 * ascending) in one launch; blob i gets generator index first_blob + i. */
int  dm_synth_fill_device_many(dm_engine *e, uint64_t seed, uint64_t first_blob, void *dev_base,
                               const uint64_t *offsets, const uint64_t *lengths, uint32_t n);

/* ---- proxy-side driver (the host half of the path, in-process) --------- */
/* What the Go side does per connection, restated in C++ threads so the
 * end-to-end path can be driven here, where no Go toolchain exists:
 * `nthreads` connection workers each pull whole blobs from a shared queue,
 * read them in `chunk`-byte pieces from caller-owned HOST memory
 * [host_base + offsets[i], host_base + offsets[i+1]) and push them through
 * dm_stream_open/write/finish.  zero_copy selects how: 0 copy + non-blocking
 * EOF (flush), 1 acquire/commit with the "socket read" landing directly in the
 * ring, 2 / 3 the blocking io.ReadCloser forms of 0 / 1 (one body per thread at
 * a time), 4 as 2 but the client disconnects half way (Close before EOF:
 * matched_out[i] = 2, nothing is published).  Streams are interleaved
 * `concurrency` at a time the way concurrent goroutines would be.
 * Returns wall seconds in *seconds. */
int dm_proxy_drive(dm_engine *e, const void *host_base, const uint64_t *offsets, uint32_t n,
                   const uint8_t *expect, size_t chunk, uint32_t concurrency, int nthreads,
                   int zero_copy, uint8_t *digests_out, uint8_t *matched_out, double *seconds);
/* Serve n cached blobs back out into caller-owned host memory in `chunk`
 * pieces (the cache-hit path), `nthreads` readers. */
int dm_proxy_serve(dm_engine *e, const uint8_t *digests, uint32_t n, void *host_base,
                   const uint64_t *offsets, size_t chunk, int nthreads, double *seconds);

/* Single-connection twins of the two hooks for callers that work with URLs (demodel_b200/csrc/proxy_hooks.hpp:
 * BodyTee::SetURL, HitReader(url), ManifestTee).
 * dm_proxy_fetch: the OnResponse tee for one body fetched under `url`; expect may be NULL (HuggingFace resolve/
 * URL: digest unknown until hashed).  A verified body is entered in the alias index under the URL.
 * dm_proxy_request: the OnRequest check - a digest in the URL (OCI `sha256:<hex>`) or the alias index.
 * DM_ENOENT = miss; DM_OK = *reader is an open cache reader over *size bytes.
 * dm_proxy_manifest: the OnResponse tee for a manifest response, Content-Encoding "gzip" or identity (NULL):
 * passes the body through, inflates, parses, prefetches.  Up to max_layers entries are returned. */
int dm_proxy_fetch(dm_engine *e, const char *url, const void *body, uint64_t len, const uint8_t *expect,
                   size_t chunk, uint8_t digest_out[32], int *matched_out);
int dm_proxy_request(dm_engine *e, const char *url, uint64_t *reader, uint64_t *size);
int dm_proxy_manifest(dm_engine *e, const void *body, uint64_t len, const char *content_encoding, size_t chunk,
                      dm_layer *layers_out, uint64_t *ids_out, uint32_t max_layers, uint32_t *n_layers);

#ifdef __cplusplus
}
#endif
#endif /* DEMODEL_B200_H */
