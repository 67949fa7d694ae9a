// The blob hash-and-cache engine behind include/demodel_b200.h.
//
// Data path (DESIGN.md §4):
//
//   dm_stream_write ──memcpy──▶ pinned ring slab ──one H2D DMA per slab──▶ the blob's
//   (many threads)              (per stream)        (copy streams)         CAS extent in HBM
//                                                                               │
//   pump thread: gathers the streams with unhashed bytes into a job table       ▼
//   (one slab-sized job per stream, at most one in flight per stream) and  sha256_{deep,group,wide}
//   launches ONE multi-buffer SHA-256 kernel over them; up to 8 launches   (reads each byte once)
//   overlap on separate CUDA streams, each ordered after the DMAs by an
//   event.  Finished streams get their digest through mapped pinned memory,
//   are compared with the expected oid and published in the CAS index; spill
//   threads write published blobs to the disk tier with D2H copies on side
//   streams; readers (hits, followers of in-flight bodies) copy out through
//   pinned read-ahead windows.
//
// The bytes land at their final CAS address straight from the DMA, so the
// ring path costs HBM one write (DMA) + one read (hash) per blob byte.  The
// device-resident path (dm_ingest_device) fuses the copy into the hash kernel.
//
// Lock order (outer → inner): reader.mu → stream.mu → {arena_mu, e->mu, work_mu};
// slab_mu → work_mu; stripe / reader-stripe mutexes are leaves taken alone.
// The pump never holds work_mu while taking a stream mutex.
//
// Reference hooks served: cmd/demodel/start.go:201-204 (ingest) and
// start.go:197-200 (hit serving); see include/demodel_b200.h.
#include "engine_internal.hpp"

#include <dirent.h>

#if defined(__x86_64__)
#include <emmintrin.h>
#endif

namespace dmi {

thread_local std::string g_last_error;

// Socket buffer -> ring slab.  The ring is written once by the CPU and read once by the DMA engine, never
// by a core, so an ordinary store stream costs a read-for-ownership of every destination line (3 memory
// transfers per byte instead of 2) and evicts the proxy's working set.  Pieces of at least nt_copy_min
// bytes go out as streaming (non-temporal) stores: tools/ubench/ntcopy.cc, +18 % (1 thread) to +55 %
// (4 threads) on 32 KiB pieces; slower for 4 KiB pieces, hence the threshold.  The fence orders the
// write-combining buffers before anything that can make the DMA engine read the slab.
void ring_copy(dm_engine *e, void *dst, const void *src, size_t n)
{
#if defined(__x86_64__)
    if (e->nt_copy_min && n >= e->nt_copy_min) {
        uint8_t *d = static_cast<uint8_t *>(dst);
        const uint8_t *s = static_cast<const uint8_t *>(src);
        size_t head = (size_t)((16 - ((uintptr_t)d & 15)) & 15);
        if (head) { memcpy(d, s, head); d += head; s += head; n -= head; }
        size_t i = 0;
        for (; i + 64 <= n; i += 64) {
            const __m128i a = _mm_loadu_si128((const __m128i *)(s + i)), b = _mm_loadu_si128((const __m128i *)(s + i + 16));
            const __m128i c = _mm_loadu_si128((const __m128i *)(s + i + 32)), f = _mm_loadu_si128((const __m128i *)(s + i + 48));
            _mm_stream_si128((__m128i *)(d + i), a); _mm_stream_si128((__m128i *)(d + i + 16), b);
            _mm_stream_si128((__m128i *)(d + i + 32), c); _mm_stream_si128((__m128i *)(d + i + 48), f);
        }
        if (i < n) memcpy(d + i, s + i, n - i);
        _mm_sfence();
        return;
    }
#endif
    memcpy(dst, src, n);
}

int fail(int code, const char *what)
{
    g_last_error = what ? what : "";
    return code;
}
// cudaEventQuery's "not ready" also lands in the runtime's per-thread last-error slot, where the next
// `cudaGetLastError()` (the launch wrappers end in one) would find it and report a launch failure that never
// happened.  Every poll goes through here.
cudaError_t poll_event(cudaEvent_t ev)
{
    const cudaError_t q = cudaEventQuery(ev);
    if (q == cudaErrorNotReady) (void)cudaGetLastError();
    return q;
}

int fail_cuda(cudaError_t err, const char *where)
{
    g_last_error = std::string(where) + ": " + cudaGetErrorString(err);
    return DM_ECUDA;
}

// dm_error_detail(): the text of the last failing call on a stream / reader id, readable from any thread.
// Bounded (the oldest ids are forgotten); misses (DM_ENOENT from a lookup) are not errors worth a slot.
int note_err(dm_engine *e, uint64_t id, int rc)
{
    if (rc >= 0 || !e || rc == DM_ENOENT) return rc;
    constexpr size_t kKeep = 4096;
    std::lock_guard<std::mutex> g(e->err_mu);
    auto it = e->err_text.find(id);
    if (it != e->err_text.end()) { it->second = g_last_error; return rc; }
    if (e->err_order.size() >= kKeep) { e->err_text.erase(e->err_order.front()); e->err_order.pop_front(); }
    e->err_text.emplace(id, g_last_error);
    e->err_order.push_back(id);
    return rc;
}


// ---- extents ---------------------------------------------------------------

// Device pointer of byte `off`, and how many bytes are contiguous from there.
uint8_t *seg_at(dm_engine *e, const std::vector<Extent> &ext, uint64_t off, uint64_t *contig)
{
    uint64_t base = 0;
    for (const Extent &x : ext) {
        if (off < base + x.len) { *contig = base + x.len - off; return e->arena_base + x.off + (off - base); }
        base += x.len;
    }
    *contig = 0;
    return nullptr;
}

void free_extents(dm_engine *e, std::vector<Extent> &ext)
{
    std::lock_guard<std::mutex> g(e->arena_mu);
    for (const Extent &x : ext) e->arena.release(x.off, x.len);
    ext.clear();
}

void lru_drop(dm_engine *e, Blob *b)
{
    if (!b->in_lru) return;
    (b->lru_prev ? b->lru_prev->lru_next : e->lru_head) = b->lru_next;
    (b->lru_next ? b->lru_next->lru_prev : e->lru_tail) = b->lru_prev;
    b->lru_prev = b->lru_next = nullptr;
    b->in_lru = false;
}

void lru_touch(dm_engine *e, Blob *b)
{
    if (b->in_lru && e->lru_tail == b) return;
    lru_drop(e, b);
    b->lru_prev = e->lru_tail;
    (e->lru_tail ? e->lru_tail->lru_next : e->lru_head) = b;
    e->lru_tail = b;
    b->in_lru = true;
}

// Evict least-recently-used unreferenced blobs until `need` bytes could fit.
// Caller holds neither e->mu nor arena_mu.  The LRU list holds exactly the HBM-resident blobs, oldest
// first, so a victim costs a walk over the pinned ones in front of it, not a scan of the whole index.
bool evict_for(dm_engine *e, uint64_t need)
{
    for (;;) {
        std::shared_ptr<Blob> victim;
        std::vector<Extent> ext;
        bool touch = false;
        {
            std::lock_guard<std::mutex> g(e->mu);
            for (Blob *b = e->lru_head; b; b = b->lru_next) {
                if (b->readers) continue;
                if (!e->cas_dir.empty() && !b->spill_done) continue;   // not yet safe on disk
                auto it = e->blobs.find(b->digest);
                if (it != e->blobs.end() && it->second.get() == b) victim = it->second;
                break;
            }
            if (!victim) return false;
            victim->in_hbm = false;
            lru_drop(e, victim.get());
            ext.swap(victim->extents);          // taken under the lock: a re-publish may install new ones at once
            if (!victim->on_disk) e->blobs.erase(victim->digest);
            else touch = true;
        }
        if (touch) tier_touch(e, victim->digest);     // leaving HBM is its last use
        free_extents(e, ext);
        std::lock_guard<std::mutex> g(e->arena_mu);
        uint64_t off;
        if (e->arena.alloc(need, &off)) { e->arena.release(off, need); return true; }
    }
}

bool arena_alloc(dm_engine *e, uint64_t len, Extent *out)
{
    len = round_up(std::max<uint64_t>(len, 1), kAlign);
    for (int attempt = 0; attempt < 4; ++attempt) {      // another thread may take what an eviction freed
        {
            std::lock_guard<std::mutex> g(e->arena_mu);
            uint64_t off;
            if (e->arena.alloc(len, &off)) { out->off = off; out->len = len; return true; }
        }
        if (!evict_for(e, len)) return false;
    }
    return false;
}

// Make sure the stream's extents cover `need` bytes.  Stream mutex held.
int ensure_capacity(dm_engine *e, Stream *s, uint64_t need)
{
    while (s->capacity < need) {
        uint64_t want = need - s->capacity;
        if (!s->extents.empty()) {   // unknown / exceeded size: grow geometrically
            const uint64_t grow = std::min<uint64_t>(std::max<uint64_t>(s->capacity, e->cfg.slab_bytes), kMaxGrow);
            want = std::max(want, grow);
        }
        Extent x;
        if (!arena_alloc(e, want, &x)) {
            if (!arena_alloc(e, need - s->capacity, &x)) return fail(DM_ENOMEM, "HBM CAS arena exhausted");
        }
        s->extents.push_back(x);
        s->capacity += x.len;
    }
    return DM_OK;
}

// ---- ring slabs --------------------------------------------------------------

Slab *slab_get(dm_engine *e)
{
    std::unique_lock<std::mutex> g(e->slab_mu);
    if (e->slab_free.empty() && !e->stop) {
        e->st_ring_waits++;
        // Every slab is out.  Usually most of them are in flight to the device and come back by
        // themselves (writers outrunning PCIe: plain back-pressure, just wait).  But if ALL of them are
        // partly filled and held by streams waiting for their next bytes, nothing moves: more live
        // streams than slabs would starve - or, with one thread driving many streams, deadlock.  The
        // pump tells the two apart (slabs_returning) and recalls partial slabs only in the second case.
        // The waiter is counted BEFORE the pump is poked: the pump acts on "asked and somebody waits",
        // and consumes the flag when it looks.
        e->ring_waiters++;
        { std::lock_guard<std::mutex> gw(e->work_mu); e->ring_starved.store(true); }   // under the pump's mutex: no lost wake-up
        e->work_cv.notify_one();
        e->slab_cv.wait(g, [&] { return !e->slab_free.empty() || e->stop; });
        e->ring_waiters--;
    }
    if (e->slab_free.empty()) return nullptr;
    Slab *s = e->slab_free.back();
    e->slab_free.pop_back();
    return s;
}

Slab *slab_try_get(dm_engine *e)
{
    std::lock_guard<std::mutex> g(e->slab_mu);
    if (e->slab_free.empty()) return nullptr;
    Slab *s = e->slab_free.back();
    e->slab_free.pop_back();
    return s;
}

void slab_put(dm_engine *e, Slab *s)
{
    {
        std::lock_guard<std::mutex> g(e->slab_mu);
        e->slab_free.push_back(s);
    }
    e->slab_cv.notify_one();
    if (e->feed_starved.load(std::memory_order_relaxed)) {        // a disk-backed read-back waits for a slab
        { std::lock_guard<std::mutex> g(e->disk_mu); e->feed_kick = true; }
        e->disk_cv.notify_one();
    }
}

void slab_return(dm_engine *e, Slab *s)
{
    e->slabs_returning.fetch_sub(1, std::memory_order_relaxed);
    slab_put(e, s);
}

// Give the stream a fresh slab.  The stream mutex is dropped while waiting for
// ring back-pressure: the pump needs it to build jobs, and only the pump's
// reaping frees slabs.
int take_slab(dm_engine *e, Stream *s, std::unique_lock<std::mutex> &g)
{
    g.unlock();
    Slab *fresh = slab_get(e);
    g.lock();
    if (!fresh) return fail(DM_ESTATE, "engine stopping");
    if (s->st != St::Open) { slab_put(e, fresh); return fail(DM_ESTATE, "stream closed while waiting for the ring"); }
    if (s->cur) { slab_put(e, fresh); return DM_OK; }
    s->cur = fresh;
    s->cur_fill = s->carry_fill;
    if (s->carry_fill) { memcpy(fresh->host, s->carry, s->carry_fill); s->carry_fill = 0; }
    if (s->small_fill) {                        // a body that outgrew its private buffer continues in a real slab
        memcpy(fresh->host, s->small.get(), s->small_fill);
        s->cur_fill = s->small_fill;
        s->small_fill = 0;
    }
    s->small.reset(); s->small_cap = 0;
    return DM_OK;
}

// Tell the pump this stream has new DMA'd bytes (or is finishing).  Stream mutex held.
void mark_dirty(dm_engine *e, const std::shared_ptr<Stream> &sp, Slab *submitted, uint64_t landed_end)
{
    const bool enqueue = !sp->queued;
    sp->queued = true;
    if (submitted) e->slabs_returning.fetch_add(1, std::memory_order_relaxed);
    {
        std::lock_guard<std::mutex> g(e->work_mu);
        if (submitted) e->pending_slabs.push_back(SentSlab{submitted, landed_end ? sp : nullptr, landed_end});
        if (enqueue) e->dirty.push_back(sp);
    }
    e->work_cv.notify_one();
}

// DMA `n` staged bytes to blob offset `base`.  Stream mutex held.  The slab is handed to the pump
// (released once its copy event completes) on success, returned to the ring on failure.
int dma_range(dm_engine *e, const std::shared_ptr<Stream> &sp, Slab *slab, uint64_t base, uint32_t n)
{
    Stream *s = sp.get();
    cudaSetDevice(e->device);       // the caller may be any OS thread (cgo)
    int rc = ensure_capacity(e, s, base + n);
    if (rc != DM_OK) { slab_put(e, slab); return rc; }
    cudaStream_t cs = e->copy_stream[s->id % kCopyStreams];
    const uint8_t *src = slab->host;
    cudaError_t err = cudaSuccess;
    for_segments(e, s->extents, base, n, [&](uint8_t *dev, uint64_t len) {
        if (err == cudaSuccess) err = cudaMemcpyAsync(dev, src, len, cudaMemcpyHostToDevice, cs);
        src += len;
    });
    if (err != cudaSuccess) {
        s->cuda_failed = true;
        cudaStreamSynchronize(cs);      // earlier segments of this slab may still be DMA-ing out of it
        slab_put(e, slab);
        return fail_cuda(err, "cudaMemcpyAsync(H2D slab)");
    }
    e->st_h2d += n;
    return DM_OK;
}

// The contiguous frontier swallows islands that now touch it.  Stream mutex held.
void absorb_islands(Stream *s)
{
    if (s->cur_fill) return;            // staged sequential bytes sit between the frontier and any island
    auto it = s->islands.begin();
    while (it != s->islands.end() && it->first <= s->dma_issued) {
        s->dma_issued = std::max(s->dma_issued, it->second);
        it = s->islands.erase(it);
    }
}

// DMA the stream's sequential slab to its place in the blob.  Stream mutex held.  A failure drops the
// staged bytes and is recorded in s->lost (sticky): whoever calls next - this may be the pump recalling a
// partial slab, with no writer to tell - learns that the stream is broken, and it is never published.
int submit_slab(dm_engine *e, const std::shared_ptr<Stream> &sp)
{
    Stream *s = sp.get();
    if (!s->cur) return DM_OK;
    Slab *slab = s->cur;
    const uint32_t n = s->cur_fill;
    s->cur = nullptr; s->cur_fill = 0;
    if (n == 0) { slab_put(e, slab); return DM_OK; }
    if (!s->check_only) e->st_ingested.fetch_add(n, std::memory_order_relaxed);   // per slab, not per write: one shared line, many writer threads
    if (s->disk) {
        disk_write(e, sp, slab, s->dma_issued, n);
        s->dma_issued += n;
        absorb_islands(s);
        return DM_OK;
    }
    if (s->verify_only) {
        cudaSetDevice(e->device);
        cudaError_t err = cudaMemcpyAsync(slab->dev, slab->host, n, cudaMemcpyHostToDevice, e->copy_stream[s->id % kCopyStreams]);
        if (err != cudaSuccess) { slab_put(e, slab); s->cuda_failed = true; return s->lost = fail_cuda(err, "cudaMemcpyAsync(H2D slab)"); }
        e->st_h2d += n;
        s->staged.emplace_back(slab, n);
        e->slabs_returning.fetch_add(1, std::memory_order_relaxed);
        s->dma_issued += n;
        mark_dirty(e, sp, nullptr);       // the slab stays out of the ring until its job has run
        return DM_OK;
    }
    int rc = dma_range(e, sp, slab, s->dma_issued, n);
    if (rc != DM_OK) return s->lost = rc;      // the staged bytes are gone: the stream can only be aborted now
    s->dma_issued += n;
    const uint64_t seq_end = s->dma_issued;      // this slab's bytes end here (before any island is absorbed)
    absorb_islands(s);
    mark_dirty(e, sp, slab, s->range_mode ? 0 : seq_end);
    if (s->followers) s->cv.notify_all();
    return DM_OK;
}

// DMA one range part.  Stream mutex held; invalidates indices into s->parts.
int submit_part(dm_engine *e, const std::shared_ptr<Stream> &sp, size_t idx)
{
    Stream *s = sp.get();
    Stream::Part pt = s->parts[idx];
    s->parts.erase(s->parts.begin() + (long)idx);
    s->range_mode = true;
    if (pt.fill == 0) { slab_put(e, pt.slab); return DM_OK; }
    e->st_ingested.fetch_add(pt.fill, std::memory_order_relaxed);
    if (s->disk) disk_write(e, sp, pt.slab, pt.base, pt.fill);
    else {
        int rc = dma_range(e, sp, pt.slab, pt.base, pt.fill);
        if (rc != DM_OK) return s->lost = rc;
    }
    if (pt.base + pt.fill <= s->resume_base) add_interval(s->prefix_cover, pt.base, pt.base + pt.fill);
    else add_interval(s->islands, pt.base, pt.base + pt.fill);
    absorb_islands(s);
    if (s->disk) return DM_OK;                  // the slab comes back from the disk thread
    mark_dirty(e, sp, pt.slab);
    if (s->followers) s->cv.notify_all();
    return DM_OK;
}

// Would [off, off+len) collide with bytes this stream already holds?  Stream mutex held.
bool range_taken(const Stream *s, uint64_t off, uint64_t len, const Stream::Part *self)
{
    const uint64_t end = off + len;
    auto hits = [&](uint64_t lo, uint64_t hi) { return lo < end && off < hi; };
    if (hits(s->resume_base, s->dma_issued + s->cur_fill) && !(self == nullptr && off == s->dma_issued + s->cur_fill)) return true;
    auto in_map = [&](const std::map<uint64_t, uint64_t> &m) {
        auto it = m.upper_bound(off);
        if (it != m.begin() && std::prev(it)->second > off) return true;
        return it != m.end() && it->first < end;
    };
    if (in_map(s->islands) || in_map(s->prefix_cover)) return true;
    for (const Stream::Part &p : s->parts)
        if (&p != self && hits(p.base, p.base + p.fill)) return true;
    return false;
}

// ---- tiny bodies: shared pack slabs (struct Pack) ---------------------------------

// Called by begin_finish with the stream mutex held.  True: the body now lives in the open pack, its own slab is
// back in the ring and its extent is reserved; false: not eligible or no pack resources right now (the caller takes
// the ordinary one-DMA-per-slab path, which is always correct).
bool pack_tiny_body(dm_engine *e, Stream *s)
{
    const uint32_t n = s->cur ? s->cur_fill : s->small_fill;
    const uint8_t *from = s->cur ? s->cur->host : s->small.get();
    if (!from || n == 0 || n > e->tiny_max || (s->verify_only && !s->check_only) || s->dma_issued || s->resume_base ||
        s->carry_fill || !s->parts.empty() || !s->islands.empty() || e->pack_dev_base == nullptr)
        return false;
    if (!s->check_only) {                      // a check is a hash-only member: no extent, its job's dst stays null
        if (ensure_capacity(e, s, n) != DM_OK) return false;          // (the ordinary path reports the ENOMEM)
        uint64_t contig = 0;
        if (!seg_at(e, s->extents, 0, &contig) || contig < n) return false;
    }
    const uint32_t need = (uint32_t)round_up(n, kAlign);
    std::shared_ptr<Pack> pk;
    uint32_t off;
    {
        std::lock_guard<std::mutex> g(e->pack_mu);
        if (e->open_pack && e->open_pack->fill + need > e->cfg.slab_bytes) {
            e->sealed_packs.push_back(e->open_pack);
            e->open_pack.reset();
        }
        if (!e->open_pack) {
            if (e->pack_dev_free.empty()) return false;
            Slab *sl = slab_try_get(e);
            if (!sl) return false;
            auto np = std::make_shared<Pack>();
            np->slab = sl;
            np->dev = e->pack_dev_free.back();
            e->pack_dev_free.pop_back();
            e->open_pack = np;
            e->st_packs++;
        }
        pk = e->open_pack;
        off = pk->fill;
        memcpy(pk->slab->host + off, from, n);
        pk->fill += need;
        pk->bytes += n;
        pk->refs.fetch_add(1);
    }
    s->pack = pk; s->pack_off = off; s->pack_len = n;
    if (s->cur) { slab_put(e, s->cur); s->cur = nullptr; s->cur_fill = 0; }     // the body's own slab is free again at once
    s->small.reset(); s->small_fill = 0; s->small_cap = 0;
    if (!s->check_only) e->st_ingested.fetch_add(n, std::memory_order_relaxed);
    e->st_packed++;
    return true;
}

void pack_release_member(dm_engine *e, Stream *s)
{
    (void)e;
    if (!s->pack) return;
    s->pack->refs.fetch_sub(1);
    s->pack.reset();
}

// ---- CAS commit --------------------------------------------------------------

std::string json_quote(const std::string &v)
{
    std::string o = "\"";
    for (unsigned char c : v) {
        if (c == '"' || c == '\\') { o += '\\'; o += (char)c; }
        else if (c < 0x20) { char t[8]; snprintf(t, sizeof t, "\\u%04x", c); o += t; }
        else o += (char)c;
    }
    return o + "\"";
}

// The sidecar: what a hit needs besides the bytes (SURVEY.md §8f-2).  The digest is over the
// identity-encoded body, which is what HF LFS oids and OCI layer digests are defined on.
std::string sidecar_json(const Blob &b)
{
    if (!b.sidecar.empty()) return b.sidecar;
    std::string o = "{\"digest\":\"sha256:" + hex_of(b.digest.b, 32) + "\",\"size\":" + std::to_string(b.size) +
                    ",\"encoding\":\"identity\",\"engine\":\"demodel_b200\",\"abi\":" + std::to_string(DM_ABI_VERSION) +
                    ",\"headers\":{";
    for (size_t i = 0; i < b.meta.size(); ++i)
        o += (i ? "," : "") + json_quote(b.meta[i].first) + ":" + json_quote(b.meta[i].second);
    return o + "}}\n";
}

bool write_sidecar(const std::string &path, const Blob &b)
{
    FILE *f = fopen(path.c_str(), "w");
    if (!f) return false;
    const std::string j = sidecar_json(b);
    const bool ok = fwrite(j.data(), 1, j.size(), f) == j.size();
    return fclose(f) == 0 && ok;
}

std::string blob_path(const dm_engine *e, const uint8_t d[32])
{
    const std::string hx = hex_of(d, 32);
    return e->cas_dir + "/blobs/sha256/" + hx.substr(0, 2) + "/" + hx;
}

// Publish a verified blob.  Returns the blob that now owns the digest (an
// earlier copy wins; the new extents are then released).
std::shared_ptr<Blob> publish(dm_engine *e, const Digest &d, uint64_t size, std::vector<Extent> &ext,
                              std::vector<std::pair<std::string, std::string>> *meta)
{
    // trim the last extent to the bytes actually held
    uint64_t keep = round_up(std::max<uint64_t>(size, 1), kAlign), base = 0;
    std::vector<Extent> kept;
    {
        std::lock_guard<std::mutex> g(e->arena_mu);
        for (Extent &x : ext) {
            if (base >= keep) { e->arena.release(x.off, x.len); }
            else if (base + x.len > keep) {
                const uint64_t k = keep - base;
                e->arena.release(x.off + k, x.len - k);
                kept.push_back({x.off, k});
            } else kept.push_back(x);
            base += x.len;
        }
    }
    ext.clear();
    std::shared_ptr<Blob> b;
    bool fresh = false;
    {
        std::lock_guard<std::mutex> g(e->mu);
        auto it = e->blobs.find(d);
        if (it != e->blobs.end() && it->second->in_hbm) {
            b = it->second;
            lru_touch(e, b.get());
        } else if (it != e->blobs.end()) {   // known on disk only: re-home into HBM
            b = it->second;
            if (b->size != size) b->sidecar.clear();     // an entry dm_cache_promote registered from an unverified file:
            b->size = size;                              // the verified length wins, and a sidecar stating another goes
            b->extents = kept; kept.clear();
            b->in_hbm = true; lru_touch(e, b.get());
        } else {
            b = std::make_shared<Blob>();
            b->digest = d; b->size = size; b->extents = kept; kept.clear();
            b->in_hbm = true; lru_touch(e, b.get());
            if (meta) b->meta.swap(*meta);
            e->blobs[d] = b;
            fresh = true;
        }
    }
    if (!kept.empty()) free_extents(e, kept);
    e->st_committed++;
    if (fresh && !e->cas_dir.empty()) {
        {
            std::lock_guard<std::mutex> g(e->spill_mu);
            e->spill_q.push_back(b);
        }
        e->spill_cv.notify_all();
    }
    return b;
}

// Batch form of publish() for dm_ingest_device: every blob has exactly one right-sized extent, so
// the index is updated under ONE lock and the arena under one more (150 k blobs per call otherwise
// spend longer in lock traffic than in the kernel).
void publish_many(dm_engine *e, const std::vector<Verified> &items)
{
    std::vector<Extent> to_free;
    std::vector<std::shared_ptr<Blob>> to_spill;
    {
        std::lock_guard<std::mutex> g(e->mu);
        e->blobs.reserve(e->blobs.size() + items.size());           // one rehash, not log(n) of them
        for (const Verified &v : items) {
            auto it = e->blobs.find(v.d);
            if (it != e->blobs.end() && it->second->in_hbm) {          // an earlier copy wins
                lru_touch(e, it->second.get());
                to_free.push_back(v.x);
            } else if (it != e->blobs.end()) {                         // on disk only: re-home
                Blob *b = it->second.get();
                b->size = v.size;
                b->extents.assign(1, v.x);
                b->in_hbm = true; lru_touch(e, b);
            } else {
                auto b = std::make_shared<Blob>();
                b->digest = v.d; b->size = v.size; b->extents.assign(1, v.x);
                b->in_hbm = true; lru_touch(e, b.get());
                e->blobs.emplace(v.d, b);
                if (!e->cas_dir.empty()) to_spill.push_back(b);
            }
        }
    }
    e->st_committed += items.size();
    if (!to_free.empty()) {
        std::lock_guard<std::mutex> g(e->arena_mu);
        for (const Extent &x : to_free) e->arena.release(x.off, x.len);
    }
    if (!to_spill.empty()) {
        {
            std::lock_guard<std::mutex> g(e->spill_mu);
            for (auto &b : to_spill) e->spill_q.push_back(b);
        }
        e->spill_cv.notify_all();
    }
}

// DM_ING_REPLACE parks a cached blob instead of evicting it: the entry stays in the index, out of sight (not in HBM,
// not in the LRU list - the state of a disk-only blob), its extent becomes the destination of the new copy.  Here the
// verified ones come back under ONE lock; the others leave for good.  While it was parked a blob may have been
// re-homed by a stream that carried the same digest - and then evicted again, which takes it out of the index: only
// an entry that still maps to this very object is revived in place, anything else goes the way of a new blob.
void unpark_many(dm_engine *e, std::vector<Parked> &verified, std::vector<Parked> &failed)
{
    std::vector<Extent> to_free;
    std::vector<Verified> anew;
    {
        std::lock_guard<std::mutex> g(e->mu);
        constexpr size_t kAhead = 16;
        for (size_t q = 0; q < verified.size(); ++q) {
            if (q + kAhead < verified.size()) e->blobs.prefetch(verified[q + kAhead].b->digest);
            Parked &k = verified[q];
            Blob *b = k.b.get();
            auto it = e->blobs.find(b->digest);
            if (it == e->blobs.end() || it->second.get() != b) { anew.push_back(Verified{b->digest, b->size, k.x}); continue; }
            b->parked = false;
            if (b->in_hbm) { to_free.push_back(k.x); continue; }       // a stream re-homed it meanwhile: that copy wins
            b->extents.assign(1, k.x);
            b->in_hbm = true; lru_touch(e, b);
        }
        for (Parked &k : failed) {
            Blob *b = k.b.get();
            b->parked = false;
            to_free.push_back(k.x);
            if (b->in_hbm || b->on_disk) continue;
            auto it = e->blobs.find(b->digest);
            if (it != e->blobs.end() && it->second.get() == b) e->blobs.erase(it);
        }
    }
    e->st_committed += verified.size() - anew.size();
    if (!anew.empty()) publish_many(e, anew);
    if (!to_free.empty()) free_extents(e, to_free);
}

// ---- pump ----------------------------------------------------------------------

// Before a stream's extents are freed or change owner: let followers' in-flight copy-outs finish.
void wait_follow_reads(Stream *s, std::unique_lock<std::mutex> &g)
{
    s->cv.wait(g, [&] { return s->follow_reads == 0; });
}

void complete_stream(dm_engine *e, const std::shared_ptr<Stream> &sp, const uint32_t *words)
{
    Stream *s = sp.get();
    std::unique_lock<std::mutex> g(s->mu);
    if (s->st == St::Aborted) return;
    words_to_digest(words, s->digest.b);
    s->matched = (!s->has_expect || s->digest == s->expect) ? 1 : 0;
    if (s->cuda_failed || s->lost != DM_OK) { s->matched = 0; memset(s->digest.b, 0, 32); }     // never publish under a digest the device may not have produced, or a body with bytes missing
    s->completing = true;                       // no new follower copy-out starts past this point
    wait_follow_reads(s, g);
    std::vector<Extent> ext;
    ext.swap(s->extents);
    s->capacity = 0;
    const uint64_t size = s->dma_issued;
    if (s->disk) {                              // the rename into the disk tier runs on a disk thread, finish waits for it
        s->publishing = true;
        g.unlock();
        disk_enqueue(e, DiskTask{DiskTask::Publish, sp});
        return;
    }
    const Digest d = s->digest;
    const int matched = s->matched;
    // a resumed stream is cacheable only if the already-hashed prefix was re-supplied
    const bool whole = s->resume_base == 0 ||
                       (s->prefix_cover.size() == 1 && s->prefix_cover.begin()->first == 0 &&
                        s->prefix_cover.begin()->second >= s->resume_base);
    std::vector<std::pair<std::string, std::string>> meta;
    meta.swap(s->meta);
    g.unlock();
    std::shared_ptr<Blob> b;
    if (matched && whole && !s->verify_only) b = publish(e, d, size, ext, &meta);
    else { free_extents(e, ext); if (!matched && !s->check_only) e->st_mismatch++; }
    g.lock();
    s->blob = b;
    s->st = St::Done;
    const bool load = s->load;
    g.unlock();
    s->cv.notify_all();
    if (load) load_wake(e);
}

void completer_main(dm_engine *e)
{
    cudaSetDevice(e->device);
    std::vector<dm_engine::DoneItem> batch;
    for (;;) {
        {
            std::unique_lock<std::mutex> g(e->done_mu);
            e->done_cv.wait(g, [&] { return !e->done_q.empty() || e->done_stop; });
            if (e->done_q.empty()) return;
            // a share of what is queued (the other completion thread takes the rest), at most 64 per lock
            size_t take = std::min<size_t>(64, (e->done_q.size() + kCompleters - 1) / kCompleters);
            while (take--) { batch.push_back(std::move(e->done_q.front())); e->done_q.pop_front(); }
        }
        for (auto &it : batch) complete_stream(e, it.sp, it.words);
        batch.clear();
    }
}

// A ring load's slab whose job has been reaped: it no longer comes back by itself (slabs_returning), and goes back to
// the ring now or once its readers are done with it.  Stream mutex held.
static void ring_reaped(dm_engine *e, const std::shared_ptr<Stream> &sp, Slab *slab)
{
    e->slabs_returning.fetch_sub(1, std::memory_order_relaxed);
    bool found = false;
    for (RingLoad::Held &h : sp->ring->held)
        if (h.slab == slab) { h.reaped = found = true; h.reaped_at = Clock::now(); break; }
    if (!found) slab_put(e, slab);              // (not kept: cannot happen, but never lose a slab)
    ring_release(e, sp);
}

void ring_release(dm_engine *e, const std::shared_ptr<Stream> &sp)
{
    RingLoad *R = sp->ring.get();
    for (auto it = R->held.begin(); it != R->held.end();) {
        bool needed = false;
        if (!R->closed)
            for (const auto &p : R->parts) if (p->needs(it->off, it->n)) { needed = true; break; }
        if (it->reaped && !needed) {
            R->low = std::max<uint64_t>(R->low, it->off + it->n);
            slab_put(e, it->slab);
            it = R->held.erase(it);
        } else ++it;
    }
}

void reap_cycle(dm_engine *e, Cycle &c)
{
    std::vector<dm_engine::DoneItem> finished;          // handed to the completion threads under ONE lock at the end
    float ms = 0.f;
    if (c.njobs) {
        cudaEventElapsedTime(&ms, c.k_start, c.k_end);
        std::lock_guard<std::mutex> g(e->stat_mu);
        e->st_kernel_ms += ms;
    }
    e->st_hashed += c.bytes;
    // (a ring load's slab may still be wanted by its reader: see ring_reaped below)
    for (size_t i = 0; i < c.job_slabs.size(); ++i) if (c.job_slabs[i] && !c.streams[i]->ring) slab_return(e, c.job_slabs[i]);
    for (size_t i = 0; i < c.streams.size(); ++i) {
        std::shared_ptr<Stream> &sp = c.streams[i];
        bool free_now = false, wake = false;
        {
            std::lock_guard<std::mutex> g(sp->mu);
            if (c.err != cudaSuccess) sp->cuda_failed = true;
            if (i < c.job_packs.size() && c.job_packs[i]) {        // tiny body: its bytes are in its own extent now
                if (c.job_packs[i]->failed.load()) sp->cuda_failed = true;
                sp->dma_issued = sp->hash_issued = sp->pack_len;
                pack_release_member(e, sp.get());
            }
            sp->jobs_inflight--;
            if (sp->ring && c.job_slabs[i]) ring_reaped(e, sp, c.job_slabs[i]);
            if (sp->disk) disk_feed(e, sp);                        // a staged slab was used up: read the next one back
            free_now = sp->st == St::Aborted && sp->jobs_inflight == 0;
            wake = sp->ckpt_waiter;
        }
        if (wake) sp->cv.notify_all();
        if (free_now) {
            // slabs written after this job was built may still be landing in the extent (see dm_stream_abort)
            cudaStreamSynchronize(e->copy_stream[sp->id % kCopyStreams]);
            { std::unique_lock<std::mutex> g(sp->mu); wait_follow_reads(sp.get(), g); }
            free_extents(e, sp->extents);
            std::lock_guard<std::mutex> g(e->slot_mu);
            e->free_slots.push_back(sp->slot);
        } else if (c.is_final[i]) {
            dm_engine::DoneItem it;
            it.sp = sp;
            memcpy(it.words, e->h_digests + 8ull * sp->slot, sizeof it.words);
            finished.push_back(std::move(it));
        }
    }
    if (!finished.empty()) {
        const bool many = finished.size() > 1;
        {
            std::lock_guard<std::mutex> g(e->done_mu);
            for (auto &it : finished) e->done_q.push_back(std::move(it));
        }
        if (many) e->done_cv.notify_all(); else e->done_cv.notify_one();
    }
    c.streams.clear(); c.is_final.clear(); c.job_packs.clear(); c.job_slabs.clear();
    c.njobs = 0; c.bytes = 0; c.busy = false; c.err = cudaSuccess;
}

// Build one job per eligible ready stream and launch ONE multi-buffer kernel
// over them on this cycle's CUDA stream.  Streams that still have unhashed
// bytes afterwards (or a job in flight) stay in `ready`.
bool run_cycle(dm_engine *e, Cycle &c, std::vector<std::shared_ptr<Stream>> &ready)
{
    c.njobs = 0; c.bytes = 0; c.needs_copy_wait = false;
    // Job length.  A launch is reaped as a whole, so it lasts as long as its longest lane and every lane
    // should be the same length: the quantum.  It is one slab while the streams are network-bound (each has
    // about a slab of backlog when it becomes ready), and grows to the smallest backlog among the streams
    // that are at least a slab behind, up to kMaxJobSlabs slabs, when the hash is the bottleneck (few
    // streams, DMA far ahead): fewer, longer launches, so the reap -> rebuild -> relaunch gap between two jobs
    // of a stream (host work, ~0.1 ms) is paid once per 8 MiB instead of once per MiB.
    const uint64_t slab = (uint64_t)e->cfg.slab_bytes;
    uint64_t quantum = slab;
    {
        uint64_t min_backlog = ~0ull;
        for (auto &sp : ready) {
            Stream *s = sp.get();
            std::lock_guard<std::mutex> g(s->mu);
            if (s->st == St::Aborted || s->st == St::Done || s->final_issued || s->jobs_inflight || s->verify_only || s->pack) continue;
            // what a job could cover right now: landed bytes where the stream tracks them, else everything enqueued
            const uint64_t upto = s->range_mode ? s->dma_issued : std::min(s->dma_issued, s->landed);
            const uint64_t backlog = upto > s->hash_issued ? upto - s->hash_issued : 0;
            if (backlog >= slab) min_backlog = std::min(min_backlog, backlog);
        }
        if (min_backlog != ~0ull) quantum = std::min<uint64_t>(min_backlog / slab, kMaxJobSlabs) * slab;
    }
    std::vector<std::shared_ptr<Stream>> again;
    for (auto &sp : ready) {
        Stream *s = sp.get();
        std::lock_guard<std::mutex> g(s->mu);
        if (s->st == St::Aborted || s->st == St::Done || s->final_issued || s->suspending) { s->queued = false; continue; }
        // one job per stream in flight: its next job chains on the state this one writes
        if (s->jobs_inflight || c.njobs >= e->max_jobs) { again.push_back(sp); continue; }
        const bool finishing = s->st == St::Finishing;
        // How much can go into this job, and does the launch have to be ordered after the copy streams for it?
        // Streams that track `landed` hash landed bytes only - no ordering, the launch starts at once - except for
        // the tail of a finishing body, which is taken whole and ordered after its DMAs.
        const uint64_t remaining = s->dma_issued - s->hash_issued;
        const bool tracks = !s->verify_only && !s->pack && !s->range_mode;
        bool wait_copy = !tracks;
        uint64_t n;
        if (tracks) {
            const uint64_t lend = std::min(s->dma_issued, s->landed);
            const uint64_t landed_n = lend > s->hash_issued ? lend - s->hash_issued : 0;
            if (finishing && landed_n == remaining) n = remaining;
            else if (finishing && landed_n < quantum) { n = remaining; wait_copy = true; }
            else n = landed_n & ~63ull;
        } else n = finishing ? remaining : (remaining & ~63ull);
        if (!finishing && n == 0) { s->queued = false; continue; }      // (bytes still in flight re-queue the stream when they land)
        uint64_t contig = 0;
        uint8_t *src = nullptr;
        bool final = finishing;
        Slab *job_slab = nullptr;
        uint8_t *dst = nullptr;
        std::shared_ptr<Pack> job_pack;
        if (s->pack) {
            // tiny body in a shared pack: wait for the pack's one DMA to be enqueued, then hash its piece out of the
            // staging buffer while the kernel copies it into the body's own extent
            if (!s->pack->dma_issued.load()) { again.push_back(sp); continue; }
            if (s->pack->failed.load()) s->cuda_failed = true;
            job_pack = s->pack;
            src = job_pack->dev + s->pack_off;
            dst = seg_at(e, s->extents, 0, &contig);
            n = s->pack_len;
            final = true;
        } else if (s->verify_only) {
            if (!s->staged.empty()) {
                job_slab = s->staged.front().first;
                n = s->staged.front().second;               // whole slab; only the last may hold a partial block
                src = job_slab->dev;
                s->staged.pop_front();
                final = finishing && s->staged.empty() && (!s->disk || disk_fed(s));
                if (!final && (n & 63)) { final = false; }   // cannot happen: mid-stream slabs are full
            } else if (!finishing || (s->disk && !disk_fed(s))) { s->queued = false; continue; }   // (a read-back re-queues it)
            else n = 0;
        } else {
            src = n ? seg_at(e, s->extents, s->hash_issued, &contig) : nullptr;
            if (n > contig && n) n = contig;                             // stop at the extent boundary
            if (n > quantum) n = quantum;
            if (n & 63 && s->hash_issued + n != s->dma_issued) n &= ~63ull;     // only the very last job may end in a partial block
            final = finishing && s->hash_issued + n == s->dma_issued;
        }
        dm::HashJob &jb = c.h_jobs[c.njobs++];
        jb.src = src; jb.dst = dst; jb.nbytes = n; jb.total_len = job_pack ? n : s->dma_issued; jb.slot = s->slot;
        jb.flags = (s->hash_issued == 0 ? dm::JOB_INIT : 0u) | (final ? dm::JOB_FINAL : 0u);
        jb.one = 1; jb.pad_ = 0;
        if (!job_pack) s->hash_issued += n;            // (a packed body's counters move when its job is reaped)
        s->jobs_inflight++;
        if (final) s->final_issued = true;
        c.bytes += n;
        c.streams.push_back(sp);
        c.is_final.push_back(final ? 1 : 0);
        c.job_slabs.push_back(job_slab);
        c.job_packs.push_back(job_pack);
        if (wait_copy) c.needs_copy_wait = true;
        if (!final && (finishing || !s->staged.empty() || (!s->verify_only && ((s->dma_issued - s->hash_issued) & ~63ull)))) again.push_back(sp);
        else s->queued = false;
    }
    ready.swap(again);
    if (c.njobs == 0) return false;

    // Jobs over landed bytes need nothing from the copy streams.  The others (range parts, verify-only staging, packs,
    // the tail of a finishing body) are ordered after everything whose DMA was enqueued before this point.
    if (c.needs_copy_wait)
        for (int i = 0; i < kCopyStreams; ++i) {
            cudaEventRecord(c.copy_ev[i], e->copy_stream[i]);
            cudaStreamWaitEvent(c.stream, c.copy_ev[i], 0);
        }
    // Launches overlap on the GPU, so what decides the kernel shape is how many jobs will be
    // co-resident (this launch + those still running), not the size of this launch alone.
    uint32_t resident = c.njobs;
    for (const Cycle &o : e->cycles) if (o.busy) resident += o.njobs;
    const int spw = e->force_spw ? e->force_spw : dm::streams_per_warp_for(resident);
    c.deep = spw == 1;
    // warp pairs only while ALL co-resident groups can have two sub-partitions each: a round warp that shares its
    // sub-partition with another one runs at half speed
    const dm::KernelShape shape = dm::kernel_shape(spw, resident, e->variant_wide, e->variant_deep);
    if (spw > 1) {
        // lanes of a warp run in lock step: keep neighbours the same length
        std::vector<uint32_t> order(c.njobs);
        for (uint32_t i = 0; i < c.njobs; ++i) order[i] = i;
        std::stable_sort(order.begin(), order.end(),
                         [&](uint32_t a, uint32_t b) { return c.h_jobs[a].nbytes > c.h_jobs[b].nbytes; });
        std::vector<dm::HashJob> tmp(c.h_jobs, c.h_jobs + c.njobs);
        std::vector<std::shared_ptr<Stream>> st2(c.njobs);
        std::vector<uint8_t> fin2(c.njobs);
        std::vector<Slab *> sl2(c.njobs);
        std::vector<std::shared_ptr<Pack>> pk2(c.njobs);
        for (uint32_t i = 0; i < c.njobs; ++i) {
            c.h_jobs[i] = tmp[order[i]]; st2[i] = c.streams[order[i]]; fin2[i] = c.is_final[order[i]];
            sl2[i] = c.job_slabs[order[i]]; pk2[i] = c.job_packs[order[i]];
        }
        c.streams.swap(st2); c.is_final.swap(fin2); c.job_slabs.swap(sl2); c.job_packs.swap(pk2);
    }
    // A failure anywhere here (or reported later by the end event) marks every stream of the launch:
    // their verdict becomes "not matched" and nothing is published (reap_cycle / complete_stream).
    (void)cudaGetLastError();           // nothing stale may be mistaken for this launch's result
    auto note = [&](cudaError_t r) { if (r != cudaSuccess && r != cudaErrorNotReady && c.err == cudaSuccess) c.err = r; };
    note(cudaMemcpyAsync(c.d_jobs, c.h_jobs, sizeof(dm::HashJob) * c.njobs, cudaMemcpyHostToDevice, c.stream));
    note(cudaEventRecord(c.k_start, c.stream));
    if (c.err != cudaSuccess) { /* the job table may not be on the device: launching would run stale jobs */ }
    else {
        note(dm::launch_sha256(c.d_jobs, c.njobs, e->d_states, e->d_digests, c.stream, shape));
        (spw == 1 ? e->st_deep : spw == 32 ? e->st_wide : e->st_group)++;
    }
    e->st_launches++;
    note(cudaEventRecord(c.k_end, c.stream));
    c.busy = true;
    return true;
}

// Ring back-pressure relief (pump thread): DMA the partly filled slabs of open streams - the sequential
// one and those of range parts (a client fetching one blob as P parallel ranges holds P of them) - so
// they return to the ring.  try_lock only: a stream busy in a write keeps its slabs this round.
void flush_partial_slabs(dm_engine *e)
{
    std::vector<std::shared_ptr<Stream>> all;
    for (int k = 0; k < kStripes; ++k) {
        std::lock_guard<std::mutex> g(e->stripe_mu[k]);
        for (auto &kv : e->streams[k]) all.push_back(kv.second);
    }
    for (auto &sp : all) {
        Stream *s = sp.get();
        std::unique_lock<std::mutex> g(s->mu, std::try_to_lock);
        if (!g.owns_lock() || s->st != St::Open || s->window_out) continue;
        // A submit that fails here (arena full while growing an unknown-size body, a failed copy) has
        // already dropped the staged bytes, and the writer is not on this thread to be told: remember it
        // in the stream, so that its next write / finish / checkpoint fails and nothing is ever published.
        auto lose = [&](int rc) {
            if (rc != DM_OK && s->lost == DM_OK) { s->lost = rc; s->cv.notify_all(); }
        };
        // a part that was sent early simply becomes an island; the range continues in a fresh part
        for (size_t i = s->parts.size(); i-- > 0;)
            if (s->parts[i].fill) lose(submit_part(e, sp, i));
        if (!s->cur || s->cur_fill == 0) continue;
        if (s->verify_only && !s->disk && (s->cur_fill & 63)) {  // slab-by-slab hashing needs whole blocks:
            const uint32_t whole = s->cur_fill & ~63u;           // send those, keep the tail in the stream
            s->carry_fill = s->cur_fill - whole;
            memcpy(s->carry, s->cur->host + whole, s->carry_fill);
            s->cur_fill = whole;                                 // (0 whole blocks: submit_slab just returns the slab)
        }
        lose(submit_slab(e, sp));
    }
}

// The pump owns all launch decisions.  Policy: at most one JOB PER STREAM in
// flight (its next job chains on the state the running one writes), but up to
// kCycles LAUNCHES in flight, each on its own CUDA stream.  A launch costs its
// longest lane however few lanes it has, so a launch that caught only a few
// early streams must not hold the others back: they go out in the next launch
// and overlap with it on the GPU (a deep launch occupies one sub-partition per
// job).  When every launch slot is busy the ready set simply accumulates.
void pump_main(dm_engine *e)
{
    cudaSetDevice(e->device);
    int n_inflight = 0;
    int b_head = 0, b_tail = 0, b_live = 0;
    std::vector<std::shared_ptr<Stream>> ready, inbox;
    std::vector<SentSlab> slabs;
    std::vector<std::shared_ptr<Pack>> live_packs, sealed;
    int starve_ticks = 0;
    bool retry_ready = false;       // ready streams blocked only by their own in-flight job
    bool launched = false;
    for (;;) {
        // 1. ring slabs whose DMA has completed go back to the writers, and their streams learn how far they have landed
        bool landed_any = false;
        while (b_live) {
            SlabBatch &b = e->batches[b_tail];
            bool done = true;
            for (int i = 0; i < kCopyStreams; ++i) done = done && poll_event(b.ev[i]) == cudaSuccess;
            if (!done) break;
            for (SentSlab &ss : b.slabs) {
                slab_return(e, ss.slab);
                if (!ss.sp) continue;
                // the copy event behind this slab has fired: the stream's bytes up to ss.end are in HBM
                bool wake = false;
                {
                    std::lock_guard<std::mutex> g(ss.sp->mu);
                    if (ss.end > ss.sp->landed) ss.sp->landed = ss.end;
                    if (!ss.sp->queued && (ss.sp->st == St::Open || ss.sp->st == St::Finishing)) { ss.sp->queued = true; wake = true; }
                }
                if (wake) { ready.push_back(ss.sp); landed_any = true; }
            }
            b.slabs.clear(); b.busy = false;
            b_tail = (b_tail + 1) % kSlabBatches; --b_live;
        }
        // Writers blocked on the ring: recall partly filled slabs only when nothing is on its way back
        // (see slabs_returning).  A recall can miss slabs (stream busy in a write, window lent out), so it
        // is repeated every 16 passes while the writers are still waiting and still nothing is in flight.
        {
            const bool asked = e->ring_starved.exchange(false);
            if ((e->ring_waiters.load() > 0 || e->feed_starved.load()) && e->slabs_returning.load() == 0) {
                if (asked || ++starve_ticks >= 16) { starve_ticks = 0; flush_partial_slabs(e); }
            } else starve_ticks = asked ? 15 : 0;      // re-check on the very next pass if somebody just asked
        }
        // 2. finished hash launches (any order)
        bool reaped = false;
        for (Cycle &c : e->cycles)
            if (c.busy) {
                const cudaError_t q = poll_event(c.k_end);
                if (q == cudaErrorNotReady) continue;
                if (q != cudaSuccess && c.err == cudaSuccess) c.err = q;       // a faulted launch must end, not hang its streams
                reap_cycle(e, c); --n_inflight; reaped = true;
            }
        // 3. inbox.  Sleep unless the previous pass launched something (more may be launchable).
        bool stopping;
        {
            std::unique_lock<std::mutex> g(e->work_mu);
            const bool idle = !n_inflight && !b_live && ready.empty() && slabs.empty() && live_packs.empty();
            if (e->dirty.empty() && e->pending_slabs.empty() && !e->stop && !launched && !reaped && !landed_any) {
                if (idle && e->ring_waiters.load() == 0 && !e->feed_starved.load())
                    e->work_cv.wait(g, [&] { return !e->dirty.empty() || !e->pending_slabs.empty() || e->stop || e->ring_starved.load(); });
                else e->work_cv.wait_for(g, std::chrono::microseconds(40));
            }
            stopping = e->stop;
            inbox.swap(e->dirty);
            if (slabs.empty()) slabs.swap(e->pending_slabs);
            else { slabs.insert(slabs.end(), e->pending_slabs.begin(), e->pending_slabs.end()); e->pending_slabs.clear(); }
        }
        launched = false;
        const bool fresh = !inbox.empty();
        for (auto &sp : inbox) ready.push_back(sp);
        inbox.clear();
        // 3b. tiny-body packs: whatever gathered in the open pack since the last pass goes to the device with ONE copy
        //     (after the inbox was taken: every stream in `ready` that sits in a pack has its pack sealed here)
        {
            std::lock_guard<std::mutex> g(e->pack_mu);
            if (e->open_pack && e->open_pack->fill) { e->sealed_packs.push_back(e->open_pack); e->open_pack.reset(); }
            sealed.swap(e->sealed_packs);
        }
        for (auto &pk : sealed) {
            const cudaError_t err = cudaMemcpyAsync(pk->dev, pk->slab->host, pk->fill, cudaMemcpyHostToDevice, e->copy_stream[0]);
            if (err != cudaSuccess) { (void)cudaGetLastError(); pk->failed.store(true); }
            else e->st_h2d += pk->bytes;
            e->slabs_returning.fetch_add(1, std::memory_order_relaxed);
            slabs.push_back(SentSlab{pk->slab, nullptr, 0});     // back to the ring with the next copy-event batch (step 4)
            pk->slab = nullptr;
            pk->dma_issued.store(true);
            live_packs.push_back(pk);
        }
        sealed.clear();
        for (size_t i = 0; i < live_packs.size();)      // staging buffers whose members have all been reaped (or aborted)
            if (live_packs[i]->refs.load() == 0) {
                { std::lock_guard<std::mutex> g(e->pack_mu); e->pack_dev_free.push_back(live_packs[i]->dev); }
                live_packs[i] = live_packs.back();
                live_packs.pop_back();
            } else ++i;
        // 4. tag the newly DMA'd slabs with copy events
        if (!slabs.empty() && b_live < kSlabBatches) {
            SlabBatch &b = e->batches[b_head];
            b.slabs.swap(slabs);
            for (int i = 0; i < kCopyStreams; ++i) cudaEventRecord(b.ev[i], e->copy_stream[i]);
            b.busy = true;
            b_head = (b_head + 1) % kSlabBatches; ++b_live;
        }
        // 5. launch on a free slot.  With launches already running, let the ready set
        //    build up to a worthwhile size first (they will all fit in one launch anyway).
        if (!ready.empty() && n_inflight < kCycles && (fresh || reaped || landed_any || !retry_ready)) {
            const uint64_t open_now = e->n_streams;
            const bool worthwhile = n_inflight == 0 || ready.size() * 8 >= open_now || ready.size() >= 4096;
            if (worthwhile) {
                for (Cycle &c : e->cycles) {
                    if (c.busy) continue;
                    const size_t before = ready.size();
                    if (run_cycle(e, c, ready)) { ++n_inflight; retry_ready = false; launched = true; }
                    else retry_ready = !ready.empty() && ready.size() == before;   // all blocked on their own jobs
                    break;
                }
            }
        }
        if (stopping && !n_inflight && !b_live && ready.empty() && slabs.empty()) {
            std::lock_guard<std::mutex> g(e->work_mu);
            if (e->dirty.empty() && e->pending_slabs.empty()) break;       // (packs still referenced belong to streams nobody will finish)
        }
    }
}

// ---- disk tier -----------------------------------------------------------------

Bounce *bounce_get(dm_engine *e)
{
    std::unique_lock<std::mutex> g(e->bounce_mu);
    e->bounce_cv.wait(g, [&] { return !e->bounce_free.empty(); });
    Bounce *b = e->bounce_free.back();
    e->bounce_free.pop_back();
    return b;
}
Bounce *bounce_try_get(dm_engine *e)      // for long-lived borrowers: leaves a reserve
{
    std::lock_guard<std::mutex> g(e->bounce_mu);
    if ((int)e->bounce_free.size() <= kBounceReserve) return nullptr;
    Bounce *b = e->bounce_free.back();
    e->bounce_free.pop_back();
    return b;
}
void bounce_put(dm_engine *e, Bounce *b)
{
    { std::lock_guard<std::mutex> g(e->bounce_mu); e->bounce_free.push_back(b); }
    e->bounce_cv.notify_one();
}

void mkdirs(const std::string &path)
{
    for (size_t i = 1; i < path.size(); ++i)
        if (path[i] == '/') { std::string p = path.substr(0, i); mkdir(p.c_str(), 0755); }
}

// Write the first `size` bytes held in `ext` to `fd` through two pinned buffers: the D2H of piece k+1 runs
// while piece k is written to the file.  Used by the disk tier (spill), dm_stream_suspend and dm_cache_export.
// *cuda_failed (when given): the failure was a copy, not a write.
bool d2h_to_fd(dm_engine *e, const std::vector<Extent> &ext, uint64_t size, int fd, bool *cuda_failed)
{
    if (cuda_failed) *cuda_failed = false;
    Bounce *bn[2] = {bounce_get(e), bounce_get(e)};
    uint64_t piece_len[2] = {0, 0};
    bool ok = true;
    auto start_piece = [&](int slot, uint64_t off) {
        const uint64_t n = std::min<uint64_t>(kBounceBytes, size - off);
        uint8_t *dst = bn[slot]->host;
        cudaError_t err = cudaSuccess;
        for_segments(e, ext, off, n, [&](uint8_t *dev, uint64_t len) {
            if (err == cudaSuccess) err = cudaMemcpyAsync(dst, dev, len, cudaMemcpyDeviceToHost, bn[slot]->stream);
            dst += len;
        });
        piece_len[slot] = n;
        if (err != cudaSuccess && cuda_failed) *cuda_failed = true;
        return err == cudaSuccess;
    };
    uint64_t issued = 0, written = 0;
    int cur = 0;
    if (size) { ok = start_piece(0, 0); issued = piece_len[0]; }
    while (ok && written < size) {
        if (issued < size) { ok = start_piece(cur ^ 1, issued); issued += piece_len[cur ^ 1]; }
        if (cudaStreamSynchronize(bn[cur]->stream) != cudaSuccess) {
            if (cuda_failed) *cuda_failed = true;
            ok = false;
            break;
        }
        const uint64_t n = piece_len[cur];
        e->st_d2h += n;
        uint64_t w = 0;
        while (w < n) {
            ssize_t r = write(fd, bn[cur]->host + w, n - w);
            if (r < 0) { if (errno == EINTR) continue; ok = false; break; }
            w += (uint64_t)r;
        }
        written += n;
        cur ^= 1;
    }
    cudaStreamSynchronize(bn[0]->stream);
    cudaStreamSynchronize(bn[1]->stream);
    bounce_put(e, bn[0]);
    bounce_put(e, bn[1]);
    return ok;
}

// ---- disk-tier limit (dm_cache_set_disk_limit) -------------------------------------------------------------------
// Host bookkeeping only: which entries exist, their bytes and their order.  Every placement reserves its bytes before
// they reach the disk, and a reservation evicts unpinned entries, least recently used first, until it fits.

static std::string tier_saved_base(const dm_engine *e, const Digest &d) { return e->cas_dir + "/partial/" + hex_of(d.b, 32); }

static uint64_t file_size(const std::string &path, struct stat *out = nullptr)
{
    struct stat st;
    if (stat(path.c_str(), &st) != 0 || !S_ISREG(st.st_mode)) return 0;
    if (out) *out = st;
    return (uint64_t)st.st_size;
}

static int64_t stamp_of(const struct stat &st) { return (int64_t)st.st_mtim.tv_sec * 1000000000 + st.st_mtim.tv_nsec; }

// tier_mu held: `k` becomes the most recently used entry; a blob's file gets the time as its mtime.
static void tier_rank(dm_engine *e, const TierKey &k, TierEntry &t, bool write_mtime)
{
    DiskTier &T = e->tier;
    if (t.seq) T.order.erase(t.seq);
    t.seq = ++T.seq;
    T.order.emplace(t.seq, k);
    if (!write_mtime || k.saved || t.linked) return;
    struct timespec now;
    clock_gettime(CLOCK_REALTIME, &now);
    const int64_t ns = std::max<int64_t>((int64_t)now.tv_sec * 1000000000 + now.tv_nsec, T.last_stamp + 1);
    T.last_stamp = ns;
    const struct timespec ts[2] = {{0, UTIME_OMIT}, {(time_t)(ns / 1000000000), (long)(ns % 1000000000)}};
    utimensat(AT_FDCWD, blob_path(e, k.d.b).c_str(), ts, 0);
}

// tier_mu held: drop the entry from the index (its files are gone or going).
static void tier_erase(dm_engine *e, const Digest &d, bool saved)
{
    DiskTier &T = e->tier;
    auto &m = saved ? T.saved : T.blobs;
    auto it = m.find(d);
    if (it == m.end()) return;
    (saved ? T.partial_bytes : T.blob_bytes) -= it->second.bytes;
    T.order.erase(it->second.seq);
    m.erase(it);
}

// tier_mu held: (re)enter the files of `d` at their current st_size.
void tier_enter(dm_engine *e, const Digest &d, bool saved, bool use)
{
    DiskTier &T = e->tier;
    uint64_t bytes;
    struct stat st{};
    if (saved) {                                // either file alone is counted (and evicted) too: a record being rewritten
        const std::string base = tier_saved_base(e, d);
        struct stat part{};
        bytes = file_size(base + ".ckpt", &st) + file_size(base + ".part", &part);
        if (!S_ISREG(st.st_mode)) st = part;
    } else {
        const std::string path = blob_path(e, d.b);
        bytes = file_size(path, &st);
        if (bytes || S_ISREG(st.st_mode)) bytes += file_size(path + ".meta");
    }
    if (!S_ISREG(st.st_mode)) { tier_erase(e, d, saved); return; }
    auto &m = saved ? T.saved : T.blobs;
    auto ins = m.emplace(d, TierEntry{});
    TierEntry &t = ins.first->second;
    (saved ? T.partial_bytes : T.blob_bytes) += bytes - t.bytes;
    t.bytes = bytes;
    t.linked = !saved && st.st_nlink > 1;
    if (ins.second || use) tier_rank(e, TierKey{d, saved}, t, use);
}

static bool tier_pinned(const DiskTier &T, const TierKey &k)
{
    const auto &p = k.saved ? T.saved_pins : T.pins;
    auto it = p.find(k.d);
    return it != p.end() && it->second > 0;
}

// tier_mu held: evict unpinned entries until `need` more bytes fit under the limit.  Disk-only entries go first, least
// recently used first; then the disk copies of HBM-resident blobs (the hot set), in HBM LRU order.  `partial`: evict as
// far as possible even when that is not enough (a new limit); otherwise nothing goes unless the placement then fits.
// A blob's index entry is updated under e->mu as the victims are taken; the files are removed afterwards (tier_mu keeps
// every pinning caller out until then).  A blob whose disk copy goes while it stays in HBM is never spilled again.
bool tier_make_room(dm_engine *e, uint64_t need, bool partial)
{
    DiskTier &T = e->tier;
    if (!T.on || T.used() + need <= T.limit) return true;
    const uint64_t over = T.used() + need - T.limit;
    std::vector<TierKey> victims;
    uint64_t freed = 0;
    {
        std::lock_guard<std::mutex> g(e->mu);
        for (auto &kv : T.order) {
            if (freed >= over) break;
            const TierKey &k = kv.second;
            if (tier_pinned(T, k)) continue;
            if (!k.saved) {
                auto it = e->blobs.find(k.d);
                if (it != e->blobs.end() && it->second->in_hbm) continue;
            }
            victims.push_back(k);
            freed += (k.saved ? T.saved : T.blobs)[k.d].bytes;
        }
        for (Blob *b = e->lru_head; b && freed < over; b = b->lru_next) {
            auto it = T.blobs.find(b->digest);
            const TierKey k{b->digest, false};
            if (it == T.blobs.end() || tier_pinned(T, k)) continue;
            victims.push_back(k);
            freed += it->second.bytes;
        }
        if (freed < over && !partial) return false;
        for (const TierKey &k : victims) {
            if (k.saved) continue;
            auto it = e->blobs.find(k.d);
            if (it == e->blobs.end()) continue;
            if (it->second->in_hbm) { it->second->on_disk = false; it->second->spill_done = true; }
            else e->blobs.erase(it);
        }
    }
    for (const TierKey &k : victims) {
        uint64_t bytes;
        if (k.saved) {
            const std::string base = tier_saved_base(e, k.d);
            unlink((base + ".ckpt").c_str());            // the record first: a .part without it is never resumed
            unlink((base + ".part").c_str());
            if (e->n_suspended) e->n_suspended--;
            bytes = T.saved[k.d].bytes;
        } else {
            const std::string path = blob_path(e, k.d.b);
            unlink(path.c_str());
            unlink((path + ".meta").c_str());
            bytes = T.blobs[k.d].bytes;
        }
        T.evicted_files++;
        T.evicted_bytes += bytes;
        tier_erase(e, k.d, k.saved);
    }
    return T.used() + need <= T.limit;
}

static void count_down(std::unordered_map<Digest, uint32_t, DigestHash> &m, const Digest &d)
{
    auto it = m.find(d);
    if (it != m.end() && --it->second == 0) m.erase(it);
}

void tier_pin(dm_engine *e, const Digest &d, bool saved, bool spill)
{
    std::lock_guard<std::mutex> g(e->tier_mu);
    (saved ? e->tier.saved_pins : e->tier.pins)[d]++;
    if (spill) e->tier.spills[d]++;
}

void tier_unpin(dm_engine *e, const Digest &d, bool saved, bool spill)
{
    std::lock_guard<std::mutex> g(e->tier_mu);
    count_down(saved ? e->tier.saved_pins : e->tier.pins, d);
    if (spill) count_down(e->tier.spills, d);
}

bool tier_reserve(dm_engine *e, uint64_t bytes, bool partial, TierRes *r)
{
    *r = TierRes{};
    if (!e->tier_on.load(std::memory_order_acquire)) return true;
    std::lock_guard<std::mutex> g(e->tier_mu);
    DiskTier &T = e->tier;
    if (!T.on) return true;
    if (!tier_make_room(e, bytes, false)) { T.refused++; return false; }
    (partial ? T.reserved_partial : T.reserved_blob) += bytes;
    *r = TierRes{bytes, T.gen, partial};
    return true;
}

static void tier_release_locked(dm_engine *e, TierRes &r)
{
    DiskTier &T = e->tier;
    if (r.gen && T.on && r.gen == T.gen) (r.partial ? T.reserved_partial : T.reserved_blob) -= r.bytes;
    r = TierRes{};
}

void tier_release(dm_engine *e, TierRes &r)
{
    if (!r.gen) return;
    std::lock_guard<std::mutex> g(e->tier_mu);
    tier_release_locked(e, r);
}

void tier_placed(dm_engine *e, const Digest &d, bool saved, TierRes *r, bool use)
{
    if (!e->tier_on.load(std::memory_order_acquire) && !(r && r->gen)) return;
    std::lock_guard<std::mutex> g(e->tier_mu);
    if (r) tier_release_locked(e, *r);
    if (e->tier.on) tier_enter(e, d, saved, use);
}

void tier_touch(dm_engine *e, const Digest &d)
{
    if (!e->tier_on.load(std::memory_order_acquire)) return;
    std::lock_guard<std::mutex> g(e->tier_mu);
    auto it = e->tier.blobs.find(d);
    if (e->tier.on && it != e->tier.blobs.end()) tier_rank(e, TierKey{d, false}, it->second, true);
}

void tier_forget(dm_engine *e, const Digest &d, bool saved)
{
    if (!e->tier_on.load(std::memory_order_acquire)) return;
    std::lock_guard<std::mutex> g(e->tier_mu);
    if (e->tier.on) tier_enter(e, d, saved, false);    // what is there now: another call may have placed files meanwhile
}

static void tier_charge(DiskTier &T, std::pair<uint64_t, uint64_t> &s, uint64_t reserved, uint64_t written)
{
    T.staging_bytes -= std::max(s.first, s.second);
    s.first = reserved; s.second = written;
    T.staging_bytes += std::max(s.first, s.second);
}

bool tier_stage(dm_engine *e, const std::string &path, uint64_t reserve, uint64_t counted)
{
    if (!e->tier_on.load(std::memory_order_acquire)) return true;
    std::lock_guard<std::mutex> g(e->tier_mu);
    DiskTier &T = e->tier;
    if (!T.on) return true;
    const uint64_t need = reserve - std::min(reserve, counted);
    if (need && !tier_make_room(e, need, false)) { T.refused++; return false; }
    tier_charge(T, T.staging[path], reserve, 0);
    return true;
}

void tier_stage_grow(dm_engine *e, const std::string &path, uint64_t written)
{
    if (!e->tier_on.load(std::memory_order_acquire)) return;
    std::lock_guard<std::mutex> g(e->tier_mu);
    DiskTier &T = e->tier;
    if (!T.on) return;
    auto &s = T.staging[path];
    if (written > s.second) tier_charge(T, s, s.first, written);
}

void tier_unstage(dm_engine *e, const std::string &path)
{
    if (!e->tier_on.load(std::memory_order_acquire)) return;
    std::lock_guard<std::mutex> g(e->tier_mu);
    DiskTier &T = e->tier;
    auto it = T.staging.find(path);
    if (it == T.staging.end()) return;
    tier_charge(T, it->second, 0, 0);
    T.staging.erase(it);
}

bool tier_stage_to_blob(dm_engine *e, const std::string &path, uint64_t size, uint64_t side, TierRes *r)
{
    *r = TierRes{};
    if (!e->tier_on.load(std::memory_order_acquire)) return true;
    std::lock_guard<std::mutex> g(e->tier_mu);
    DiskTier &T = e->tier;
    uint64_t granted = 0;                       // room reserved for the body when it was staged
    auto it = T.staging.find(path);
    if (it != T.staging.end()) { granted = it->second.first; tier_charge(T, it->second, 0, 0); T.staging.erase(it); }
    if (!T.on) return true;
    // A body whose room was reserved up front keeps it: it is placed even when unknown-size bodies have run the tier
    // over the limit meanwhile (its sidecar then adds to that overshoot), unless the limit has since been lowered below
    // what it needs.  Anything else must fit now.
    const uint64_t bytes = size + side;
    if (!tier_make_room(e, bytes, false) && (granted < size || bytes > T.limit)) { T.refused++; return false; }
    T.reserved_blob += bytes;
    *r = TierRes{bytes, T.gen, false};
    return true;
}

// tier_mu held: the one walk of blobs/, incoming/ and partial/ that builds the index.  Removes spill leftovers
// (<hex>.part under blobs/ with no spill of this engine running), sidecars without their blob and the incoming/ files
// of processes that are gone.  Entries are ranked by mtime.
void tier_build(dm_engine *e)
{
    DiskTier &T = e->tier;
    T.blobs.clear(); T.saved.clear(); T.order.clear(); T.staging.clear();
    T.blob_bytes = T.partial_bytes = T.staging_bytes = T.reserved_blob = T.reserved_partial = 0;
    T.gen++;
    std::vector<std::pair<int64_t, TierKey>> ranked;
    const std::string root = e->cas_dir + "/blobs/sha256/";
    for (int p = 0; p < 256; ++p) {
        char aa[3];
        snprintf(aa, sizeof aa, "%02x", p);
        const std::string dir = root + aa + "/";
        DIR *d = opendir(dir.c_str());
        if (!d) continue;
        std::vector<std::string> names;
        while (struct dirent *de = readdir(d)) if (de->d_name[0] != '.') names.emplace_back(de->d_name);
        closedir(d);
        std::unordered_map<Digest, uint64_t, DigestHash> metas;
        for (const std::string &n : names) {
            Digest dg;
            const bool named = n.size() >= 64 && n.compare(0, 2, aa) == 0 && digest_from_hex(n.substr(0, 64).c_str(), dg.b) &&
                               hex_of(dg.b, 32) == n.substr(0, 64);
            struct stat st;
            if (stat((dir + n).c_str(), &st) != 0 || !S_ISREG(st.st_mode)) continue;
            const std::string tail = named ? n.substr(64) : n;
            if (named && tail.empty()) {
                auto &t = T.blobs[dg];
                t.bytes += (uint64_t)st.st_size;
                t.linked = st.st_nlink > 1;
                ranked.push_back({stamp_of(st), TierKey{dg, false}});
            } else if (named && tail == ".meta") {
                metas[dg] = (uint64_t)st.st_size;
            } else if (named && tail == ".part") {
                if (!T.spills.count(dg)) unlink((dir + n).c_str());       // (a running spill's file is counted when placed)
            } else {
                T.blob_bytes += (uint64_t)st.st_size;     // not ours to remove; counted so the total is the tier's
            }
        }
        for (auto &kv : metas) {
            auto it = T.blobs.find(kv.first);
            if (it != T.blobs.end()) it->second.bytes += kv.second;
            else unlink((dir + hex_of(kv.first.b, 32) + ".meta").c_str());
        }
    }
    for (auto &kv : T.blobs) T.blob_bytes += kv.second.bytes;
    if (DIR *d = opendir((e->cas_dir + "/partial").c_str())) {
        std::vector<std::string> names;
        while (struct dirent *de = readdir(d)) if (de->d_name[0] != '.') names.emplace_back(de->d_name);
        closedir(d);
        for (const std::string &n : names) {
            struct stat st;
            if (stat((e->cas_dir + "/partial/" + n).c_str(), &st) != 0 || !S_ISREG(st.st_mode)) continue;
            Digest dg;
            const bool rec = n.size() == 69 && (n.compare(64, 5, ".ckpt") == 0 || n.compare(64, 5, ".part") == 0) &&
                             digest_from_hex(n.substr(0, 64).c_str(), dg.b);
            if (!rec) { T.partial_bytes += (uint64_t)st.st_size; continue; }
            auto ins = T.saved.emplace(dg, TierEntry{});
            ins.first->second.bytes += (uint64_t)st.st_size;
            T.partial_bytes += (uint64_t)st.st_size;
            if (ins.second) ranked.push_back({stamp_of(st), TierKey{dg, true}});
        }
    }
    const std::string inc = e->cas_dir + "/incoming";
    sweep_incoming(inc);
    if (DIR *d = opendir(inc.c_str())) {
        std::vector<std::string> names;
        while (struct dirent *de = readdir(d)) if (de->d_name[0] != '.') names.emplace_back(de->d_name);
        closedir(d);
        for (const std::string &n : names) {
            const uint64_t sz = file_size(inc + "/" + n);
            tier_charge(T, T.staging[inc + "/" + n], 0, sz);
        }
    }
    std::stable_sort(ranked.begin(), ranked.end(), [](const auto &a, const auto &b) { return a.first < b.first; });
    for (auto &r : ranked) {
        TierEntry &t = (r.second.saved ? T.saved : T.blobs)[r.second.d];
        t.seq = ++T.seq;
        T.order.emplace(t.seq, r.second);
        T.last_stamp = std::max(T.last_stamp, r.first);
    }
    T.on = true;
}

bool spill_one(dm_engine *e, Blob *b)
{
    const std::string path = blob_path(e, b->digest.b), tmp = path + ".part";
    mkdirs(path);
    int fd = open(tmp.c_str(), O_CREAT | O_TRUNC | O_WRONLY, 0644);
    if (fd < 0) return false;
    bool ok = d2h_to_fd(e, b->extents, b->size, fd);
    close(fd);
    bool removed = false;                       // dm_cache_remove took the blob out meanwhile: its file must not appear
    if (ok) {
        std::lock_guard<std::mutex> g(e->mu);
        removed = b->removed;
        b->renaming = !removed;
    }
    if (ok && !removed) {
        ok = rename(tmp.c_str(), path.c_str()) == 0;
        if (ok) write_sidecar(path + ".meta", *b);
        { std::lock_guard<std::mutex> g(e->mu); b->renaming = false; }
        e->remove_cv.notify_all();
    }
    if (!ok || removed) unlink(tmp.c_str());
    return ok && !removed;
}

void spill_main(dm_engine *e)
{
    cudaSetDevice(e->device);
    for (;;) {
        std::shared_ptr<Blob> b;
        {
            std::unique_lock<std::mutex> g(e->spill_mu);
            e->spill_cv.wait(g, [&] { return !e->spill_q.empty() || e->stop; });
            if (e->spill_q.empty()) break;
            b = e->spill_q.front();
            e->spill_q.pop_front();
        }
        tier_pin(e, b->digest, false, true);   // a running spill: its .part is not a leftover, its digest not a victim
        bool have;
        std::string side;
        {
            std::lock_guard<std::mutex> g(e->mu);
            have = b->in_hbm;
            if (have) { b->readers++; side = sidecar_json(*b); }   // pin against eviction while copying out
        }
        TierRes res;
        bool ok = have && tier_reserve(e, b->size + side.size(), false, &res) && spill_one(e, b.get());
        if (ok) tier_placed(e, b->digest, false, &res, true);
        else tier_release(e, res);
        std::vector<Extent> gone;
        {
            std::lock_guard<std::mutex> g(e->mu);
            if (have) gone = reader_gone(b.get());
            b->on_disk = b->on_disk || ok;     // (a disk-backed publish or an import may have placed a copy meanwhile)
            b->spill_done = true;
        }
        if (!gone.empty()) free_extents(e, gone);
        tier_unpin(e, b->digest, false, true);
        {
            std::lock_guard<std::mutex> g(e->spill_mu);
        }
        e->spill_done_cv.notify_all();
    }
}

// The device mirror of the ring exists from the start with DM_F_NO_HBM_CAS, otherwise it is
// allocated the first time a blob too large for the arena shows up.
int ensure_dev_ring(dm_engine *e)
{
    std::lock_guard<std::mutex> g(e->slab_mu);
    if (e->dev_ring) return DM_OK;
    cudaSetDevice(e->device);
    const uint64_t bytes = (uint64_t)e->slab_store.size() * e->cfg.slab_bytes;
    CU_TRY(cudaMalloc(&e->dev_ring, bytes));
    for (size_t i = 0; i < e->slab_store.size(); ++i) e->slab_store[i].dev = e->dev_ring + i * e->cfg.slab_bytes;
    return DM_OK;
}

// ---- disk-backed streams (DM_F_DISK_DIRECT) and checks of disk-tier files (dm_cache_verify) ---------------
// The client writes into ring slabs as on every stream; a full slab (or a recalled partial one, or a range part)
// is pwritten at its blob offset by a disk thread and returns to the ring when the write completes, so the
// client runs at the speed of the network and the disk.  The hash follows from the file: a disk thread reads
// the contiguous written prefix back into a ring slab, copies it to the slab's device mirror and stages it,
// and the pump hashes it exactly as a verify-only slab (one slab per job).  The digest is therefore over the
// bytes of the file that gets published.

std::string incoming_path(const dm_engine *e, uint64_t id)
{
    return e->cas_dir + "/incoming/" + std::to_string((long)getpid()) + "-" + std::to_string(e->device) + "-" +
           std::to_string(id) + ".part";
}

void disk_enqueue(dm_engine *e, DiskTask t)
{
    { std::lock_guard<std::mutex> g(e->disk_mu); e->disk_q.push_back(std::move(t)); }
    e->disk_cv.notify_one();
}

void disk_write(dm_engine *e, const std::shared_ptr<Stream> &sp, Slab *slab, uint64_t off, uint32_t n)
{
    e->slabs_returning.fetch_add(1, std::memory_order_relaxed);     // comes back by itself once written
    sp->disk_writes++;
    disk_enqueue(e, DiskTask{DiskTask::Write, sp, slab, sp->fd, off, n});
}

bool disk_fed(const Stream *s)
{
    return s->disk_writes == 0 && s->disk_reads == 0 &&
           (s->staged_to == s->dma_issued || s->lost != DM_OK || s->cuda_failed);
}

void disk_feed(dm_engine *e, const std::shared_ptr<Stream> &sp)
{
    Stream *s = sp.get();
    // at most two slabs on the hash side per stream, counting the one its running job reads: with the writer's slab
    // a disk-backed body never holds more than three
    if (!s->disk || s->disk_reads || s->staged.size() + s->jobs_inflight >= 2 || s->suspending || s->lost != DM_OK ||
        s->cuda_failed)
        return;
    // a ring load also counts the slabs its reader has not finished with: a slow reader slows its own load only
    if (s->ring && (s->ring->closed || s->ring->held.size() >= s->ring->cap)) return;
    if (s->st != St::Open && s->st != St::Finishing) return;
    uint64_t end = s->staged_to;
    auto it = s->written.upper_bound(s->staged_to);
    if (it != s->written.begin() && std::prev(it)->second > s->staged_to) end = std::prev(it)->second;
    uint64_t n = std::min<uint64_t>(end - s->staged_to, e->cfg.slab_bytes);
    // whole blocks only (jobs chain block by block); the final partial block once nothing more can arrive
    const bool last = s->st == St::Finishing && s->disk_writes == 0 && s->staged_to + n == s->dma_issued;
    if (!last) n &= ~63ull;
    if (n == 0) return;
    Slab *sl = slab_try_get(e);
    if (!sl) {
        { std::lock_guard<std::mutex> g(e->disk_mu); e->disk_starved.push_back(sp); e->feed_starved.store(true); }
        { std::lock_guard<std::mutex> g(e->work_mu); e->ring_starved.store(true); }     // the pump may recall partial slabs
        e->work_cv.notify_one();
        e->disk_cv.notify_one();
        return;
    }
    e->slabs_returning.fetch_add(1, std::memory_order_relaxed);     // staged: back to the ring when its job is reaped
    s->disk_reads++;
    disk_enqueue(e, DiskTask{DiskTask::Read, sp, sl, s->fd, s->staged_to, (uint32_t)n});
    s->staged_to += n;
}

static int pwrite_all(int fd, const uint8_t *p, uint64_t n, uint64_t off)
{
    while (n) {
        const ssize_t r = pwrite(fd, p, n, (off_t)off);
        if (r < 0 && errno == EINTR) continue;
        if (r <= 0) return r < 0 ? errno : ENOSPC;
        p += r; n -= (uint64_t)r; off += (uint64_t)r;
    }
    return 0;
}

static bool pread_all(int fd, uint8_t *p, uint64_t n, uint64_t off)
{
    while (n) {
        const ssize_t r = pread(fd, p, n, (off_t)off);
        if (r < 0 && errno == EINTR) continue;
        if (r <= 0) return false;
        p += r; n -= (uint64_t)r; off += (uint64_t)r;
    }
    return true;
}

static void disk_task_write(dm_engine *e, DiskTask &t)
{
    Stream *s = t.sp.get();
    const int err = pwrite_all(t.fd, t.slab->host, t.n, t.off);
    slab_return(e, t.slab);
    if (!err) tier_stage_grow(e, s->path, t.off + t.n);     // (the path is stable while a write is in flight)
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (err && s->lost == DM_OK) s->lost = fail(DM_EIO, "write to the disk-backed stream's file failed");
        if (!err) add_interval(s->written, t.off, t.off + t.n);
        s->disk_writes--;
        disk_feed(e, t.sp);
        if (s->st == St::Finishing) mark_dirty(e, t.sp, nullptr);   // a failed write still has to end in a (failed) verdict
    }
    s->cv.notify_all();
}

static void disk_task_read(dm_engine *e, DiskTask &t)
{
    Stream *s = t.sp.get();
    cudaStream_t cs = e->copy_stream[s->id % kCopyStreams];
    const bool got = pread_all(t.fd, t.slab->host, t.n, t.off);
    const cudaError_t err = got ? cudaMemcpyAsync(t.slab->dev, t.slab->host, t.n, cudaMemcpyHostToDevice, cs) : cudaSuccess;
    if (err != cudaSuccess) (void)cudaGetLastError();
    bool keep;
    {
        std::lock_guard<std::mutex> g(s->mu);
        s->disk_reads--;
        if (!got && s->lost == DM_OK) s->lost = fail(DM_EIO, "read-back of the disk-backed stream's file failed");
        if (err != cudaSuccess) s->cuda_failed = true;
        keep = got && err == cudaSuccess && s->st != St::Aborted && !s->suspending;
        if (keep) {
            e->st_h2d += t.n;
            s->staged.emplace_back(t.slab, t.n);
            if (s->ring) s->ring->held.push_back(RingLoad::Held{t.slab, t.off, t.n, false});
            disk_feed(e, t.sp);
        }
        if (keep || s->st == St::Finishing) mark_dirty(e, t.sp, nullptr);
    }
    if (!keep) {
        cudaStreamSynchronize(cs);               // the copy out of the slab may still be running
        slab_return(e, t.slab);
    }
    s->cv.notify_all();
}

// The final job has been reaped.  Matched and whole: the file becomes the blob in the disk tier; anything else
// (a mismatch, a failed copy or launch, a lost write, an abort): the file is removed.
static void disk_task_publish(dm_engine *e, DiskTask &t)
{
    Stream *s = t.sp.get();
    std::unique_lock<std::mutex> g(s->mu);
    if (s->check_only) {                        // dm_cache_verify: the verdict is all; the file is the caller's to judge
        if (s->fd >= 0) { close(s->fd); s->fd = -1; }
        s->publishing = false;
        const bool ring = s->ring && s->st != St::Aborted;
        if (s->st != St::Aborted) s->st = St::Done;
        g.unlock();
        s->cv.notify_all();
        if (ring) ring_load_settle(e, t.sp);    // (its reader waits for this, not for Done)
        return;
    }
    const bool whole = s->resume_base == 0 ||
                       (s->prefix_cover.size() == 1 && s->prefix_cover.begin()->first == 0 &&
                        s->prefix_cover.begin()->second >= s->resume_base);
    const bool keep = s->st != St::Aborted && s->matched && whole && s->lost == DM_OK && !s->cuda_failed;
    const int fd = s->fd;
    s->fd = -1;
    const std::string path = s->path;
    const uint64_t size = s->dma_issued;
    auto b = std::make_shared<Blob>();
    b->digest = s->digest; b->size = size;
    b->meta.swap(s->meta);
    const bool counted_mismatch = !s->matched;
    g.unlock();
    std::string side = sidecar_json(*b);
    bool ok = keep && ftruncate(fd, (off_t)size) == 0 && (!(e->cfg.flags & DM_F_DISK_SYNC) || fsync(fd) == 0);
    if (fd >= 0) close(fd);
    std::shared_ptr<Blob> pub;
    bool refused = false;                       // no room under the disk-tier limit: verified, not cached
    if (ok) {
        const std::string dst = blob_path(e, b->digest.b);
        mkdirs(dst);
        tier_pin(e, b->digest);                 // not a victim while it is placed
        TierRes res;
        struct stat st;
        const bool had = stat(dst.c_str(), &st) == 0;          // already in the disk tier: keep that copy
        if (had) { unlink(path.c_str()); tier_unstage(e, path); tier_touch(e, b->digest); }
        else if (!tier_stage_to_blob(e, path, size, side.size(), &res)) refused = true;
        else ok = rename(path.c_str(), dst.c_str()) == 0;
        if (ok && !had && !refused) {
            write_sidecar(dst + ".meta", *b);
            tier_placed(e, b->digest, false, &res, true);
        } else tier_release(e, res);
        if (refused) ok = false;
        if (ok) {                               // still pinned: the file the index now names cannot be evicted first
            std::lock_guard<std::mutex> gi(e->mu);
            auto it = e->blobs.find(b->digest);
            if (it != e->blobs.end()) pub = it->second;
            else {
                b->on_disk = b->spill_done = true;
                e->blobs[b->digest] = b;
                pub = b;
            }
            if (!pub->on_disk) { pub->on_disk = true; pub->spill_done = true; }
        }
        tier_unpin(e, b->digest);
    }
    if (!ok) { unlink(path.c_str()); tier_unstage(e, path); }
    if (ok) e->st_committed++;
    else if (counted_mismatch || (keep && !refused)) e->st_mismatch++;
    g.lock();
    if (keep && !ok && !refused) { s->matched = 0; if (s->lost == DM_OK) s->lost = fail(DM_EIO, "could not move the verified file into the disk tier"); }
    s->publishing = false;
    s->blob = pub;
    s->sidecar.swap(side);
    if (s->st != St::Aborted) s->st = St::Done;
    g.unlock();
    s->cv.notify_all();
}

void disk_main(dm_engine *e)
{
    cudaSetDevice(e->device);
    for (;;) {
        DiskTask t;
        std::vector<std::weak_ptr<Stream>> retry;
        {
            std::unique_lock<std::mutex> g(e->disk_mu);
            // A starved read-back may be queued by any thread (the pump's reap, a finishing client, resume) while every
            // disk thread sleeps: it is work of its own, retried at once, then whenever a slab is put back (slab_put
            // notifies) and at least every millisecond while the ring stays empty.
            auto work = [&] { return !e->disk_q.empty() || e->disk_stop; };
            if (e->disk_starved.empty()) e->disk_cv.wait(g, [&] { return work() || !e->disk_starved.empty(); });
            else e->disk_cv.wait_for(g, std::chrono::milliseconds(1), [&] { return work() || e->feed_kick; });
            e->feed_kick = false;
            if (e->disk_q.empty() && e->disk_stop) break;
            if (!e->disk_starved.empty()) { retry.swap(e->disk_starved); e->feed_starved.store(false); }
            if (!e->disk_q.empty()) { t = std::move(e->disk_q.front()); e->disk_q.pop_front(); }
        }
        for (auto &w : retry)
            if (auto sp = w.lock()) { std::lock_guard<std::mutex> g(sp->mu); disk_feed(e, sp); }
        if (!t.sp) continue;
        if (t.kind == DiskTask::Write) disk_task_write(e, t);
        else if (t.kind == DiskTask::Read) disk_task_read(e, t);
        else disk_task_publish(e, t);
    }
}

void ensure_disk_threads(dm_engine *e)
{
    std::lock_guard<std::mutex> g(e->disk_mu);
    if (!e->disk_threads.empty() || e->disk_stop) return;
    for (int i = 0; i < kDiskThreads; ++i) e->disk_threads.emplace_back(disk_main, e);
}

std::shared_ptr<Stream> find_stream(dm_engine *e, uint64_t id)
{
    const int k = (int)(id % kStripes);
    std::lock_guard<std::mutex> g(e->stripe_mu[k]);
    auto it = e->streams[k].find(id);
    return it == e->streams[k].end() ? nullptr : it->second;
}

void drop_stream(dm_engine *e, const std::shared_ptr<Stream> &sp, bool release_slot)
{
    const int k = (int)(sp->id % kStripes);
    bool erased;
    {
        std::lock_guard<std::mutex> g(e->stripe_mu[k]);
        erased = e->streams[k].erase(sp->id) != 0;
        if (erased) e->n_streams--;
    }
    // exactly one caller takes the stream out of the table, and only that one may give its state slot
    // back (two finishes on one id, or a finish racing an abort, would otherwise release it twice and
    // two later streams would share one state / digest slot)
    if (release_slot && erased) {
        std::lock_guard<std::mutex> g(e->slot_mu);
        e->free_slots.push_back(sp->slot);
    }
    if (sp->has_expect) {                            // only streams with an expected digest are in the follow index
        std::lock_guard<std::mutex> g(e->mu);
        auto it = e->inflight.find(sp->expect);
        if (it != e->inflight.end() && (it->second.expired() || it->second.lock() == sp)) e->inflight.erase(it);
    }
    if (sp->held && erased) release_digest(e, sp->expect);
}

void hold_digest(dm_engine *e, const Digest &d, const char *what)
{
    std::lock_guard<std::mutex> g(e->mu);
    auto &h = e->holds[d];
    h.n++;
    h.what = what;
}

void release_digest(dm_engine *e, const Digest &d)
{
    std::lock_guard<std::mutex> g(e->mu);
    auto it = e->holds.find(d);
    if (it != e->holds.end() && --it->second.n == 0) e->holds.erase(it);
}

std::vector<Extent> reader_gone(Blob *b)
{
    std::vector<Extent> ext;
    if (--b->readers == 0 && b->removed) ext.swap(b->extents);
    return ext;
}

int ensure_ingest_scratch(dm_engine *e, uint32_t n)
{
    if (n <= e->ing_cap) return DM_OK;
    const uint32_t cap = std::max<uint32_t>(n, 4096);
    // free and forget: if one of the allocations below fails, the next call (or dm_engine_destroy) must not
    // free these a second time
    e->ing_cap = 0;
    if (e->ing_states) { cudaFree(e->ing_states); e->ing_states = nullptr; }
    if (e->ing_digests) { cudaFree(e->ing_digests); e->ing_digests = nullptr; }
    if (e->ing_jobs_d) { cudaFree(e->ing_jobs_d); e->ing_jobs_d = nullptr; }
    if (e->ing_jobs_h) { cudaFreeHost(e->ing_jobs_h); e->ing_jobs_h = nullptr; }
    if (e->ing_digests_h) { cudaFreeHost(e->ing_digests_h); e->ing_digests_h = nullptr; }
    CU_TRY(cudaMalloc(&e->ing_states, 32ull * cap));
    CU_TRY(cudaMalloc(&e->ing_digests, 32ull * cap));
    CU_TRY(cudaMalloc(&e->ing_jobs_d, sizeof(dm::HashJob) * (uint64_t)cap));
    CU_TRY(cudaHostAlloc(&e->ing_jobs_h, sizeof(dm::HashJob) * (uint64_t)cap, cudaHostAllocDefault));
    CU_TRY(cudaHostAlloc(&e->ing_digests_h, 32ull * cap, cudaHostAllocDefault));
    e->ing_cap = cap;
    return DM_OK;
}

}  // namespace dmi
