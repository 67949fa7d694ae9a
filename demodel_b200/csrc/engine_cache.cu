// C-ABI, part 2: hit serving (readers, followers), device-resident ingest, the synthetic generator.
#include "engine_internal.hpp"

extern "C" {

// ---- hit serving ---------------------------------------------------------------

int dm_cache_contains(dm_engine *e, const uint8_t digest[32], uint64_t *size)
{
    if (!e || !digest) return fail(DM_EINVAL, "null argument");
    Digest d;
    memcpy(d.b, digest, 32);
    {
        std::lock_guard<std::mutex> g(e->mu);
        auto it = e->blobs.find(d);
        if (it != e->blobs.end() && (it->second->in_hbm || it->second->on_disk)) {
            if (size) *size = it->second->size;
            return DM_OK;
        }
    }
    if (!e->cas_dir.empty()) {
        struct stat st;
        if (stat(blob_path(e, digest).c_str(), &st) == 0) { if (size) *size = (uint64_t)st.st_size; return DM_OK; }
    }
    return DM_ENOENT;
}

static int cache_open_impl(dm_engine *e, const uint8_t digest[32], uint64_t *reader, uint64_t *size)
{
    if (!e || !digest || !reader) return fail(DM_EINVAL, "null argument");
    Digest d;
    memcpy(d.b, digest, 32);
    auto r = std::make_shared<Reader>();
    {
        std::lock_guard<std::mutex> g(e->mu);
        auto it = e->blobs.find(d);
        if (it != e->blobs.end() && it->second->in_hbm) {
            r->blob = it->second;
            r->blob->readers++;
            lru_touch(e, r->blob.get());
            r->size = r->blob->size;
        }
    }
    if (!r->blob) {
        if (e->cas_dir.empty()) return DM_ENOENT;
        r->fd = open(blob_path(e, digest).c_str(), O_RDONLY);
        if (r->fd < 0) return DM_ENOENT;
        struct stat st;
        fstat(r->fd, &st);
        r->size = (uint64_t)st.st_size;
        if (FILE *mf = fopen((blob_path(e, digest) + ".meta").c_str(), "r")) {
            char tmp[4096];
            size_t k;
            while ((k = fread(tmp, 1, sizeof tmp, mf)) > 0) r->disk_meta.append(tmp, k);
            fclose(mf);
        }
    }
    const uint64_t id = e->next_id.fetch_add(1);
    {
        std::lock_guard<std::mutex> g(e->reader_mu[id % kStripes]);
        e->readers[id % kStripes][id] = r;
    }
    *reader = id;
    if (size) *size = r->size;
    return DM_OK;
}

static std::shared_ptr<Reader> find_reader(dm_engine *e, uint64_t id)
{
    std::lock_guard<std::mutex> g(e->reader_mu[id % kStripes]);
    auto it = e->readers[id % kStripes].find(id);
    return it == e->readers[id % kStripes].end() ? nullptr : it->second;
}

// Read from a body that is still arriving (request coalescing).  Blocks until bytes past `off` have
// been DMA'd, the body completes, or it fails.  Returns DM_OK with *nread set, a dm_err, or 1 when the
// body has completed and been published (the reader has been switched to the blob; caller continues).
static int follow_read(dm_engine *e, Reader *r, uint64_t off, void *buf, size_t len, size_t *nread)
{
    std::lock_guard<std::mutex> gr(r->mu);
    if (!r->follow) return 1;
    Stream *s = r->follow.get();
    std::vector<std::pair<uint8_t *, uint64_t>> segs;
    size_t n = 0;
    {
        std::unique_lock<std::mutex> g(s->mu);
        s->followers++;
        s->cv.wait(g, [&] {
            return s->st == St::Done || s->st == St::Aborted || (off < s->dma_issued && !s->completing) || len == 0;
        });
        s->followers--;
        if (s->st == St::Aborted) return fail(DM_ESTATE, "the upstream body this reader followed was aborted");
        if (s->st == St::Done) {
            std::shared_ptr<Blob> b = s->blob;
            g.unlock();
            if (!b) return fail(DM_ESTATE, "the upstream body this reader followed failed verification");
            std::lock_guard<std::mutex> g2(e->mu);
            if (!b->in_hbm) return fail(DM_ENOENT, "blob evicted before the follower switched over");
            b->readers++;
            r->blob = b;
            r->size = b->size;
            r->follow.reset();
            return 1;
        }
        if (len == 0) return DM_OK;
        n = (size_t)std::min<uint64_t>(len, s->dma_issued - off);
        for_segments(e, s->extents, off, n, [&](uint8_t *dev, uint64_t l) { segs.emplace_back(dev, l); });
        s->follow_reads++;                      // pins the extents until the copy-out below is done
    }
    struct Unpin {
        Stream *s;
        ~Unpin() { { std::lock_guard<std::mutex> g(s->mu); s->follow_reads--; } s->cv.notify_all(); }
    } unpin{s};
    // the bytes may still be in flight on the body's copy stream: order the read-back after them
    cudaSetDevice(e->device);
    Bounce *bn = bounce_get(e);
    cudaEvent_t ev;
    cudaError_t err = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    if (err == cudaSuccess) err = cudaEventRecord(ev, e->copy_stream[s->id % kCopyStreams]);
    if (err == cudaSuccess) err = cudaStreamWaitEvent(bn->stream, ev, 0);
    uint8_t *out = static_cast<uint8_t *>(buf);
    size_t done = 0;
    for (auto &sg : segs) {
        uint64_t left = sg.second;
        uint8_t *dev = sg.first;
        while (left && err == cudaSuccess) {
            const size_t m = (size_t)std::min<uint64_t>(left, kBounceBytes);
            err = cudaMemcpyAsync(bn->host, dev, m, cudaMemcpyDeviceToHost, bn->stream);
            if (err == cudaSuccess) err = cudaStreamSynchronize(bn->stream);
            if (err == cudaSuccess) memcpy(out + done, bn->host, m);
            done += m; dev += m; left -= m;
        }
    }
    if (ev) cudaEventDestroy(ev);
    bounce_put(e, bn);
    if (err != cudaSuccess) return fail_cuda(err, "follow_read D2H");
    e->st_d2h += done; e->st_served += done;
    if (nread) *nread = done;
    return DM_OK;
}

// Start the D2H of [start, start + <=4 MiB) of the blob into a read-ahead window.
static cudaError_t window_fill(dm_engine *e, Reader *r, Window &w, uint64_t start)
{
    const uint64_t n = std::min<uint64_t>(kBounceBytes, r->size - start);
    uint8_t *dst = w.b->host;
    cudaError_t err = cudaSuccess;
    for_segments(e, r->blob->extents, start, n, [&](uint8_t *dev, uint64_t l) {
        if (err == cudaSuccess) err = cudaMemcpyAsync(dst, dev, l, cudaMemcpyDeviceToHost, w.b->stream);
        dst += l;
    });
    if (err != cudaSuccess) {           // a retry must not find a partly filled window that looks valid
        cudaStreamSynchronize(w.b->stream);
        w.off = 0; w.len = 0; w.pending = false;
        return err;
    }
    w.off = start; w.len = n; w.pending = true;
    e->st_d2h += n;
    return err;
}

static int cache_read_impl(dm_engine *e, uint64_t reader, uint64_t off, void *buf, size_t len, size_t *nread)
{
    if (!e || (!buf && len)) return fail(DM_EINVAL, "null argument");
    std::shared_ptr<Reader> r = find_reader(e, reader);
    if (!r) return fail(DM_EINVAL, "unknown reader id");
    if (nread) *nread = 0;
    if (r->follow) {
        int rc = follow_read(e, r.get(), off, buf, len, nread);
        if (rc != 1) return rc;                 // 1: the body completed and was published: fall through to the blob
    }
    if (off > r->size) return fail(DM_ERANGE, "offset beyond blob end");
    len = (size_t)std::min<uint64_t>(len, r->size - off);
    if (len == 0) return DM_OK;
    uint8_t *out = static_cast<uint8_t *>(buf);
    if (!r->blob) {
        size_t got = 0;
        while (got < len) {
            ssize_t n = pread(r->fd, out + got, len - got, (off_t)(off + got));
            if (n < 0) { if (errno == EINTR) continue; return fail(DM_EIO, "pread failed"); }
            if (n == 0) break;
            got += (size_t)n;
        }
        if (nread) *nread = got;
        e->st_served += got;
        return DM_OK;
    }
    cudaSetDevice(e->device);
    std::lock_guard<std::mutex> g(r->mu);
    if (!r->tried_windows) {
        r->tried_windows = true;
        Bounce *a = bounce_try_get(e), *b = a ? bounce_try_get(e) : nullptr;
        if (a && b) { r->win[0].b = a; r->win[1].b = b; }
        else if (a) bounce_put(e, a);
    }
    size_t done = 0;
    int rc = DM_OK;
    if (r->win[0].b) {
        // HTTP bodies are read front to back in small pieces (io.Copy: 32 KiB): serve them from two
        // 4 MiB pinned windows, the next one filling by DMA while this one is copied out.
        while (done < len) {
            const uint64_t pos = off + done;
            Window *w = nullptr;
            for (Window &c : r->win) if (c.len && pos >= c.off && pos < c.off + c.len) w = &c;
            cudaError_t err = cudaSuccess;
            if (!w) {                                              // miss: restart the pipeline at pos
                for (Window &c : r->win) if (c.pending) { cudaStreamSynchronize(c.b->stream); c.pending = false; }
                err = window_fill(e, r.get(), r->win[0], pos);
                r->win[1].len = 0;
                if (err == cudaSuccess && pos + r->win[0].len < r->size)
                    err = window_fill(e, r.get(), r->win[1], pos + r->win[0].len);
                if (err != cudaSuccess) { rc = fail_cuda(err, "cudaMemcpyAsync(D2H)"); break; }
                w = &r->win[0];
            }
            if (w->pending) {
                err = cudaStreamSynchronize(w->b->stream);
                w->pending = false;
                if (err != cudaSuccess) { rc = fail_cuda(err, "cudaStreamSynchronize(D2H)"); break; }
            }
            const size_t n = (size_t)std::min<uint64_t>(len - done, w->off + w->len - pos);
            memcpy(out + done, w->b->host + (pos - w->off), n);
            done += n;
            if (pos + n == w->off + w->len) {                      // window drained: refill it behind the other one
                Window &other = (w == &r->win[0]) ? r->win[1] : r->win[0];
                const uint64_t next = other.len ? other.off + other.len : w->off + w->len;
                if (next < r->size && other.len && other.off == w->off + w->len) {
                    err = window_fill(e, r.get(), *w, next);
                    if (err != cudaSuccess) { rc = fail_cuda(err, "cudaMemcpyAsync(D2H)"); break; }
                } else w->len = 0;
            }
        }
    } else {
        Bounce *bn = bounce_get(e);                                // no windows left: one-shot staging
        while (done < len) {
            const size_t n = std::min(len - done, kBounceBytes);
            uint8_t *dst = bn->host;
            cudaError_t err = cudaSuccess;
            for_segments(e, r->blob->extents, off + done, n, [&](uint8_t *dev, uint64_t l) {
                if (err == cudaSuccess) err = cudaMemcpyAsync(dst, dev, l, cudaMemcpyDeviceToHost, bn->stream);
                dst += l;
            });
            if (err == cudaSuccess) err = cudaStreamSynchronize(bn->stream);
            if (err != cudaSuccess) { rc = fail_cuda(err, "cudaMemcpyAsync(D2H)"); break; }
            memcpy(out + done, bn->host, n);
            done += n;
            e->st_d2h += n;
        }
        bounce_put(e, bn);
    }
    e->st_served.fetch_add(done, std::memory_order_relaxed);
    if (nread) *nread = done;
    return rc;
}

static int cache_meta_impl(dm_engine *e, uint64_t reader, char *buf, size_t cap, size_t *len)
{
    if (!e || !len || (!buf && cap)) return fail(DM_EINVAL, "null argument");
    std::shared_ptr<Reader> r = find_reader(e, reader);
    if (!r) return fail(DM_EINVAL, "unknown reader id");
    std::string j;
    if (r->blob) {
        std::lock_guard<std::mutex> g(e->mu);
        j = sidecar_json(*r->blob);
    } else j = r->disk_meta;
    *len = j.size();
    if (cap) {
        const size_t n = std::min(cap - 1, j.size());
        memcpy(buf, j.data(), n);
        buf[n] = 0;
    }
    return DM_OK;
}

static int cache_close_impl(dm_engine *e, uint64_t reader)
{
    if (!e) return fail(DM_EINVAL, "null argument");
    std::shared_ptr<Reader> r;
    {
        std::lock_guard<std::mutex> g(e->reader_mu[reader % kStripes]);
        auto it = e->readers[reader % kStripes].find(reader);
        if (it == e->readers[reader % kStripes].end()) return fail(DM_EINVAL, "unknown reader id");
        r = it->second;
        e->readers[reader % kStripes].erase(it);
    }
    {
        std::lock_guard<std::mutex> g(r->mu);
        for (Window &w : r->win) {
            if (!w.b) continue;
            if (w.pending) cudaStreamSynchronize(w.b->stream);
            bounce_put(e, w.b);
            w.b = nullptr;
        }
    }
    if (r->blob) {
        std::lock_guard<std::mutex> g(e->mu);
        r->blob->readers--;
    }
    if (r->fd >= 0) close(r->fd);
    return DM_OK;
}

static int cache_follow_impl(dm_engine *e, const uint8_t digest[32], uint64_t *reader, uint64_t *size_hint)
{
    if (!e || !digest || !reader) return fail(DM_EINVAL, "null argument");
    Digest d;
    memcpy(d.b, digest, 32);
    auto r = std::make_shared<Reader>();
    uint64_t id;
    {
        std::lock_guard<std::mutex> g(e->mu);
        auto it = e->inflight.find(d);
        if (it == e->inflight.end()) return DM_ENOENT;
        r->follow = it->second.lock();
        if (!r->follow) { e->inflight.erase(it); return DM_ENOENT; }
        id = e->next_id.fetch_add(1);
    }
    r->size = r->follow->size_hint;
    {
        std::lock_guard<std::mutex> g(e->reader_mu[id % kStripes]);
        e->readers[id % kStripes][id] = r;
    }
    *reader = id;
    if (size_hint) *size_hint = r->size;
    return DM_OK;
}

static int cache_evict_impl(dm_engine *e, const uint8_t digest[32])
{
    if (!e || !digest) return fail(DM_EINVAL, "null argument");
    Digest d;
    memcpy(d.b, digest, 32);
    std::shared_ptr<Blob> b;
    std::vector<Extent> ext;
    {
        std::lock_guard<std::mutex> g(e->mu);
        auto it = e->blobs.find(d);
        if (it == e->blobs.end() || !it->second->in_hbm) return DM_ENOENT;
        if (it->second->readers) return fail(DM_ESTATE, "blob has open readers");
        b = it->second;
        b->in_hbm = false;
        lru_drop(e, b.get());
        ext.swap(b->extents);                       // under the lock (see evict_for)
        if (!b->on_disk) e->blobs.erase(it);
    }
    free_extents(e, ext);
    return DM_OK;
}

static int cache_device_extents_impl(dm_engine *e, uint64_t reader, void **dev_ptrs, uint64_t *lens, uint32_t max_ext)
{
    if (!e) return fail(DM_EINVAL, "null argument");
    std::shared_ptr<Reader> r = find_reader(e, reader);
    if (!r) return fail(DM_EINVAL, "unknown reader id");
    if (!r->blob) return fail(DM_ESTATE, "blob is on the disk tier only");
    const auto &ext = r->blob->extents;
    uint64_t left = r->blob->size;
    for (uint32_t i = 0; i < ext.size() && i < max_ext; ++i) {
        if (dev_ptrs) dev_ptrs[i] = e->arena_base + ext[i].off;
        if (lens) lens[i] = std::min(left, ext[i].len);
        left -= std::min(left, ext[i].len);
    }
    return (int)ext.size();
}

// ---- URL -> digest aliases -----------------------------------------------------------
// The OnRequest hook (start.go:197-200) sees a URL.  OCI URLs name the digest; HuggingFace resolve/ URLs do
// not, so a hit needs URL (or ETag) -> digest.  In memory: one hash map.  On the disk tier: an append-only
// text log, one "<64 hex>\t<key>\n" per put, replayed at start (later lines win) and compacted when more
// than half of it is dead.

}  // extern "C"

namespace dmi {

bool digest_from_hex(const char *hex, uint8_t out[32])
{
    auto nib = [](char c) { return c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : c >= 'A' && c <= 'F' ? c - 'A' + 10 : -1; };
    for (int i = 0; i < 32; ++i) {
        const int h = nib(hex[2 * i]);
        if (h < 0) return false;
        const int l = nib(hex[2 * i + 1]);
        if (l < 0) return false;
        out[i] = (uint8_t)(h << 4 | l);
    }
    return true;
}

static bool alias_key_ok(const char *key)
{
    if (!key || !*key) return false;
    size_t n = 0;
    for (const unsigned char *p = (const unsigned char *)key; *p; ++p, ++n)
        if (*p < 0x20 || *p == 0x7f || n >= 4096) return false;      // one key per log line
    return true;
}

void alias_load(dm_engine *e)
{
    if (e->cas_dir.empty()) return;
    const std::string path = e->cas_dir + "/aliases.log";
    size_t lines = 0;
    if (FILE *f = fopen(path.c_str(), "r")) {
        std::string line;
        char buf[8192];
        while (fgets(buf, sizeof buf, f)) {
            line += buf;
            if (line.empty() || line.back() != '\n') continue;        // long line: keep reading
            line.pop_back();
            ++lines;
            Digest d;
            if (line.size() > 65 && line[64] == '\t' && digest_from_hex(line.c_str(), d.b) && alias_key_ok(line.c_str() + 65))
                e->aliases[line.substr(65)] = d;                       // a torn last line simply fails these checks
            line.clear();
        }
        fclose(f);
    }
    if (lines > 2 * e->aliases.size() + 1024) {                        // mostly superseded entries: rewrite
        const std::string tmp = path + ".tmp";
        if (FILE *f = fopen(tmp.c_str(), "w")) {
            for (auto &kv : e->aliases) fprintf(f, "%s\t%s\n", hex_of(kv.second.b, 32).c_str(), kv.first.c_str());
            const bool ok = fflush(f) == 0;
            fclose(f);
            if (!ok || rename(tmp.c_str(), path.c_str()) != 0) unlink(tmp.c_str());
        }
    }
    e->alias_log = fopen(path.c_str(), "a");
}

}  // namespace dmi

extern "C" {

int dm_cache_alias_put(dm_engine *e, const char *key, const uint8_t digest[32])
{
    if (!e || !digest) return fail(DM_EINVAL, "null argument");
    if (!alias_key_ok(key)) return note_err(e, 0, fail(DM_EINVAL, "alias key must be 1..4096 bytes without control characters"));
    Digest d;
    memcpy(d.b, digest, 32);
    std::lock_guard<std::mutex> g(e->alias_mu);
    auto it = e->aliases.find(key);
    if (it != e->aliases.end() && it->second == d) return DM_OK;      // already known: nothing to log
    e->aliases[key] = d;
    if (e->alias_log) {
        const bool ok = fprintf(e->alias_log, "%s\t%s\n", hex_of(d.b, 32).c_str(), key) > 0 && fflush(e->alias_log) == 0;
        if (!ok) return note_err(e, 0, fail(DM_EIO, "could not append to aliases.log (the alias is held in memory only)"));
    }
    return DM_OK;
}

int dm_cache_alias_get(dm_engine *e, const char *key, uint8_t digest_out[32])
{
    if (!e || !key || !digest_out) return fail(DM_EINVAL, "null argument");
    std::lock_guard<std::mutex> g(e->alias_mu);
    auto it = e->aliases.find(key);
    if (it == e->aliases.end()) return DM_ENOENT;
    memcpy(digest_out, it->second.b, 32);
    return DM_OK;
}

// ---- device-resident ingest -------------------------------------------------------

namespace {

// One dm_ingest_device call.  Jobs are addressed by POSITION p in launch order (longest first when the kernel shape
// wants that); caller_index(p) is the blob the caller knows.  HashJob::slot = p, so a chunk's digests are contiguous.
struct IngestBatch {
    dm_engine *e;
    const uint8_t *base;
    const uint64_t *offsets, *lengths;
    const uint8_t *expect;
    uint8_t *digests_out, *matched_out;
    bool hash_only, replace;
    const uint32_t *order = nullptr;         // position -> caller index; nullptr = identity
    std::vector<Extent> ext;                 // by position: where the blob's CAS copy goes
    std::vector<std::shared_ptr<Blob>> parked;   // by position: the cached copy whose extent is being rewritten (REPLACE)
    uint32_t published = 0;                  // positions from here on may hold an extent or a parked blob nothing else knows about
    uint32_t caller_index(uint32_t p) const { return order ? order[p] : p; }
};

// Before the launch of positions [lo, hi): extents and the job table.
int ingest_prepare(IngestBatch &B, uint32_t lo, uint32_t hi)
{
    dm_engine *e = B.e;
    if (!B.hash_only) {
        std::vector<Extent> freed;
        if (B.replace && B.expect) {
            // The previous copy of a blob we are about to re-ingest goes out of sight, and - when its one extent has
            // the right size - that extent is simply written again: no arena traffic, no new index entry, and the
            // blob comes back by pointer (unpark_many).  Anything else is evicted the ordinary way.
            std::lock_guard<std::mutex> g(e->mu);
            auto digest_at = [&](uint32_t p) { Digest d; memcpy(d.b, B.expect + 32ull * B.caller_index(p), 32); return d; };
            constexpr uint32_t kAhead = 16;                          // the index slot of a digest is known from the digest alone
            for (uint32_t p = lo; p < hi; ++p) {
                if (p + kAhead < hi) e->blobs.prefetch(digest_at(p + kAhead));
                const uint32_t i = B.caller_index(p);
                const Digest d = digest_at(p);
                auto it = e->blobs.find(d);
                if (it == e->blobs.end() || !it->second->in_hbm || it->second->readers) continue;
                Blob *b = it->second.get();
                const uint64_t want = round_up(std::max<uint64_t>(B.lengths[i], 1), kAlign);
                const bool disk_safe = e->cas_dir.empty() || (b->on_disk && b->spill_done);
                b->in_hbm = false;
                lru_drop(e, b);
                if (disk_safe && b->extents.size() == 1 && b->extents[0].len == want) {
                    B.ext[p] = b->extents[0];
                    b->extents.clear();
                    B.parked[p] = it->second;
                } else {
                    freed.insert(freed.end(), b->extents.begin(), b->extents.end());
                    b->extents.clear();                              // under the lock (see evict_for)
                    if (!b->on_disk) e->blobs.erase(it);
                }
            }
        }
        uint32_t p = lo;
        {                                                            // all extents of the chunk under one arena lock
            std::lock_guard<std::mutex> g(e->arena_mu);
            for (const Extent &x : freed) e->arena.release(x.off, x.len);
            for (; p < hi; ++p) {
                if (B.parked[p]) continue;
                const uint64_t want = round_up(std::max<uint64_t>(B.lengths[B.caller_index(p)], 1), kAlign);
                uint64_t off;
                if (!e->arena.alloc(want, &off)) break;
                B.ext[p] = Extent{off, want};
            }
        }
        for (; p < hi; ++p) {                                        // arena full: evict LRU blobs one allocation at a time
            if (!B.parked[p]) {
                Extent x;
                if (!arena_alloc(e, B.lengths[B.caller_index(p)], &x)) return fail(DM_ENOMEM, "HBM CAS arena exhausted");
                B.ext[p] = x;
            }
        }
    }
    for (uint32_t p = lo; p < hi; ++p) {
        const uint32_t i = B.caller_index(p);
        dm::HashJob &jb = e->ing_jobs_h[p];
        jb.src = B.base + B.offsets[i]; jb.dst = B.hash_only ? nullptr : e->arena_base + B.ext[p].off;
        jb.nbytes = B.lengths[i]; jb.total_len = B.lengths[i];
        jb.slot = p; jb.flags = dm::JOB_INIT | dm::JOB_FINAL; jb.one = 1; jb.pad_ = 0;
    }
    return DM_OK;
}

// After the digests of positions [lo, hi) are back: verdicts out, verified copies published, the others released.
void ingest_publish(IngestBatch &B, uint32_t lo, uint32_t hi)
{
    dm_engine *e = B.e;
    std::vector<Verified> good;
    std::vector<Parked> back, gone;
    std::vector<Extent> bad;
    if (!B.hash_only) { good.reserve(hi - lo); if (B.replace) back.reserve(hi - lo); }
    for (uint32_t p = lo; p < hi; ++p) {
        const uint32_t i = B.caller_index(p);
        Digest d;
        words_to_digest(e->ing_digests_h + 8ull * p, d.b);
        if (B.digests_out) memcpy(B.digests_out + 32ull * i, d.b, 32);
        const int ok = (!B.expect || memcmp(B.expect + 32ull * i, d.b, 32) == 0) ? 1 : 0;
        if (B.matched_out) B.matched_out[i] = (uint8_t)ok;
        if (B.hash_only) continue;
        if (!ok) e->st_mismatch++;
        if (B.parked[p]) (ok ? back : gone).push_back(Parked{std::move(B.parked[p]), B.ext[p]});   // parked under expect[i]: ok means it IS that blob
        else if (ok) good.push_back(Verified{d, B.lengths[i], B.ext[p]});
        else bad.push_back(B.ext[p]);
    }
    B.published = hi;
    if (!good.empty()) publish_many(e, good);
    if (!back.empty() || !gone.empty()) unpark_many(e, back, gone);
    if (!bad.empty()) free_extents(e, bad);
}

// A failed call: whatever was prepared and not yet published goes back (the caller has synchronised the streams).
void ingest_unwind(IngestBatch &B)
{
    if (B.hash_only) return;
    std::vector<Parked> none, gone;
    std::vector<Extent> ext;
    for (uint32_t p = B.published; p < B.ext.size(); ++p) {
        if (B.parked[p]) gone.push_back(Parked{std::move(B.parked[p]), B.ext[p]});
        else if (B.ext[p].len) ext.push_back(B.ext[p]);              // allocated extents are never empty
        B.ext[p] = Extent{0, 0};
    }
    if (!gone.empty()) unpark_many(B.e, none, gone);
    if (!ext.empty()) free_extents(B.e, ext);
}

}  // namespace

static int ingest_device_impl(dm_engine *e, const void *dev_base, const uint64_t *offsets, const uint64_t *lengths,
                              uint32_t n, const uint8_t *expect, uint8_t *digests_out, uint8_t *matched_out,
                              uint32_t flags, double *kernel_ms)
{
    if (!e || ((!offsets || !lengths || !dev_base) && n)) return fail(DM_EINVAL, "null argument");
    if (kernel_ms) *kernel_ms = 0.0;
    if (n == 0) return DM_OK;
    if (((uintptr_t)dev_base) & 15) return fail(DM_EINVAL, "dev_base must be 16-byte aligned");
    uint64_t total = 0;
    bool sorted = true;                                  // equal-sized batches (the common bulk case) need no reordering
    for (uint32_t i = 0; i < n; ++i) {
        if (offsets[i] & 15) return fail(DM_EINVAL, "offsets must be multiples of 16");
        total += lengths[i];
        if (i && lengths[i - 1] < lengths[i]) sorted = false;
    }
    cudaSetDevice(e->device);
    std::lock_guard<std::mutex> gi(e->ingest_mu);
    int rc = ensure_ingest_scratch(e, n);
    if (rc != DM_OK) return rc;
    IngestBatch B;
    B.e = e; B.base = static_cast<const uint8_t *>(dev_base); B.offsets = offsets; B.lengths = lengths; B.expect = expect;
    B.digests_out = digests_out; B.matched_out = matched_out;
    B.hash_only = (flags & DM_ING_HASH_ONLY) != 0; B.replace = (flags & DM_ING_REPLACE) != 0;
    if (!B.hash_only) {
        B.ext.assign(n, Extent{0, 0});
        B.parked.resize(n);
    }
    int spw = e->force_spw ? e->force_spw : dm::streams_per_warp_for(n);
    if (flags & DM_ING_FORCE_WIDE) spw = 32;
    if (flags & DM_ING_FORCE_DEEP) spw = 1;
    if (flags & DM_ING_SPW_MASK) spw = 1 << (((flags & DM_ING_SPW_MASK) >> DM_ING_SPW_SHIFT) - 1);
    std::vector<uint32_t> order;
    if (spw > 1 && !sorted) {                            // lanes of a warp should end together: longest first
        order.resize(n);
        for (uint32_t i = 0; i < n; ++i) order[i] = i;
        std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return lengths[a] > lengths[b]; });
        B.order = order.data();
    }
    // A batch whose sizes are badly skewed (a few multi-GiB layers among thousands of small files) is two batches: the
    // launch lasts as long as its longest chain, and a chain runs fastest with a warp of its own, so the long jobs
    // (within 4x of the longest, at most one per sub-partition) get a warp-per-stream launch on a second CUDA
    // stream while the rest go through the kernel their own count calls for.  (The stream path does this by itself:
    // short bodies finish early and the pump sizes each later launch by who is left.)
    uint32_t n_long = 0;
    const bool forced = e->force_spw || (flags & (DM_ING_FORCE_WIDE | DM_ING_FORCE_DEEP | DM_ING_SPW_MASK));
    if (spw > 1 && !forced && n > 1) {
        const uint64_t longest = lengths[B.caller_index(0)];        // positions are longest first here
        while (n_long < n && n_long < dm::kSubPartitions && lengths[B.caller_index(n_long)] * 4 >= longest) ++n_long;
        // not skewed (everything is "long", or more long jobs than sub-partitions), or nothing long enough to matter
        if (n_long == n || longest < e->split_min || lengths[B.caller_index(n_long)] * 4 >= longest) n_long = 0;
    }
    const uint32_t n_rest = n - n_long;
    // the two launches of a split batch share the chip: the rest runs one warp per group (the long jobs keep their
    // warp pairs while there are at most kMaxWarpPairs of them)
    const int spw_rest = n_long ? dm::streams_per_warp_unpaired(n_rest) : spw;
    const dm::KernelShape rest_shape = dm::kernel_shape(spw_rest, n_long ? 0 : n, e->variant_wide, e->variant_deep);
    // Very large lane-per-stream batches go out in chunks, each on a stream of its own: at 10^5 blobs the host work
    // around the launch (extents, index) is of the order of the kernel itself, and this way all but the first
    // chunk's preparation and the last chunk's publication happens while kernels run.  The launches overlap on the
    // device (together they are the same CTAs), so the GPU side costs nothing.
    uint32_t nchunks = 1;
    if (!n_long && spw_rest == 32) {
        // (a forced kernel shape is a measurement of that kernel: one launch, unless DM_INGEST_CHUNKS says otherwise)
        nchunks = e->ingest_chunks ? std::min<uint32_t>(e->ingest_chunks, n) : forced ? 1 : std::min<uint32_t>(kIngestMaxChunks, n / kIngestChunkMin);
        nchunks = std::max<uint32_t>(1, nchunks);
    }
    cudaStream_t st = e->ingest_stream, st2 = e->util_stream;
    (void)cudaGetLastError();           // the caller's thread may carry a stale "not ready" from its own event polling
    cudaError_t err = cudaSuccess;
    float ms = 0.f;
    if (nchunks > 1) {
        uint32_t per = (n + nchunks - 1) / nchunks;
        if (per >= 64) per = (per + 31) / 32 * 32;                                // whole warps per chunk
        uint32_t lo_of[kIngestMaxChunks + 1];
        for (uint32_t c = 0; c <= nchunks; ++c) lo_of[c] = std::min<uint64_t>(n, (uint64_t)c * per);
        uint32_t launched = 0, reaped = 0;
        auto reap = [&]() {                                 // digests of the oldest chunk in flight
            err = cudaEventSynchronize(e->ing_cev_done[reaped]);
            if (err != cudaSuccess) return;
            ingest_publish(B, lo_of[reaped], lo_of[reaped + 1]);
            ++reaped;
        };
        while (launched < nchunks && lo_of[launched] < n) {
            const uint32_t c = launched, lo = lo_of[c], hi = lo_of[c + 1];
            rc = ingest_prepare(B, lo, hi);
            if (rc != DM_OK) break;
            cudaStream_t cs = e->ing_streams[c];
            err = cudaMemcpyAsync(e->ing_jobs_d + lo, e->ing_jobs_h + lo, sizeof(dm::HashJob) * (uint64_t)(hi - lo), cudaMemcpyHostToDevice, cs);
            if (err == cudaSuccess && c == 0) err = cudaEventRecord(e->ing_ev0, cs);
            if (err == cudaSuccess) err = dm::launch_sha256(e->ing_jobs_d + lo, hi - lo, e->ing_states, e->ing_digests, cs, rest_shape);
            if (err == cudaSuccess) err = cudaEventRecord(e->ing_cev_k[c], cs);
            if (err == cudaSuccess) err = cudaMemcpyAsync(e->ing_digests_h + 8ull * lo, e->ing_digests + 8ull * lo, 32ull * (hi - lo), cudaMemcpyDeviceToHost, cs);
            if (err == cudaSuccess) err = cudaEventRecord(e->ing_cev_done[c], cs);
            ++launched;                                     // whatever did get enqueued is waited for, also on failure
            while (reaped < launched && err == cudaSuccess) {           // publish what has finished meanwhile, without waiting
                const cudaError_t q = cudaEventQuery(e->ing_cev_done[reaped]);
                if (q == cudaErrorNotReady) { (void)cudaGetLastError(); break; }     // not an error, but it sticks to the thread
                if (q != cudaSuccess) { err = q; break; }
                reap();
            }
            if (err != cudaSuccess) break;
        }
        while (err == cudaSuccess && reaped < launched) reap();     // also when a later chunk found no room: these are done
        if (rc != DM_OK || err != cudaSuccess) {
            for (uint32_t c = 0; c < launched; ++c) cudaStreamSynchronize(e->ing_streams[c]);
            ingest_unwind(B);
            return rc != DM_OK ? rc : fail_cuda(err, "dm_ingest_device launch");
        }
        for (uint32_t c = 0; c < launched; ++c) {           // the pass lasted from the first launch to the last one's end
            float t = 0.f;
            cudaEventElapsedTime(&t, e->ing_ev0, e->ing_cev_k[c]);
            ms = std::max(ms, t);
        }
        e->st_launches += launched; e->st_wide += launched;
    } else {
        rc = ingest_prepare(B, 0, n);
        if (rc != DM_OK) { ingest_unwind(B); return rc; }
        err = cudaMemcpyAsync(e->ing_jobs_d, e->ing_jobs_h, sizeof(dm::HashJob) * (uint64_t)n, cudaMemcpyHostToDevice, st);
        if (err == cudaSuccess) err = cudaEventRecord(e->ing_ev0, st);
        if (err == cudaSuccess && n_long) {
            err = cudaStreamWaitEvent(st2, e->ing_ev0, 0);              // the job table is in place
            if (err == cudaSuccess)
                err = dm::launch_sha256(e->ing_jobs_d, n_long, e->ing_states, e->ing_digests, st2,
                                        dm::kernel_shape(1, n_long, e->variant_wide, e->variant_deep));
            if (err == cudaSuccess) err = cudaEventRecord(e->ing_ev2, st2);
        }
        if (err == cudaSuccess) err = dm::launch_sha256(e->ing_jobs_d + n_long, n_rest, e->ing_states, e->ing_digests, st, rest_shape);
        if (err == cudaSuccess) err = cudaEventRecord(e->ing_ev1, st);
        if (err == cudaSuccess && n_long) err = cudaStreamWaitEvent(st, e->ing_ev2, 0);       // digests of both launches
        if (err == cudaSuccess) err = cudaMemcpyAsync(e->ing_digests_h, e->ing_digests, 32ull * n, cudaMemcpyDeviceToHost, st);
        if (err == cudaSuccess) err = cudaStreamSynchronize(st);
        if (err != cudaSuccess) {
            cudaStreamSynchronize(st);      // whatever was enqueued before the failure still uses the job table and the extents
            cudaStreamSynchronize(st2);
            ingest_unwind(B);
            return fail_cuda(err, "dm_ingest_device launch");
        }
        cudaEventElapsedTime(&ms, e->ing_ev0, e->ing_ev1);
        if (n_long) {                       // two overlapping launches: the pass lasted until the later one ended
            float ms2 = 0.f;
            cudaEventElapsedTime(&ms2, e->ing_ev0, e->ing_ev2);
            ms = std::max(ms, ms2);
            e->st_launches++; e->st_deep++;
        }
        e->st_launches++; (spw_rest == 1 ? e->st_deep : spw_rest == 32 ? e->st_wide : e->st_group)++;
        ingest_publish(B, 0, n);
    }
    if (kernel_ms) *kernel_ms = ms;
    { std::lock_guard<std::mutex> g(e->stat_mu); e->st_kernel_ms += ms; }
    e->st_hashed += total;
    return DM_OK;
}

// ---- synthetic bytes ---------------------------------------------------------------

void dm_synth_fill_host(uint64_t seed, uint64_t blob, uint64_t byte_off, void *dst, size_t len)
{
    const uint64_t key = dm_blob_key(seed, blob);
    uint8_t *p = static_cast<uint8_t *>(dst);
    uint64_t j = byte_off;
    while (len && (j & 7)) { *p++ = (uint8_t)(dm_blob_word_k(key, j >> 3) >> (8 * (j & 7))); ++j; --len; }
    while (len >= 8) { const uint64_t w = dm_blob_word_k(key, j >> 3); memcpy(p, &w, 8); p += 8; j += 8; len -= 8; }
    while (len) { *p++ = (uint8_t)(dm_blob_word_k(key, j >> 3) >> (8 * (j & 7))); ++j; --len; }
}

int dm_synth_fill_device(dm_engine *e, uint64_t seed, uint64_t blob, uint64_t byte_off, void *dev_dst, size_t len)
{
    if (!e || (!dev_dst && len)) return fail(DM_EINVAL, "null argument");
    cudaSetDevice(e->device);
    CU_TRY(dm::launch_synth_fill(seed, blob, byte_off, dev_dst, len, e->util_stream));
    CU_TRY(cudaStreamSynchronize(e->util_stream));
    return DM_OK;
}

int dm_synth_fill_device_many(dm_engine *e, uint64_t seed, uint64_t first_blob, void *dev_base,
                              const uint64_t *offsets, const uint64_t *lengths, uint32_t n)
{
    if (!e || ((!offsets || !lengths || !dev_base) && n)) return fail(DM_EINVAL, "null argument");
    if (n == 0) return DM_OK;
    for (uint32_t i = 0; i < n; ++i) {
        if (offsets[i] & 15) return fail(DM_EINVAL, "offsets must be multiples of 16");
        if (i && offsets[i] < offsets[i - 1] + lengths[i - 1]) return fail(DM_EINVAL, "blobs must be ascending and disjoint");
    }
    cudaSetDevice(e->device);
    uint64_t *d_tab = nullptr;
    CU_TRY(cudaMalloc(&d_tab, 16ull * n));
    cudaError_t err = cudaMemcpyAsync(d_tab, offsets, 8ull * n, cudaMemcpyHostToDevice, e->util_stream);
    if (err == cudaSuccess) err = cudaMemcpyAsync(d_tab + n, lengths, 8ull * n, cudaMemcpyHostToDevice, e->util_stream);
    if (err == cudaSuccess)
        err = dm::launch_synth_fill_many(seed, first_blob, dev_base, d_tab, d_tab + n, n, offsets[0],
                                         offsets[n - 1] + lengths[n - 1] - offsets[0], e->util_stream);
    const cudaError_t sync = cudaStreamSynchronize(e->util_stream);     // also on failure: the table may still be in use
    if (err == cudaSuccess) err = sync;
    cudaFree(d_tab);
    if (err != cudaSuccess) return fail_cuda(err, "dm_synth_fill_device_many");
    return DM_OK;
}

// ---- exported wrappers: file the error text under the reader id (dm_error_detail) ----
int dm_cache_open(dm_engine *e, const uint8_t digest[32], uint64_t *reader, uint64_t *size) { return note_err(e, 0, cache_open_impl(e, digest, reader, size)); }
int dm_cache_read(dm_engine *e, uint64_t reader, uint64_t off, void *buf, size_t len, size_t *nread) { return note_err(e, reader, cache_read_impl(e, reader, off, buf, len, nread)); }
int dm_cache_meta(dm_engine *e, uint64_t reader, char *buf, size_t cap, size_t *len) { return note_err(e, reader, cache_meta_impl(e, reader, buf, cap, len)); }
int dm_cache_close(dm_engine *e, uint64_t reader) { return note_err(e, reader, cache_close_impl(e, reader)); }
int dm_cache_follow(dm_engine *e, const uint8_t digest[32], uint64_t *reader, uint64_t *size_hint) { return note_err(e, 0, cache_follow_impl(e, digest, reader, size_hint)); }
int dm_cache_evict(dm_engine *e, const uint8_t digest[32]) { return note_err(e, 0, cache_evict_impl(e, digest)); }
int dm_cache_device_extents(dm_engine *e, uint64_t reader, void **dev_ptrs, uint64_t *lens, uint32_t max_ext) { return note_err(e, reader, cache_device_extents_impl(e, reader, dev_ptrs, lens, max_ext)); }
int dm_ingest_device(dm_engine *e, const void *dev_base, const uint64_t *offsets, const uint64_t *lengths,
                     uint32_t n, const uint8_t *expect, uint8_t *digests_out, uint8_t *matched_out,
                     uint32_t flags, double *kernel_ms)
{
    return note_err(e, 0, ingest_device_impl(e, dev_base, offsets, lengths, n, expect, digests_out, matched_out, flags, kernel_ms));
}

}  // extern "C"
