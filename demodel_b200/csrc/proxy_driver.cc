// dm_proxy_drive / dm_proxy_serve: the per-connection work of the proxy,
// restated as C++ threads over the hook wrappers in proxy_hooks.hpp.
//
// In the reference, net/http runs one goroutine per client connection
// (demodel/cmd/demodel/start.go:210-215) and goproxy reads the
// response body on that goroutine in 32 KiB pieces.  Here `nthreads` OS
// threads play `concurrency` such goroutines the way the Go scheduler runs
// them on GOMAXPROCS threads: each thread round-robins one piece at a time
// over its share of live connections (a BodyTee over an "upstream body" that
// is a region of caller-owned host memory), starts the final hash at EOF
// without blocking (dm_stream_flush) and collects verdicts afterwards.
#include "proxy_hooks.hpp"

#include <algorithm>
#include <atomic>
#include <memory>
#include <chrono>
#include <thread>
#include <vector>

namespace {

struct MemUpstream : dm::Upstream {
    const uint8_t *p;
    uint64_t left;
    MemUpstream(const uint8_t *base, uint64_t n) : p(base), left(n) {}
    long Read(void *dst, size_t n) override
    {
        if (n > left) n = (size_t)left;
        if (n) memcpy(dst, p, n);
        p += n; left -= n;
        return (long)n;
    }
};

double now_s()
{
    return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

}  // namespace

extern "C" int dm_proxy_drive(dm_engine *e, const void *host_base, const uint64_t *offsets, uint32_t n,
                              const uint8_t *expect, size_t chunk, uint32_t concurrency, int nthreads,
                              int zero_copy, uint8_t *digests_out, uint8_t *matched_out, double *seconds)
{
    if (!e || !offsets || (!host_base && n)) return DM_EINVAL;
    if (chunk == 0) chunk = 32768;                    // io.Copy's buffer
    if (concurrency == 0) concurrency = 1;
    if (concurrency > n) concurrency = n ? n : 1;
    // `nthreads` OS threads play `concurrency` goroutines, like GOMAXPROCS; 0 = one thread per connection
    uint32_t workers = nthreads > 0 ? (uint32_t)nthreads : concurrency;
    if (workers > concurrency) workers = concurrency;
    std::atomic<uint32_t> next{0};
    std::atomic<int> first_err{DM_OK};
    const uint8_t *base = static_cast<const uint8_t *>(host_base);

    struct Conn {
        uint32_t blob;
        MemUpstream up;
        dm::BodyTee tee;
        Conn(dm_engine *e, uint32_t i, const uint8_t *p, uint64_t len, const uint8_t *exp)
            : blob(i), up(p, len), tee(e, &up, exp, len) {}
    };

    auto worker = [&](uint32_t share) {
        std::vector<uint8_t> buf(chunk);                       // goproxy's copy buffer
        std::vector<std::unique_ptr<Conn>> live, draining;
        auto note_err = [&](int rc) { int exp = DM_OK; first_err.compare_exchange_strong(exp, rc); };
        auto open_next = [&]() -> bool {
            const uint32_t i = next.fetch_add(1);
            if (i >= n) return false;
            live.emplace_back(new Conn(e, i, base + offsets[i], offsets[i + 1] - offsets[i],
                                       expect ? expect + 32ull * i : nullptr));
            return true;
        };
        auto collect = [&](Conn &c) {
            if (c.tee.Wait() != DM_OK) { note_err(c.tee.status()); return; }
            if (digests_out) memcpy(digests_out + 32ull * c.blob, c.tee.digest(), 32);
            if (matched_out) matched_out[c.blob] = c.tee.matched() ? 1 : 0;
        };
        bool more = true;
        while (more && live.size() < share) more = open_next();
        while (!live.empty()) {
            if (zero_copy >= 2) {
                // io.ReadCloser exactly as goproxy drives it: this thread IS the goroutine of one
                // connection and blocks in Read() at EOF (modes 2/3), or the client goes away half
                // way and Close() aborts the stream (mode 4).
                Conn &c = *live.back();
                const uint64_t len = offsets[c.blob + 1] - offsets[c.blob];
                uint64_t seen = 0;
                long got = 1;
                const void *view = nullptr;
                while (got > 0) {
                    if (zero_copy == 4 && seen >= len / 2) { c.tee.Close(); break; }
                    got = zero_copy == 3 ? c.tee.ReadInPlace(&view, chunk) : c.tee.Read(buf.data(), chunk);
                    if (got > 0) seen += (uint64_t)got;
                }
                if (got < 0) note_err((int)got);
                else if (zero_copy == 4) { if (matched_out) matched_out[c.blob] = 2; }      // 2 = aborted by the client
                else {
                    if (digests_out) memcpy(digests_out + 32ull * c.blob, c.tee.digest(), 32);
                    if (matched_out) matched_out[c.blob] = c.tee.matched() ? 1 : 0;
                }
                live.pop_back();
                if (more) more = open_next();
                continue;
            }
            for (size_t k = 0; k < live.size();) {             // one piece per connection per turn
                Conn &c = *live[k];
                const long got = c.tee.Pump(buf.data(), chunk, zero_copy == 1);
                if (got > 0) { ++k; continue; }
                if (got < 0) note_err((int)got); else draining.push_back(std::move(live[k]));
                live[k] = std::move(live.back());
                live.pop_back();
                if (more) more = open_next();
            }
            if (draining.size() >= 4 * (size_t)share) {        // bound the slots held by finished bodies
                for (auto &c : draining) collect(*c);
                draining.clear();
            }
        }
        for (auto &c : draining) collect(*c);
    };

    const double t0 = now_s();
    std::vector<std::thread> th;
    th.reserve(workers);
    for (uint32_t t = 0; t < workers; ++t) {
        const uint32_t share = concurrency / workers + (t < concurrency % workers ? 1 : 0);
        th.emplace_back(worker, share ? share : 1);
    }
    for (auto &t : th) t.join();
    if (seconds) *seconds = now_s() - t0;
    return first_err.load();
}

extern "C" int dm_proxy_serve(dm_engine *e, const uint8_t *digests, uint32_t n, void *host_base,
                              const uint64_t *offsets, size_t chunk, int nthreads, double *seconds)
{
    if (!e || !digests || !offsets || (!host_base && n)) return DM_EINVAL;
    if (chunk == 0) chunk = 32768;
    uint32_t workers = nthreads > 0 ? (uint32_t)nthreads : 1;
    if (workers > n) workers = n ? n : 1;
    std::atomic<uint32_t> next{0};
    std::atomic<int> first_err{DM_OK};
    uint8_t *base = static_cast<uint8_t *>(host_base);

    auto worker = [&]() {
        for (;;) {
            const uint32_t i = next.fetch_add(1);
            if (i >= n) break;
            dm::HitReader hr(e, digests + 32ull * i);
            int exp = DM_OK;
            if (!hr.hit()) { first_err.compare_exchange_strong(exp, DM_ENOENT); continue; }
            const uint64_t want = offsets[i + 1] - offsets[i];
            if (hr.size() != want) { first_err.compare_exchange_strong(exp, DM_ERANGE); continue; }
            uint8_t *dst = base + offsets[i];
            uint64_t off = 0;
            long got;
            while (off < want && (got = hr.Read(dst + off, (size_t)std::min<uint64_t>(chunk, want - off))) > 0)
                off += (uint64_t)got;
            if (off != want) first_err.compare_exchange_strong(exp, DM_EIO);
        }
    };

    const double t0 = now_s();
    std::vector<std::thread> th;
    th.reserve(workers);
    for (uint32_t t = 0; t < workers; ++t) th.emplace_back(worker);
    for (auto &t : th) t.join();
    if (seconds) *seconds = now_s() - t0;
    return first_err.load();
}

// ---- single-connection twins of the two hooks, for callers (tests) that work with URLs ----------------

// OnResponse for one body fetched under `url`: tee it into the engine in `chunk`-byte reads.  expect may be
// NULL (HuggingFace resolve/ URL: digest unknown until hashed); a verified body is entered in the alias
// index under the URL.
extern "C" int dm_proxy_fetch(dm_engine *e, const char *url, const void *body, uint64_t len, const uint8_t *expect,
                              size_t chunk, uint8_t digest_out[32], int *matched_out)
{
    if (!e || (!body && len)) return DM_EINVAL;
    if (chunk == 0) chunk = 32768;
    MemUpstream up(static_cast<const uint8_t *>(body), len);
    dm::BodyTee tee(e, &up, expect, len);
    if (tee.status() != DM_OK) return tee.status();
    tee.SetURL(url);
    std::vector<uint8_t> buf(chunk);
    long got;
    while ((got = tee.Read(buf.data(), chunk)) > 0) {}
    if (got < 0) return (int)got;
    if (digest_out) memcpy(digest_out, tee.digest(), 32);
    if (matched_out) *matched_out = tee.matched() ? 1 : 0;
    return tee.status();
}

// OnRequest: does this URL name something in the cache?  DM_ENOENT = miss (go upstream); DM_OK = *reader is
// an open cache reader (dm_cache_read / dm_cache_close) over *size bytes.
extern "C" int dm_proxy_request(dm_engine *e, const char *url, uint64_t *reader, uint64_t *size)
{
    if (!e || !url || !reader) return DM_EINVAL;
    dm::HitReader hr(e, url);
    if (!hr.hit()) return DM_ENOENT;
    if (size) *size = hr.size();
    *reader = hr.Release();
    return DM_OK;
}

// OnResponse for a manifest body (possibly Content-Encoding: gzip): pass it through in `chunk` reads, then
// parse and prefetch.  layers_out / ids_out receive up to max_layers entries, *n_layers the count found.
extern "C" int dm_proxy_manifest(dm_engine *e, const void *body, uint64_t len, const char *content_encoding, size_t chunk,
                                 dm_layer *layers_out, uint64_t *ids_out, uint32_t max_layers, uint32_t *n_layers)
{
    if (!e || (!body && len) || !n_layers) return DM_EINVAL;
    if (chunk == 0) chunk = 32768;
    MemUpstream up(static_cast<const uint8_t *>(body), len);
    dm::ManifestTee tee(e, &up, content_encoding);
    std::vector<uint8_t> buf(chunk);
    uint64_t seen = 0;
    long got;
    while ((got = tee.Read(buf.data(), chunk)) > 0) seen += (uint64_t)got;      // goproxy's copy loop: bytes reach the client unchanged
    if (got < 0 || seen != len) return DM_EIO;
    *n_layers = (uint32_t)tee.layers().size();
    for (uint32_t i = 0; i < *n_layers && i < max_layers; ++i) {
        if (layers_out) layers_out[i] = tee.layers()[i];
        if (ids_out) ids_out[i] = tee.ids()[i];
    }
    return tee.status();
}
