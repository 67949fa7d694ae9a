// TEST INFRASTRUCTURE ONLY — soak of dm_cache_remove through the C-ABI, linked against the fake CUDA runtime
// (fake_cuda.cc) so it runs on a CPU-only box under ThreadSanitizer / AddressSanitizer.  Worker threads ingest blobs,
// read them (dm_cache_open, dm_cache_open_verified, dm_cache_follow onto a body being ingested), promote, verify,
// import, change the disk-tier limit and remove random digests with random flags while readers have them open.  Half
// way the engine is restarted over the same cas_dir.  Every byte a reader got is its blob's.  At rest: the limit index
// equals a walk of blobs/, incoming/ and partial/; hbm_cas_used equals the extents of the blobs still in HBM (no reader
// is open by then, so no removed blob holds one); no ring slab, stream slot or reader is leaked; and once every digest
// is removed with nothing publishing, every digest is a miss on both tiers.
//
// usage: remove_soak <seconds> <cas_dir>        (FAKE_CUDA_JITTER_US: device jitter)
#include "../../include/demodel_b200.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <filesystem>
#include <random>
#include <string>
#include <thread>
#include <vector>

extern "C" void dmo_sha256(const void *data, size_t len, uint8_t out[32]);

#define CHECK(c) do { if (!(c)) { fprintf(stderr, "FAILED %s:%d: %s (last error: %s)\n", __FILE__, __LINE__, #c, dm_last_error()); \
                                   failures.fetch_add(1); return; } } while (0)

namespace fs = std::filesystem;

static std::atomic<int> failures{0};
static std::atomic<long> reads{0}, removed{0}, refused{0}, imported{0}, followed{0};
static std::string g_cas;
static const uint64_t kArena = 4u << 20;
static const uint32_t kMaxStreams = 256;
static const int kThreads = 6;

struct Body { std::vector<uint8_t> bytes; uint8_t digest[32]; std::string src; };
static std::vector<Body> bodies;

static void make_bodies()
{
    const size_t sizes[] = {0, 1, 1000, 70000, 300001, 900000};
    for (int rep = 0; rep < 2; ++rep)
        for (size_t s : sizes) {
            Body b;
            b.bytes.resize(s);
            dm_synth_fill_host(0xDE1E7E, 700 + bodies.size(), 0, b.bytes.data(), s);
            dmo_sha256(b.bytes.data(), s, b.digest);
            b.src = g_cas + "-src/" + std::to_string(bodies.size());       // the file dm_cache_import reads
            FILE *f = fopen(b.src.c_str(), "wb");
            if (f) { if (s) fwrite(b.bytes.data(), 1, s, f); fclose(f); }
            bodies.push_back(std::move(b));
        }
}

static dm_engine *make_engine()
{
    dm_config cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.struct_size = sizeof cfg;
    cfg.hbm_cas_bytes = kArena;
    cfg.ring_bytes = 1u << 20;
    cfg.slab_bytes = 64u << 10;
    cfg.max_streams = kMaxStreams;
    cfg.cas_dir = g_cas.c_str();
    dm_engine *e = nullptr;
    if (dm_engine_create(&cfg, &e) != DM_OK) { fprintf(stderr, "create failed: %s\n", dm_last_error()); return nullptr; }
    return e;
}

static void ingest(dm_engine *e, const Body &b, std::mt19937_64 &rng)
{
    uint64_t id = 0;
    int rc = dm_stream_open(e, b.digest, b.bytes.size(), &id);
    if (rc != DM_OK) { CHECK(rc == DM_ENOMEM); return; }
    uint64_t fid = 0, hint = 0;                           // a follower coalesced onto this body, read after it completes
    const bool follow = rng() % 2 && dm_cache_follow(e, b.digest, &fid, &hint) == DM_OK;
    for (size_t off = 0; rc == DM_OK && off < b.bytes.size(); off += 100000)
        rc = dm_stream_write(e, id, b.bytes.data() + off, std::min<size_t>(100000, b.bytes.size() - off));
    uint8_t got[32];
    int matched = 0;
    if (rc == DM_OK) rc = dm_stream_finish(e, id, got, &matched);
    if (rc != DM_OK) { CHECK(rc == DM_ENOMEM); dm_stream_abort(e, id); }
    if (follow) {
        std::vector<uint8_t> buf(b.bytes.size() + 1);
        size_t pos = 0, n = 0;
        int r2;
        while ((r2 = dm_cache_read(e, fid, pos, buf.data() + pos, buf.size() - pos, &n)) == DM_OK && n) pos += n;
        // DM_ENOENT / DM_ESTATE: the published blob left HBM (eviction, removal) before the follower switched over
        CHECK(r2 == DM_OK || r2 == DM_ENOENT || r2 == DM_ESTATE);
        if (r2 == DM_OK) { CHECK(pos == b.bytes.size() && (pos == 0 || memcmp(buf.data(), b.bytes.data(), pos) == 0)); followed++; }
        CHECK(dm_cache_close(e, fid) == DM_OK);
    }
}

// Open (plain or verified), read part of the blob, maybe remove it half way, read the rest: every byte is the blob's.
static void reader(dm_engine *e, const Body &b, std::mt19937_64 &rng)
{
    uint64_t rid = 0, size = 0;
    const bool verified = rng() % 2;
    const int orc = verified ? dm_cache_open_verified(e, b.digest, &rid, &size) : dm_cache_open(e, b.digest, &rid, &size);
    if (orc != DM_OK) { CHECK(orc == DM_ENOENT || orc == DM_ENOMEM); return; }
    CHECK(size == b.bytes.size());
    std::vector<uint8_t> buf(size + 1);
    size_t pos = 0, n = 0;
    int rc = DM_OK;
    bool removed_mid = false;
    while (pos < size) {
        const size_t want = 1 + rng() % 90000;
        rc = dm_cache_read(e, rid, pos, buf.data() + pos, std::min(want, size - pos), &n);
        if (rc != DM_OK) break;
        CHECK(n > 0);
        pos += n;
        if (!removed_mid && rng() % 4 == 0) {
            int32_t st = 0;
            CHECK(dm_cache_remove(e, b.digest, 1, (uint32_t)(rng() % 4), &st) == DM_OK);
            CHECK(st == DM_OK || st == DM_ENOENT || st == DM_ESTATE);
            removed_mid = true;
        }
    }
    int eof = DM_OK;
    if (rc == DM_OK) eof = dm_cache_read(e, rid, size, buf.data(), 1, &n);
    CHECK(dm_cache_close(e, rid) == DM_OK);
    // a verified reader whose blob left HBM (evicted, removed) before it switched over: DM_ESTATE, at any read from the
    // last byte on; the bytes it got are still checked
    CHECK(rc == DM_OK || (verified && rc == DM_ESTATE));
    CHECK(pos == 0 || memcmp(buf.data(), b.bytes.data(), pos) == 0);
    if (rc == DM_OK) {
        CHECK((eof == DM_OK && n == 0) || (verified && eof == DM_ESTATE));
        reads++;
    }
}

static void remover(dm_engine *e, std::mt19937_64 &rng)
{
    uint8_t digs[4 * 32];
    int32_t st[4];
    const uint32_t n = 1 + rng() % 4;
    for (uint32_t i = 0; i < n; ++i) memcpy(digs + 32 * i, bodies[rng() % bodies.size()].digest, 32);
    CHECK(dm_cache_remove(e, digs, n, (uint32_t)(rng() % 4), st) == DM_OK);
    for (uint32_t i = 0; i < n; ++i) {
        CHECK(st[i] == DM_OK || st[i] == DM_ENOENT || st[i] == DM_ESTATE);
        if (st[i] == DM_OK) removed++;
        if (st[i] == DM_ESTATE) refused++;
    }
}

static void worker(dm_engine *e, int seed, std::chrono::steady_clock::time_point until)
{
    std::mt19937_64 rng(seed);
    while (std::chrono::steady_clock::now() < until && failures.load() == 0) {
        const int r = (int)(rng() % 20);
        const Body &b = bodies[rng() % bodies.size()];
        if (r < 6) reader(e, b, rng);
        else if (r < 9) ingest(e, b, rng);
        else if (r < 13) remover(e, rng);
        else if (r == 13) {
            int32_t st = 0;
            CHECK(dm_cache_promote(e, b.digest, 1, &st) == DM_OK);
            CHECK(st == DM_OK || st == DM_ENOENT || st == DM_ENOMEM);
        } else if (r == 14) {
            int32_t st = 0;
            CHECK(dm_cache_verify(e, b.digest, 1, &st) == DM_OK);
            CHECK(st == DM_OK || st == DM_ENOENT || st == DM_ENOMEM);
        } else if (r == 15) {
            const char *path = b.src.c_str();
            int32_t st = 0;
            uint8_t got[32];
            CHECK(dm_cache_import(e, &path, b.digest, nullptr, 1, 0, got, &st) == DM_OK);
            CHECK(st == DM_OK || st == DM_ENOMEM);
            if (st == DM_OK) imported++;
        } else if (r == 16) {
            const uint64_t lim = rng() % 3 == 0 ? 1 : 1 + rng() % (8u << 20);
            CHECK(dm_cache_set_disk_limit(e, rng() % 4 == 0 ? 0 : lim) == DM_OK);
        } else {
            const int rc = dm_cache_evict(e, b.digest);
            CHECK(rc == DM_OK || rc == DM_ENOENT || rc == DM_ESTATE);
        }
    }
}

static uint64_t walk()
{
    uint64_t total = 0;
    for (const char *sub : {"blobs", "incoming", "partial"}) {
        std::error_code ec;
        for (auto it = fs::recursive_directory_iterator(g_cas + "/" + sub, ec); !ec && it != fs::recursive_directory_iterator(); it.increment(ec))
            if (it->is_regular_file()) total += it->file_size();
    }
    return total;
}

static void quiesce_and_check(dm_engine *e)
{
    dm_stats st;
    for (int i = 0; i < 12000; ++i) {                             // up to a minute: sanitizers and jitter slow the drain
        dm_engine_stats(e, &st);
        if (st.ring_slabs_free == st.ring_slabs_total && st.free_stream_slots == kMaxStreams && st.open_streams == 0 &&
            st.open_readers == 0)
            break;
        std::this_thread::sleep_for(std::chrono::milliseconds(5));
    }
    CHECK(st.ring_slabs_free == st.ring_slabs_total && st.free_stream_slots == kMaxStreams && st.open_streams == 0 &&
          st.open_readers == 0);
    CHECK(dm_cache_set_disk_limit(e, 1ull << 40) == DM_OK);
    dm_disk_usage u;
    memset(&u, 0, sizeof u);
    u.struct_size = sizeof u;
    uint64_t w = 0;
    for (int i = 0; i < 2000; ++i) {                              // spills still running are counted at their reservation
        CHECK(dm_cache_disk_usage(e, &u) == DM_OK);
        w = walk();
        if (u.used_bytes == w) break;
        std::this_thread::sleep_for(std::chrono::milliseconds(5));
    }
    if (u.used_bytes != w) fprintf(stderr, "limit index %llu, walk %llu\n", (unsigned long long)u.used_bytes, (unsigned long long)w);
    CHECK(u.used_bytes == w);
    // hbm_cas_used = the extents of the blobs in HBM (every reader is closed, so no removed blob keeps one)
    uint64_t in_hbm = 0;
    for (const Body &b : bodies) {
        uint64_t rid = 0, size = 0;
        if (dm_cache_open(e, b.digest, &rid, &size) != DM_OK) continue;
        if (dm_cache_device_extents(e, rid, nullptr, nullptr, 0) > 0) in_hbm += (std::max<uint64_t>(size, 1) + 255) / 256 * 256;
        CHECK(dm_cache_close(e, rid) == DM_OK);
    }
    dm_engine_stats(e, &st);
    CHECK(st.hbm_cas_used == in_hbm);
    // remove everything with nothing publishing: every digest is a miss, on both tiers, and nothing is left to count
    std::vector<uint8_t> all;
    for (const Body &b : bodies) all.insert(all.end(), b.digest, b.digest + 32);
    std::vector<int32_t> status(bodies.size());
    CHECK(dm_cache_remove(e, all.data(), (uint32_t)bodies.size(), DM_RM_ALIASES | DM_RM_PARTIAL, status.data()) == DM_OK);
    for (size_t i = 0; i < bodies.size(); ++i) {
        CHECK(status[i] == DM_OK || status[i] == DM_ENOENT);
        uint64_t size = 0;
        CHECK(dm_cache_contains(e, bodies[i].digest, &size) == DM_ENOENT);
    }
    uint32_t n = 0;
    uint8_t d[32];
    CHECK(dm_cache_list(e, nullptr, d, nullptr, 1, &n) == DM_OK && n == 0);
    dm_engine_stats(e, &st);
    CHECK(st.hbm_cas_used == 0 && st.suspended == 0);
    CHECK(dm_cache_disk_usage(e, &u) == DM_OK && u.used_bytes == walk());
    CHECK(dm_cache_set_disk_limit(e, 0) == DM_OK);
    printf("quiescent: slabs %llu/%llu, slots %llu, readers %llu\n", (unsigned long long)st.ring_slabs_free,
           (unsigned long long)st.ring_slabs_total, (unsigned long long)st.free_stream_slots,
           (unsigned long long)st.open_readers);
}

static void phase(double secs, int seed)
{
    dm_engine *e = make_engine();
    if (!e) { failures++; return; }
    {
        std::mt19937_64 rng(seed);
        for (const Body &b : bodies) ingest(e, b, rng);
    }
    const auto until = std::chrono::steady_clock::now() + std::chrono::milliseconds((long)(secs * 1000));
    std::vector<std::thread> th;
    for (int t = 0; t < kThreads; ++t) th.emplace_back(worker, e, seed + t, until);
    for (auto &t : th) t.join();
    quiesce_and_check(e);
    // destroyed with readers of removed blobs still open: neither hangs nor leaks
    std::mt19937_64 rng(seed + 99);
    for (const Body &b : bodies) ingest(e, b, rng);
    std::vector<uint64_t> rids;
    for (const Body &b : bodies) {
        uint64_t rid = 0, size = 0;
        if (dm_cache_open(e, b.digest, &rid, &size) == DM_OK) rids.push_back(rid);
        int32_t st = 0;
        dm_cache_remove(e, b.digest, 1, 0, &st);
    }
    dm_engine_destroy(e);
}

int main(int argc, char **argv)
{
    if (argc < 3) { fprintf(stderr, "usage: %s <seconds> <cas_dir>\n", argv[0]); return 2; }
    const double secs = atof(argv[1]);
    g_cas = argv[2];
    fs::remove_all(g_cas);
    fs::remove_all(g_cas + "-src");
    fs::create_directories(g_cas);
    fs::create_directories(g_cas + "-src");
    make_bodies();
    phase(secs / 2, 100);
    phase(secs / 2, 200);                                         // restart over the same cas_dir
    printf("complete reads %ld, followers %ld, removed %ld, refused %ld, imported %ld\n", reads.load(), followed.load(),
           removed.load(), refused.load(), imported.load());
    if (failures.load()) { printf("REMOVE SOAK FAILED (%d)\n", failures.load()); return 1; }
    if (reads.load() == 0 || removed.load() == 0) { printf("REMOVE SOAK FAILED (nothing was exercised)\n"); return 1; }
    printf("REMOVE SOAK OK\n");
    return 0;
}
