// TEST INFRASTRUCTURE ONLY — soak of followers of disk-backed bodies (dm_cache_follow on DM_F_DISK_DIRECT streams)
// through the C-ABI, linked against the fake CUDA runtime (fake_cuda.cc) so it runs on a CPU-only box under
// ThreadSanitizer / AddressSanitizer.  Owner threads write bodies sequentially, as out-of-order range parts, of known
// and unknown size, slowly enough to be followed; some abort half way, some are opened with an expected digest their
// bytes do not have (the last byte is never written), some are suspended and resumed from the saved file.  Follower
// threads attach at random times and offsets and read to EOF or an error.  Other threads change the disk-tier limit,
// down to 1 byte, and verify blobs.  Half way the engine is restarted as a verify-only engine whose every stream is
// disk-backed.  Every byte a follower returned must be the body's byte at that offset, and only a body whose verdict
// matched may end in a clean EOF.  At rest no slab, stream slot or reader is leaked, incoming/ is empty, and a limit of
// 1 byte empties blobs/ (no follower left a pin behind).
//
// usage: disk_follow_soak <seconds> <threads> <cas_dir>        (FAKE_CUDA_JITTER_US: device jitter)
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
static std::atomic<long> owned{0}, follows{0}, eofs{0}, estates{0}, suspends{0};
static std::atomic<int> g_hot{0};                // the body an owner opened last: followers prefer it
static std::string g_cas;
static const uint64_t kArena = 1u << 20;         // bodies above it are disk-backed on the HBM engine
static const uint32_t kMaxStreams = 256;
static const uint64_t kLimitHi = 16u << 20;

struct Body { std::vector<uint8_t> bytes; uint8_t digest[32]; };
static std::vector<Body> bodies;

static void make_bodies()
{
    const size_t sizes[] = {300001, 1100000, 1500007, 2000003};
    for (int rep = 0; rep < 2; ++rep)
        for (size_t s : sizes) {
            Body b;
            b.bytes.resize(s);
            dm_synth_fill_host(0xF011, 700 + bodies.size(), 0, b.bytes.data(), s);
            dmo_sha256(b.bytes.data(), s, b.digest);
            bodies.push_back(std::move(b));
        }
}

static dm_engine *make_engine(uint32_t flags)
{
    dm_config cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.struct_size = sizeof cfg;
    cfg.hbm_cas_bytes = kArena;
    cfg.ring_bytes = 1u << 20;
    cfg.slab_bytes = 64u << 10;
    cfg.max_streams = kMaxStreams;
    cfg.cas_dir = g_cas.c_str();
    cfg.flags = flags;
    dm_engine *e = nullptr;
    if (dm_engine_create(&cfg, &e) != DM_OK) { fprintf(stderr, "create failed: %s\n", dm_last_error()); return nullptr; }
    return e;
}

static void pause(std::mt19937_64 &rng) { if (rng() % 4 == 0) std::this_thread::sleep_for(std::chrono::microseconds(rng() % 400)); }

// Writes [from, end) of the body in random pieces: in order, or as two to four range parts in a random order.
static int write_body(dm_engine *e, uint64_t id, const Body &b, size_t from, size_t end, bool ranged, std::mt19937_64 &rng)
{
    std::vector<std::pair<size_t, size_t>> parts;
    const size_t k = ranged ? 2 + rng() % 3 : 1;
    for (size_t i = 0; i < k; ++i) parts.emplace_back(from + (end - from) * i / k, from + (end - from) * (i + 1) / k);
    std::shuffle(parts.begin(), parts.end(), rng);
    int rc = DM_OK;
    for (auto &p : parts)
        for (size_t off = p.first; rc == DM_OK && off < p.second;) {
            const size_t n = std::min<size_t>(1 + rng() % 90000, p.second - off);
            rc = ranged ? dm_stream_write_at(e, id, off, b.bytes.data() + off, n) : dm_stream_write(e, id, b.bytes.data() + off, n);
            off += n;
            pause(rng);
        }
    return rc;
}

static void owner(dm_engine *e, int bi, std::mt19937_64 &rng)
{
    const Body &b = bodies[bi];
    const size_t size = b.bytes.size();
    const bool known = rng() % 3 != 0, ranged = rng() % 3 == 0;
    const int mode = (int)(rng() % 10);                  // 0: abort half way, 1: wrong digest, 2: suspend + resume
    const size_t end = mode == 1 ? size - 1 : size;      // (the body without its last byte does not have its digest)
    uint64_t id = 0;
    if (dm_stream_open(e, b.digest, known ? size : 0, &id) != DM_OK) return;
    g_hot = bi;
    owned++;
    const size_t cut = mode == 0 || mode == 2 ? size / 2 : end;
    int rc = write_body(e, id, b, 0, cut, ranged, rng);
    if (rc == DM_OK && mode == 2) {
        uint64_t from = 0;
        rc = dm_stream_suspend(e, id, &from);
        if (rc != DM_OK) { dm_stream_abort(e, id); return; }          // another thread saves the same digest, no room, ...
        suspends++;
        if (dm_stream_resume_saved(e, b.digest, known ? size : 0, &id, &from) != DM_OK) return;   // evicted, taken over
        g_hot = bi;
        rc = write_body(e, id, b, from, size, ranged, rng);
    } else if (rc == DM_OK && mode == 0) {
        CHECK(dm_stream_abort(e, id) == DM_OK);
        return;
    }
    uint8_t got[32];
    int matched = 0;
    if (rc == DM_OK) rc = dm_stream_finish(e, id, got, &matched);
    if (rc != DM_OK) { dm_stream_abort(e, id); return; }
    CHECK(matched == (mode == 1 ? 0 : 1));
}

static void follower(dm_engine *e, int bi, std::mt19937_64 &rng)
{
    const Body &b = bodies[bi];
    const size_t size = b.bytes.size();
    uint64_t rid = 0, hint = 0;
    if (dm_cache_follow(e, b.digest, &rid, &hint) != DM_OK) return;
    follows++;
    CHECK(hint == 0 || hint == size);
    size_t pos = rng() % 3 ? 0 : rng() % size;
    const bool early_close = rng() % 8 == 0;
    std::vector<uint8_t> buf(70000);
    int rc = DM_OK;
    bool eof = false;
    for (;;) {
        size_t n = 0;
        rc = dm_cache_read(e, rid, pos, buf.data(), 1 + rng() % buf.size(), &n);
        eof = rc == DM_OK && n == 0;
        if (rc != DM_OK || n == 0) break;
        CHECK(pos + n <= size && memcmp(buf.data(), b.bytes.data() + pos, n) == 0);   // the body's bytes, never others
        pos += n;
        if (early_close && rng() % 4 == 0) break;
        if (rng() % 8 == 0) std::this_thread::sleep_for(std::chrono::microseconds(rng() % 300));
    }
    if (eof) {                                           // a clean EOF: only after a matched verdict
        CHECK(pos == size);
        eofs++;
        size_t n = 0;
        const size_t off = rng() % size;
        CHECK(dm_cache_read(e, rid, off, buf.data(), buf.size(), &n) == DM_OK);
        CHECK(n == std::min(buf.size(), size - off) && memcmp(buf.data(), b.bytes.data() + off, n) == 0);
        char meta[512];
        size_t len = 0;
        CHECK(dm_cache_meta(e, rid, meta, sizeof meta, &len) == DM_OK);
        char hex[65];
        for (int i = 0; i < 32; ++i) snprintf(hex + 2 * i, 3, "%02x", b.digest[i]);
        CHECK(strstr(meta, hex) != nullptr);
    } else if (rc != DM_OK) {
        CHECK(rc == DM_ESTATE || rc == DM_ENOENT);       // a failed body; ENOENT: an HBM follower's blob evicted first
        estates++;
    } else CHECK(early_close);
    CHECK(dm_cache_close(e, rid) == DM_OK);
}

static void worker(dm_engine *e, int seed, std::chrono::steady_clock::time_point until)
{
    std::mt19937_64 rng(seed);
    while (std::chrono::steady_clock::now() < until && failures.load() == 0) {
        const int r = (int)(rng() % 10);
        const int bi = rng() % 3 ? g_hot.load() : (int)(rng() % bodies.size());
        if (r < 3) owner(e, (int)(rng() % bodies.size()), rng);
        else if (r < 8) follower(e, bi, rng);
        else if (r == 8) {
            const uint64_t lim = rng() % 4 == 0 ? 1 : 1 + rng() % kLimitHi;
            CHECK(dm_cache_set_disk_limit(e, rng() % 5 == 0 ? 0 : lim) == DM_OK);
        } else {
            int32_t st = 0;
            CHECK(dm_cache_verify(e, bodies[bi].digest, 1, &st) == DM_OK);
            CHECK(st == DM_OK || st == DM_ENOENT || st == DM_ENOMEM);
        }
    }
}

static size_t blob_files()
{
    size_t n = 0;
    std::error_code ec;
    for (auto &p : fs::recursive_directory_iterator(g_cas + "/blobs", ec))
        if (p.is_regular_file(ec) && p.path().filename().string().size() == 64) ++n;
    return n;
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
    std::error_code ec;
    CHECK(fs::is_empty(g_cas + "/incoming", ec));
    // evict everything: with every reader closed nothing is pinned (spills of HBM blobs may still be finishing)
    for (int i = 0; i < 12000; ++i) {
        CHECK(dm_cache_set_disk_limit(e, 1) == DM_OK);
        if (blob_files() == 0) break;
        std::this_thread::sleep_for(std::chrono::milliseconds(5));
    }
    CHECK(blob_files() == 0);
    CHECK(dm_cache_set_disk_limit(e, 0) == DM_OK);
    printf("quiescent: slabs %llu/%llu, readers %llu\n", (unsigned long long)st.ring_slabs_free,
           (unsigned long long)st.ring_slabs_total, (unsigned long long)st.open_readers);
}

static void phase(uint32_t flags, double secs, int nthreads)
{
    dm_engine *e = make_engine(flags);
    if (!e) { failures++; return; }
    const auto until = std::chrono::steady_clock::now() + std::chrono::milliseconds((long)(secs * 1000));
    std::vector<std::thread> th;
    for (int t = 0; t < nthreads; ++t) th.emplace_back(worker, e, 1000 * (int)flags + t, until);
    for (auto &t : th) t.join();
    quiesce_and_check(e);
    dm_engine_destroy(e);
}

int main(int argc, char **argv)
{
    if (argc < 4) { fprintf(stderr, "usage: %s <seconds> <threads> <cas_dir>\n", argv[0]); return 2; }
    const double secs = atof(argv[1]);
    const int nthreads = atoi(argv[2]);
    g_cas = argv[3];
    fs::remove_all(g_cas);
    fs::create_directories(g_cas);
    make_bodies();
    phase(DM_F_DISK_DIRECT, secs / 2, nthreads);                          // HBM engine; large bodies disk-backed
    phase(DM_F_DISK_DIRECT | DM_F_NO_HBM_CAS, secs / 2, nthreads);        // restart: every stream disk-backed
    printf("owned %ld, follows %ld, clean EOFs %ld, failed reads %ld, suspends %ld\n", owned.load(), follows.load(),
           eofs.load(), estates.load(), suspends.load());
    if (failures.load()) { printf("DISK FOLLOW SOAK FAILED (%d)\n", failures.load()); return 1; }
    if (eofs.load() == 0 || estates.load() == 0) { printf("DISK FOLLOW SOAK FAILED (nothing was followed)\n"); return 1; }
    printf("DISK FOLLOW SOAK OK\n");
    return 0;
}
