// TEST INFRASTRUCTURE ONLY — soak of shared ring loads (dm_cache_open_verified_range) through the C-ABI, linked against
// the fake CUDA runtime (fake_cuda.cc) so it runs on a CPU-only box under ThreadSanitizer / AddressSanitizer.  Two
// engines, each starting with every blob on the disk tier only: one with an arena smaller than most blobs, one without
// an HBM tier (DM_F_NO_HBM_CAS | DM_F_DISK_DIRECT).  Reader threads open random ranges of blobs, so that they attach to
// running shared loads, join late and start loads of their own, and read them forward in random pieces; some stall
// (some past the detach grace, so that they are detached while others wait), some close early (also before the
// verdict), some try a read backwards or outside their range.  Other threads flip a byte of a tier file in place,
// ingest blobs again, verify, remove, evict from HBM and set the disk-tier limit.  Every piece a reader got is what the
// load hashed: a reader that saw a damaged piece never gets the last byte or a clean EOF.  At rest every ring slab and
// stream slot is back, no reader or stream is open, no digest is held against removal, hbm_cas_used is what it was,
// and after the engine is destroyed with range readers open no descriptor is left open.
//
// usage: range_open_soak <seconds> <threads> <cas_dir>        (FAKE_CUDA_JITTER_US: device jitter)
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

#include <fcntl.h>
#include <unistd.h>

extern "C" void dmo_sha256(const void *data, size_t len, uint8_t out[32]);

#define CHECK(c) do { if (!(c)) { fprintf(stderr, "FAILED %s:%d: %s (last error: %s)\n", __FILE__, __LINE__, #c, dm_last_error()); \
                                   failures.fetch_add(1); return; } } while (0)

namespace fs = std::filesystem;

static std::atomic<int> failures{0};
static std::atomic<long> opens{0}, eofs{0}, corrupt{0}, last_bytes{0}, flips{0}, closed_early{0}, backwards{0}, stalls{0},
    refused{0}, outside{0}, long_stalls{0};
static std::string g_cas;
static const uint64_t kArena = 256u << 10;
static const uint32_t kMaxStreams = 64;

struct Body { std::vector<uint8_t> bytes; uint8_t digest[32]; };
static std::vector<Body> bodies;

static void make_bodies()
{
    const size_t sizes[] = {0, 1, 1000, 16384, 70000, 300001, 900000, 2000000};
    for (int rep = 0; rep < 2; ++rep)
        for (size_t s : sizes) {
            Body b;
            b.bytes.resize(s);
            dm_synth_fill_host(0xA11, 700 + bodies.size(), 0, b.bytes.data(), s);
            dmo_sha256(b.bytes.data(), s, b.digest);
            bodies.push_back(std::move(b));
        }
}

static std::string blob_file(const Body &b)
{
    char hex[65];
    for (int i = 0; i < 32; ++i) snprintf(hex + 2 * i, 3, "%02x", b.digest[i]);
    return g_cas + "/blobs/sha256/" + std::string(hex, 2) + "/" + hex;
}

static dm_engine *make_engine(uint32_t flags)
{
    dm_config cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.struct_size = sizeof cfg;
    cfg.hbm_cas_bytes = kArena;
    cfg.ring_bytes = 4u << 20;
    cfg.slab_bytes = 64u << 10;                                   // 64 slabs: ring loads may hold 16, four loads at once
    cfg.max_streams = kMaxStreams;
    cfg.cas_dir = g_cas.c_str();
    cfg.flags = flags;
    dm_engine *e = nullptr;
    if (dm_engine_create(&cfg, &e) != DM_OK) { fprintf(stderr, "create failed: %s\n", dm_last_error()); return nullptr; }
    return e;
}

static int ingest(dm_engine *e, const Body &b)
{
    uint64_t id = 0;
    int rc = dm_stream_open(e, b.digest, b.bytes.size(), &id);
    if (rc != DM_OK) return rc;
    for (size_t off = 0; rc == DM_OK && off < b.bytes.size(); off += 100000)
        rc = dm_stream_write(e, id, b.bytes.data() + off, std::min<size_t>(100000, b.bytes.size() - off));
    uint8_t got[32];
    int matched = 0;
    if (rc == DM_OK) rc = dm_stream_finish(e, id, got, &matched);
    if (rc != DM_OK) dm_stream_abort(e, id);
    return rc;
}

static void reader(dm_engine *e, const Body &b, std::mt19937_64 &rng)
{
    const size_t size = b.bytes.size();
    // a Range: request: mostly parts of the blob, some from an offset to the end, some the whole blob
    const int shape = (int)(rng() % 3);
    const uint64_t off = shape == 2 ? 0 : rng() % (size + 1);
    const uint64_t len = shape == 0 ? rng() % (size - off + 1) : 0;
    const uint64_t end = len ? off + len : size;
    uint64_t rid = 0, got_size = 0;
    const int orc = dm_cache_open_verified_range(e, b.digest, off, len, &rid, &got_size);
    if (orc != DM_OK) {                                   // a miss (removed, or a corrupt file dropped), or no share left
        CHECK(orc == DM_ENOENT || orc == DM_ENOMEM || orc == DM_ECORRUPT);
        if (orc == DM_ENOMEM) refused++;
        return;
    }
    opens++;
    CHECK(got_size == size);
    const bool ring = dm_cache_device_extents(e, rid, nullptr, nullptr, 0) == DM_ESTATE;   // else an HBM hit
    const int mode = (int)(rng() % 8);                    // 0: closes early, 1: stalls, 2: tries a backward read, 3: outside
    std::vector<uint8_t> buf(200000);
    bool bad_piece = false, eof = false;
    size_t pos = off;
    int rc = DM_OK;
    for (int step = 0; step < 2000; ++step) {
        const size_t want = 1 + rng() % (rng() % 4 == 0 ? buf.size() : 4096);
        size_t n = 0;
        rc = dm_cache_read(e, rid, pos, buf.data(), want, &n);
        if (rc != DM_OK) break;
        CHECK(pos + n <= end && n <= want);
        if (n && memcmp(buf.data(), b.bytes.data() + pos, n) != 0) bad_piece = true;   // a damaged file, before its verdict   // a damaged file, before its verdict
        if (n && pos + n == size) { last_bytes++; CHECK(!bad_piece); }  // the last byte: only after a verdict that matched  // the last byte: only after a verdict that matched
        if (n == 0) { CHECK(pos == end); eof = end == size; break; }
        if (ring && mode == 2 && pos > off && rng() % 16 == 0) {
            size_t m = 0;
            CHECK(dm_cache_read(e, rid, pos - 1, buf.data(), 1, &m) == DM_ESTATE);
            char why[256];
            size_t wl = 0;
            CHECK(dm_error_detail(e, rid, why, sizeof why, &wl) == DM_OK && wl > 0);
            backwards++;
        }
        if (mode == 3 && rng() % 8 == 0) {
            size_t m = 0;
            if (off > 0) CHECK(dm_cache_read(e, rid, off - 1, buf.data(), 1, &m) == DM_ERANGE);
            if (end < size) CHECK(dm_cache_read(e, rid, end + 1, buf.data(), 1, &m) == DM_ERANGE);
            outside++;
        }
        pos += n;
        if (mode == 0 && rng() % 6 == 0) { closed_early++; break; }
        if (mode == 1 && rng() % 16 == 0) {
            stalls++;
            // past the detach grace (the first few always): others waiting for bytes of its load detach it
            const bool long_stall = long_stalls.load() < 3 || rng() % 8 == 0;
            if (long_stall) long_stalls++;
            std::this_thread::sleep_for(std::chrono::milliseconds(long_stall ? 600 + rng() % 200 : 1 + rng() % 20));
        }
    }
    if (eof) { CHECK(!bad_piece); eofs++; }
    // DM_ESTATE: detached, and the blob was gone (removed, or dropped as corrupt) when its next read started a load
    if (rc != DM_OK && rc != DM_ESTATE) {
        CHECK(rc == DM_ECORRUPT);
        corrupt++;
        size_t n = 0;
        CHECK(dm_cache_read(e, rid, pos, buf.data(), 1, &n) == DM_ECORRUPT);   // sticky
    }
    CHECK(dm_cache_close(e, rid) == DM_OK);
}

static void flip(const Body &b, std::mt19937_64 &rng)
{
    if (b.bytes.empty()) return;
    const int fd = open(blob_file(b).c_str(), O_WRONLY);
    if (fd < 0) return;
    const size_t at = rng() % 2 ? b.bytes.size() - 1 : rng() % b.bytes.size();
    const uint8_t v = (uint8_t)(b.bytes[at] ^ 0x41);
    if (pwrite(fd, &v, 1, (off_t)at) == 1) flips++;
    close(fd);
}

static void worker(dm_engine *e, int seed, std::chrono::steady_clock::time_point until)
{
    std::mt19937_64 rng(seed);
    while (std::chrono::steady_clock::now() < until && failures.load() == 0) {
        const int r = (int)(rng() % 24);
        const Body &b = bodies[rng() % bodies.size()];
        if (r < 14) reader(e, b, rng);
        else if (r == 14) flip(b, rng);
        else if (r < 17) { const int rc = ingest(e, b); CHECK(rc == DM_OK || rc == DM_ENOMEM); }
        else if (r == 17) {
            int32_t st = 0;
            CHECK(dm_cache_verify(e, b.digest, 1, &st) == DM_OK);
            CHECK(st == DM_OK || st == DM_ENOENT || st == DM_ENOMEM || st == DM_ECORRUPT);
        } else if (r == 18) {
            int32_t st = 0;
            CHECK(dm_cache_remove(e, b.digest, 1, 0, &st) == DM_OK);
            CHECK(st == DM_OK || st == DM_ENOENT || st == DM_ESTATE);
        } else if (r == 19) {
            const uint64_t lim = rng() % 3 == 0 ? 1 : 1 + rng() % (16u << 20);
            CHECK(dm_cache_set_disk_limit(e, rng() % 4 == 0 ? 0 : lim) == DM_OK);
        } else {
            const int rc = dm_cache_evict(e, b.digest);
            CHECK(rc == DM_OK || rc == DM_ENOENT || rc == DM_ESTATE);
        }
    }
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
    CHECK(dm_cache_set_disk_limit(e, 0) == DM_OK);
    for (const Body &b : bodies) dm_cache_evict(e, b.digest);
    dm_engine_stats(e, &st);
    CHECK(st.hbm_cas_used == 0);                                  // ring loads took no extent
    // every blob that is still cached reads back whole, as three parts that share one load
    for (const Body &b : bodies) {
        const uint64_t size = b.bytes.size(), cut[4] = {0, size / 3, 2 * size / 3, size};
        uint64_t rid[3] = {0, 0, 0}, got_size = 0;
        dm_stats s0, s1;
        dm_engine_stats(e, &s0);
        int rc = DM_OK;
        auto empty = [&](int k) { return k < 2 && cut[k + 1] == cut[k]; };   // (len 0 would mean: to the end)
        for (int k = 0; k < 3 && rc == DM_OK; ++k)
            if (!empty(k)) rc = dm_cache_open_verified_range(e, b.digest, cut[k], cut[k + 1] - cut[k], &rid[k], &got_size);
        if (rc != DM_OK) {
            CHECK(rc == DM_ENOENT || rc == DM_ECORRUPT);
            for (uint64_t r : rid) if (r) dm_cache_close(e, r);
            continue;
        }
        std::vector<uint8_t> all(size + 1);
        std::atomic<int> r2{DM_OK};
        std::vector<std::thread> th;
        for (int k = 0; k < 3; ++k)                               // all at once: the later parts wait for the front
            if (!empty(k)) th.emplace_back([&, k] {
                size_t got = cut[k], n = 0;
                int r = DM_OK;
                while ((r = dm_cache_read(e, rid[k], got, all.data() + got, cut[k + 1] - got + 1, &n)) == DM_OK && n) got += n;
                if (r != DM_OK) r2 = r;
                else if (got != cut[k + 1]) r2 = DM_EIO;
            });
        for (auto &t : th) t.join();
        dm_engine_stats(e, &s1);
        CHECK(r2.load() == DM_OK || r2.load() == DM_ECORRUPT);
        if (r2.load() == DM_OK) {
            CHECK(size == 0 || memcmp(all.data(), b.bytes.data(), size) == 0);
            CHECK(s1.bytes_hashed - s0.bytes_hashed <= size);      // one load for the three parts (none in HBM: evicted)
        }
        for (uint64_t r : rid) if (r) CHECK(dm_cache_close(e, r) == DM_OK);
    }
    for (size_t i = 0; i < bodies.size() / 2; ++i) {          // no shared load holds a digest any more (the other
        int32_t st2 = 0;                                          // half stays for the destroy below)
        CHECK(dm_cache_remove(e, bodies[i].digest, 1, 0, &st2) == DM_OK && st2 != DM_ESTATE);
    }
    dm_engine_stats(e, &st);
    CHECK(st.ring_slabs_free == st.ring_slabs_total && st.free_stream_slots == kMaxStreams && st.hbm_cas_used == 0);
    printf("quiescent: slabs %llu/%llu, slots %llu, readers %llu\n", (unsigned long long)st.ring_slabs_free,
           (unsigned long long)st.ring_slabs_total, (unsigned long long)st.free_stream_slots,
           (unsigned long long)st.open_readers);
}

static size_t open_fds()
{
    size_t n = 0;
    for (auto &ent : fs::directory_iterator("/proc/self/fd")) { (void)ent; ++n; }
    return n;
}

static void phase(double secs, int nthreads, int seed, uint32_t flags)
{
    const size_t fds0 = open_fds();
    {                                                             // every blob on the disk tier only, undamaged
        dm_engine *p = make_engine(flags);
        if (!p) { failures++; return; }
        for (const Body &b : bodies) {
            std::error_code ec;
            fs::remove(blob_file(b), ec);
            fs::remove(blob_file(b) + ".meta", ec);
            if (ingest(p, b) != DM_OK) { fprintf(stderr, "populate failed: %s\n", dm_last_error()); failures++; }
        }
        dm_engine_destroy(p);                                     // its spills drain first
    }
    dm_engine *e = make_engine(flags);
    if (!e) { failures++; return; }
    const auto until = std::chrono::steady_clock::now() + std::chrono::milliseconds((long)(secs * 1000));
    std::vector<std::thread> th;
    for (int t = 0; t < nthreads; ++t) th.emplace_back(worker, e, seed + t, until);
    for (auto &t : th) t.join();
    quiesce_and_check(e);
    // destroyed with ring loads running and their readers open, some part way through: neither hangs nor leaks
    for (const Body &b : bodies) {
        uint64_t rid = 0, size = 0;
        if (dm_cache_open_verified_range(e, b.digest, 0, 0, &rid, &size) == DM_OK && size > 1) {
            std::vector<uint8_t> buf(size / 2);
            size_t n = 0;
            dm_cache_read(e, rid, 0, buf.data(), buf.size(), &n);
        }
    }
    dm_engine_destroy(e);
    if (open_fds() != fds0) { fprintf(stderr, "FAILED: %zu descriptors open before the phase, %zu after\n", fds0, open_fds()); failures++; }
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
    phase(secs / 2, nthreads, 100, 0);                                          // most blobs larger than the arena
    phase(secs / 2, nthreads, 200, DM_F_NO_HBM_CAS | DM_F_DISK_DIRECT);         // no HBM tier at all
    printf("opens %ld (refused %ld), clean EOFs %ld, last bytes %ld, DM_ECORRUPT %ld, flips %ld, early closes %ld, "
           "stalls %ld (past the grace %ld), backward reads %ld, reads outside the range %ld\n", opens.load(), refused.load(),
           eofs.load(), last_bytes.load(), corrupt.load(), flips.load(), closed_early.load(), stalls.load(),
           long_stalls.load(), backwards.load(), outside.load());
    if (failures.load()) { printf("RANGE OPEN SOAK FAILED (%d)\n", failures.load()); return 1; }
    if (eofs.load() == 0 || corrupt.load() == 0 || closed_early.load() == 0 || backwards.load() == 0 ||
        outside.load() == 0 || long_stalls.load() == 0) {
        printf("RANGE OPEN SOAK FAILED (nothing was exercised)\n");
        return 1;
    }
    printf("RANGE OPEN SOAK OK\n");
    return 0;
}
