// TEST INFRASTRUCTURE ONLY — soak of dm_cache_verify through the C-ABI, linked against the fake CUDA runtime
// (fake_cuda.cc) so it runs on a CPU-only box under ThreadSanitizer / AddressSanitizer.  The bodies are cached
// through ordinary streams and the engine is restarted, so that every blob is on the disk tier only.  Then worker
// threads verify random subsets (with duplicates) while others ingest the same digests through streams, open / read /
// close readers, evict, promote, and damage files on disk (a flipped byte, a truncation, bytes appended), with one
// more restart half way.  A reader of the HBM tier must always get the body's bytes (everything there was verified);
// a reader of the disk tier may see damage.  At the end a fresh engine verifies every digest in one call: each status
// must be DM_OK, DM_ECORRUPT or DM_ENOENT, the HBM arena stays empty, and after that every file under blobs/ must hash
// to its name and no slab, stream slot or reader may be leaked.  Bodies of 64 KiB slabs and less than a quarter of a
// slab are checked through packs, the others by read-backs through the disk threads.
//
// usage: verify_soak <seconds> <threads> <cas_dir>         (FAKE_CUDA_JITTER_US: device jitter)
#include "../../include/demodel_b200.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <filesystem>
#include <fstream>
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
static std::atomic<long> ops{0}, verified{0}, corrupt{0}, damaged{0}, enomem{0};
static std::string g_cas;
static const uint64_t kArena = 2u << 20;         // smaller than the bodies together: ingests and promotions evict each other
static const uint32_t kMaxStreams = 256;

struct Body { std::vector<uint8_t> bytes; uint8_t digest[32]; };
static std::vector<Body> bodies;

static void make_bodies()
{
    const size_t sizes[] = {0, 1, 63, 64, 65, 4096, 65536, 65537, 70000, 262145, 300001, 1048577};
    for (int rep = 0; rep < 2; ++rep)
        for (size_t s : sizes) {
            Body b;
            b.bytes.resize(s);
            dm_synth_fill_host(0x9A0F, 700 + bodies.size(), 0, b.bytes.data(), s);
            dmo_sha256(b.bytes.data(), s, b.digest);
            bodies.push_back(std::move(b));
        }
}

static std::string blob_file(const uint8_t d[32])
{
    char hex[65];
    for (int i = 0; i < 32; ++i) snprintf(hex + 2 * i, 3, "%02x", d[i]);
    return g_cas + "/blobs/sha256/" + std::string(hex, 2) + "/" + hex;
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

static int pull(dm_engine *e, const Body &b, size_t chunk)
{
    uint64_t id = 0;
    int rc = dm_stream_open(e, b.digest, b.bytes.size(), &id);
    if (rc != DM_OK) return rc;
    for (size_t off = 0; rc == DM_OK && off < b.bytes.size(); off += chunk)
        rc = dm_stream_write(e, id, b.bytes.data() + off, std::min(chunk, b.bytes.size() - off));
    uint8_t got[32];
    int matched = 0;
    if (rc == DM_OK) rc = dm_stream_finish(e, id, got, &matched);
    if (rc != DM_OK) { dm_stream_abort(e, id); return rc; }
    return matched == 1 && memcmp(got, b.digest, 32) == 0 ? DM_OK : DM_EINVAL;
}

// Open, read whole, close.  strict: the bytes must be the body's (HBM-tier readers always; disk-tier ones when no
// file can have been damaged).
static void read_check(dm_engine *e, const Body &b, bool strict_disk)
{
    uint64_t rid = 0, size = 0;
    if (dm_cache_open(e, b.digest, &rid, &size) != DM_OK) return;
    void *ptrs[8];
    uint64_t lens[8];
    const int ne = dm_cache_device_extents(e, rid, ptrs, lens, 8);
    CHECK(ne >= 0 || ne == DM_ESTATE);
    const bool strict = ne >= 0 || strict_disk;
    std::vector<uint8_t> got(size);
    size_t off = 0;
    while (off < size) {
        size_t n = 0;
        if (dm_cache_read(e, rid, off, got.data() + off, std::min<size_t>(50000, size - off), &n) != DM_OK || n == 0) break;
        off += n;
    }
    if (strict) CHECK(size == b.bytes.size() && off == size && (size == 0 || memcmp(got.data(), b.bytes.data(), size) == 0));
    CHECK(dm_cache_close(e, rid) == DM_OK);
}

static void damage(std::mt19937_64 &rng, const Body &b)
{
    const std::string path = blob_file(b.digest);
    const int fd = open(path.c_str(), O_RDWR);
    if (fd < 0) return;
    const off_t size = lseek(fd, 0, SEEK_END);
    const int how = (int)(rng() % 3);
    if (how == 0 && size > 0) {
        const off_t at = (off_t)(rng() % (uint64_t)size);
        uint8_t c;
        if (pread(fd, &c, 1, at) == 1) { c ^= 0x10; if (pwrite(fd, &c, 1, at) == 1) damaged++; }
    } else if (how == 1 && size > 0) {
        if (ftruncate(fd, size - 1 - (off_t)(rng() % (uint64_t)size)) == 0) damaged++;
    } else if (how == 2) {
        if (pwrite(fd, "xyz", 3, size) == 3) damaged++;
    }
    close(fd);
}

static void worker(dm_engine *e, int tid, double seconds)
{
    std::mt19937_64 rng(500 + tid);
    const auto deadline = std::chrono::steady_clock::now() + std::chrono::duration<double>(seconds);
    while (std::chrono::steady_clock::now() < deadline && !failures.load()) {
        const Body &b = bodies[rng() % bodies.size()];
        const int op = (int)(rng() % 11);
        if (op < 5) {                                                  // verify or promote a random subset, duplicates included
            const bool verify = op < 4;
            const uint32_t n = 1 + (uint32_t)(rng() % 12);
            std::vector<uint8_t> dig(32 * n);
            std::vector<const Body *> which(n);
            for (uint32_t i = 0; i < n; ++i) {
                which[i] = &bodies[rng() % bodies.size()];
                memcpy(&dig[32 * i], which[i]->digest, 32);
            }
            std::vector<int32_t> st(n, 1);
            CHECK((verify ? dm_cache_verify : dm_cache_promote)(e, dig.data(), n, st.data()) == DM_OK);
            for (uint32_t i = 0; i < n; ++i) {
                if (!(st[i] == DM_OK || st[i] == DM_ENOENT || st[i] == DM_ENOMEM || st[i] == DM_ECORRUPT || st[i] == DM_EIO))
                    fprintf(stderr, "unexpected %s status %d\n", verify ? "verify" : "promotion", st[i]);
                // DM_EIO: the file was cut short by a damaging thread while it was being read
                CHECK(st[i] == DM_OK || st[i] == DM_ENOENT || st[i] == DM_ENOMEM || st[i] == DM_ECORRUPT || st[i] == DM_EIO);
                for (uint32_t j = 0; j < i; ++j)
                    if (which[j] == which[i]) CHECK(st[j] == st[i]);              // a duplicate shares its status
                if (verify && st[i] == DM_OK) verified++;
                if (st[i] == DM_ECORRUPT) corrupt++;
                if (st[i] == DM_ENOMEM) enomem++;
            }
        } else if (op < 7) {
            const int rc = pull(e, b, 1 + rng() % 40000);
            if (rc == DM_ENOMEM) enomem++;
            else CHECK(rc == DM_OK);
        } else if (op < 9) {
            read_check(e, b, false);
        } else if (op == 9) {
            const int rc = dm_cache_evict(e, b.digest);
            CHECK(rc == DM_OK || rc == DM_ENOENT || rc == DM_ESTATE);
        } else {
            damage(rng, b);
        }
        ops++;
    }
}

static bool engine_clean(dm_engine *e)
{
    dm_stats st;
    for (int i = 0; i < 1000; ++i) {
        dm_engine_stats(e, &st);
        if (st.ring_slabs_free == st.ring_slabs_total && st.free_stream_slots == kMaxStreams && st.open_streams == 0 &&
            st.open_readers == 0)
            return true;
        std::this_thread::sleep_for(std::chrono::milliseconds(5));
    }
    printf("NOT CLEAN: open_streams=%llu slabs free/total=%llu/%llu free_stream_slots=%llu open_readers=%llu\n",
           (unsigned long long)st.open_streams, (unsigned long long)st.ring_slabs_free,
           (unsigned long long)st.ring_slabs_total, (unsigned long long)st.free_stream_slots,
           (unsigned long long)st.open_readers);
    return false;
}

static void run_workers(dm_engine *e, int threads, double seconds)
{
    std::vector<std::thread> th;
    for (int t = 0; t < threads; ++t) th.emplace_back(worker, e, t, seconds);
    std::atomic<bool> done{false};
    std::thread dog([&] {                                // a stuck engine fails with a report instead of hanging
        long last = -1;
        int still = 0;
        while (!done.load()) {
            std::this_thread::sleep_for(std::chrono::milliseconds(500));
            const long now = ops.load();
            still = now == last ? still + 1 : 0;
            last = now;
            if (still == 60) {
                dm_stats w;
                dm_engine_stats(e, &w);
                fprintf(stderr, "STUCK for 30 s: open_streams=%llu slabs free/total=%llu/%llu\nVERIFY SOAK FAILED (stuck)\n",
                        (unsigned long long)w.open_streams, (unsigned long long)w.ring_slabs_free,
                        (unsigned long long)w.ring_slabs_total);
                _Exit(3);
            }
        }
    });
    for (auto &t : th) t.join();
    done = true;
    dog.join();
}

static void final_verify()
{
    dm_engine *e = make_engine();
    CHECK(e);
    // one call over every digest, twice: nothing else runs, so every status says what its file holds, and a second
    // call finds exactly the files the first one kept
    std::vector<uint8_t> all;
    for (const Body &b : bodies) all.insert(all.end(), b.digest, b.digest + 32);
    std::vector<int32_t> st(bodies.size(), 1), again(bodies.size(), 1);
    CHECK(dm_cache_verify(e, all.data(), (uint32_t)bodies.size(), st.data()) == DM_OK);
    CHECK(dm_cache_verify(e, all.data(), (uint32_t)bodies.size(), again.data()) == DM_OK);
    for (size_t i = 0; i < bodies.size(); ++i) {
        CHECK(st[i] == DM_OK || st[i] == DM_ECORRUPT || st[i] == DM_ENOENT);
        CHECK(again[i] == (st[i] == DM_OK ? DM_OK : DM_ENOENT));
        if (st[i] == DM_OK) read_check(e, bodies[i], true);
        else { uint64_t sz; CHECK(dm_cache_contains(e, bodies[i].digest, &sz) == DM_ENOENT); }
    }
    dm_stats s;
    dm_engine_stats(e, &s);
    CHECK(s.hbm_cas_used == 0 && s.blobs_mismatched == 0);
    CHECK(engine_clean(e));
    dm_engine_destroy(e);
}

int main(int argc, char **argv)
{
    const double seconds = argc > 1 ? atof(argv[1]) : 3.0;
    const int threads = argc > 2 ? atoi(argv[2]) : 6;
    if (argc < 4) { fprintf(stderr, "usage: verify_soak <seconds> <threads> <cas_dir>\n"); return 2; }
    g_cas = argv[3];
    make_bodies();
    dm_engine *e = make_engine();
    if (!e) return 1;
    for (const Body &b : bodies)
        if (pull(e, b, 32768) != DM_OK) { printf("seeding failed: %s\nVERIFY SOAK FAILED\n", dm_last_error()); return 1; }
    dm_engine_destroy(e);                                // the spills drain: every body is on disk only now
    {
        dm_engine *f = make_engine();                    // clean files: every check passes, nothing goes into HBM
        if (!f) return 1;
        std::vector<uint8_t> all;
        for (const Body &b : bodies) all.insert(all.end(), b.digest, b.digest + 32);
        std::vector<int32_t> st(bodies.size(), 1);
        if (dm_cache_verify(f, all.data(), (uint32_t)bodies.size(), st.data()) != DM_OK) { printf("VERIFY SOAK FAILED\n"); return 1; }
        dm_stats s;
        dm_engine_stats(f, &s);
        for (size_t i = 0; i < bodies.size(); ++i) {
            if (st[i] != DM_OK) { printf("clean body %zu: status %d\nVERIFY SOAK FAILED\n", i, st[i]); return 1; }
            read_check(f, bodies[i], true);
        }
        if (s.hbm_cas_used != 0 || !engine_clean(f)) { printf("clean run left state behind\nVERIFY SOAK FAILED\n"); return 1; }
        dm_engine_destroy(f);
        if (failures.load()) { printf("VERIFY SOAK FAILED\n"); return 1; }
    }
    for (int round = 0; round < 2 && !failures.load(); ++round) {   // restart half way
        e = make_engine();
        if (!e) return 1;
        run_workers(e, threads, seconds / 2);
        const bool clean = engine_clean(e);
        dm_engine_destroy(e);
        if (!clean) failures++;
    }
    if (!failures.load()) final_verify();
    long files = 0, bad = 0;
    for (auto &ent : fs::recursive_directory_iterator(g_cas)) {
        if (!ent.is_regular_file()) continue;
        const std::string name = ent.path().filename().string();
        if (name.size() != 64) continue;
        std::ifstream f(ent.path(), std::ios::binary);
        std::vector<uint8_t> bytes((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
        uint8_t d[32];
        dmo_sha256(bytes.data(), bytes.size(), d);
        char hex[65];
        for (int i = 0; i < 32; ++i) snprintf(hex + 2 * i, 3, "%02x", d[i]);
        ++files;
        if (name != hex) { ++bad; fprintf(stderr, "disk tier file %s does not hash to its name\n", ent.path().c_str()); }
    }
    printf("ops=%ld verified=%ld corrupt=%ld damaged=%ld enomem=%ld files=%ld wrong=%ld failures=%d\n", ops.load(),
           verified.load(), corrupt.load(), damaged.load(), enomem.load(), files, bad, failures.load());
    if (failures.load() || bad || files == 0) { printf("VERIFY SOAK FAILED\n"); return 1; }
    printf("VERIFY SOAK OK\n");
    return 0;
}
