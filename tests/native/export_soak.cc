// TEST INFRASTRUCTURE ONLY — soak of dm_cache_export through the C-ABI, linked against the fake CUDA runtime
// (fake_cuda.cc) so it runs on a CPU-only box under ThreadSanitizer / AddressSanitizer.  Worker threads export random
// subsets of the bodies (duplicates, digests that are not cached, destinations in shared directories) while others
// ingest them through streams, promote, evict, remove, damage tier files in place and change the disk-tier limit, with
// an engine restart half way.  Destinations are named by the digest they must hold.  At the end every destination file
// must hash to its name, no staged file may be left, every tier file that does not hash to its name must be one this
// soak damaged (export never writes the tier), and no slab, stream slot or reader may leak.
//
// usage: export_soak <seconds> <threads> <cas_dir> <out_dir>         (FAKE_CUDA_JITTER_US: device jitter)
#include "../../include/demodel_b200.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <filesystem>
#include <fstream>
#include <mutex>
#include <random>
#include <set>
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
static std::atomic<long> ops{0}, exported{0}, corrupt{0}, missing{0}, enomem{0}, damaged{0}, refused{0};
static std::string g_cas, g_out;
static const uint64_t kArena = 2u << 20;
static const uint32_t kMaxStreams = 256;
static const int kDirs = 3;                      // destination directories the workers share
static std::mutex damaged_mu;
static std::set<std::string> damaged_names;      // tier files this soak flipped a byte of

struct Body { std::vector<uint8_t> bytes; uint8_t digest[32]; };
static std::vector<Body> bodies;

static std::string hex_of(const uint8_t d[32])
{
    char hex[65];
    for (int i = 0; i < 32; ++i) snprintf(hex + 2 * i, 3, "%02x", d[i]);
    return hex;
}

static void make_bodies()
{
    const size_t sizes[] = {0, 1, 55, 64, 65, 4096, 16383, 16385, 65536, 70000, 262145, 300001, 1000003};
    for (size_t s : sizes) {
        Body b;
        b.bytes.resize(s);
        dm_synth_fill_host(0xE4F0, 1900 + bodies.size(), 0, b.bytes.data(), s);
        dmo_sha256(b.bytes.data(), s, b.digest);
        bodies.push_back(std::move(b));
    }
}

static std::string tier_file(const uint8_t d[32])
{
    const std::string h = hex_of(d);
    return g_cas + "/blobs/sha256/" + h.substr(0, 2) + "/" + h;
}

static bool file_hash(const std::string &path, uint8_t out[32])
{
    std::ifstream f(path, std::ios::binary);
    if (!f) return false;
    std::vector<uint8_t> bytes((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    dmo_sha256(bytes.data(), bytes.size(), out);
    return true;
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

static void export_some(dm_engine *e, std::mt19937_64 &rng)
{
    const uint32_t n = 1 + (uint32_t)(rng() % 10);
    std::vector<uint8_t> digs(32 * n);
    std::vector<std::string> names(n);
    std::vector<const char *> dests(n);
    std::vector<int32_t> st(n, 1);
    for (uint32_t i = 0; i < n; ++i) {
        if (i && rng() % 4 == 0) {                             // a duplicate pair
            memcpy(&digs[32 * i], &digs[32 * (i - 1)], 32);
            names[i] = names[i - 1];
        } else {
            memcpy(&digs[32 * i], bodies[rng() % bodies.size()].digest, 32);
            if (rng() % 8 == 0) digs[32 * i + rng() % 32] ^= 0x40;     // never cached
            names[i] = g_out + "/d" + std::to_string(rng() % kDirs) + "/" + hex_of(&digs[32 * i]);
        }
    }
    for (uint32_t i = 0; i < n; ++i) dests[i] = names[i].c_str();
    CHECK(dm_cache_export(e, digs.data(), dests.data(), n, st.data()) == DM_OK);
    for (uint32_t i = 0; i < n; ++i) {
        if (!(st[i] == DM_OK || st[i] == DM_ENOENT || st[i] == DM_ECORRUPT || st[i] == DM_ENOMEM))
            fprintf(stderr, "unexpected export status %d\n", st[i]);
        CHECK(st[i] == DM_OK || st[i] == DM_ENOENT || st[i] == DM_ECORRUPT || st[i] == DM_ENOMEM);
        for (uint32_t j = 0; j < i; ++j)
            if (names[j] == names[i]) CHECK(st[j] == st[i]);   // a duplicate shares its verdict
        if (st[i] == DM_OK) {
            uint8_t got[32];
            CHECK(file_hash(names[i], got) && memcmp(got, &digs[32 * i], 32) == 0);
            exported++;
        }
        if (st[i] == DM_ENOENT) missing++;
        if (st[i] == DM_ECORRUPT) corrupt++;
        if (st[i] == DM_ENOMEM) enomem++;
    }
}

// Flip one byte of a tier file in place: what bit rot or a stray writer would do.
static void damage(const Body &b, std::mt19937_64 &rng)
{
    if (b.bytes.empty()) return;
    const std::string path = tier_file(b.digest);
    std::lock_guard<std::mutex> g(damaged_mu);                 // (recorded before the flip: the end check may not race it)
    const int fd = open(path.c_str(), O_RDWR);
    if (fd < 0) return;
    const off_t off = (off_t)(rng() % b.bytes.size());
    uint8_t c;
    if (pread(fd, &c, 1, off) == 1) {
        damaged_names.insert(hex_of(b.digest));
        c ^= 0x10;
        if (pwrite(fd, &c, 1, off) == 1) damaged++;
    }
    close(fd);
}

static void worker(dm_engine *e, int tid, double seconds)
{
    std::mt19937_64 rng(900 + tid);
    const auto deadline = std::chrono::steady_clock::now() + std::chrono::duration<double>(seconds);
    while (std::chrono::steady_clock::now() < deadline && !failures.load()) {
        const Body &b = bodies[rng() % bodies.size()];
        const int op = (int)(rng() % 16);
        if (op < 6) {
            export_some(e, rng);
        } else if (op < 9) {
            const int rc = pull(e, b, 1 + rng() % 40000);
            if (rc == DM_ENOMEM) enomem++;
            else CHECK(rc == DM_OK);
        } else if (op < 10) {
            int32_t st = 1;
            CHECK(dm_cache_promote(e, b.digest, 1, &st) == DM_OK);
            CHECK(st == DM_OK || st == DM_ENOENT || st == DM_ENOMEM || st == DM_ECORRUPT);
        } else if (op < 11) {
            const int rc = dm_cache_evict(e, b.digest);
            CHECK(rc == DM_OK || rc == DM_ENOENT || rc == DM_ESTATE);
        } else if (op < 13) {
            int32_t st = 1;
            CHECK(dm_cache_remove(e, b.digest, 1, 0, &st) == DM_OK);
            CHECK(st == DM_OK || st == DM_ENOENT || st == DM_ESTATE);
            if (st == DM_ESTATE) refused++;
        } else if (op < 14) {
            damage(b, rng);
        } else if (op < 15) {
            const uint64_t limits[] = {0, 256u << 10, 1u << 20, 64u << 20};
            CHECK(dm_cache_set_disk_limit(e, limits[rng() % 4]) == DM_OK);
        } else {
            int32_t st = 1;
            CHECK(dm_cache_verify(e, b.digest, 1, &st) == DM_OK);
            CHECK(st == DM_OK || st == DM_ENOENT || st == DM_ENOMEM || st == DM_ECORRUPT);
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
                fprintf(stderr, "STUCK for 30 s\nEXPORT SOAK FAILED (stuck)\n");
                _Exit(3);
            }
        }
    });
    for (auto &t : th) t.join();
    done = true;
    dog.join();
}

int main(int argc, char **argv)
{
    if (argc < 5) { fprintf(stderr, "usage: export_soak <seconds> <threads> <cas_dir> <out_dir>\n"); return 2; }
    const double seconds = atof(argv[1]);
    const int threads = atoi(argv[2]);
    g_cas = argv[3];
    g_out = argv[4];
    make_bodies();
    for (int round = 0; round < 2 && !failures.load(); ++round) {   // restart half way
        dm_engine *e = make_engine();
        if (!e) return 1;
        run_workers(e, threads, seconds / 2);
        const bool clean = engine_clean(e);
        dm_engine_destroy(e);
        if (!clean) failures++;
    }
    long dests = 0, bad = 0, staged = 0, tier = 0, foreign = 0;
    for (auto &ent : fs::recursive_directory_iterator(g_out)) {
        if (!ent.is_regular_file()) continue;
        const std::string name = ent.path().filename().string();
        if (name.find(".dm-export-") != std::string::npos) { ++staged; fprintf(stderr, "staged file left: %s\n", ent.path().c_str()); continue; }
        uint8_t d[32];
        ++dests;
        if (!file_hash(ent.path().string(), d) || name != hex_of(d)) { ++bad; fprintf(stderr, "%s does not hash to its name\n", ent.path().c_str()); }
    }
    for (auto &ent : fs::recursive_directory_iterator(g_cas)) {
        if (!ent.is_regular_file()) continue;
        const std::string name = ent.path().filename().string();
        if (name.size() != 64) continue;
        uint8_t d[32];
        ++tier;
        if (file_hash(ent.path().string(), d) && name == hex_of(d)) continue;
        if (!damaged_names.count(name)) { ++foreign; fprintf(stderr, "tier file %s changed by something other than this soak\n", ent.path().c_str()); }
    }
    printf("ops=%ld exported=%ld missing=%ld corrupt=%ld enomem=%ld damaged=%ld remove_refused=%ld dests=%ld wrong=%ld "
           "staged=%ld tier_files=%ld foreign=%ld failures=%d\n", ops.load(), exported.load(), missing.load(), corrupt.load(),
           enomem.load(), damaged.load(), refused.load(), dests, bad, staged, tier, foreign, failures.load());
    if (failures.load() || bad || staged || foreign || dests == 0 || exported.load() == 0) { printf("EXPORT SOAK FAILED\n"); return 1; }
    printf("EXPORT SOAK OK\n");
    return 0;
}
