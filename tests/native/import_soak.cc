// TEST INFRASTRUCTURE ONLY — soak of dm_cache_import through the C-ABI, linked against the fake CUDA runtime
// (fake_cuda.cc) so it runs on a CPU-only box under ThreadSanitizer / AddressSanitizer.  Worker threads import random
// subsets of source files (duplicates, wrong digests, unknown digests, hard-link and copy mode) while others ingest
// the same bodies through streams, verify, promote, evict, open / read / close readers and rewrite the source files,
// with an engine restart half way.  Half of the sources are replaced by rename (a new inode: they may be hard-linked
// into the tier), the other half rewritten in place while they may be being copied (those are imported by copy only:
// a linked file rewritten in place would change the tier's bytes, which is what DM_IMP_LINK documents).  At the end
// every file under blobs/ must hash to its name, incoming/ must be empty, and no slab, stream slot or reader may leak.
//
// usage: import_soak <seconds> <threads> <cas_dir> <source_dir>         (FAKE_CUDA_JITTER_US: device jitter)
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
static std::atomic<long> ops{0}, imported{0}, corrupt{0}, enomem{0}, rewrites{0};
static std::string g_cas, g_src;
static const uint64_t kArena = 2u << 20;
static const uint32_t kMaxStreams = 256;
static const int kSources = 16;                  // 0..7 replaced by rename (linkable), 8..15 rewritten in place (copied)

struct Body { std::vector<uint8_t> bytes; uint8_t digest[32]; };
static std::vector<Body> bodies;

static void make_bodies()
{
    const size_t sizes[] = {0, 1, 55, 64, 65, 4096, 16383, 16385, 65536, 70000, 262145, 300001};
    for (size_t s : sizes) {
        Body b;
        b.bytes.resize(s);
        dm_synth_fill_host(0x1A0F, 900 + bodies.size(), 0, b.bytes.data(), s);
        dmo_sha256(b.bytes.data(), s, b.digest);
        bodies.push_back(std::move(b));
    }
}

static std::string source(int i) { return g_src + "/s" + std::to_string(i); }

static bool write_file(const std::string &path, const Body &b)
{
    FILE *f = fopen(path.c_str(), "wb");
    if (!f) return false;
    const bool ok = b.bytes.empty() || fwrite(b.bytes.data(), 1, b.bytes.size(), f) == b.bytes.size();
    return fclose(f) == 0 && ok;
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

// Open, read whole, close: a blob of the set must read back as its body.
static void read_check(dm_engine *e, const Body &b)
{
    uint64_t rid = 0, size = 0;
    if (dm_cache_open(e, b.digest, &rid, &size) != DM_OK) return;
    std::vector<uint8_t> got(size);
    size_t off = 0;
    while (off < size) {
        size_t n = 0;
        if (dm_cache_read(e, rid, off, got.data() + off, std::min<size_t>(50000, size - off), &n) != DM_OK || n == 0) break;
        off += n;
    }
    CHECK(size == b.bytes.size() && off == size && (size == 0 || memcmp(got.data(), b.bytes.data(), size) == 0));
    CHECK(dm_cache_close(e, rid) == DM_OK);
}

static void rewrite(std::mt19937_64 &rng, int i)
{
    const Body &b = bodies[rng() % bodies.size()];
    if (i < kSources / 2) {                                    // a new inode, renamed over the old one
        const std::string tmp = source(i) + ".new" + std::to_string(rng());
        if (write_file(tmp, b) && rename(tmp.c_str(), source(i).c_str()) == 0) rewrites++;
        else unlink(tmp.c_str());
    } else {                                                   // in place: a copy running now may see any mix
        const int fd = open(source(i).c_str(), O_WRONLY | O_TRUNC);
        if (fd < 0) return;
        size_t off = 0;
        while (off < b.bytes.size()) {
            const ssize_t k = pwrite(fd, b.bytes.data() + off, std::min<size_t>(7000, b.bytes.size() - off), (off_t)off);
            if (k <= 0) break;
            off += (size_t)k;
        }
        close(fd);
        rewrites++;
    }
}

static void import_some(dm_engine *e, std::mt19937_64 &rng)
{
    const bool link = rng() % 2;
    const uint32_t n = 1 + (uint32_t)(rng() % 10);
    std::vector<std::string> names(n);
    std::vector<const char *> paths(n), keys(n);
    std::vector<uint8_t> expect(32 * n, 0), digs(32 * n, 0xAA);
    std::vector<int32_t> st(n, 1);
    std::vector<int> kind(n);                                  // 0 unknown, 1 a body's digest, 2 a wrong digest
    std::vector<std::string> keytext(n);
    for (uint32_t i = 0; i < n; ++i) {
        const int s = link ? (int)(rng() % (kSources / 2)) : (int)(rng() % kSources);
        names[i] = source(s);
        if (i && rng() % 4 == 0) { names[i] = names[i - 1]; memcpy(&expect[32 * i], &expect[32 * (i - 1)], 32); kind[i] = kind[i - 1]; }
        else {
            kind[i] = (int)(rng() % 3);
            if (kind[i]) memcpy(&expect[32 * i], bodies[rng() % bodies.size()].digest, 32);
            if (kind[i] == 2) expect[32 * i + rng() % 32] ^= 0x40;
        }
        paths[i] = names[i].c_str();
        keytext[i] = "https://soak.example/" + std::to_string(rng() % 64);
        keys[i] = rng() % 2 ? keytext[i].c_str() : nullptr;
    }
    CHECK(dm_cache_import(e, paths.data(), expect.data(), keys.data(), n, link ? DM_IMP_LINK : 0, digs.data(), st.data()) == DM_OK);
    static const uint8_t zero[32] = {0};
    for (uint32_t i = 0; i < n; ++i) {
        if (!(st[i] == DM_OK || st[i] == DM_ECORRUPT || st[i] == DM_ENOMEM)) fprintf(stderr, "unexpected import status %d\n", st[i]);
        CHECK(st[i] == DM_OK || st[i] == DM_ECORRUPT || st[i] == DM_ENOMEM);
        if (kind[i] == 2) CHECK(st[i] != DM_OK);               // nothing hashes to a flipped digest
        if (st[i] == DM_OK && kind[i]) CHECK(memcmp(&digs[32 * i], &expect[32 * i], 32) == 0);
        if (st[i] == DM_ECORRUPT) CHECK(kind[i] && memcmp(&digs[32 * i], &expect[32 * i], 32) != 0);
        if (st[i] == DM_ENOMEM) CHECK(memcmp(&digs[32 * i], zero, 32) == 0);
        for (uint32_t j = 0; j < i; ++j)
            if (names[j] == names[i] && memcmp(&expect[32 * j], &expect[32 * i], 32) == 0)
                CHECK(st[j] == st[i] && memcmp(&digs[32 * j], &digs[32 * i], 32) == 0);   // a duplicate shares its verdict
        if (st[i] == DM_OK) {
            imported++;
            if (keys[i]) {
                uint8_t a[32];
                (void)dm_cache_alias_get(e, keys[i], a);       // (another thread may have re-pointed the key since)
            }
        }
        if (st[i] == DM_ECORRUPT) corrupt++;
        if (st[i] == DM_ENOMEM) enomem++;
    }
}

static void worker(dm_engine *e, int tid, double seconds)
{
    std::mt19937_64 rng(700 + tid);
    const auto deadline = std::chrono::steady_clock::now() + std::chrono::duration<double>(seconds);
    while (std::chrono::steady_clock::now() < deadline && !failures.load()) {
        const Body &b = bodies[rng() % bodies.size()];
        const int op = (int)(rng() % 12);
        if (op < 4) {
            import_some(e, rng);
        } else if (op < 6) {
            const int rc = pull(e, b, 1 + rng() % 40000);
            if (rc == DM_ENOMEM) enomem++;
            else CHECK(rc == DM_OK);
        } else if (op < 8) {
            const uint32_t n = 1 + (uint32_t)(rng() % 6);
            std::vector<uint8_t> dig(32 * n);
            for (uint32_t i = 0; i < n; ++i) memcpy(&dig[32 * i], bodies[rng() % bodies.size()].digest, 32);
            std::vector<int32_t> st(n, 1);
            CHECK((op == 6 ? dm_cache_verify : dm_cache_promote)(e, dig.data(), n, st.data()) == DM_OK);
            for (uint32_t i = 0; i < n; ++i)                   // nothing damages the tier here: no file can be corrupt
                CHECK(st[i] == DM_OK || st[i] == DM_ENOENT || st[i] == DM_ENOMEM);
        } else if (op < 9) {
            read_check(e, b);
        } else if (op < 10) {
            const int rc = dm_cache_evict(e, b.digest);
            CHECK(rc == DM_OK || rc == DM_ENOENT || rc == DM_ESTATE);
        } else {
            rewrite(rng, (int)(rng() % kSources));
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
                fprintf(stderr, "STUCK for 30 s\nIMPORT SOAK FAILED (stuck)\n");
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
    if (argc < 5) { fprintf(stderr, "usage: import_soak <seconds> <threads> <cas_dir> <source_dir>\n"); return 2; }
    const double seconds = atof(argv[1]);
    const int threads = atoi(argv[2]);
    g_cas = argv[3];
    g_src = argv[4];
    fs::create_directories(g_src);
    make_bodies();
    for (int i = 0; i < kSources; ++i)
        if (!write_file(source(i), bodies[i % bodies.size()])) { printf("could not write sources\nIMPORT SOAK FAILED\n"); return 1; }
    {
        dm_engine *f = make_engine();                    // every source by its own digest: all DM_OK, nothing in HBM
        if (!f) return 1;
        std::vector<std::string> names;
        std::vector<const char *> paths;
        std::vector<uint8_t> expect, digs(32 * kSources);
        std::vector<int32_t> st(kSources, 1);
        for (int i = 0; i < kSources; ++i) names.push_back(source(i));
        for (int i = 0; i < kSources; ++i) {
            paths.push_back(names[i].c_str());
            expect.insert(expect.end(), bodies[i % bodies.size()].digest, bodies[i % bodies.size()].digest + 32);
        }
        if (dm_cache_import(f, paths.data(), expect.data(), nullptr, kSources, 0, digs.data(), st.data()) != DM_OK) { printf("IMPORT SOAK FAILED\n"); return 1; }
        dm_stats s;
        dm_engine_stats(f, &s);
        for (int i = 0; i < kSources; ++i) {
            if (st[i] != DM_OK) { printf("clean source %d: status %d\nIMPORT SOAK FAILED\n", i, st[i]); return 1; }
            read_check(f, bodies[i % bodies.size()]);
        }
        if (s.hbm_cas_used != 0 || !engine_clean(f)) { printf("clean run left state behind\nIMPORT SOAK FAILED\n"); return 1; }
        dm_engine_destroy(f);
        if (failures.load()) { printf("IMPORT SOAK FAILED\n"); return 1; }
    }
    for (int round = 0; round < 2 && !failures.load(); ++round) {   // restart half way
        dm_engine *e = make_engine();
        if (!e) return 1;
        run_workers(e, threads, seconds / 2);
        const bool clean = engine_clean(e);
        dm_engine_destroy(e);
        if (!clean) failures++;
    }
    long files = 0, bad = 0, staged = 0;
    for (auto &ent : fs::recursive_directory_iterator(g_cas)) {
        if (!ent.is_regular_file()) continue;
        if (ent.path().parent_path().filename() == "incoming") { ++staged; fprintf(stderr, "left in incoming/: %s\n", ent.path().c_str()); }
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
    printf("ops=%ld imported=%ld corrupt=%ld enomem=%ld rewrites=%ld files=%ld wrong=%ld staged=%ld failures=%d\n",
           ops.load(), imported.load(), corrupt.load(), enomem.load(), rewrites.load(), files, bad, staged, failures.load());
    if (failures.load() || bad || staged || files == 0) { printf("IMPORT SOAK FAILED\n"); return 1; }
    printf("IMPORT SOAK OK\n");
    return 0;
}
