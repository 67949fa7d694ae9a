// TEST INFRASTRUCTURE ONLY — soak of the disk-tier limit (dm_cache_set_disk_limit) through the C-ABI, linked against the
// fake CUDA runtime (fake_cuda.cc) so it runs on a CPU-only box under ThreadSanitizer / AddressSanitizer.  Worker
// threads mix streams of known and unknown size (HBM and disk-backed), reads from disk and from HBM, evict, promote,
// verify, import, suspend / resume and changes of the limit.  Half way the engine is restarted as a verify-only engine
// whose every stream is disk-backed.  At each quiescence the tier's usage must equal a walk of blobs/, incoming/ and
// partial/ and, once the limit is applied again, be within it; every file under blobs/ must hash to its name, every
// completed read must have returned the body's bytes, incoming/ must be empty and no slab, stream slot or reader may be
// leaked.
//
// usage: disk_limit_soak <seconds> <threads> <cas_dir>        (FAKE_CUDA_JITTER_US: device jitter)
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

extern "C" void dmo_sha256(const void *data, size_t len, uint8_t out[32]);

#define CHECK(c) do { if (!(c)) { fprintf(stderr, "FAILED %s:%d: %s (last error: %s)\n", __FILE__, __LINE__, #c, dm_last_error()); \
                                   failures.fetch_add(1); return; } } while (0)

namespace fs = std::filesystem;

static std::atomic<int> failures{0};
static std::atomic<long> ops{0}, reads_ok{0};
static std::string g_cas, g_src;
static const uint64_t kArena = 1u << 20;         // bodies above it are disk-backed (DM_F_DISK_DIRECT)
static const uint32_t kMaxStreams = 256;
static const uint64_t kLimitLo = 256u << 10, kLimitHi = 4u << 20;

struct Body { std::vector<uint8_t> bytes; uint8_t digest[32]; std::string src; };
static std::vector<Body> bodies;

static void make_bodies()
{
    const size_t sizes[] = {1, 4096, 65537, 200000, 700001, 1100000, 1500007};
    fs::create_directories(g_src);
    for (int rep = 0; rep < 3; ++rep)
        for (size_t s : sizes) {
            Body b;
            b.bytes.resize(s);
            dm_synth_fill_host(0xD15C, 900 + bodies.size(), 0, b.bytes.data(), s);
            dmo_sha256(b.bytes.data(), s, b.digest);
            b.src = g_src + "/f" + std::to_string(bodies.size());
            std::ofstream(b.src, std::ios::binary).write((const char *)b.bytes.data(), (std::streamsize)s);
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

static dm_disk_usage usage(dm_engine *e)
{
    dm_disk_usage u;
    memset(&u, 0, sizeof u);
    u.struct_size = sizeof u;
    dm_cache_disk_usage(e, &u);
    return u;
}

static uint64_t walk()
{
    uint64_t t = 0;
    for (const char *sub : {"/blobs", "/incoming", "/partial"}) {
        std::error_code ec;
        for (auto &p : fs::recursive_directory_iterator(g_cas + sub, ec))
            if (p.is_regular_file(ec) && !p.is_symlink(ec)) t += p.file_size(ec);
    }
    return t;
}

// A whole body through one stream; known or unknown size.  DM_OK also when the limit left no room (verified, not
// cached): *matched must still be 1.
static int pull(dm_engine *e, const Body &b, bool known, size_t chunk)
{
    uint64_t id = 0;
    int rc = dm_stream_open(e, b.digest, known ? b.bytes.size() : 0, &id);
    if (rc != DM_OK) return rc;
    for (size_t off = 0; rc == DM_OK && off < b.bytes.size(); off += chunk)
        rc = dm_stream_write(e, id, b.bytes.data() + off, std::min(chunk, b.bytes.size() - off));
    uint8_t got[32];
    int matched = 0;
    if (rc == DM_OK) rc = dm_stream_finish(e, id, got, &matched);
    if (rc != DM_OK) { dm_stream_abort(e, id); return rc; }
    return matched == 1 && memcmp(got, b.digest, 32) == 0 ? DM_OK : DM_EINVAL;
}

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
        if (off < size && (off / 50000) % 3 == 1) std::this_thread::sleep_for(std::chrono::microseconds(200));
    }
    CHECK(size == b.bytes.size() && off == size && memcmp(got.data(), b.bytes.data(), size) == 0);   // eviction never reaches an open reader
    CHECK(dm_cache_close(e, rid) == DM_OK);
    reads_ok++;
}

static void suspend_resume(dm_engine *e, const Body &b, std::mt19937_64 &rng)
{
    uint64_t id = 0;
    if (dm_stream_open(e, b.digest, b.bytes.size(), &id) != DM_OK) return;
    const size_t half = b.bytes.size() / 2;
    if (dm_stream_write(e, id, b.bytes.data(), half) != DM_OK) { dm_stream_abort(e, id); return; }
    uint64_t from = 0;
    const int rc = dm_stream_suspend(e, id, &from);
    if (rc != DM_OK) {                                   // DM_EIO: another thread saves the same digest under the same names
        dm_stream_abort(e, id);
        CHECK(rc == DM_ENOMEM || rc == DM_ESTATE || rc == DM_EIO);
        return;
    }
    if (rng() % 3 == 0) return;                          // left saved: a later limit may evict it
    uint64_t rid = 0;
    if (dm_stream_resume_saved(e, b.digest, b.bytes.size(), &rid, &from) != DM_OK) return;   // evicted meanwhile
    int w = DM_OK;
    for (size_t off = from; w == DM_OK && off < b.bytes.size(); off += 40000)
        w = dm_stream_write_at(e, rid, off, b.bytes.data() + off, std::min<size_t>(40000, b.bytes.size() - off));
    uint8_t got[32];
    int matched = 0;
    if (w == DM_OK) w = dm_stream_finish(e, rid, got, &matched);
    if (w != DM_OK) { dm_stream_abort(e, rid); return; }
    CHECK(matched == 1 && memcmp(got, b.digest, 32) == 0);
}

static void worker(dm_engine *e, int seed, std::chrono::steady_clock::time_point until)
{
    std::mt19937_64 rng(seed);
    while (std::chrono::steady_clock::now() < until && failures.load() == 0) {
        const Body &b = bodies[rng() % bodies.size()];
        ops++;
        switch (rng() % 10) {
        case 0: case 1: {
            const int rc = pull(e, b, true, 1 + rng() % 70000);
            CHECK(rc == DM_OK || rc == DM_ENOMEM);
            break;
        }
        case 2: {
            const int rc = pull(e, b, false, 1 + rng() % 70000);
            CHECK(rc == DM_OK || rc == DM_ENOMEM);
            break;
        }
        case 3: case 4: read_check(e, b); break;
        case 5: dm_cache_evict(e, b.digest); break;
        case 6: {
            int32_t st = 0;
            const int rc = dm_cache_promote(e, b.digest, 1, &st);
            CHECK(rc == DM_OK || rc == DM_ESTATE);
            if (rc == DM_OK) CHECK(st == DM_OK || st == DM_ENOENT || st == DM_ENOMEM);
            break;
        }
        case 7: {
            uint8_t digs[3 * 32];
            for (int k = 0; k < 3; ++k) memcpy(digs + 32 * k, bodies[rng() % bodies.size()].digest, 32);
            int32_t st[3];
            CHECK(dm_cache_verify(e, digs, 3, st) == DM_OK);
            for (int k = 0; k < 3; ++k) CHECK(st[k] == DM_OK || st[k] == DM_ENOENT || st[k] == DM_ENOMEM);
            break;
        }
        case 8: {
            const char *p = b.src.c_str();
            uint8_t got[32];
            int32_t st = 0;
            CHECK(dm_cache_import(e, &p, b.digest, nullptr, 1, rng() % 2 ? DM_IMP_LINK : 0, got, &st) == DM_OK);
            CHECK(st == DM_OK || st == DM_ENOMEM);
            break;
        }
        default:
            if (rng() % 2) suspend_resume(e, b, rng);
            else CHECK(dm_cache_set_disk_limit(e, kLimitLo + rng() % (kLimitHi - kLimitLo)) == DM_OK);
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
    dm_disk_usage u = usage(e);
    for (int i = 0; i < 12000 && u.used_bytes != walk(); ++i) {     // spills still being written
        std::this_thread::sleep_for(std::chrono::milliseconds(5));
        u = usage(e);
    }
    CHECK(u.used_bytes == walk());
    CHECK(u.used_bytes == u.blob_bytes + u.staging_bytes + u.partial_bytes && u.staging_bytes == 0);
    CHECK(dm_cache_set_disk_limit(e, u.limit_bytes) == DM_OK);     // nothing is pinned now: the limit holds
    u = usage(e);
    CHECK(u.used_bytes <= u.limit_bytes && u.used_bytes == walk());
    std::error_code ec;
    CHECK(fs::is_empty(g_cas + "/incoming", ec));
    for (const Body &b : bodies) {                                 // no index entry outlives its evicted file
        uint64_t rid = 0, size = 0;
        if (dm_cache_contains(e, b.digest, &size) != DM_OK) continue;
        CHECK(dm_cache_open(e, b.digest, &rid, &size) == DM_OK);
        CHECK(dm_cache_close(e, rid) == DM_OK);
    }
    for (auto &p : fs::recursive_directory_iterator(g_cas + "/blobs", ec)) {
        const std::string name = p.path().filename().string();
        if (!p.is_regular_file(ec) || name.size() != 64) continue;
        std::ifstream f(p.path(), std::ios::binary);
        std::vector<uint8_t> bytes((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
        uint8_t d[32];
        dmo_sha256(bytes.data(), bytes.size(), d);
        char hex[65];
        for (int i = 0; i < 32; ++i) snprintf(hex + 2 * i, 3, "%02x", d[i]);
        CHECK(name == hex);
    }
    printf("quiescent: used %llu of %llu, %llu blobs, evicted %llu, refused %llu\n", (unsigned long long)u.used_bytes,
           (unsigned long long)u.limit_bytes, (unsigned long long)u.blob_files, (unsigned long long)u.evicted_files,
           (unsigned long long)u.refused);
}

static void phase(uint32_t flags, double secs, int nthreads)
{
    dm_engine *e = make_engine(flags);
    if (!e) { failures++; return; }
    if (dm_cache_set_disk_limit(e, kLimitHi) != DM_OK) failures++;
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
    g_src = g_cas + "_src";
    fs::remove_all(g_cas);
    fs::create_directories(g_cas);
    make_bodies();
    phase(DM_F_DISK_DIRECT, secs / 2, nthreads);                          // HBM engine; large bodies disk-backed
    phase(DM_F_DISK_DIRECT | DM_F_NO_HBM_CAS, secs / 2, nthreads);        // restart: every stream disk-backed
    printf("ops %ld, reads %ld\n", ops.load(), reads_ok.load());
    if (failures.load()) { printf("DISK LIMIT SOAK FAILED (%d)\n", failures.load()); return 1; }
    printf("DISK LIMIT SOAK OK\n");
    return 0;
}
