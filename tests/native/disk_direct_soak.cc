// TEST INFRASTRUCTURE ONLY — soak of disk-backed streams (DM_F_DISK_DIRECT) through the C-ABI, linked against
// the fake CUDA runtime (fake_cuda.cc) so it runs on a CPU-only box under ThreadSanitizer / AddressSanitizer.
// A small arena makes most bodies disk-backed.  Several threads mix sequential and zero-copy writes, 2..16
// range parts in random order, aborts, wrong expected digests and flush + finish racing an abort; then
// downloads are suspended, the engine is destroyed, and a new engine (with the flag, or without it and with
// room in HBM) resumes them; then file writes are made to fail with RLIMIT_FSIZE; then disk-backed bodies must
// finish while HBM writers hold a small ring, and 16 of them at once over 32 slabs.  At the end every file
// under blobs/ must hash to its own name, incoming/ must be empty, and no slab or stream slot may be leaked.
//
// usage: disk_direct_soak <seconds> <threads> <cas_dir> [no_hbm]    (RIG_SLAB / RIG_RING: ring geometry)
#include "../../include/demodel_b200.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <filesystem>
#include <fstream>
#include <map>
#include <random>
#include <string>
#include <thread>
#include <vector>

#include <signal.h>
#include <sys/resource.h>

extern "C" void dmo_sha256(const void *data, size_t len, uint8_t out[32]);

#define CHECK(c) do { if (!(c)) { fprintf(stderr, "FAILED %s:%d: %s (last error: %s)\n", __FILE__, __LINE__, #c, dm_last_error()); \
                                   failures.fetch_add(1); return; } } while (0)

namespace fs = std::filesystem;

static std::atomic<int> failures{0};
static std::atomic<long> ops{0}, enomem{0}, committed{0};
static std::string g_cas;
static uint32_t g_flags = 0;
static uint64_t g_slab = 64u << 10, g_ring = 1u << 20;
static const uint64_t kArena = 256u << 10;      // bodies above this are disk-backed

struct Body { std::vector<uint8_t> bytes; uint8_t digest[32]; };
static std::vector<Body> bodies;

static void make_bodies()
{
    const size_t sizes[] = {0, 1, 63, 64, 65, 4096, 70000, 262145, 300001, 524288, 700000, 1048577, 1500000};
    for (int rep = 0; rep < 2; ++rep)
        for (size_t s : sizes) {
            Body b;
            b.bytes.resize(s);
            dm_synth_fill_host(0xD15C, 900 + bodies.size(), 0, b.bytes.data(), s);
            dmo_sha256(b.bytes.data(), s, b.digest);
            bodies.push_back(std::move(b));
        }
}

static dm_engine *make_engine(uint32_t flags, uint64_t arena, uint64_t ring = g_ring, uint64_t slab = g_slab)
{
    dm_config cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.struct_size = sizeof cfg;
    cfg.hbm_cas_bytes = arena;
    cfg.ring_bytes = ring;
    cfg.slab_bytes = (uint32_t)slab;
    cfg.max_streams = 256;
    cfg.cas_dir = g_cas.c_str();
    cfg.flags = flags;
    dm_engine *e = nullptr;
    if (dm_engine_create(&cfg, &e) != DM_OK) { fprintf(stderr, "create failed: %s\n", dm_last_error()); return nullptr; }
    return e;
}

static bool read_back_equals(dm_engine *e, const Body &b)
{
    uint64_t rid = 0, size = 0;
    if (dm_cache_open(e, b.digest, &rid, &size) != DM_OK) return false;
    std::vector<uint8_t> got(size);
    size_t off = 0;
    bool ok = size == b.bytes.size();
    while (ok && off < size) {
        size_t n = 0;
        ok = dm_cache_read(e, rid, off, got.data() + off, std::min<size_t>(100000, size - off), &n) == DM_OK && n > 0;
        off += n;
    }
    dm_cache_close(e, rid);
    return ok && (size == 0 || memcmp(got.data(), b.bytes.data(), size) == 0);
}

// [lo, hi) pieces of a body in 2..16 parts, shuffled
static std::vector<std::pair<uint64_t, uint64_t>> split_parts(std::mt19937_64 &rng, uint64_t size)
{
    const int k = 2 + (int)(rng() % 15);
    std::vector<uint64_t> cuts = {0, size};
    for (int i = 1; i < k; ++i) cuts.push_back(size ? rng() % size : 0);
    std::sort(cuts.begin(), cuts.end());
    std::vector<std::pair<uint64_t, uint64_t>> parts;
    for (size_t i = 0; i + 1 < cuts.size(); ++i) if (cuts[i] < cuts[i + 1]) parts.push_back({cuts[i], cuts[i + 1]});
    std::shuffle(parts.begin(), parts.end(), rng);
    return parts;
}

// Write the parts interleaved, in pieces of up to `chunk` bytes.
static int write_parts(dm_engine *e, uint64_t id, const Body &b, std::vector<std::pair<uint64_t, uint64_t>> parts,
                       std::mt19937_64 &rng, size_t chunk)
{
    while (!parts.empty()) {
        const size_t i = rng() % parts.size();
        auto &p = parts[i];
        const uint64_t n = std::min<uint64_t>(chunk, p.second - p.first);
        const int rc = dm_stream_write_at(e, id, p.first, b.bytes.data() + p.first, n);
        if (rc != DM_OK) return rc;
        p.first += n;
        if (p.first == p.second) parts.erase(parts.begin() + (long)i);
    }
    return DM_OK;
}

static void worker(dm_engine *e, int tid, double seconds)
{
    std::mt19937_64 rng(7000 + tid);
    const auto deadline = std::chrono::steady_clock::now() + std::chrono::duration<double>(seconds);
    while (std::chrono::steady_clock::now() < deadline && !failures.load()) {
        const Body &b = bodies[rng() % bodies.size()];
        const int op = (int)(rng() % 7);
        const bool wrong = op == 3;
        uint8_t bad[32];
        memcpy(bad, b.digest, 32);
        bad[5] ^= 0x40;
        uint64_t id = 0;
        int rc = dm_stream_open(e, wrong ? bad : b.digest, b.bytes.size(), &id);
        if (rc == DM_ENOMEM) { enomem++; continue; }
        CHECK(rc == DM_OK);
        const size_t chunk = 1 + rng() % 40000;
        if (op == 0 || op == 3) {                                   // sequential
            for (size_t off = 0; rc == DM_OK && off < b.bytes.size(); off += chunk)
                rc = dm_stream_write(e, id, b.bytes.data() + off, std::min(chunk, b.bytes.size() - off));
        } else if (op == 1) {                                       // zero-copy windows
            size_t off = 0;
            while (rc == DM_OK && off < b.bytes.size()) {
                void *p = nullptr;
                size_t cap = 0;
                rc = dm_stream_acquire(e, id, &p, &cap);
                if (rc != DM_OK) break;
                const size_t n = std::min({cap, chunk, b.bytes.size() - off});
                memcpy(p, b.bytes.data() + off, n);
                rc = dm_stream_commit(e, id, n);
                off += n;
            }
        } else if (op == 2 || op == 5) {                            // range parts, any order
            rc = write_parts(e, id, b, split_parts(rng, b.bytes.size()), rng, chunk);
        } else if (op == 4) {                                       // abort mid-body
            const size_t cut = b.bytes.size() / 2;
            for (size_t off = 0; rc == DM_OK && off < cut; off += chunk)
                rc = dm_stream_write(e, id, b.bytes.data() + off, std::min(chunk, cut - off));
            if (rc == DM_ENOMEM) enomem++;
            CHECK(rc == DM_OK || rc == DM_ENOMEM);
            CHECK(dm_stream_abort(e, id) == DM_OK);
            ops++;
            continue;
        } else {                                                    // flush + finish racing an abort
            for (size_t off = 0; rc == DM_OK && off < b.bytes.size(); off += chunk)
                rc = dm_stream_write(e, id, b.bytes.data() + off, std::min(chunk, b.bytes.size() - off));
            if (rc == DM_OK) {
                std::thread other([&] { dm_stream_abort(e, id); });
                uint8_t got[32];
                int matched = 0;
                const int f = dm_stream_flush(e, id);
                const int g = f == DM_OK ? dm_stream_finish(e, id, got, &matched) : f;
                other.join();
                CHECK(g == DM_OK || g == DM_ESTATE || g == DM_EINVAL);
                CHECK(g != DM_OK || !matched || memcmp(got, b.digest, 32) == 0);
                ops++;
                continue;
            }
        }
        if (rc == DM_ENOMEM) { enomem++; dm_stream_abort(e, id); continue; }
        CHECK(rc == DM_OK);
        uint8_t got[32];
        int matched = -1;
        if (rng() & 1) CHECK(dm_stream_flush(e, id) == DM_OK);
        rc = dm_stream_finish(e, id, got, &matched);
        if (rc == DM_ENOMEM) { enomem++; dm_stream_abort(e, id); continue; }
        CHECK(rc == DM_OK);
        if (memcmp(got, b.digest, 32) != 0) fprintf(stderr, "wrong digest: op %d, %zu bytes, chunk %zu\n", op, b.bytes.size(), chunk);
        CHECK(memcmp(got, b.digest, 32) == 0);
        CHECK(matched == (wrong ? 0 : 1));
        if (!wrong) {
            committed++;
            // a disk-backed body is in its final place when finish returns; an HBM one may have been evicted already
            if (b.bytes.size() > kArena || (g_flags & DM_F_NO_HBM_CAS)) CHECK(fs::exists(g_cas + "/blobs/sha256/" + [&] {
                char h[65];
                for (int i = 0; i < 32; ++i) snprintf(h + 2 * i, 3, "%02x", b.digest[i]);
                return std::string(h, 2) + "/" + h;
            }()));
            uint64_t size = 0;
            if (dm_cache_contains(e, b.digest, &size) == DM_OK && (b.bytes.size() > kArena || (g_flags & DM_F_NO_HBM_CAS)))
                CHECK(read_back_equals(e, b));
        }
        ops++;
    }
}

static bool engine_clean(dm_engine *e)
{
    dm_stats st;
    for (int i = 0; i < 1000; ++i) {
        dm_engine_stats(e, &st);
        if (st.ring_slabs_free == st.ring_slabs_total && st.free_stream_slots == 256 && st.open_streams == 0) return true;
        std::this_thread::sleep_for(std::chrono::milliseconds(5));
    }
    printf("NOT CLEAN: open_streams=%llu slabs free/total=%llu/%llu free_stream_slots=%llu\n", (unsigned long long)st.open_streams,
           (unsigned long long)st.ring_slabs_free, (unsigned long long)st.ring_slabs_total, (unsigned long long)st.free_stream_slots);
    return false;
}

// suspend -> dm_engine_destroy -> new engine -> resume_saved: resume_from is the contiguous prefix rounded down to 64
static void suspend_and_resume_phase(uint32_t flags)
{
    std::mt19937_64 rng(4242);
    std::vector<std::pair<const Body *, uint64_t>> saved;
    dm_engine *e = make_engine(flags, kArena);
    CHECK(e);
    for (const Body &b : bodies) {
        if (b.bytes.size() <= kArena) continue;
        uint64_t id = 0;
        CHECK(dm_stream_open(e, b.digest, b.bytes.size(), &id) == DM_OK);
        // a sequential head, then a few parts beyond it
        const uint64_t head = rng() % (b.bytes.size() / 2);
        CHECK(dm_stream_write(e, id, b.bytes.data(), head) == DM_OK);
        std::map<uint64_t, uint64_t> have = {{0, head}};
        for (int k = 0; k < 3; ++k) {
            const uint64_t lo = head + 1 + rng() % (b.bytes.size() - head - 1);
            const uint64_t hi = std::min<uint64_t>(b.bytes.size(), lo + 1 + rng() % 100000);
            bool clash = false;
            for (auto &h : have) clash = clash || (lo < h.second + 1 && h.first < hi + 1);
            if (clash) continue;
            CHECK(dm_stream_write_at(e, id, lo, b.bytes.data() + lo, hi - lo) == DM_OK);
            have[lo] = hi;
        }
        uint64_t contiguous = 0;
        for (auto &h : have) if (h.first <= contiguous) contiguous = std::max(contiguous, h.second);
        uint64_t from = ~0ull;
        CHECK(dm_stream_suspend(e, id, &from) == DM_OK);
        CHECK(from == (contiguous & ~63ull));
        saved.push_back({&b, from});
    }
    CHECK(engine_clean(e));
    dm_engine_destroy(e);
    // the same flags, or an engine without the flag whose arena now holds the blob
    const bool to_hbm = (flags & DM_F_NO_HBM_CAS) == 0;
    e = make_engine(to_hbm ? 0 : flags, to_hbm ? 16u << 20 : kArena);
    CHECK(e);
    for (auto &sv : saved) {
        const Body &b = *sv.first;
        uint64_t id = 0, from = ~0ull;
        CHECK(dm_stream_resume_saved(e, b.digest, 0, &id, &from) == DM_OK);
        CHECK(from == sv.second);
        CHECK(dm_stream_write(e, id, b.bytes.data() + from, b.bytes.size() - from) == DM_OK);
        uint8_t got[32];
        int matched = 0;
        CHECK(dm_stream_finish(e, id, got, &matched) == DM_OK);
        CHECK(matched == 1 && memcmp(got, b.digest, 32) == 0);
        CHECK(read_back_equals(e, b));
    }
    CHECK(engine_clean(e));
    dm_stats st;
    dm_engine_stats(e, &st);
    CHECK(st.suspended == 0);
    dm_engine_destroy(e);
}

// File writes that fail (RLIMIT_FSIZE: EFBIG) surface as DM_EIO and never as a published file.
static void write_failure_phase(uint32_t flags)
{
    signal(SIGXFSZ, SIG_IGN);
    dm_engine *e = make_engine(flags, kArena);
    CHECK(e);
    struct rlimit old;
    getrlimit(RLIMIT_FSIZE, &old);
    struct rlimit lim = old;
    lim.rlim_cur = 400000;
    CHECK(setrlimit(RLIMIT_FSIZE, &lim) == 0);
    long eio = 0;
    for (const Body &b : bodies) {
        if (b.bytes.size() <= 400000) continue;
        char h[65];
        for (int i = 0; i < 32; ++i) snprintf(h + 2 * i, 3, "%02x", b.digest[i]);
        const std::string path = g_cas + "/blobs/sha256/" + std::string(h, 2) + "/" + h;
        std::error_code ec;
        fs::remove(path, ec);
        fs::remove(path + ".meta", ec);
        uint64_t id = 0;
        CHECK(dm_stream_open(e, b.digest, b.bytes.size(), &id) == DM_OK);
        int rc = DM_OK;
        for (size_t off = 0; rc == DM_OK && off < b.bytes.size(); off += 32768)
            rc = dm_stream_write(e, id, b.bytes.data() + off, std::min<size_t>(32768, b.bytes.size() - off));
        uint8_t got[32];
        int matched = 0;
        if (rc == DM_OK) rc = dm_stream_finish(e, id, got, &matched);
        CHECK(rc == DM_EIO);
        dm_stream_abort(e, id);                              // (DM_EINVAL if finish already released the id)
        CHECK(!fs::exists(path));
        ++eio;
    }
    CHECK(setrlimit(RLIMIT_FSIZE, &old) == 0);
    CHECK(eio > 0);
    CHECK(engine_clean(e));
    dm_engine_destroy(e);
}

// Bodies that must all finish within `seconds`, or the rig fails with a report instead of hanging.
static void must_finish(dm_engine *e, const char *what, std::atomic<int> &done, int want, double seconds)
{
    const auto deadline = std::chrono::steady_clock::now() + std::chrono::duration<double>(seconds);
    while (done.load() < want && !failures.load()) {
        if (std::chrono::steady_clock::now() > deadline) {
            dm_stats w;
            dm_engine_stats(e, &w);
            fprintf(stderr, "STUCK in %s: %d of %d bodies finished, open_streams=%llu slabs free/total=%llu/%llu\nDISK SOAK FAILED (stuck)\n",
                    what, done.load(), want, (unsigned long long)w.open_streams, (unsigned long long)w.ring_slabs_free,
                    (unsigned long long)w.ring_slabs_total);
            _Exit(3);
        }
        std::this_thread::sleep_for(std::chrono::milliseconds(20));
    }
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
    if (rc == DM_OK) rc = dm_stream_flush(e, id);
    if (rc == DM_OK) rc = dm_stream_finish(e, id, got, &matched);
    if (rc != DM_OK) { dm_stream_abort(e, id); return rc; }
    return matched == 1 && memcmp(got, b.digest, 32) == 0 ? DM_OK : DM_EINVAL;
}

// One disk-backed body at a time finishing while HBM writers keep an 8-slab ring busy: its read-backs find the ring
// empty again and again, and only slabs coming back through the HBM copy path (no disk work at all) can restart them.
static void disk_body_under_hbm_pressure()
{
    dm_engine *e = make_engine(DM_F_DISK_DIRECT, 1u << 20, 8 * 4096, 4096);
    CHECK(e);
    std::vector<const Body *> hbm, disk;
    for (const Body &b : bodies) {
        if (b.bytes.size() > 4096 && b.bytes.size() <= 70000) hbm.push_back(&b);
        if (b.bytes.size() > (1u << 20)) disk.push_back(&b);
    }
    std::atomic<bool> stop{false};
    std::atomic<int> done{0};
    std::vector<std::thread> th;
    for (int t = 0; t < 6; ++t)
        th.emplace_back([&, t] {
            for (size_t k = t; !stop.load() && !failures.load(); ++k) {
                const int rc = pull(e, *hbm[k % hbm.size()], 1000);
                if (rc == DM_ENOMEM) { enomem++; continue; }
                CHECK(rc == DM_OK);
            }
        });
    th.emplace_back([&] {
        for (const Body *b : disk) {
            CHECK(pull(e, *b, 32768) == DM_OK);
            done++;
        }
    });
    must_finish(e, "disk body under HBM pressure", done, (int)disk.size(), 120);
    stop = true;
    for (auto &t : th) t.join();
    CHECK(engine_clean(e));
    dm_engine_destroy(e);
}

// 16 disk-backed bodies at once over a 32-slab ring: each body's writer, running job and staged slab compete for
// the ring with the other fifteen.  Run with FAKE_CUDA_JITTER_US set, the hash trails the writers.
static void sixteen_bodies_over_32_slabs()
{
    dm_engine *e = make_engine(g_flags, kArena, 32 * 65536, 65536);
    CHECK(e);
    std::vector<const Body *> big;
    for (const Body &b : bodies) if (b.bytes.size() > kArena) big.push_back(&b);
    std::atomic<int> done{0};
    std::vector<std::thread> th;
    for (int t = 0; t < 16; ++t)
        th.emplace_back([&, t] {
            for (int k = 0; k < 2 && !failures.load(); ++k) {
                CHECK(pull(e, *big[(t + k) % big.size()], 32768) == DM_OK);
                done++;
            }
        });
    must_finish(e, "16 bodies over 32 slabs", done, 32, 180);
    for (auto &t : th) t.join();
    CHECK(engine_clean(e));
    dm_engine_destroy(e);
}

int main(int argc, char **argv)
{
    const double seconds = argc > 1 ? atof(argv[1]) : 3.0;
    const int threads = argc > 2 ? atoi(argv[2]) : 6;
    if (argc < 4) { fprintf(stderr, "usage: disk_direct_soak <seconds> <threads> <cas_dir> [no_hbm]\n"); return 2; }
    g_cas = argv[3];
    g_flags = DM_F_DISK_DIRECT | (argc > 4 && atoi(argv[4]) ? DM_F_NO_HBM_CAS : 0u);
    auto env_u64 = [](const char *name, uint64_t dflt) { const char *v = getenv(name); return v && *v ? strtoull(v, nullptr, 0) : dflt; };
    g_slab = env_u64("RIG_SLAB", 64u << 10);
    g_ring = env_u64("RIG_RING", 1u << 20);
    make_bodies();
    {
        dm_config cfg;                                   // the flag needs a disk tier
        memset(&cfg, 0, sizeof cfg);
        cfg.struct_size = sizeof cfg;
        cfg.flags = DM_F_DISK_DIRECT;
        dm_engine *none = nullptr;
        if (dm_engine_create(&cfg, &none) != DM_EINVAL || none) { printf("DM_F_DISK_DIRECT without cas_dir was accepted\nDISK SOAK FAILED\n"); return 1; }
    }
    // a leftover of a process that is gone is removed at create; a live process's file is not
    fs::create_directories(g_cas + "/incoming");
    const std::string dead = g_cas + "/incoming/999999999-0-7.part", live = g_cas + "/incoming/" + std::to_string(getppid()) + "-0-7.part";
    std::ofstream(dead) << "x";
    std::ofstream(live) << "x";
    dm_engine *e = make_engine(g_flags, kArena);
    if (!e) return 1;
    if (fs::exists(dead) || !fs::exists(live)) { printf("incoming/ sweep wrong\nDISK SOAK FAILED\n"); return 1; }
    fs::remove(live);
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
            if (still == 40) {
                dm_stats w;
                dm_engine_stats(e, &w);
                fprintf(stderr, "STUCK for 20 s: open_streams=%llu slabs free/total=%llu/%llu launches=%llu\nDISK SOAK FAILED (stuck)\n",
                        (unsigned long long)w.open_streams, (unsigned long long)w.ring_slabs_free,
                        (unsigned long long)w.ring_slabs_total, (unsigned long long)w.kernel_launches);
                _Exit(3);
            }
        }
    });
    for (auto &t : th) t.join();
    done = true;
    dog.join();
    const bool clean = engine_clean(e);
    dm_stats st;
    dm_engine_stats(e, &st);
    printf("ops=%ld enomem=%ld committed=%ld launches=%llu mismatched=%llu ring_waits=%llu clean=%d failures=%d\n", ops.load(),
           enomem.load(), committed.load(), (unsigned long long)st.kernel_launches, (unsigned long long)st.blobs_mismatched,
           (unsigned long long)st.ring_waits, (int)clean, failures.load());
    dm_engine_destroy(e);
    if (!failures.load()) suspend_and_resume_phase(g_flags);
    if (!failures.load()) write_failure_phase(g_flags);
    if (!failures.load() && !(g_flags & DM_F_NO_HBM_CAS)) disk_body_under_hbm_pressure();
    if (!failures.load()) sixteen_bodies_over_32_slabs();
    long files = 0, bad = 0, incoming = 0;
    for (auto &ent : fs::recursive_directory_iterator(g_cas)) {
        if (!ent.is_regular_file()) continue;
        if (ent.path().parent_path().filename() == "incoming") { ++incoming; fprintf(stderr, "left in incoming/: %s\n", ent.path().c_str()); }
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
    printf("disk tier: %ld blob files, %ld wrong, %ld left in incoming/\n", files, bad, incoming);
    if (failures.load() || !clean || bad || incoming || files == 0) { printf("DISK SOAK FAILED\n"); return 1; }
    printf("DISK SOAK OK\n");
    return 0;
}
