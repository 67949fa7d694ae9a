// C-ABI, part 1: engine lifecycle and the ingest side (streams).  See engine_internal.hpp for the layout of the engine.
#include "engine_internal.hpp"

#include <dirent.h>
#include <functional>
#include <sched.h>
#include <signal.h>

namespace {

// DM_F_NUMA_LOCAL: the CPUs of the NUMA node the GPU hangs off (sysfs), or false when the topology is not
// visible (container without /sys/bus/pci, single-node box reporting -1).
bool numa_cpus_of_device(int device, cpu_set_t *set, int *node_out)
{
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) { (void)cudaGetLastError(); return false; }
    for (char *c = bus; *c; ++c) if (*c >= 'A' && *c <= 'Z') *c = (char)(*c - 'A' + 'a');
    char path[160];
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE *f = fopen(path, "r");
    if (!f) return false;
    int node = -1;
    const int got = fscanf(f, "%d", &node);
    fclose(f);
    if (got != 1 || node < 0) return false;
    snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
    f = fopen(path, "r");
    if (!f) return false;
    char list[4096] = {0};
    const size_t k = fread(list, 1, sizeof list - 1, f);
    fclose(f);
    list[k] = 0;
    cpu_set_t allowed;
    CPU_ZERO(&allowed);
    if (sched_getaffinity(0, sizeof allowed, &allowed) != 0) return false;
    CPU_ZERO(set);
    int n_set = 0;
    for (char *tok = strtok(list, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
        int lo = 0, hi = 0;
        const int m = sscanf(tok, "%d-%d", &lo, &hi);
        if (m < 1) continue;
        if (m == 1) hi = lo;
        for (int c = lo; c <= hi && c < CPU_SETSIZE; ++c)
            if (CPU_ISSET(c, &allowed)) { CPU_SET(c, set); ++n_set; }
    }
    *node_out = node;
    return n_set > 0;
}

}  // namespace

namespace dmi {

// Files of disk-backed streams are named <pid>-<device>-<id>.part: remove those of processes that are gone, and
// leave every live process's alone (other engines may share the directory).
void sweep_incoming(const std::string &dir)
{
    DIR *d = opendir(dir.c_str());
    if (!d) return;
    while (struct dirent *de = readdir(d)) {
        char *end = nullptr;
        const long pid = strtol(de->d_name, &end, 10);
        if (end == de->d_name || *end != '-' || pid <= 0) continue;
        if (kill((pid_t)pid, 0) == 0 || errno == EPERM) continue;        // alive (EPERM: alive, another user's)
        unlink((dir + "/" + de->d_name).c_str());
    }
    closedir(d);
}

}  // namespace dmi

extern "C" {

uint32_t dm_abi_version(void) { return DM_ABI_VERSION; }

const char *dm_last_error(void) { return g_last_error.c_str(); }

// Detail text by id instead of by thread.  cgo: a goroutine may run on a different OS thread by the time it
// asks for the text of a call that failed, so the thread-local dm_last_error() can return another
// connection's message; every failing stream / reader call also files its text under its id (0 for calls
// that have none), where any thread finds it.  e == NULL: the last dm_engine_create failure of the process.
static std::mutex g_create_err_mu;
static std::string g_create_err;
int dm_error_detail(dm_engine *e, uint64_t id, char *buf, size_t cap, size_t *len)
{
    if (!buf && cap) return fail(DM_EINVAL, "null argument");
    std::string t;
    if (!e) { std::lock_guard<std::mutex> g(g_create_err_mu); t = g_create_err; }
    else {
        std::lock_guard<std::mutex> g(e->err_mu);
        auto it = e->err_text.find(id);
        if (it != e->err_text.end()) t = it->second;
    }
    if (len) *len = t.size();
    if (cap) {
        const size_t n = std::min(cap - 1, t.size());
        memcpy(buf, t.data(), n);
        buf[n] = 0;
    }
    return DM_OK;
}
static int note_create_err(int rc)
{
    if (rc != DM_OK) { std::lock_guard<std::mutex> g(g_create_err_mu); g_create_err = g_last_error; }
    return rc;
}

const char *dm_strerror(int err)
{
    switch (err) {
    case DM_OK: return "ok";
    case DM_EINVAL: return "invalid argument";
    case DM_ENOMEM: return "out of HBM arena, pinned ring or stream slots";
    case DM_ENOENT: return "digest not in the content-addressed store";
    case DM_ECUDA: return "CUDA runtime error";
    case DM_ESTATE: return "call not valid in this stream state";
    case DM_EIO: return "disk tier I/O error";
    case DM_ENODEV: return "no usable CUDA device";
    case DM_ERANGE: return "offset beyond blob end";
    case DM_ECORRUPT: return "disk tier copy does not hash to its name";
    default: return "unknown error";
    }
}

int dm_device_count(void)
{
    int n = 0;
    cudaError_t err = cudaGetDeviceCount(&n);
    if (err != cudaSuccess) { fail_cuda(err, "cudaGetDeviceCount"); return DM_ENODEV; }
    return n;
}

uint32_t dm_default_kernel_variant(int which) { return (uint32_t)(which ? dm::kDefaultDeepVariant : dm::kDefaultWideVariant); }

uint32_t dm_streams_per_warp(uint32_t n_resident) { return (uint32_t)dm::streams_per_warp_for(n_resident); }

uint32_t dm_shard_of(const uint8_t digest[32], uint32_t n_shards)
{
    if (!digest || n_shards <= 1) return 0;
    const uint32_t prefix = ((uint32_t)digest[0] << 8) | digest[1];
    return (uint32_t)(((uint64_t)prefix * n_shards) >> 16);
}

void dm_engine_destroy(dm_engine *e)
{
    if (!e) return;
    cudaSetDevice(e->device);
    load_stop_all(e);                             // first: a loader may be waiting for ring slabs the pump gives back
    {
        std::lock_guard<std::mutex> g(e->work_mu);
        e->stop = true;
    }
    e->work_cv.notify_all();
    e->slab_cv.notify_all();
    if (e->pump.joinable()) e->pump.join();
    { std::lock_guard<std::mutex> g(e->done_mu); e->done_stop = true; }       // the pump has reaped everything: drain, then stop
    e->done_cv.notify_all();
    for (auto &t : e->completers) if (t.joinable()) t.join();
    {
        std::lock_guard<std::mutex> g(e->spill_mu);
    }
    e->spill_cv.notify_all();
    for (auto &t : e->spillers) if (t.joinable()) t.join();
    { std::lock_guard<std::mutex> g(e->disk_mu); e->disk_stop = true; }     // after the completers: they queue publications
    e->disk_cv.notify_all();
    for (auto &t : e->disk_threads) if (t.joinable()) t.join();
    for (auto &m : e->streams)                    // disk-backed streams nobody finished: their files go with the engine
        for (auto &kv : m)
            if (kv.second->fd >= 0) {
                close(kv.second->fd);
                if (!kv.second->check_only) unlink(kv.second->path.c_str());     // (a check's file is a blob of the tier)
            }
    cudaDeviceSynchronize();
    for (auto &m : e->readers) for (auto &kv : m) if (kv.second->fd >= 0) close(kv.second->fd);
    for (Cycle &c : e->cycles) {
        for (int i = 0; i < kCopyStreams; ++i) if (c.copy_ev[i]) cudaEventDestroy(c.copy_ev[i]);
        if (c.stream) cudaStreamDestroy(c.stream);
        if (c.k_start) cudaEventDestroy(c.k_start);
        if (c.k_end) cudaEventDestroy(c.k_end);
        if (c.h_jobs) cudaFreeHost(c.h_jobs);
        if (c.d_jobs) cudaFree(c.d_jobs);
    }
    for (SlabBatch &b : e->batches)
        for (int i = 0; i < kCopyStreams; ++i) if (b.ev[i]) cudaEventDestroy(b.ev[i]);
    for (Bounce &b : e->bounce_store) { if (b.host) cudaFreeHost(b.host); if (b.stream) cudaStreamDestroy(b.stream); }
    if (e->ing_states) cudaFree(e->ing_states);
    if (e->ing_digests) cudaFree(e->ing_digests);
    if (e->ing_jobs_d) cudaFree(e->ing_jobs_d);
    if (e->ing_jobs_h) cudaFreeHost(e->ing_jobs_h);
    if (e->ing_digests_h) cudaFreeHost(e->ing_digests_h);
    if (e->alias_log) fclose(e->alias_log);
    if (e->ckpt_stream) cudaStreamDestroy(e->ckpt_stream);
    if (e->ckpt_pinned) cudaFreeHost(e->ckpt_pinned);
    if (e->ing_ev0) cudaEventDestroy(e->ing_ev0);
    if (e->ing_ev1) cudaEventDestroy(e->ing_ev1);
    if (e->ing_ev2) cudaEventDestroy(e->ing_ev2);
    for (int i = 0; i < kIngestMaxChunks; ++i) {
        if (e->ing_cev_k[i]) cudaEventDestroy(e->ing_cev_k[i]);
        if (e->ing_cev_done[i]) cudaEventDestroy(e->ing_cev_done[i]);
        if (e->ing_streams[i]) cudaStreamDestroy(e->ing_streams[i]);
    }
    if (e->pack_dev_base) cudaFree(e->pack_dev_base);
    if (e->d_states) cudaFree(e->d_states);
    if (e->h_digests) cudaFreeHost(e->h_digests);
    if (e->ring) cudaFreeHost(e->ring);
    if (e->dev_ring) cudaFree(e->dev_ring);
    if (e->arena_base) cudaFree(e->arena_base);
    for (int i = 0; i < kCopyStreams; ++i) if (e->copy_stream[i]) cudaStreamDestroy(e->copy_stream[i]);
    if (e->ingest_stream) cudaStreamDestroy(e->ingest_stream);
    if (e->util_stream) cudaStreamDestroy(e->util_stream);
    delete e;
}

static int engine_create(const dm_config *cfg, dm_engine **out);
int dm_engine_create(const dm_config *cfg, dm_engine **out) { return note_create_err(engine_create(cfg, out)); }
static int engine_create(const dm_config *cfg, dm_engine **out)
{
    if (!cfg || !out || cfg->struct_size != sizeof(dm_config)) return fail(DM_EINVAL, "dm_config missing or wrong struct_size");
    *out = nullptr;
    int ndev = 0;
    cudaError_t err = cudaGetDeviceCount(&ndev);
    if (err != cudaSuccess || ndev == 0) {
        fail_cuda(err, "cudaGetDeviceCount");
        return DM_ENODEV;   // no CPU fallback on the hash path
    }
    if (cfg->device < 0 || cfg->device >= ndev) return fail(DM_ENODEV, "device ordinal out of range");
    if (cfg->slab_bytes && (cfg->slab_bytes % 256)) return fail(DM_EINVAL, "slab_bytes must be a multiple of 256");
    if ((cfg->flags & DM_F_DISK_DIRECT) && !(cfg->cas_dir && cfg->cas_dir[0])) return fail(DM_EINVAL, "DM_F_DISK_DIRECT needs a cas_dir");

    dm_engine *e = new dm_engine();
    e->cfg = *cfg;
    e->device = cfg->device;
    if (cfg->cas_dir) e->cas_dir = cfg->cas_dir;
    e->cfg.cas_dir = nullptr;
    if (const char *v = getenv("DM_FORCE_SPW")) {
        const int f = atoi(v);
        if (f == 1 || f == 2 || f == 4 || f == 8 || f == 16 || f == 32) e->force_spw = f;
    }
    if (const char *v = getenv("DM_KERNEL_VARIANT")) {   // "wide,deep" variant numbers; experiments only
        int w = -1, d = -1;
        if (sscanf(v, "%d,%d", &w, &d) >= 1) {
            if (w >= 0 && w < 24) e->variant_wide = w;
            if (d >= 0 && d <= 10) e->variant_deep = d;   // 4..7 = short-chain rounds (deep and group kernels)
        }
    }
    // Streaming stores for the socket -> ring copy from 16 KiB pieces up (io.Copy moves 32 KiB); DM_NT_COPY_MIN=0
    // turns them off, any other value moves the threshold (A/B runs).
    e->nt_copy_min = 16384;
    if (const char *v = getenv("DM_NT_COPY_MIN")) e->nt_copy_min = (uint32_t)strtoul(v, nullptr, 10);
    if (const char *v = getenv("DM_INGEST_CHUNKS")) e->ingest_chunks = (uint32_t)std::min<long>(std::max<long>(atol(v), 0), kIngestMaxChunks);   // tuning / tests only
    if (const char *v = getenv("DM_SPLIT_MIN_BYTES")) e->split_min = strtoull(v, nullptr, 10);       // tuning / tests only
    if (!e->cfg.slab_bytes) e->cfg.slab_bytes = 1u << 20;
    if (!e->cfg.ring_bytes) e->cfg.ring_bytes = 256ull << 20;
    if (!e->cfg.max_streams) e->cfg.max_streams = 65536;
    if (e->cfg.ring_bytes < 4ull * e->cfg.slab_bytes) e->cfg.ring_bytes = 4ull * e->cfg.slab_bytes;

#define CU_INIT(expr)                                                                   \
    do {                                                                                \
        cudaError_t cu_err_ = (expr);                                                   \
        if (cu_err_ != cudaSuccess) { fail_cuda(cu_err_, #expr); dm_engine_destroy(e); return DM_ECUDA; } \
    } while (0)

    CU_INIT(cudaSetDevice(e->device));
    // DM_F_NUMA_LOCAL: everything the engine pins (ring, bounce buffers, job tables) is first touched, and
    // every thread it starts (pump, spill) is created, while this thread is confined to the GPU's NUMA node;
    // the caller's affinity is restored before returning.  At 8 GPUs the ingest path is bound by host
    // memory traffic, and a ring on the wrong socket costs ~40 % (DESIGN.md section 6).
    cpu_set_t saved_aff, node_aff;
    bool rebind = false;
    if ((e->cfg.flags & DM_F_NUMA_LOCAL) && sched_getaffinity(0, sizeof saved_aff, &saved_aff) == 0 &&
        numa_cpus_of_device(e->device, &node_aff, &e->numa_node) && sched_setaffinity(0, sizeof node_aff, &node_aff) == 0)
        rebind = true;
    else e->numa_node = -1;
    struct Restore {
        bool on; cpu_set_t *set;
        ~Restore() { if (on) sched_setaffinity(0, sizeof *set, set); }
    } restore{rebind, &saved_aff};
    cudaDeviceProp prop;
    CU_INIT(cudaGetDeviceProperties(&prop, e->device));
    e->sm_count = prop.multiProcessorCount;
    // sm_90a SASS (no PTX in the fat binary) loads on compute capability 9.0 only
    if (prop.major != 9 || prop.minor != 0) { fail(DM_ENODEV, "kernels are built for sm_90a only"); dm_engine_destroy(e); return DM_ENODEV; }

    for (int i = 0; i < kCopyStreams; ++i) CU_INIT(cudaStreamCreateWithFlags(&e->copy_stream[i], cudaStreamNonBlocking));
    CU_INIT(cudaStreamCreateWithFlags(&e->ingest_stream, cudaStreamNonBlocking));
    CU_INIT(cudaStreamCreateWithFlags(&e->util_stream, cudaStreamNonBlocking));
    CU_INIT(cudaStreamCreateWithFlags(&e->ckpt_stream, cudaStreamNonBlocking));
    CU_INIT(cudaHostAlloc(&e->ckpt_pinned, 64, cudaHostAllocDefault));
    CU_INIT(cudaEventCreate(&e->ing_ev0));
    CU_INIT(cudaEventCreate(&e->ing_ev1));
    CU_INIT(cudaEventCreate(&e->ing_ev2));
    for (int i = 0; i < kIngestMaxChunks; ++i) {
        CU_INIT(cudaStreamCreateWithFlags(&e->ing_streams[i], cudaStreamNonBlocking));
        CU_INIT(cudaEventCreate(&e->ing_cev_k[i]));
        CU_INIT(cudaEventCreateWithFlags(&e->ing_cev_done[i], cudaEventDisableTiming));
    }

    if ((e->cfg.flags & DM_F_NO_HBM_CAS) && !e->cfg.hbm_cas_bytes) e->cfg.hbm_cas_bytes = 1u << 20;   // only dm_ingest_device would use it
    if (!e->cfg.hbm_cas_bytes) {
        size_t fr = 0, tot = 0;
        CU_INIT(cudaMemGetInfo(&fr, &tot));
        e->cfg.hbm_cas_bytes = fr / 2;
    }
    e->cfg.hbm_cas_bytes = round_up(e->cfg.hbm_cas_bytes, kAlign);
    CU_INIT(cudaMalloc(&e->arena_base, e->cfg.hbm_cas_bytes));
    e->arena.reset(e->cfg.hbm_cas_bytes);

    const uint64_t nslab = e->cfg.ring_bytes / e->cfg.slab_bytes;
    CU_INIT(cudaHostAlloc(&e->ring, nslab * e->cfg.slab_bytes, cudaHostAllocDefault));
    e->slab_store.resize(nslab);
    if (e->cfg.flags & DM_F_NO_HBM_CAS) CU_INIT(cudaMalloc(&e->dev_ring, nslab * e->cfg.slab_bytes));
    for (uint64_t i = 0; i < nslab; ++i) {
        e->slab_store[i].host = e->ring + i * e->cfg.slab_bytes;
        e->slab_store[i].dev = e->dev_ring ? e->dev_ring + i * e->cfg.slab_bytes : nullptr;
        e->slab_free.push_back(&e->slab_store[i]);
    }

    if (!(e->cfg.flags & DM_F_NO_HBM_CAS) && e->cfg.slab_bytes >= 1024) {      // staging for tiny-body packs
        e->tiny_max = std::min<uint32_t>(kTinyMax, e->cfg.slab_bytes / 4);
        CU_INIT(cudaMalloc(&e->pack_dev_base, (uint64_t)kPackDevBufs * e->cfg.slab_bytes));
        for (int i = 0; i < kPackDevBufs; ++i) e->pack_dev_free.push_back(e->pack_dev_base + (uint64_t)i * e->cfg.slab_bytes);
    }
    CU_INIT(cudaMalloc(&e->d_states, 32ull * e->cfg.max_streams));
    CU_INIT(cudaHostAlloc(&e->h_digests, 32ull * e->cfg.max_streams, cudaHostAllocMapped));
    CU_INIT(cudaHostGetDevicePointer((void **)&e->d_digests, e->h_digests, 0));
    e->free_slots.reserve(e->cfg.max_streams);
    for (uint32_t i = e->cfg.max_streams; i-- > 0;) e->free_slots.push_back(i);

    e->max_jobs = e->cfg.max_streams;
    for (Cycle &c : e->cycles) {
        for (int i = 0; i < kCopyStreams; ++i) CU_INIT(cudaEventCreateWithFlags(&c.copy_ev[i], cudaEventDisableTiming));
        CU_INIT(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
        CU_INIT(cudaEventCreate(&c.k_start));
        CU_INIT(cudaEventCreate(&c.k_end));
        CU_INIT(cudaHostAlloc(&c.h_jobs, sizeof(dm::HashJob) * (uint64_t)e->max_jobs, cudaHostAllocDefault));
        CU_INIT(cudaMalloc(&c.d_jobs, sizeof(dm::HashJob) * (uint64_t)e->max_jobs));
    }
    for (SlabBatch &b : e->batches)
        for (int i = 0; i < kCopyStreams; ++i) CU_INIT(cudaEventCreateWithFlags(&b.ev[i], cudaEventDisableTiming));
    e->bounce_store.resize(kBounces);
    for (Bounce &b : e->bounce_store) {
        CU_INIT(cudaHostAlloc(&b.host, kBounceBytes, cudaHostAllocDefault));
        CU_INIT(cudaStreamCreateWithFlags(&b.stream, cudaStreamNonBlocking));
        e->bounce_free.push_back(&b);
    }
#undef CU_INIT
    if (!e->cas_dir.empty()) {
        mkdirs(e->cas_dir + "/blobs/sha256/x");
        mkdirs(e->cas_dir + "/partial/x");
        alias_load(e);
        if (DIR *dir = opendir((e->cas_dir + "/partial").c_str())) {      // downloads suspended by an earlier process
            while (struct dirent *de = readdir(dir)) {
                const size_t n = strlen(de->d_name);
                if (n == 69 && strcmp(de->d_name + 64, ".ckpt") == 0) e->n_suspended++;
            }
            closedir(dir);
        }
        if (e->cfg.flags & DM_F_DISK_DIRECT) {
            mkdirs(e->cas_dir + "/incoming/x");
            sweep_incoming(e->cas_dir + "/incoming");
        }
    }
    e->pump = std::thread(pump_main, e);
    if (!e->cas_dir.empty())          // disk-backed streams, and dm_cache_verify on any engine with a disk tier
        for (int i = 0; i < kDiskThreads; ++i) e->disk_threads.emplace_back(disk_main, e);
    for (int i = 0; i < kCompleters; ++i) e->completers.emplace_back(completer_main, e);
    if (!e->cas_dir.empty())
        for (int i = 0; i < kSpillThreads; ++i) e->spillers.emplace_back(spill_main, e);
    *out = e;
    return DM_OK;
}

int dm_engine_stats(dm_engine *e, dm_stats *o)
{
    if (!e || !o) return fail(DM_EINVAL, "null argument");
    memset(o, 0, sizeof *o);
    o->bytes_ingested = e->st_ingested; o->bytes_hashed = e->st_hashed; o->bytes_served = e->st_served;
    o->blobs_committed = e->st_committed; o->blobs_mismatched = e->st_mismatch;
    o->kernel_launches = e->st_launches; o->launches_wide = e->st_wide; o->launches_deep = e->st_deep;
    { std::lock_guard<std::mutex> g(e->stat_mu); o->kernel_ms = e->st_kernel_ms; }
    o->h2d_bytes = e->st_h2d; o->d2h_bytes = e->st_d2h;
    { std::lock_guard<std::mutex> g(e->arena_mu); o->hbm_cas_used = e->arena.used(); o->hbm_cas_capacity = e->arena.capacity(); }
    o->open_streams = e->n_streams;
    o->ring_waits = e->st_ring_waits;
    o->launches_group = e->st_group;
    { std::lock_guard<std::mutex> g(e->slab_mu); o->ring_slabs_total = e->slab_store.size(); o->ring_slabs_free = e->slab_free.size(); }
    for (int k = 0; k < kStripes; ++k) { std::lock_guard<std::mutex> g(e->reader_mu[k]); o->open_readers += e->readers[k].size(); }
    { std::lock_guard<std::mutex> g(e->slot_mu); o->free_stream_slots = e->free_slots.size(); }
    o->numa_node = e->numa_node;
    { std::lock_guard<std::mutex> g(e->alias_mu); o->aliases = e->aliases.size(); }
    o->suspended = e->n_suspended;
    o->packed_bodies = e->st_packed; o->packs = e->st_packs;
    return DM_OK;
}

// ---- ingest ------------------------------------------------------------------

// `followable`: index the stream by its expected digest so that dm_cache_follow can attach to it.  A
// resumed stream is registered by dm_stream_resume itself, and only when it starts at byte 0: a follower
// reads from offset 0, and nothing before resume_base is ever written.
// `saved`: bytes of this body already counted in the disk tier (a saved download being resumed): a disk-backed stream
// makes room only for the rest of its size_hint.
// `internal`: the stream of a load (e->loads already keeps dm_cache_remove off its digest); any other stream with an
// expected digest holds it (e->holds) until it is dropped.
static int stream_open_impl(dm_engine *e, const uint8_t expect[32], uint64_t size_hint, uint64_t *id, bool followable,
                            uint64_t saved = 0, bool internal = false)
{
    if (!e || !id) return fail(DM_EINVAL, "null argument");
    auto sp = std::make_shared<Stream>();
    if (expect) { sp->has_expect = true; memcpy(sp->expect.b, expect, 32); }
    {
        std::lock_guard<std::mutex> g(e->slot_mu);
        if (e->free_slots.empty()) return fail(DM_ENOMEM, "max_streams reached");
        sp->slot = e->free_slots.back();
        e->free_slots.pop_back();
    }
    sp->id = e->next_id.fetch_add(1);
    sp->verify_only = (e->cfg.flags & DM_F_NO_HBM_CAS) != 0;
    if (!sp->verify_only && size_hint > e->cfg.hbm_cas_bytes) {
        // can never be cached here: still verify it, through the device mirror of the ring
        int rc = ensure_dev_ring(e);
        if (rc != DM_OK) {
            std::lock_guard<std::mutex> g2(e->slot_mu);
            e->free_slots.push_back(sp->slot);
            return rc;
        }
        sp->verify_only = true;
    }
    // kept after all: in a file of the disk tier, when the disk-tier limit leaves room for the announced size (a body
    // of unknown size is charged as it grows); otherwise it stays verify-only: verified, not cached
    sp->path = incoming_path(e, sp->id);
    if (sp->verify_only && (e->cfg.flags & DM_F_DISK_DIRECT) && tier_stage(e, sp->path, size_hint, saved)) {
        sp->disk = true;
        sp->fd = open(sp->path.c_str(), O_CREAT | O_TRUNC | O_RDWR | O_CLOEXEC, 0644);
        if (sp->fd < 0) {
            tier_unstage(e, sp->path);
            std::lock_guard<std::mutex> g2(e->slot_mu);
            e->free_slots.push_back(sp->slot);
            return fail(DM_EIO, "could not create the stream's file under <cas_dir>/incoming");
        }
    }
    if (!sp->disk) sp->path.clear();
    if (size_hint && !sp->verify_only) {
        cudaSetDevice(e->device);
        std::lock_guard<std::mutex> g(sp->mu);
        Extent x;
        if (!arena_alloc(e, size_hint, &x)) {
            std::lock_guard<std::mutex> g2(e->slot_mu);
            e->free_slots.push_back(sp->slot);
            return fail(DM_ENOMEM, "HBM CAS arena exhausted");
        }
        sp->extents.push_back(x);
        sp->capacity = x.len;
    }
    sp->size_hint = size_hint;
    if (size_hint && size_hint <= e->tiny_max && !sp->verify_only) {       // announced tiny: no ring slab (see Stream::small)
        sp->small.reset(new uint8_t[size_hint]);
        sp->small_cap = (uint32_t)size_hint;
    }
    if (sp->has_expect && !internal) {
        sp->held = true;
        hold_digest(e, sp->expect, "a stream opened with it as its expected digest");
    }
    {
        const int k = (int)(sp->id % kStripes);
        std::lock_guard<std::mutex> g(e->stripe_mu[k]);
        e->streams[k][sp->id] = sp;
        e->n_streams++;
    }
    // followable: a stream that keeps its bytes, in HBM or in its file (a verify-only stream retains nothing to serve)
    if (followable && sp->has_expect && (!sp->verify_only || sp->disk)) {   // first opener wins; later duplicates are not followable
        std::lock_guard<std::mutex> g(e->mu);
        auto &slot = e->inflight[sp->expect];
        if (slot.expired()) slot = sp;
    }
    *id = sp->id;
    return DM_OK;
}

int dm_stream_open(dm_engine *e, const uint8_t expect[32], uint64_t size_hint, uint64_t *id)
{
    return note_err(e, 0, stream_open_impl(e, expect, size_hint, id, true));
}

static const char *kLostText = "bytes this stream had accepted were dropped by an earlier failure (HBM arena full or a failed copy): abort it";

static int stream_write_impl(dm_engine *e, uint64_t id, const void *buf, size_t len)
{
    if (!e || (!buf && len)) return fail(DM_EINVAL, "null argument");
    auto sp = find_stream(e, id);
    if (!sp) return fail(DM_EINVAL, "unknown stream id");
    Stream *s = sp.get();
    std::unique_lock<std::mutex> g(s->mu);
    if (s->st != St::Open || s->window_out) return fail(DM_ESTATE, "stream not open for write");
    if (s->lost != DM_OK) return fail(s->lost, kLostText);
    const uint8_t *p = static_cast<const uint8_t *>(buf);
    const uint32_t slab_bytes = e->cfg.slab_bytes;
    if (s->small_cap && !s->cur && s->small_fill + len <= s->small_cap) {     // announced-tiny body: private buffer, no slab
        if (len) memcpy(s->small.get() + s->small_fill, p, len);
        s->small_fill += (uint32_t)len; s->received += len;
        return DM_OK;
    }
    while (len) {
        if (s->lost != DM_OK) return fail(s->lost, kLostText);
        if (!s->cur) {
            int rc = take_slab(e, s, g);
            if (rc != DM_OK) return rc;
            continue;                                       // the pump may have marked the stream while we waited
        }
        const size_t n = std::min<size_t>(len, slab_bytes - s->cur_fill);
        if ((!s->islands.empty() || !s->parts.empty()) && range_taken(s, s->dma_issued + s->cur_fill, n, nullptr))
            return fail(DM_EINVAL, "write overlaps a range already received");
        ring_copy(e, s->cur->host + s->cur_fill, p, n);
        s->cur_fill += (uint32_t)n; s->received += n; p += n; len -= n;
        if (s->cur_fill == slab_bytes) {
            int rc = submit_slab(e, sp);
            if (rc != DM_OK) return rc;
        }
    }
    return DM_OK;
}

static int stream_write_at_impl(dm_engine *e, uint64_t id, uint64_t offset, const void *buf, size_t len)
{
    if (!e || (!buf && len)) return fail(DM_EINVAL, "null argument");
    if (offset + len < offset) return fail(DM_ERANGE, "offset + len overflows");
    auto sp = find_stream(e, id);
    if (!sp) return fail(DM_EINVAL, "unknown stream id");
    Stream *s = sp.get();
    std::unique_lock<std::mutex> g(s->mu);
    if (s->st != St::Open || s->window_out) return fail(DM_ESTATE, "stream not open for write");
    if (s->lost != DM_OK) return fail(s->lost, kLostText);
    if (s->small_cap && !s->cur) {                       // range parts need real slabs: move the private buffer's bytes into one
        int rc = take_slab(e, s, g);
        if (rc != DM_OK) return rc;
    }
    if (offset < s->resume_base && offset + len > s->resume_base) {
        // A re-supplied prefix that runs across the resume point: the part below it is kept for caching
        // only (prefix_cover), the part above it is hashed.  Treat them as the two writes they are.
        const uint64_t below = s->resume_base - offset;
        g.unlock();
        int rc = stream_write_at_impl(e, id, offset, buf, (size_t)below);
        if (rc != DM_OK) return rc;
        return stream_write_at_impl(e, id, offset + below, static_cast<const uint8_t *>(buf) + below, len - (size_t)below);
    }
    if (offset == s->dma_issued + s->cur_fill + s->carry_fill && s->parts.empty() && s->islands.empty()) {
        g.unlock();
        return stream_write_impl(e, id, buf, len);          // plain sequential continuation
    }
    if (s->verify_only && !s->disk) return fail(DM_ESTATE, "out-of-order ranges need the HBM store (engine is verify-only)");
    const uint8_t *p = static_cast<const uint8_t *>(buf);
    const uint32_t slab_bytes = e->cfg.slab_bytes;
    while (len) {
        // the part that ends exactly here, or a new one
        size_t idx = s->parts.size();
        for (size_t i = 0; i < s->parts.size(); ++i)
            if (s->parts[i].base + s->parts[i].fill == offset) { idx = i; break; }
        if (idx == s->parts.size()) {
            if (offset == s->dma_issued + s->cur_fill) {
                // continues the contiguous run: use the sequential cursor
                if (!s->cur) {
                    int rc = take_slab(e, s, g);
                    if (rc != DM_OK) return rc;
                    continue;                               // state may have moved while unlocked
                }
                const size_t n = std::min<size_t>(len, slab_bytes - s->cur_fill);
                if (range_taken(s, offset, n, nullptr)) return fail(DM_EINVAL, "write overlaps a range already received");
                ring_copy(e, s->cur->host + s->cur_fill, p, n);
                s->cur_fill += (uint32_t)n; s->received += n; p += n; len -= n; offset += n;
                if (s->cur_fill == slab_bytes) { int rc = submit_slab(e, sp); if (rc != DM_OK) return rc; }
                continue;
            }
            if (s->parts.size() >= 64) return fail(DM_ENOMEM, "too many concurrent range parts on one stream");
            if (range_taken(s, offset, 1, nullptr)) return fail(DM_EINVAL, "write overlaps a range already received");
            g.unlock();
            Slab *fresh = slab_get(e);
            g.lock();
            if (!fresh) return fail(DM_ESTATE, "engine stopping");
            if (s->st != St::Open) { slab_put(e, fresh); return fail(DM_ESTATE, "stream closed while waiting for the ring"); }
            s->parts.push_back({offset, fresh, 0});
            s->range_mode = true;
            continue;                                       // re-find (the vector may have changed while unlocked)
        }
        Stream::Part &pt = s->parts[idx];
        size_t n = std::min<size_t>(len, slab_bytes - pt.fill);
        // a part never straddles the resume point (submit_part files it as prefix cover OR as an island)
        const bool below = pt.base < s->resume_base;
        if (below) n = (size_t)std::min<uint64_t>(n, s->resume_base - offset);
        if (range_taken(s, offset, n, &pt)) return fail(DM_EINVAL, "write overlaps a range already received");
        ring_copy(e, pt.slab->host + pt.fill, p, n);
        pt.fill += (uint32_t)n; s->received += n; p += n; len -= n; offset += n;
        if (pt.fill == slab_bytes || (below && offset == s->resume_base)) { int rc = submit_part(e, sp, idx); if (rc != DM_OK) return rc; }
    }
    return DM_OK;
}

// The SHA-256 chaining value in state slot `slot` after `hashed` bytes (the IV when nothing is hashed).  No job of
// the stream may be running.  Used by dm_stream_checkpoint and by the suspend of a disk-backed stream.
static int read_chain_state(dm_engine *e, uint32_t slot, uint64_t hashed, uint32_t h[8])
{
    if (hashed == 0) {
        static const uint32_t iv[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au,
                                       0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
        memcpy(h, iv, sizeof iv);
        return DM_OK;
    }
    cudaSetDevice(e->device);
    std::lock_guard<std::mutex> gc(e->ckpt_mu);
    CU_TRY(cudaMemcpyAsync(e->ckpt_pinned, e->d_states + 8ull * slot, 32, cudaMemcpyDeviceToHost, e->ckpt_stream));
    CU_TRY(cudaStreamSynchronize(e->ckpt_stream));
    memcpy(h, e->ckpt_pinned, 32);
    return DM_OK;
}

static int stream_checkpoint_impl(dm_engine *e, uint64_t id, dm_checkpoint *out)
{
    if (!e || !out) return fail(DM_EINVAL, "null argument");
    auto sp = find_stream(e, id);
    if (!sp) return fail(DM_EINVAL, "unknown stream id");
    Stream *s = sp.get();
    std::unique_lock<std::mutex> g(s->mu);
    if (s->st != St::Open || s->window_out) return fail(DM_ESTATE, "stream not open");
    if (s->cuda_failed) return fail(DM_ECUDA, "a CUDA copy or launch failed earlier on this stream: its state is not trusted");
    if (s->lost != DM_OK) return fail(s->lost, kLostText);
    if (s->small_fill && !s->cur) {                      // bytes still in the private buffer of an announced-tiny body
        int rc = take_slab(e, s, g);
        if (rc != DM_OK) return rc;
        if (s->st != St::Open) return fail(DM_ESTATE, "stream closed during checkpoint");
    }
    if (!s->verify_only || s->disk || (s->cur_fill & 63) == 0) {
        // push out what is staged so the checkpoint covers every whole block received in order
        // (a verify-only stream hashes slab by slab, so only a block-aligned partial slab may go early)
        int rc = submit_slab(e, sp);
        if (rc != DM_OK) return rc;
    }
    // everything DMA'd so far in whole blocks must be hashed and no job may be running
    s->ckpt_waiter = true;
    s->cv.wait(g, [&] {
        return s->st != St::Open || (s->disk && s->lost != DM_OK) ||      // (a failed file write leaves a hole the hash never passes)
               (s->jobs_inflight == 0 && ((s->dma_issued - s->hash_issued) & ~63ull) == 0);
    });
    s->ckpt_waiter = false;
    if (s->st != St::Open) return fail(DM_ESTATE, "stream closed during checkpoint");
    if (s->cuda_failed) return fail(DM_ECUDA, "a CUDA copy or launch failed on this stream: its state is not trusted");
    if (s->lost != DM_OK) return fail(s->lost, kLostText);
    memset(out, 0, sizeof *out);
    out->abi = DM_ABI_VERSION;
    out->bytes = s->hash_issued;
    return read_chain_state(e, s->slot, s->hash_issued, out->h);
}

static int stream_resume_impl(dm_engine *e, const dm_checkpoint *ck, const uint8_t expect[32], uint64_t size_hint, uint64_t *id,
                              uint64_t saved = 0);
int dm_stream_resume(dm_engine *e, const dm_checkpoint *ck, const uint8_t expect[32], uint64_t size_hint, uint64_t *id)
{
    return note_err(e, 0, stream_resume_impl(e, ck, expect, size_hint, id));
}
static int stream_resume_impl(dm_engine *e, const dm_checkpoint *ck, const uint8_t expect[32], uint64_t size_hint, uint64_t *id,
                              uint64_t saved)
{
    if (!e || !ck || !id) return fail(DM_EINVAL, "null argument");
    if (ck->abi != DM_ABI_VERSION || (ck->bytes & 63)) return fail(DM_EINVAL, "bad checkpoint");
    // Not followable while it is being set up (a follower attaching now would read [0, ck->bytes) out of an
    // extent nothing has been written to), and never when it starts past byte 0: the prefix may not be
    // re-supplied at all, so there is nothing to serve from offset 0.
    int rc = stream_open_impl(e, expect, size_hint, id, false, saved);
    if (rc != DM_OK) return rc;
    auto sp = find_stream(e, *id);
    if (!sp) return fail(DM_ESTATE, "stream closed while resuming");
    Stream *s = sp.get();
    std::unique_lock<std::mutex> g(s->mu);
    s->resume_base = s->dma_issued = s->hash_issued = s->landed = s->staged_to = ck->bytes;
    // (a disk-backed stream taking over a saved file is registered by dm_stream_resume_saved once the file holds [0, C))
    if (ck->bytes == 0 && s->has_expect && (!s->verify_only || (s->disk && saved == 0))) {
        std::lock_guard<std::mutex> g2(e->mu);
        auto &slot = e->inflight[s->expect];
        if (slot.expired()) slot = sp;
    }
    if (ck->bytes) {
        // The state must be IN device memory before this returns: the stream's first job may launch at
        // once on another CUDA stream.  (A plain cudaMemcpy from pageable memory returns when the bytes
        // are staged, not when they have landed — found by tools/soak.py.)
        cudaSetDevice(e->device);
        std::lock_guard<std::mutex> gc(e->ckpt_mu);
        memcpy(e->ckpt_pinned, ck->h, 32);
        cudaError_t err = cudaMemcpyAsync(e->d_states + 8ull * s->slot, e->ckpt_pinned, 32, cudaMemcpyHostToDevice, e->ckpt_stream);
        if (err == cudaSuccess) err = cudaStreamSynchronize(e->ckpt_stream);
        if (err != cudaSuccess) {
            // nothing of this stream is in flight yet: give back its extent, state slot and id
            s->st = St::Aborted;
            if (s->disk) { close(s->fd); s->fd = -1; unlink(s->path.c_str()); tier_unstage(e, s->path); }
            g.unlock();
            free_extents(e, s->extents);
            drop_stream(e, sp, true);
            *id = 0;
            return fail_cuda(err, "cudaMemcpyAsync(checkpoint state)");
        }
    }
    return DM_OK;
}

// ---- checkpoints that survive a restart (SURVEY.md section 8f-3) ------------------------------------
// <cas_dir>/partial/<hex of the expected digest>.ckpt   the record below
// <cas_dir>/partial/<hex>.part                           the first `bytes` bytes of the body
// The .ckpt is renamed into place last, so a record always has its bytes.

namespace {
struct SavedCkpt {
    char magic[8];          // "DMCKPT\0\2"
    uint32_t abi, reserved;
    uint64_t bytes;         // multiple of 64: hashed AND saved
    uint64_t size_hint;     // Content-Length the stream was opened with (0 = unknown)
    uint32_t h[8];          // SHA-256 chaining value after `bytes`
    uint8_t expect[32];
};
const char kCkptMagic[8] = {'D', 'M', 'C', 'K', 'P', 'T', 0, 2};
// A disk-backed stream's record: the hash stopped at ck.bytes, the .part holds the first `saved` bytes (saved >= ck.bytes)
struct SavedDiskCkpt {
    SavedCkpt ck;           // magic "DMCKPT\0\3"
    uint64_t saved;         // multiple of 64
};
const char kDiskCkptMagic[8] = {'D', 'M', 'C', 'K', 'P', 'T', 0, 3};
std::string partial_base(const dm_engine *e, const uint8_t d[32]) { return e->cas_dir + "/partial/" + hex_of(d, 32); }
}  // namespace

static int stream_abort_impl(dm_engine *e, uint64_t id);
static int stream_checkpoint_impl(dm_engine *e, uint64_t id, dm_checkpoint *out);

// dm_stream_suspend of a disk-backed stream: no wait for the hash, no copy.  The state at the hashed position H
// is saved with H and C (the contiguous written prefix, rounded down to 64); the file, cut to C, is renamed.
static int suspend_disk(dm_engine *e, const std::shared_ptr<Stream> &sp, uint64_t *resume_from)
{
    Stream *s = sp.get();
    uint64_t hashed, saved, hint;
    int fd;
    std::string path;
    auto unsuspend = [&](std::unique_lock<std::mutex> &g) { s->suspending = false; disk_feed(e, sp); mark_dirty(e, sp, nullptr); g.unlock(); };
    {
        std::unique_lock<std::mutex> g(s->mu);
        if (s->st != St::Open || s->window_out) return fail(DM_ESTATE, "stream not open");
        int rc = submit_slab(e, sp);                      // what sits in the ring goes to the file first
        while (rc == DM_OK && !s->parts.empty()) rc = submit_part(e, sp, s->parts.size() - 1);
        if (rc != DM_OK) return rc;
        s->suspending = true;
        s->ckpt_waiter = true;
        s->cv.wait(g, [&] { return s->st != St::Open || (s->jobs_inflight == 0 && s->disk_writes == 0 && s->disk_reads == 0); });
        s->ckpt_waiter = false;
        if (s->st != St::Open) return fail(DM_ESTATE, "stream closed during suspend");
        if (s->cuda_failed) { unsuspend(g); return fail(DM_ECUDA, "a CUDA copy or launch failed on this stream: its state is not trusted"); }
        if (s->lost != DM_OK) { unsuspend(g); return fail(s->lost, kLostText); }
        if (!s->staged.empty()) {                         // read back but not hashed: the resumed stream reads them again
            cudaSetDevice(e->device);
            cudaStreamSynchronize(e->copy_stream[s->id % kCopyStreams]);
            for (auto &ps : s->staged) slab_return(e, ps.first);
            s->staged.clear();
        }
        s->staged_to = s->hash_issued;
        hashed = s->hash_issued;
        saved = 0;
        if (!s->written.empty() && s->written.begin()->first == 0) saved = s->written.begin()->second & ~63ull;
        hint = s->size_hint;
        fd = s->fd;
        path = s->path;
    }
    dm_checkpoint ck;
    memset(&ck, 0, sizeof ck);
    ck.bytes = hashed;
    if (int rc = read_chain_state(e, s->slot, hashed, ck.h); rc != DM_OK) {
        std::unique_lock<std::mutex> g(s->mu);
        unsuspend(g);
        return rc;
    }
    const std::string base = partial_base(e, s->expect.b);
    SavedDiskCkpt rec;
    memset(&rec, 0, sizeof rec);
    memcpy(rec.ck.magic, kDiskCkptMagic, 8);
    rec.ck.abi = DM_ABI_VERSION; rec.ck.bytes = hashed; rec.ck.size_hint = hint; rec.saved = saved;
    memcpy(rec.ck.h, ck.h, sizeof rec.ck.h);
    memcpy(rec.ck.expect, s->expect.b, 32);
    struct stat st;
    const bool fresh = stat((base + ".ckpt").c_str(), &st) != 0;
    unlink((base + ".ckpt").c_str());                    // an older record must not pair with the new bytes
    { std::lock_guard<std::mutex> g(s->mu); s->cuts++; }     // followers: what they read past C from now on is not the body's
    s->cv.notify_all();
    bool ok = ftruncate(fd, (off_t)saved) == 0 && rename(path.c_str(), (base + ".part").c_str()) == 0;
    const bool moved = ok;
    FILE *f = ok ? fopen((base + ".ckpt.tmp").c_str(), "wb") : nullptr;
    ok = f && fwrite(&rec, sizeof rec, 1, f) == 1 && fflush(f) == 0;
    if (f) fclose(f);
    ok = ok && rename((base + ".ckpt.tmp").c_str(), (base + ".ckpt").c_str()) == 0;
    if (!ok) {
        unlink((base + ".ckpt.tmp").c_str());
        if (moved) rename((base + ".part").c_str(), path.c_str());     // the stream keeps its file
        if (!fresh && e->n_suspended) e->n_suspended--;               // the older record went with the attempt
        tier_placed(e, s->expect, true, nullptr, false);
        std::unique_lock<std::mutex> g(s->mu);
        unsuspend(g);
        return fail(DM_EIO, "could not save the checkpoint under <cas_dir>/partial (the stream is still open)");
    }
    {
        std::lock_guard<std::mutex> g(s->mu);            // the file is the saved download now, not the stream's
        close(s->fd);
        s->fd = -1;
        s->path.clear();
    }
    tier_unstage(e, path);                               // its bytes moved from incoming/ to partial/
    tier_placed(e, s->expect, true, nullptr, true);
    if (fresh) e->n_suspended++;
    stream_abort_impl(e, s->id);                         // releases the id, the state slot and the staged slabs
    if (resume_from) *resume_from = saved;
    return DM_OK;
}

static int stream_suspend_saving(dm_engine *e, const std::shared_ptr<Stream> &sp, uint64_t *resume_from);
static int stream_suspend_impl(dm_engine *e, uint64_t id, uint64_t *resume_from)
{
    if (!e) return fail(DM_EINVAL, "null argument");
    if (resume_from) *resume_from = 0;
    if (e->cas_dir.empty()) return fail(DM_ESTATE, "dm_stream_suspend needs a disk tier (cas_dir)");
    auto sp = find_stream(e, id);
    if (!sp) return fail(DM_EINVAL, "unknown stream id");
    {
        std::lock_guard<std::mutex> g(sp->mu);
        if (!sp->has_expect) return fail(DM_ESTATE, "only a stream opened with an expected digest can be suspended (the digest names the saved files)");
    }
    tier_pin(e, sp->expect, true);                       // the saved download it writes is not a victim meanwhile
    const int rc = stream_suspend_saving(e, sp, resume_from);
    tier_unpin(e, sp->expect, true);
    return rc;
}

static int stream_suspend_saving(dm_engine *e, const std::shared_ptr<Stream> &sp, uint64_t *resume_from)
{
    Stream *s = sp.get();
    const uint64_t id = s->id;
    bool disk;
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (s->verify_only && !s->disk) return fail(DM_ESTATE, "a verify-only stream retains no bytes to save");
        const bool whole = s->resume_base == 0 ||
                           (s->prefix_cover.size() == 1 && s->prefix_cover.begin()->first == 0 &&
                            s->prefix_cover.begin()->second >= s->resume_base);
        if (!whole) return fail(DM_ESTATE, "the stream was resumed without its prefix: there is nothing whole to save");
        disk = s->disk;
    }
    if (disk) return suspend_disk(e, sp, resume_from);
    dm_checkpoint ck;
    int rc = stream_checkpoint_impl(e, id, &ck);        // every whole block received in order is hashed now
    if (rc != DM_OK) return rc;
    TierRes res;
    if (!tier_reserve(e, ck.bytes + sizeof(SavedCkpt), true, &res))
        return fail(DM_ENOMEM, "no room under the disk-tier limit for the saved download (the stream is still open)");
    std::vector<Extent> ext;
    uint64_t hint;
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (s->st != St::Open) { tier_release(e, res); return fail(DM_ESTATE, "stream closed during suspend"); }
        ext = s->extents;
        hint = s->size_hint;
        s->follow_reads++;                               // pins the extents against abort / completion while they are copied out
    }
    cudaSetDevice(e->device);
    const std::string base = partial_base(e, s->expect.b);
    bool ok = cudaStreamSynchronize(e->copy_stream[s->id % kCopyStreams]) == cudaSuccess;     // the saved bytes have landed
    int fd = ok ? open((base + ".part.tmp").c_str(), O_CREAT | O_TRUNC | O_WRONLY, 0644) : -1;
    ok = ok && fd >= 0 && d2h_to_fd(e, ext, ck.bytes, fd);
    if (fd >= 0) ok = (close(fd) == 0) && ok;
    { std::lock_guard<std::mutex> g(s->mu); s->follow_reads--; }
    s->cv.notify_all();
    bool fresh = false;
    if (ok) {
        SavedCkpt rec;
        memset(&rec, 0, sizeof rec);
        memcpy(rec.magic, kCkptMagic, 8);
        rec.abi = DM_ABI_VERSION; rec.bytes = ck.bytes; rec.size_hint = hint;
        memcpy(rec.h, ck.h, sizeof rec.h);
        memcpy(rec.expect, s->expect.b, 32);
        struct stat st;
        fresh = stat((base + ".ckpt").c_str(), &st) != 0;
        unlink((base + ".ckpt").c_str());                // an older record must not pair with the new bytes
        ok = rename((base + ".part.tmp").c_str(), (base + ".part").c_str()) == 0;
        FILE *f = ok ? fopen((base + ".ckpt.tmp").c_str(), "wb") : nullptr;
        ok = f && fwrite(&rec, sizeof rec, 1, f) == 1 && fflush(f) == 0;
        if (f) fclose(f);
        ok = ok && rename((base + ".ckpt.tmp").c_str(), (base + ".ckpt").c_str()) == 0;
    }
    if (!ok) {
        unlink((base + ".part.tmp").c_str());
        unlink((base + ".ckpt.tmp").c_str());
        struct stat st;
        if (!fresh && stat((base + ".ckpt").c_str(), &st) != 0 && e->n_suspended) e->n_suspended--;    // the older record went with the attempt
        tier_placed(e, s->expect, true, &res, false);    // (what is left of an older record, if anything)
        return fail(DM_EIO, "could not save the checkpoint under <cas_dir>/partial (the stream is still open)");
    }
    tier_placed(e, s->expect, true, &res, true);
    if (fresh) e->n_suspended++;
    stream_abort_impl(e, id);                            // releases the id, the state slot and the extent
    if (resume_from) *resume_from = ck.bytes;
    return DM_OK;
}

static int resume_saved_pinned(dm_engine *e, const uint8_t expect[32], uint64_t size_hint, uint64_t *id, uint64_t *resume_from);
static int stream_resume_saved_impl(dm_engine *e, const uint8_t expect[32], uint64_t size_hint, uint64_t *id, uint64_t *resume_from)
{
    if (!e || !expect || !id) return fail(DM_EINVAL, "null argument");
    if (resume_from) *resume_from = 0;
    if (e->cas_dir.empty()) return DM_ENOENT;
    Digest d;
    memcpy(d.b, expect, 32);
    DigestHold held(e, d, "dm_stream_resume_saved is taking its saved download over");
    tier_pin(e, d, true);                                // the saved download being taken over is not a victim
    const int rc = resume_saved_pinned(e, expect, size_hint, id, resume_from);
    tier_unpin(e, d, true);
    return rc;
}

static int resume_saved_pinned(dm_engine *e, const uint8_t expect[32], uint64_t size_hint, uint64_t *id, uint64_t *resume_from)
{
    Digest dg;
    memcpy(dg.b, expect, 32);
    const std::string base = partial_base(e, expect);
    SavedCkpt rec;
    uint64_t saved;                                      // bytes in the .part: == rec.bytes, or more for a disk-backed stream's record
    {
        FILE *f = fopen((base + ".ckpt").c_str(), "rb");
        if (!f) return DM_ENOENT;
        SavedDiskCkpt any;
        memset(&any, 0, sizeof any);
        const size_t got = fread(&any, 1, sizeof any, f);
        fclose(f);
        rec = any.ck;
        const bool v2 = got == sizeof(SavedCkpt) && memcmp(rec.magic, kCkptMagic, 8) == 0;
        const bool v3 = got == sizeof(SavedDiskCkpt) && memcmp(rec.magic, kDiskCkptMagic, 8) == 0;
        saved = v3 ? any.saved : rec.bytes;
        if (!(v2 || v3) || rec.abi != DM_ABI_VERSION || (rec.bytes & 63) || (saved & 63) || saved < rec.bytes ||
            memcmp(rec.expect, expect, 32) != 0) {
            unlink((base + ".ckpt").c_str()); unlink((base + ".part").c_str());
            if (e->n_suspended) e->n_suspended--;
            tier_forget(e, dg, true);
            return fail(DM_EIO, "saved checkpoint is damaged or from another ABI: discarded");
        }
    }
    dm_checkpoint ck;
    memset(&ck, 0, sizeof ck);
    memcpy(ck.h, rec.h, sizeof ck.h);
    ck.bytes = rec.bytes; ck.abi = DM_ABI_VERSION;
    int rc = stream_resume_impl(e, &ck, expect, size_hint ? size_hint : rec.size_hint, id, saved);
    if (rc != DM_OK) return rc;
    // Re-supply the saved prefix [0, rec.bytes) (cached, not re-hashed) and the saved bytes past it (hashed) through
    // the ordinary range path: ring -> DMA -> extent, or ring -> file.  A blob too large for the arena continues
    // verify-only: it retains nothing, so only the bytes still to be hashed are loaded.  A disk-backed stream
    // resuming a disk-backed record adopts the saved file instead: renamed back, nothing copied.
    bool retains = true, adopted = false;
    if (auto sp = find_stream(e, *id)) {
        std::lock_guard<std::mutex> g(sp->mu);
        Stream *s = sp.get();
        retains = !s->verify_only || s->disk;
        if (s->disk && saved) {
            close(s->fd);
            s->fd = -1;
            bool moved = rename((base + ".part").c_str(), s->path.c_str()) == 0;
            if (moved) s->fd = open(s->path.c_str(), O_RDWR | O_CLOEXEC);
            if (moved && s->fd < 0) {                    // adopted but not openable: give the saved bytes back untouched
                if (rename(s->path.c_str(), (base + ".part").c_str()) != 0) s->path.clear();   // (then never unlinked)
                moved = false;
            }
            // not adopted: a fresh file of the stream's own, the saved bytes are loaded into it below
            if (!moved && !s->path.empty()) s->fd = open(s->path.c_str(), O_CREAT | O_TRUNC | O_RDWR | O_CLOEXEC, 0644);
            if (moved) {
                adopted = true;
                add_interval(s->written, 0, saved);
                if (rec.bytes) add_interval(s->prefix_cover, 0, rec.bytes);
                s->dma_issued = s->landed = s->received = saved;
                disk_feed(e, sp);
                tier_stage_grow(e, s->path, saved);      // its bytes moved from partial/ back to incoming/
            }
        }
    }
    const uint64_t from = retains ? 0 : rec.bytes;
    int fd = saved > from && !adopted ? open((base + ".part").c_str(), O_RDONLY) : -1;
    bool ok = adopted || saved == from || fd >= 0;
    if (ok && !adopted && saved > from) {
        std::vector<uint8_t> buf(1u << 20);
        uint64_t off = from;
        while (ok && off < saved) {
            const size_t want = (size_t)std::min<uint64_t>(buf.size(), saved - off);
            const ssize_t got = pread(fd, buf.data(), want, (off_t)off);
            if (got < 0 && errno == EINTR) continue;
            if (got <= 0) { ok = false; break; }
            rc = stream_write_at_impl(e, *id, off, buf.data(), (size_t)got);
            if (rc != DM_OK) ok = false;
            off += (uint64_t)got;
        }
    }
    if (fd >= 0) close(fd);
    if (!ok) {
        stream_abort_impl(e, *id);
        *id = 0;
        return rc != DM_OK ? rc : fail(DM_EIO, "could not read the saved bytes back from <cas_dir>/partial");
    }
    unlink((base + ".ckpt").c_str());                    // the stream owns the download again
    unlink((base + ".part").c_str());
    if (e->n_suspended) e->n_suspended--;
    tier_forget(e, dg, true);
    if (auto sp = find_stream(e, *id)) {
        // a disk-backed stream's file holds the saved bytes from byte 0 now (adopted, or written back above as they
        // land): followable from byte 0, first opener wins
        bool disk;
        { std::lock_guard<std::mutex> g(sp->mu); disk = sp->disk && sp->fd >= 0 && sp->st == St::Open; }
        if (disk) {
            std::lock_guard<std::mutex> g(e->mu);
            auto &slot = e->inflight[sp->expect];
            if (slot.expired()) slot = sp;
        }
    }
    if (resume_from) *resume_from = saved;
    return DM_OK;
}

static int stream_set_meta_impl(dm_engine *e, uint64_t id, const char *key, const char *value)
{
    if (!e || !key || !value) return fail(DM_EINVAL, "null argument");
    auto sp = find_stream(e, id);
    if (!sp) return fail(DM_EINVAL, "unknown stream id");
    std::lock_guard<std::mutex> g(sp->mu);
    if (sp->st != St::Open) return fail(DM_ESTATE, "stream not open");
    if (sp->meta.size() >= 64) return fail(DM_ENOMEM, "too many metadata entries");
    for (auto &kv : sp->meta) if (kv.first == key) { kv.second = value; return DM_OK; }
    sp->meta.emplace_back(key, value);
    return DM_OK;
}

static int stream_acquire_impl(dm_engine *e, uint64_t id, void **ptr, size_t *cap)
{
    if (!e || !ptr || !cap) return fail(DM_EINVAL, "null argument");
    auto sp = find_stream(e, id);
    if (!sp) return fail(DM_EINVAL, "unknown stream id");
    Stream *s = sp.get();
    std::unique_lock<std::mutex> g(s->mu);
    if (s->st != St::Open || s->window_out) return fail(DM_ESTATE, "stream not open or window outstanding");
    if (!s->cur) {
        int rc = take_slab(e, s, g);
        if (rc != DM_OK) return rc;
    }
    if (s->lost != DM_OK) return fail(s->lost, kLostText);
    *ptr = s->cur->host + s->cur_fill;
    *cap = e->cfg.slab_bytes - s->cur_fill;
    s->window_out = true;
    return DM_OK;
}

static int stream_commit_impl(dm_engine *e, uint64_t id, size_t len)
{
    if (!e) return fail(DM_EINVAL, "null argument");
    auto sp = find_stream(e, id);
    if (!sp) return fail(DM_EINVAL, "unknown stream id");
    Stream *s = sp.get();
    std::lock_guard<std::mutex> g(s->mu);
    if (!s->window_out) return fail(DM_ESTATE, "no window outstanding");
    if (len > e->cfg.slab_bytes - s->cur_fill) return fail(DM_EINVAL, "commit larger than the window");
    s->window_out = false;
    s->cur_fill += (uint32_t)len; s->received += len;
    if (s->cur_fill == e->cfg.slab_bytes) return submit_slab(e, sp);
    return DM_OK;
}

// Flush the partial slab and hand the stream to the pump for its final job.  Stream mutex held.
static int begin_finish(dm_engine *e, const std::shared_ptr<Stream> &sp, std::unique_lock<std::mutex> &g)
{
    Stream *s = sp.get();
    if (s->st == St::Finishing || s->st == St::Done) return DM_OK;
    if (s->st != St::Open || s->window_out) return fail(DM_ESTATE, "stream not open");
    if (s->cuda_failed) return fail(DM_ECUDA, "a CUDA copy or launch failed earlier on this stream (bytes may be missing): abort it");
    if (s->lost != DM_OK) return fail(s->lost, kLostText);
    int rc = DM_OK;
    if (s->carry_fill && !s->cur) {                  // a recalled slab left a sub-block tail: it needs a slab to travel in
        rc = take_slab(e, s, g);
        if (rc != DM_OK) return rc;
        if (s->st == St::Finishing || s->st == St::Done) return DM_OK;      // someone else finished it while we waited
    }
    if (!pack_tiny_body(e, s)) {                       // tiny bodies share one DMA (struct Pack); everything else: its own
        if (s->small_fill && !s->cur) {                  // no pack to be had right now: the private buffer's bytes need a slab
            rc = take_slab(e, s, g);
            if (rc != DM_OK) return rc;
            if (s->st == St::Finishing || s->st == St::Done) return DM_OK;
        }
        rc = submit_slab(e, sp);
        if (rc != DM_OK) return rc;
    }
    while (!s->parts.empty()) {
        rc = submit_part(e, sp, s->parts.size() - 1);
        if (rc != DM_OK) return rc;
    }
    if (!s->islands.empty()) return fail(DM_ESTATE, "blob has holes: ranges missing before the last byte");
    if (s->lost != DM_OK) return fail(s->lost, kLostText);      // the pump may have recalled (and lost) a slab while take_slab waited
    s->st = St::Finishing;
    disk_feed(e, sp);                                  // a disk-backed body's last partial block may be read back now
    mark_dirty(e, sp, nullptr);
    return DM_OK;
}

static int stream_flush_impl(dm_engine *e, uint64_t id)
{
    if (!e) return fail(DM_EINVAL, "null argument");
    auto sp = find_stream(e, id);
    if (!sp) return fail(DM_EINVAL, "unknown stream id");
    std::unique_lock<std::mutex> g(sp->mu);
    return begin_finish(e, sp, g);
}

static int stream_finish_impl(dm_engine *e, uint64_t id, uint8_t digest_out[32], int *matched)
{
    if (!e) return fail(DM_EINVAL, "null argument");
    auto sp = find_stream(e, id);
    if (!sp) return fail(DM_EINVAL, "unknown stream id");
    Stream *s = sp.get();
    std::shared_ptr<Blob> blob;
    bool failed = false;
    int disk_rc = DM_OK;
    {
        std::unique_lock<std::mutex> g(s->mu);
        int rc = begin_finish(e, sp, g);
        if (rc != DM_OK) return rc;
        s->cv.wait(g, [&] { return s->st == St::Done || s->st == St::Aborted; });
        // another thread closed the stream (BodyTee.Close from the client side) while this one waited for the
        // final hash: the abort owns the clean-up (id, state slot, extents); nothing was published
        if (s->st == St::Aborted) return fail(DM_ESTATE, "stream aborted while finishing");
        if (digest_out) memcpy(digest_out, s->digest.b, 32);
        if (matched) *matched = s->matched;
        blob = s->blob;
        failed = s->cuda_failed;
        if (s->disk) disk_rc = s->lost;
    }
    drop_stream(e, sp, true);
    if (failed) return fail(DM_ECUDA, "a CUDA copy or launch failed while this stream was being hashed; nothing was cached");
    if (disk_rc != DM_OK) return fail(disk_rc, "the disk-backed stream's file could not be written or published; nothing was cached");
    if (blob && (e->cfg.flags & DM_F_DISK_SYNC) && !e->cas_dir.empty()) {
        std::unique_lock<std::mutex> g(e->spill_mu);
        e->spill_done_cv.wait(g, [&] { std::lock_guard<std::mutex> g2(e->mu); return blob->spill_done; });
        std::lock_guard<std::mutex> g2(e->mu);
        if (!blob->on_disk) return fail(DM_EIO, "disk tier write failed");
    }
    return DM_OK;
}

static int stream_abort_impl(dm_engine *e, uint64_t id)
{
    if (!e) return fail(DM_EINVAL, "null argument");
    auto sp = find_stream(e, id);
    if (!sp) return fail(DM_EINVAL, "unknown stream id");
    Stream *s = sp.get();
    bool free_now = false;
    {
        std::unique_lock<std::mutex> g(s->mu);
        if (s->st == St::Done || s->st == St::Aborted) return fail(DM_ESTATE, "stream already closed");
        if (s->cur) { slab_put(e, s->cur); s->cur = nullptr; s->cur_fill = 0; }
        s->carry_fill = 0;
        s->small.reset(); s->small_fill = 0; s->small_cap = 0;
        for (Stream::Part &pt : s->parts) slab_put(e, pt.slab);
        s->parts.clear();
        if (s->disk) {
            // writes and read-backs in flight use the file and ring slabs (a read-back of an aborted stream returns
            // its slab itself), and a publication may be renaming the file: let them end first.  Who releases the
            // slot is decided here, where the state changes: the pump's reap sees Aborted as soon as it is set.
            s->st = St::Aborted;
            free_now = s->jobs_inflight == 0;
            s->cv.wait(g, [&] { return s->disk_writes == 0 && s->disk_reads == 0 && !s->publishing; });
            if (s->fd >= 0) { close(s->fd); s->fd = -1; }
            if (!s->path.empty() && !s->check_only) { unlink(s->path.c_str()); tier_unstage(e, s->path); }
        }
        if (!s->staged.empty()) {            // their DMAs may be in flight: drain before the ring reuses them
            cudaSetDevice(e->device);
            cudaStreamSynchronize(e->copy_stream[s->id % kCopyStreams]);
            for (auto &ps : s->staged) slab_return(e, ps.first);
            s->staged.clear();
        }
        if (!s->disk) {
            s->st = St::Aborted;
            free_now = s->jobs_inflight == 0;
        }
        if (free_now) pack_release_member(e, s);         // (a job already built keeps the pack until it is reaped)
    }
    if (free_now) {
        // A slab DMA into this extent may still be in flight; the range must not be handed to
        // another blob before it lands (the stale copy would overwrite the new owner's bytes).
        cudaSetDevice(e->device);
        cudaStreamSynchronize(e->copy_stream[s->id % kCopyStreams]);
        { std::unique_lock<std::mutex> g(s->mu); wait_follow_reads(s, g); }
        free_extents(e, s->extents);
    }
    drop_stream(e, sp, free_now);   // otherwise the pump releases slot + extents at reap (after the kernel,
                                    // which itself waited for every DMA enqueued before its launch)
    s->cv.notify_all();
    return DM_OK;
}

// ---- loads: disk tier -> HBM (dm_cache_promote, dm_cache_open_verified) -----------------
// Each blob is an internal stream opened with expect = its digest and size_hint = its file size: the file is pread
// into acquired ring windows, flushed, and the next file starts while the pump hashes it.  The blob is registered as
// disk-only first, so publish() re-homes it into HBM without queueing a spill: the verified file keeps its inode.
// A running load is in e->loads under its digest (struct Load): a second promotion or verified open of the digest waits
// for it or reads along instead of loading the file again.

namespace {

constexpr int kLoadThreads = 4;           // the engine's loader threads (dm_cache_open_verified)
const char *kCorruptText = "the disk tier file does not hash to its digest: file and sidecar removed";

// The stream slots of the tier calls (dm_cache_promote, verify, import and export, verified opens, ring loads), slot_mu
// held: take up to `want` of the free slots that no other such call has reserved, at most half of them, so none with
// one or none left, which stays dm_stream_open's.  Returns how many were taken; slots_release gives them back.
size_t slots_reserve(dm_engine *e, size_t want)
{
    const size_t free = e->free_slots.size();
    const size_t n = std::min(want, free > e->slots_reserved ? (free - e->slots_reserved) / 2 : 0);
    e->slots_reserved += n;
    return n;
}

void slots_release(dm_engine *e, size_t n)
{
    e->slots_reserved -= n;
}

// pread exactly n bytes at offset 0: false on a read error, or when the file ends first.
bool pread_full(int fd, uint8_t *buf, uint64_t n)
{
    for (uint64_t off = 0; off < n;) {
        const ssize_t got = pread(fd, buf + off, n - off, (off_t)off);
        if (got < 0 && errno == EINTR) continue;
        if (got <= 0) return false;
        off += (uint64_t)got;
    }
    return true;
}

// The sidecar's top-level "size" (it precedes "headers", so the first match is it).  The number must be followed by
// ',' or '}': a sidecar read while write_sidecar is still writing it may end in the middle of the number.
bool sidecar_size(const std::string &j, uint64_t *size)
{
    const size_t p = j.find("\"size\":");
    if (p == std::string::npos) return false;
    const char *s = j.c_str() + p + 7;
    char *end = nullptr;
    *size = strtoull(s, &end, 10);
    return end != s && (*end == ',' || *end == '}');
}

// The disk copy under the index entry of `d` is bad or unchecked: forget an entry that is not in HBM, and spill
// one that a stream has re-homed into HBM meanwhile again, from its verified HBM copy.  `only`: touch the entry only
// if it is this object.
void forget_disk_copy(dm_engine *e, const Digest &d, const Blob *only)
{
    std::shared_ptr<Blob> respill;
    {
        std::lock_guard<std::mutex> g(e->mu);
        auto it = e->blobs.find(d);
        if (it == e->blobs.end() || (only && it->second.get() != only)) return;
        if (!it->second->in_hbm) e->blobs.erase(it);
        else if (it->second->on_disk) {
            respill = it->second;
            respill->on_disk = respill->spill_done = false;
        }
    }
    if (respill) {
        { std::lock_guard<std::mutex> g(e->spill_mu); e->spill_q.push_back(respill); }
        e->spill_cv.notify_all();
    }
}

// The disk copy that was read (`seen`) does not hash to its name.  Remove it and its sidecar only while the path still
// names that file: one a spill or a disk-backed stream renamed into place meanwhile is verified and stays.
void drop_corrupt(dm_engine *e, const Digest &d, const struct stat &seen)
{
    const std::string path = blob_path(e, d.b);
    struct stat now;
    const bool exists = stat(path.c_str(), &now) == 0;
    const bool same = exists && now.st_dev == seen.st_dev && now.st_ino == seen.st_ino;
    if (same) { unlink(path.c_str()); unlink((path + ".meta").c_str()); }
    if (!exists || same) { tier_forget(e, d); forget_disk_copy(e, d, nullptr); }
}

// The load ended without a verdict on the file (no slot or room, a failed read, copy or launch): take back the
// entry it registered, which carries the file's unverified size.
void load_undo(dm_engine *e, Load &L)
{
    if (L.mine) forget_disk_copy(e, L.d, L.mine.get());
}

// Open the disk copy of `d` for a check: *fd open O_RDONLY, `seen` its fstat, `side` its sidecar text ("" if none).
// DM_ENOENT without a file (or a cas_dir), DM_EIO when it cannot be opened, DM_ECORRUPT (file and sidecar dropped
// unless `keep`) when its size is not the one its sidecar states.
int open_disk_copy(dm_engine *e, const Digest &d, int *fd, struct stat *seen, std::string *side, bool keep = false)
{
    *fd = -1;
    if (e->cas_dir.empty()) return DM_ENOENT;
    const std::string path = blob_path(e, d.b);
    const int f = open(path.c_str(), O_RDONLY | O_CLOEXEC);
    if (f < 0) return errno == ENOENT ? DM_ENOENT : fail(DM_EIO, "could not open the disk tier file");
    if (fstat(f, seen) != 0) { close(f); return fail(DM_EIO, "could not stat the disk tier file"); }
    side->clear();
    if (FILE *mf = fopen((path + ".meta").c_str(), "r")) {
        char tmp[4096];
        size_t k;
        while ((k = fread(tmp, 1, sizeof tmp, mf)) > 0) side->append(tmp, k);
        fclose(mf);
    }
    uint64_t claimed;
    if (!side->empty() && sidecar_size(*side, &claimed) && claimed != (uint64_t)seen->st_size) {
        close(f);
        if (!keep) drop_corrupt(e, d, *seen);
        return fail(DM_ECORRUPT, "disk tier file is not the size its sidecar says");
    }
    *fd = f;
    return DM_OK;
}

// Every outcome of a claimed load ends here: it leaves the index, and whoever waits for it (readers, promotions) wakes.
void load_end(dm_engine *e, Load &L, int status, const char *why)
{
    {
        std::lock_guard<std::mutex> g(e->mu);
        auto it = e->loads.find(L.d);
        if (it != e->loads.end() && it->second.get() == &L) e->loads.erase(it);
    }
    {
        std::lock_guard<std::mutex> g(L.mu);
        L.done = true;
        L.status = status;
        if (status != DM_OK) L.why = why;
    }
    L.cv.notify_all();
}

int load_wait(Load &L)
{
    std::unique_lock<std::mutex> g(L.mu);
    L.cv.wait(g, [&] { return L.done; });
    return L.status;
}

// Open the stream of a claimed load on the calling thread: the file and its sidecar, the size checks, the stream (its
// HBM extent reserved, evicting LRU blobs) and the disk-only index entry.  Returns 1 with the stream open and L.fd left
// open for load_fill, or the load's final status (L.fd closed): DM_OK when a stream published the blob meanwhile.
// `may_open`: false when the call has no stream slot to spare.
int load_open(dm_engine *e, Load &L, bool may_open)
{
    std::string side;
    if (int rc = open_disk_copy(e, L.d, &L.fd, &L.seen, &side); rc != DM_OK) return rc;
    const uint64_t size = (uint64_t)L.seen.st_size;
    auto shut = [&] { close(L.fd); L.fd = -1; };
    // checked here: a stream with this size_hint would silently become verify-only or disk-backed
    if (size > e->cfg.hbm_cas_bytes) { shut(); return fail(DM_ENOMEM, "blob is larger than the HBM arena"); }
    if (!may_open) { shut(); return fail(DM_ENOMEM, "no stream slot to spare for a load of a disk tier blob"); }
    uint64_t id = 0;
    int rc = stream_open_impl(e, L.d.b, size, &id, false, 0, true);
    if (rc != DM_OK) { shut(); return rc; }
    bool in_hbm = false;                                 // a stream published it meanwhile
    {
        // registered before the verdict (publish() then re-homes it without a spill); taken back on every outcome
        // that does not verify the file
        std::lock_guard<std::mutex> g(e->mu);
        auto it = e->blobs.find(L.d);
        if (it != e->blobs.end() && it->second->in_hbm) in_hbm = true;
        else if (it == e->blobs.end()) {
            L.mine = std::make_shared<Blob>();
            L.mine->digest = L.d; L.mine->size = size;
            L.mine->on_disk = L.mine->spill_done = true;
            L.mine->sidecar = side;
            e->blobs[L.d] = L.mine;
        }
    }
    if (in_hbm) { shut(); stream_abort_impl(e, id); return DM_OK; }
    std::shared_ptr<Stream> sp = find_stream(e, id);
    { std::lock_guard<std::mutex> g(sp->mu); sp->load = true; }
    L.stream = id;
    L.tiny = size <= e->tiny_max;
    {
        std::lock_guard<std::mutex> g(L.mu);
        L.sp = sp;
        L.size = size;
        L.side.swap(side);
        L.opened = true;
    }
    L.cv.notify_all();
    return 1;
}

// Read the file of an opened load into its stream and close it: a tiny one into the stream's private buffer (flushed
// here when `flush_tiny`, else by the caller), anything else through acquired ring windows, flushed.  DM_OK, or the
// load's final status (its stream aborted, the entry it registered taken back).
int load_fill(dm_engine *e, Load &L, uint8_t *tiny_buf, bool flush_tiny)
{
    const uint64_t size = L.size;
    const uint64_t id = L.stream;
    int rc = DM_OK;
    if (L.tiny && size)
        rc = pread_full(L.fd, tiny_buf, size) ? stream_write_impl(e, id, tiny_buf, size)
                                              : fail(DM_EIO, "could not read the disk tier file");
    for (uint64_t off = 0; !L.tiny && rc == DM_OK && off < size;) {
        if (e->load_stop) { rc = fail(DM_ESTATE, "the engine is being destroyed"); break; }
        void *win = nullptr;
        size_t cap = 0;
        rc = stream_acquire_impl(e, id, &win, &cap);
        if (rc != DM_OK) break;
        const size_t want = (size_t)std::min<uint64_t>(cap, size - off);
        ssize_t got;
        do got = pread(L.fd, win, want, (off_t)off); while (got < 0 && errno == EINTR);
        if (got <= 0) {                                  // a read error, or the file shrank while it was read
            stream_commit_impl(e, id, 0);
            rc = fail(DM_EIO, "could not read the disk tier file");
            break;
        }
        rc = stream_commit_impl(e, id, (size_t)got);
        off += (uint64_t)got;
    }
    close(L.fd);
    L.fd = -1;
    if (rc == DM_OK && (!L.tiny || flush_tiny)) rc = stream_flush_impl(e, id);
    if (rc != DM_OK) { stream_abort_impl(e, id); load_undo(e, L); }
    return rc;
}

// Collect the digest of a flushed stream that checks a file (waits for it): DM_OK with got[] what the file hashed to,
// or the error of a failed read, copy or launch (the stream is aborted then).
int check_finish(dm_engine *e, uint64_t stream, uint8_t got[32], int *matched)
{
    const int rc = stream_finish_impl(e, stream, got, matched);
    if (rc != DM_OK) stream_abort_impl(e, stream);       // (an id finish released just says so)
    return rc;
}

// The verdict on the tier file `seen` of `d`, checked by a flushed stream (a load's, or dm_cache_verify's): DM_OK when
// it hashed to `d` (a load's blob is in HBM then), DM_ECORRUPT with the file dropped, or the error of check_finish with
// the file left untouched and the entry `load` registered taken back.
int tier_verdict(dm_engine *e, uint64_t stream, const Digest &d, const struct stat &seen, Load *load = nullptr)
{
    uint8_t got[32];
    int matched = 0;
    const int rc = check_finish(e, stream, got, &matched);
    if (rc != DM_OK) {
        if (load) load_undo(e, *load);
        return rc;
    }
    if (matched) return DM_OK;
    drop_corrupt(e, d, seen);
    return DM_ECORRUPT;
}

// The end of a load dm_cache_open_verified began: its stream slot and disk-tier pin go, a verified blob counts as
// used, and the load ends.
void load_release(dm_engine *e, Load &L, int status)
{
    const std::string why = status == DM_ECORRUPT ? kCorruptText : g_last_error;
    if (L.reserved) { std::lock_guard<std::mutex> g(e->slot_mu); slots_release(e, 1); L.reserved = false; }
    if (status == DM_OK) tier_touch(e, L.d);
    tier_unpin(e, L.d);
    load_end(e, L, status, why.c_str());
}

// A loader thread: reads opened loads' files into their streams, and collects the verdicts of loads whose streams
// have completed.  Verdicts go first: they are quick, and readers wait for them.  One thread scans load_wait at a time:
// a load it has taken out of the list is invisible to the others, so a kick that arrives meanwhile stays set for the
// scanner's next round rather than being spent on a scan that cannot see that load.
void load_main(dm_engine *e)
{
    cudaSetDevice(e->device);
    std::vector<uint8_t> tiny_buf(e->tiny_max);
    std::unique_lock<std::mutex> g(e->load_mu);
    for (;;) {
        e->load_cv.wait(g, [&] { return e->load_stop || (e->load_kick && !e->load_scanning) || !e->load_q.empty(); });
        if (e->load_stop) return;
        if (e->load_kick && !e->load_scanning) {
            e->load_kick = false;
            e->load_scanning = true;
            std::vector<std::shared_ptr<Load>> wait, rest;
            wait.swap(e->load_wait);
            g.unlock();
            for (auto &L : wait) {
                bool over;
                { std::lock_guard<std::mutex> gs(L->sp->mu); over = L->sp->st == St::Done || L->sp->st == St::Aborted; }
                if (over) load_release(e, *L, tier_verdict(e, L->stream, L->d, L->seen, L.get()));
                else rest.push_back(std::move(L));
            }
            g.lock();
            e->load_wait.insert(e->load_wait.end(), rest.begin(), rest.end());
            e->load_scanning = false;
            continue;
        }
        std::shared_ptr<Load> L = std::move(e->load_q.front());
        e->load_q.pop_front();
        g.unlock();
        const int rc = load_fill(e, *L, tiny_buf.data(), true);
        if (rc != DM_OK) load_release(e, *L, rc);
        g.lock();
        if (rc == DM_OK) {
            e->load_wait.push_back(std::move(L));
            e->load_kick = true;                         // its stream may have completed already
        }
    }
}

}  // namespace

}  // extern "C"

namespace dmi {

int load_claim(dm_engine *e, const Digest &d, std::shared_ptr<Load> *L)
{
    auto it = e->blobs.find(d);
    if (it != e->blobs.end() && it->second->in_hbm) return DM_OK;
    std::shared_ptr<Load> &slot = e->loads[d];
    if (slot) { *L = slot; return 2; }
    slot = std::make_shared<Load>();
    slot->d = d;
    *L = slot;
    return 1;
}

int load_begin(dm_engine *e, const std::shared_ptr<Load> &L)
{
    { std::lock_guard<std::mutex> g(e->slot_mu); L->reserved = slots_reserve(e, 1) == 1; }
    tier_pin(e, L->d);                                   // not a disk-tier victim until its verdict
    const int rc = load_open(e, *L, L->reserved);
    if (rc != 1) { load_release(e, *L, rc); return rc; }
    {
        std::lock_guard<std::mutex> g(e->load_mu);
        if (e->loaders.empty())
            for (int i = 0; i < kLoadThreads; ++i) e->loaders.emplace_back(load_main, e);
        e->load_q.push_back(L);
    }
    e->load_cv.notify_all();
    return 1;
}

void load_wake(dm_engine *e)
{
    { std::lock_guard<std::mutex> g(e->load_mu); e->load_kick = true; }
    e->load_cv.notify_all();
}

void load_stop_all(dm_engine *e)
{
    std::vector<std::thread> th;
    {
        std::lock_guard<std::mutex> g(e->load_mu);
        e->load_stop = true;
        th.swap(e->loaders);
    }
    e->load_cv.notify_all();
    for (auto &t : th) t.join();
    // loads nobody will read in or collect: their files close, and whoever waits for them wakes (their streams go with
    // the engine)
    std::vector<std::shared_ptr<Load>> left(e->load_q.begin(), e->load_q.end());
    left.insert(left.end(), e->load_wait.begin(), e->load_wait.end());
    e->load_q.clear();
    e->load_wait.clear();
    for (auto &L : left) {
        if (L->fd >= 0) { close(L->fd); L->fd = -1; }
        load_end(e, *L, DM_ESTATE, "the engine was destroyed before the load's verdict");
    }
}

}  // namespace dmi

extern "C" {

// ---- batch calls (dm_cache_promote, dm_cache_verify, dm_cache_import, dm_cache_export) ---------------------------

namespace {

constexpr int kBatchThreads = 4;          // threads of a batch call: reads of different files overlap
// Tiny items are flushed this many at a time.  Their hash takes less time than reading the next file, so one by one
// each would be a launch of its own; together they share a pack DMA and a launch.
constexpr size_t kTinyBatch = 256;

// An item of a batch call: a blob to promote or verify, or a file to import or export, and the stream that checks it.
struct Check {
    Digest d;                             // the expected digest (when `known`)
    bool known = true;
    int32_t status = DM_ENOENT;
    uint64_t stream = 0;                  // open: the verdict is still to be collected
    bool tiny = false;                    // in its stream's private buffer until flushed, then in a pack
    bool disk = false;                    // disk-backed: read back through ring slabs by the disk threads
    struct stat seen{};                   // the file that was read (st_dev / st_ino), of a check of a file
};

// One entry per distinct key among the n inputs of a batch call, in order of first appearance: key(i, &k) sets the key
// of input i or returns the error that fails the call, and add(i) appends the entry of the first input with its key.
// DM_OK with (*slot_of)[i] the index of input i's entry, or key's error.
int dedup(uint32_t n, std::vector<uint32_t> *slot_of, const std::function<int(uint32_t, std::string *)> &key,
          const std::function<void(uint32_t)> &add)
{
    std::unordered_map<std::string, uint32_t> first;
    slot_of->resize(n);
    for (uint32_t i = 0; i < n; ++i) {
        std::string k;
        if (const int rc = key(i, &k)) return rc;
        auto ins = first.emplace(std::move(k), (uint32_t)first.size());
        if (ins.second) add(i);
        (*slot_of)[i] = ins.first->second;
    }
    return DM_OK;
}

// Collects verdicts of a batch thread's open items, oldest first, until it may open one more (`disk`: disk-backed).
using MakeRoom = std::function<void(bool disk)>;

// The loop of a batch call: up to kBatchThreads threads take the items in turn and open each.  A thread keeps at most
// budget / threads items open (the call's stream slots), at most disk_share / threads of them disk-backed, flushes tiny
// ones kTinyBatch at a time and collects verdicts oldest first.
//   open(c, room, tiny_buf): 1 with c.stream open (c.tiny and c.disk set), or c's final status.  It calls room before
//     it takes a stream slot.  tiny_buf is tiny_max bytes of the thread's own.
//   settle(c): c's final status, once c's stream is flushed.
void run_batch(dm_engine *e, std::vector<Check> &work, size_t budget, size_t disk_share,
               const std::function<int(Check &, const MakeRoom &, uint8_t *)> &open,
               const std::function<int(Check &)> &settle)
{
    const size_t nthreads = std::min<size_t>({(size_t)kBatchThreads, work.size(), std::max<size_t>(budget, 1), disk_share});
    const size_t per_thread = std::max<size_t>(1, budget / std::max<size_t>(nthreads, 1));
    const size_t disk_per_thread = std::max<size_t>(1, disk_share / std::max<size_t>(nthreads, 1));
    std::atomic<size_t> next{0};
    auto worker = [&] {
        cudaSetDevice(e->device);
        std::vector<uint8_t> tiny_buf(e->tiny_max);
        std::deque<Check *> opened;                      // verdict not collected yet (oldest first)
        std::vector<Check *> unflushed;                  // tiny ones among them, flushed together
        size_t open_disk = 0;
        // a flush that fails leaves the stream open: its finish fails the same way and the verdict aborts it
        auto flush = [&] { for (Check *c : unflushed) stream_flush_impl(e, c->stream); unflushed.clear(); };
        auto collect = [&] {
            flush();
            Check *c = opened.front();
            opened.pop_front();
            if (c->disk) --open_disk;
            c->status = settle(*c);
        };
        const MakeRoom room = [&](bool disk) {
            while (!opened.empty() && (opened.size() >= per_thread || (disk && open_disk >= disk_per_thread))) collect();
        };
        for (size_t k; (k = next.fetch_add(1)) < work.size();) {
            Check &c = work[k];
            const int rc = open(c, room, tiny_buf.data());
            if (rc != 1) { c.status = rc; continue; }
            opened.push_back(&c);
            if (c.tiny) unflushed.push_back(&c);
            if (c.disk) ++open_disk;
            if (unflushed.size() >= kTinyBatch) flush();
        }
        flush();
        while (!opened.empty()) collect();
    };
    std::vector<std::thread> th;
    for (size_t t = 1; t < nthreads; ++t) th.emplace_back(worker);
    if (nthreads) worker();
    for (auto &t : th) t.join();
}

}  // namespace

static int cache_promote_impl(dm_engine *e, const uint8_t *digests, uint32_t n, int32_t *status_out)
{
    if (!e || (n && (!digests || !status_out))) return fail(DM_EINVAL, "null argument");
    if (e->cfg.flags & DM_F_NO_HBM_CAS) return fail(DM_ESTATE, "the engine has no HBM tier (DM_F_NO_HBM_CAS)");
    std::vector<Check> work;
    std::vector<uint32_t> slot_of;
    dedup(n, &slot_of, [&](uint32_t i, std::string *k) { k->assign((const char *)digests + 32ull * i, 32); return DM_OK; },
          [&](uint32_t i) { work.emplace_back(); memcpy(work.back().d.b, digests + 32ull * i, 32); });
    std::vector<std::shared_ptr<Load>> loads(work.size());   // the load each promotion runs, or the running one it waits for
    size_t budget;
    { std::lock_guard<std::mutex> g(e->slot_mu); budget = slots_reserve(e, SIZE_MAX); }
    for (Check &p : work) hold_digest(e, p.d, "a running dm_cache_promote");
    for (Check &p : work) tier_pin(e, p.d);            // held by this call: not disk-tier victims until it returns
    // A load reads its file into its stream on the calling thread: none is disk-backed, and the ring share is no bound.
    run_batch(e, work, budget, SIZE_MAX,
              [&](Check &p, const MakeRoom &room, uint8_t *tiny_buf) -> int {
                  room(false);
                  std::shared_ptr<Load> &L = loads[&p - work.data()];
                  int rc;
                  { std::lock_guard<std::mutex> g(e->mu); rc = load_claim(e, p.d, &L); }
                  if (rc != 1) return rc;                // DM_OK: in HBM; 2: another load's, collected below
                  rc = load_open(e, *L, budget > 0);
                  if (rc == 1 && (rc = load_fill(e, *L, tiny_buf, false)) == DM_OK) {
                      p.stream = L->stream;
                      p.tiny = L->tiny;
                      return 1;
                  }
                  load_end(e, *L, rc, g_last_error.c_str());
                  return rc;
              },
              [&](Check &p) -> int {
                  Load &L = *loads[&p - work.data()];
                  const int st = tier_verdict(e, L.stream, L.d, L.seen, &L);
                  load_end(e, L, st, st == DM_ECORRUPT ? kCorruptText : g_last_error.c_str());
                  return st;
              });
    { std::lock_guard<std::mutex> g(e->slot_mu); slots_release(e, budget); }
    for (size_t k = 0; k < work.size(); ++k)           // a load that was already running reports its own verdict
        if (work[k].status == 2) work[k].status = load_wait(*loads[k]);
    for (Check &p : work) {
        if (p.status == DM_OK) tier_touch(e, p.d);
        tier_unpin(e, p.d);
        release_digest(e, p.d);
    }
    for (uint32_t i = 0; i < n; ++i) status_out[i] = work[slot_of[i]].status;
    return DM_OK;
}

// ---- checks of files already written (dm_cache_verify, dm_cache_import, dm_cache_export) ------------------------
// A stored file is a disk-backed stream whose every byte is already written.  Each check is an internal stream opened
// with expect = the digest (when it is known): its fd is the file, [0, size) counts as written, and it is finished at
// once, so the disk threads read the file back into ring slabs (at most two per check on the hash side) and the pump
// hashes them as verify-only jobs.  Files of at most tiny_max bytes are read here instead and travel in packs as
// hash-only members, many to a launch.  No check holds an arena extent, and a verdict is all a check produces.

namespace {

bool blob_in_hbm(dm_engine *e, const Digest &d)
{
    std::lock_guard<std::mutex> g(e->mu);
    auto it = e->blobs.find(d);
    return it != e->blobs.end() && it->second->in_hbm;
}

// Open the check of the file `fd` at `path` (c.seen is its fstat).  The stream takes over fd, or it is closed here.
// Returns 1 with c.stream open (a disk-backed check already finishing, a tiny one waiting for its flush) or c's final
// status.  `ring`: the check is a ring load (dm_cache_open_verified_ring), always read back through ring slabs, never
// packed; it takes over the caller's hold on c.d (released when it is dropped), and *out is its stream.
int check_open(dm_engine *e, Check &c, int fd, const std::string &path, std::unique_ptr<RingLoad> ring = nullptr,
               std::shared_ptr<Stream> *out = nullptr)
{
    const uint64_t size = (uint64_t)c.seen.st_size;
    auto sp = std::make_shared<Stream>();
    sp->has_expect = c.known;
    if (c.known) sp->expect = c.d;
    sp->check_only = sp->verify_only = true;
    sp->size_hint = size;
    c.tiny = !ring && e->tiny_max && size <= e->tiny_max;
    if (c.tiny) {
        sp->small.reset(new uint8_t[std::max<uint64_t>(size, 1)]);
        sp->small_cap = (uint32_t)size;
        const bool read = pread_full(fd, sp->small.get(), size);    // (false also when the file shrank since fstat)
        close(fd);
        if (!read) return fail(DM_EIO, "could not read the disk tier file");
        sp->small_fill = (uint32_t)size;
        sp->received = size;
    } else {
        c.disk = true;
        sp->disk = true;
        sp->fd = fd;
        sp->path = path;
        if (size) add_interval(sp->written, 0, size);
        sp->dma_issued = sp->landed = sp->received = size;
    }
    {
        std::lock_guard<std::mutex> g(e->slot_mu);
        if (e->free_slots.empty()) {
            if (sp->fd >= 0) close(sp->fd);
            return fail(DM_ENOMEM, "max_streams reached");
        }
        sp->slot = e->free_slots.back();
        e->free_slots.pop_back();
    }
    sp->id = e->next_id.fetch_add(1);
    if (ring) { sp->ring = std::move(ring); sp->held = true; }
    {
        const int k = (int)(sp->id % kStripes);
        std::lock_guard<std::mutex> g(e->stripe_mu[k]);
        e->streams[k][sp->id] = sp;
        e->n_streams++;
    }
    if (out) *out = sp;
    if (!c.tiny) {                                       // flushed straight away: every byte is already in the file
        std::lock_guard<std::mutex> g(sp->mu);
        sp->st = St::Finishing;
        disk_feed(e, sp);
        mark_dirty(e, sp, nullptr);
    }
    c.stream = sp->id;
    return 1;
}

// The ring slabs a batch call's disk-backed checks may hold, and the ones all ring loads together may hold: a quarter
// of the ring each.
size_t ring_quarter(dm_engine *e)
{
    return std::max<size_t>(1, e->slab_store.size() / 4);
}

// What dm_cache_verify, dm_cache_import and dm_cache_export share: the ring's device mirror (read-backs, and a tiny
// check that finds no pack, stage slabs there), the call's stream slots, and run_batch.  The live proxy keeps its ring:
// at most a quarter of the slabs' worth of disk-backed checks are open at once, and each holds at most two slabs.  Ring
// loads (below) have a quarter of their own, so checks and ring loads together never hold more than half of the ring.
class CheckRun {
public:
    CheckRun(dm_engine *e, size_t n_work) : e_(e)
    {
        ring_ok_ = e->cas_dir.empty() || n_work == 0 || ensure_dev_ring(e) == DM_OK;
        std::lock_guard<std::mutex> g(e->slot_mu);
        budget_ = slots_reserve(e, SIZE_MAX);
    }
    ~CheckRun() { std::lock_guard<std::mutex> g(e_->slot_mu); slots_release(e_, budget_); }
    CheckRun(const CheckRun &) = delete;
    CheckRun &operator=(const CheckRun &) = delete;

    // DM_OK, or the status of every check this call cannot run
    int blocked() const
    {
        if (!ring_ok_) return fail(DM_ECUDA, "could not allocate the ring's device mirror");
        if (budget_ == 0) return fail(DM_ENOMEM, "no stream slot to spare for a check");
        return DM_OK;
    }

    // prepare(c, &fd, &path): 1 with fd open on the file to check, `path` its name and c.seen its fstat; or c's final
    // status.  settle(c, rc): c's final status, where rc is 1 when c's check is open and its verdict is due, or the
    // status with which it could not be opened (fd is closed by then).
    void run(std::vector<Check> &work, const std::function<int(Check &, int *, std::string *)> &prepare,
             const std::function<int(Check &, int)> &settle)
    {
        dm_engine *e = e_;
        run_batch(e, work, budget_, ring_quarter(e),
                  [&](Check &c, const MakeRoom &room, uint8_t *) -> int {
                      int fd = -1;
                      std::string path;
                      const int rc = prepare(c, &fd, &path);
                      if (rc != 1) return rc;
                      if (const int b = blocked()) { close(fd); return settle(c, b); }
                      room(!(e->tiny_max && (uint64_t)c.seen.st_size <= e->tiny_max));
                      const int st = check_open(e, c, fd, path);
                      return st == 1 ? 1 : settle(c, st);
                  },
                  [&](Check &c) { return settle(c, 1); });
    }

private:
    dm_engine *e_;
    bool ring_ok_ = true;
    size_t budget_ = 0;
};

// A directory entry of blobs/sha256/<aa>/ that names a blob: 64 lowercase hex digits starting with <aa>.
bool blob_name(const char *name, const char aa[2], Digest *d)
{
    return strlen(name) == 64 && name[0] == aa[0] && name[1] == aa[1] && digest_from_hex(name, d->b) &&
           hex_of(d->b, 32) == name;
}

}  // namespace

static int cache_verify_impl(dm_engine *e, const uint8_t *digests, uint32_t n, int32_t *status_out)
{
    if (!e || (n && (!digests || !status_out))) return fail(DM_EINVAL, "null argument");
    std::vector<Check> work;
    std::vector<uint32_t> slot_of;
    dedup(n, &slot_of, [&](uint32_t i, std::string *k) { k->assign((const char *)digests + 32ull * i, 32); return DM_OK; },
          [&](uint32_t i) { work.emplace_back(); memcpy(work.back().d.b, digests + 32ull * i, 32); });
    CheckRun run(e, work.size());
    for (Check &c : work) hold_digest(e, c.d, "a running dm_cache_verify");
    for (Check &c : work) tier_pin(e, c.d);
    run.run(work,
            [&](Check &c, int *fd, std::string *path) -> int {
                std::string side;
                const int rc = open_disk_copy(e, c.d, fd, &c.seen, &side);
                if (rc == DM_ENOENT) return blob_in_hbm(e, c.d) ? DM_OK : DM_ENOENT;     // (verified at ingest)
                if (rc != DM_OK) return rc;
                *path = blob_path(e, c.d.b);
                return 1;
            },
            [&](Check &c, int rc) -> int { return rc == 1 ? tier_verdict(e, c.stream, c.d, c.seen) : rc; });
    for (Check &c : work) tier_unpin(e, c.d);
    for (Check &c : work) release_digest(e, c.d);
    for (uint32_t i = 0; i < n; ++i) status_out[i] = work[slot_of[i]].status;
    return DM_OK;
}

// ---- ring loads (dm_cache_open_verified_ring) -------------------------------------------------------------------
// A check of a tier file (above) whose read-back slabs also serve one reader (struct RingLoad).  Each load holds at
// most kRingLoadSlabs slabs: the two of the hash side (disk_feed) and two that the reader may still be copying from.
// All ring loads together hold at most a quarter of the ring's slabs (their own quarter: checks have another), and each
// takes one stream slot of the tier calls' (slots_reserve).

}  // extern "C"

namespace dmi {

constexpr uint32_t kRingLoadSlabs = 4;

static uint32_t ring_load_cap(dm_engine *e)
{
    return (uint32_t)std::min<size_t>(kRingLoadSlabs, ring_quarter(e));
}

int ring_load_reserve(dm_engine *e, size_t n)
{
    if (const size_t got = slots_reserve(e, n); got < n) { slots_release(e, got); return 1; }
    if (e->ring_load_slabs + n * ring_load_cap(e) > ring_quarter(e)) { slots_release(e, n); return 2; }
    e->ring_load_slabs += n * ring_load_cap(e);
    return 0;
}

void ring_load_unreserve(dm_engine *e, size_t n)
{
    slots_release(e, n);
    e->ring_load_slabs -= n * ring_load_cap(e);
}

int ring_load_open(dm_engine *e, const Digest &d, const std::shared_ptr<RingPart> &part, bool shared, uint64_t off,
                   uint64_t len, bool reserved, std::shared_ptr<Stream> *out)
{
    if (!reserved) {
        std::lock_guard<std::mutex> g(e->slot_mu);
        const int why = ring_load_reserve(e, 1);
        if (why == 1) return fail(DM_ENOMEM, "no stream slot to spare for a ring load");
        if (why == 2) return fail(DM_ENOMEM, "the ring slabs ring loads may hold are all taken: retry later, or serve the blob with dm_cache_open");
    }
    auto unreserve = [&] { std::lock_guard<std::mutex> g(e->slot_mu); ring_load_unreserve(e, 1); };
    if (const int rc = ensure_dev_ring(e); rc != DM_OK) { unreserve(); return rc; }
    hold_digest(e, d, shared ? "a running shared ring load (dm_cache_open_verified_range)"
                             : "a running ring load (dm_cache_open_verified_ring)");
    Check c;
    c.d = d;
    int fd = -1;
    auto R = std::make_unique<RingLoad>();
    int rc = open_disk_copy(e, d, &fd, &c.seen, &R->side);
    if (rc == DM_OK) {
        const uint64_t size = (uint64_t)c.seen.st_size;
        if (shared && (off > size || len > size - off)) {
            close(fd);
            rc = fail(DM_ERANGE, "the range is not within the blob");
        } else {
            R->cap = ring_load_cap(e);
            R->seen = c.seen;
            R->size = size;
            R->shared = shared;
            R->parts.push_back(part);
            rc = check_open(e, c, fd, blob_path(e, d.b), std::move(R), out);
        }
    }
    if (rc != 1) { release_digest(e, d); unreserve(); return rc; }
    if (shared) {                                               // (unless it has already failed: a tiny file)
        bool live;
        { std::lock_guard<std::mutex> g((*out)->mu); live = !(*out)->ring->settled || (*out)->ring->status == DM_OK; }
        if (live) e->ring_shared.emplace(d, *out);
    }
    return DM_OK;
}

// A shared load leaves e->ring_shared (it failed, or its last reader closed)
static void ring_unlist(dm_engine *e, const std::shared_ptr<Stream> &sp)
{
    std::lock_guard<std::mutex> g(e->ring_mu);
    for (auto [it, end] = e->ring_shared.equal_range(sp->expect); it != end; ++it)
        if (it->second == sp) { e->ring_shared.erase(it); return; }
}

void ring_load_settle(dm_engine *e, const std::shared_ptr<Stream> &sp)
{
    Stream *s = sp.get();
    RingLoad *R = s->ring.get();
    int status;
    {
        std::lock_guard<std::mutex> g(s->mu);
        status = s->cuda_failed ? DM_ECUDA : s->lost != DM_OK ? s->lost : s->matched ? DM_OK : DM_ECORRUPT;
    }
    if (status == DM_OK) tier_touch(e, s->expect);              // a use of the blob, as a verified open is
    else if (status == DM_ECORRUPT) drop_corrupt(e, s->expect, R->seen);
    drop_stream(e, sp, true);                                   // its slot, and its hold on the digest
    bool unreserve;
    {
        std::lock_guard<std::mutex> g(s->mu);
        unreserve = R->slot_reserved;
        R->slot_reserved = false;
        R->status = status;
        R->settled = true;
    }
    if (R->shared && status != DM_OK) ring_unlist(e, sp);      // (a verified one serves attachments until its last close)
    if (unreserve) { std::lock_guard<std::mutex> g(e->slot_mu); slots_release(e, 1); }
    s->cv.notify_all();
}

// One reader leaves the load: `part` (attached), or a reader detached from it (nullptr).  The last one stops it.
static void ring_load_leave(dm_engine *e, const std::shared_ptr<Stream> &sp, const std::shared_ptr<RingPart> &part)
{
    Stream *s = sp.get();
    RingLoad *R = s->ring.get();
    bool last, stop, unreserve = false;
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (part) R->parts.erase(std::find(R->parts.begin(), R->parts.end(), part));
        else R->dependents--;
        last = R->parts.empty() && R->dependents == 0;
        R->closed = last;
        ring_release(e, sp);
        disk_feed(e, sp);                                       // (other readers may be waiting for what it held back)
        stop = last && !R->settled && s->st != St::Done && s->st != St::Aborted;
        if (last) { unreserve = R->slot_reserved; R->slot_reserved = false; }
    }
    if (!last) return;
    if (R->shared) ring_unlist(e, sp);
    // slabs still staged come back from the abort, those being hashed when their jobs are reaped (R->closed)
    if (stop) stream_abort_impl(e, s->id);
    s->cv.notify_all();                                         // (readers detached from it may wait for its verdict)
    std::lock_guard<std::mutex> g(e->slot_mu);
    if (unreserve) slots_release(e, 1);
    e->ring_load_slabs -= R->cap;
}

void ring_load_close(dm_engine *e, const std::shared_ptr<Stream> &sp, const std::shared_ptr<RingPart> &part)
{
    bool detached, reservation;
    {
        std::lock_guard<std::mutex> g(sp->mu);
        detached = part->detached;
        reservation = part->reserved;
        part->reserved = false;
    }
    if (reservation) { std::lock_guard<std::mutex> g(e->slot_mu); ring_load_unreserve(e, 1); }
    ring_load_leave(e, sp, detached ? nullptr : part);
    for (const auto &f : part->from) ring_load_leave(e, f, nullptr);
}

}  // namespace dmi

extern "C" {

// ---- importing files from outside the cache (dm_cache_import) ---------------------------------------------------
// Each source is first copied (or hard-linked) to a private file under <cas_dir>/incoming/.  That file is checked the
// way dm_cache_verify checks a tier file and, once it hashes to what was expected, renamed into blobs/ by the thread
// that collected its verdict: the bytes that get published are the bytes that were hashed, whatever happens to the
// source meanwhile.  A bad source says nothing about the tier, so nothing here goes through drop_corrupt.

namespace {

struct Import {
    const char *src = nullptr;
    std::string staged;                   // the private copy, while it exists
    uint8_t got[32] = {0};                // what it hashed to (DM_OK, DM_ECORRUPT)
};

bool on_either_tier(dm_engine *e, const Digest &d)
{
    {
        std::lock_guard<std::mutex> g(e->mu);
        if (e->blobs.find(d) != e->blobs.end()) return true;
    }
    struct stat st;
    return stat(blob_path(e, d.b).c_str(), &st) == 0;
}

// What a failed copy_into says: the source could not be copied, read or written.
struct StageTexts { const char *copy, *read, *write; };
constexpr StageTexts kImportTexts = {"could not copy the file into <cas_dir>/incoming", "could not read the file to import",
                                     "could not write the staged copy under <cas_dir>/incoming"};

// Copy `src` into the new, empty file `out` and close it: copy_file_range (a reflink on XFS and btrfs), pread / pwrite
// where the kernel or the filesystems cannot do that.  Copies up to the end of file as it is now.
int copy_into(int src, int out, const StageTexts &t)
{
    bool plain = false;
    std::unique_ptr<uint8_t[]> buf;
    constexpr size_t kBuf = 1 << 20;
    loff_t off = 0;
    int rc = DM_OK;
    for (;;) {
        if (!plain) {
            loff_t in_off = off, out_off = off;
            const ssize_t r = copy_file_range(src, &in_off, out, &out_off, 1 << 30, 0);
            if (r > 0) { off += r; continue; }
            if (r == 0) break;
            if (errno == EINTR) continue;
            if (errno != EXDEV && errno != ENOSYS && errno != EINVAL && errno != EOPNOTSUPP) {
                rc = fail(DM_EIO, t.copy);
                break;
            }
            plain = true;
            buf.reset(new uint8_t[kBuf]);
        }
        const ssize_t r = pread(src, buf.get(), kBuf, off);
        if (r < 0 && errno == EINTR) continue;
        if (r < 0) { rc = fail(DM_EIO, t.read); break; }
        if (r == 0) break;
        ssize_t w = 0;
        while (w < r) {
            const ssize_t k = pwrite(out, buf.get() + w, (size_t)(r - w), off + w);
            if (k < 0 && errno == EINTR) continue;
            if (k <= 0) break;
            w += k;
        }
        if (w < r) { rc = fail(DM_EIO, t.write); break; }
        off += r;
    }
    if (close(out) != 0 && rc == DM_OK) rc = fail(DM_EIO, t.write);
    return rc;
}

// fsync the file (`dir`: the directory) at `path`: false when it cannot be opened or synced.
bool fsync_path(const char *path, bool dir = false)
{
    const int f = open(path, O_RDONLY | O_CLOEXEC | (dir ? O_DIRECTORY : 0));
    const bool synced = f >= 0 && fsync(f) == 0;
    if (f >= 0) close(f);
    return synced;
}

int stage_copy(int src, const std::string &dst)
{
    const int out = open(dst.c_str(), O_CREAT | O_TRUNC | O_WRONLY | O_CLOEXEC, 0644);
    if (out < 0) return fail(DM_EIO, "could not create the staged copy under <cas_dir>/incoming");
    return copy_into(src, out, kImportTexts);
}

// Open the source of `im`, stage it and open the staged file for its check (prepare of CheckRun::run).
int import_prepare(dm_engine *e, const CheckRun &run, uint32_t flags, Check &c, Import &im, int *fd, std::string *path)
{
    if (c.known && on_either_tier(e, c.d)) {             // checking the copy that is there is dm_cache_verify's job
        memcpy(im.got, c.d.b, 32);
        return DM_OK;
    }
    // O_NONBLOCK: opening a FIFO must not wait for a writer (it is refused below like every other non-regular file)
    const int src = open(im.src, O_RDONLY | O_CLOEXEC | O_NONBLOCK);
    if (src < 0)
        return errno == ENOENT || errno == ENOTDIR ? fail(DM_ENOENT, "no such file") : fail(DM_EIO, "could not open the file to import");
    struct stat st;
    if (fstat(src, &st) != 0) { close(src); return fail(DM_EIO, "could not stat the file to import"); }
    if (!S_ISREG(st.st_mode)) { close(src); return fail(DM_EINVAL, "not a regular file"); }
    if (const int b = run.blocked()) { close(src); return b; }
    im.staged = incoming_path(e, e->next_id.fetch_add(1));
    if (!tier_stage(e, im.staged, (uint64_t)st.st_size)) {
        close(src);
        im.staged.clear();
        return fail(DM_ENOMEM, "no room under the disk-tier limit for the file to import");
    }
    bool linked = false;
    if (flags & DM_IMP_LINK) {
        // ENOENT: the source was replaced (renamed over) since it was opened, and the file that is open has no name
        // left to link: it is copied from the open descriptor like one on another filesystem
        linked = linkat(AT_FDCWD, im.src, AT_FDCWD, im.staged.c_str(), AT_SYMLINK_FOLLOW) == 0;
        if (!linked && errno != EXDEV && errno != EPERM && errno != ENOENT) {
            close(src);
            tier_unstage(e, im.staged);
            im.staged.clear();
            return fail(DM_EIO, "could not link the file into <cas_dir>/incoming");
        }
    }
    int rc = linked ? DM_OK : stage_copy(src, im.staged);
    close(src);
    if (rc == DM_OK) {
        *fd = open(im.staged.c_str(), O_RDONLY | O_CLOEXEC);
        if (*fd < 0) rc = fail(DM_EIO, "could not open the staged copy");
        else if (fstat(*fd, &c.seen) != 0) { close(*fd); rc = fail(DM_EIO, "could not stat the staged copy"); }
    }
    if (rc != DM_OK) {
        unlink(im.staged.c_str());
        tier_unstage(e, im.staged);
        im.staged.clear();
        return rc;
    }
    *path = im.staged;
    return 1;
}

// The verdict of an import's check is due: publish the staged file when it hashed to what was expected.
int import_publish(dm_engine *e, Check &c, Import &im)
{
    int matched = 0;
    const int rc = check_finish(e, c.stream, im.got, &matched);
    if (rc != DM_OK) { memset(im.got, 0, 32); return rc; }
    if (!matched) return fail(DM_ECORRUPT, "the file does not hash to the digest it was imported under");
    if ((e->cfg.flags & DM_F_DISK_SYNC) && !fsync_path(im.staged.c_str()))
        return fail(DM_EIO, "could not fsync the imported copy");
    Digest d;
    memcpy(d.b, im.got, 32);
    const uint64_t size = (uint64_t)c.seen.st_size;
    const std::string dst = blob_path(e, d.b);
    mkdirs(dst);
    struct TierHold {                                    // not a disk-tier victim while it is placed
        dm_engine *e; Digest d;
        ~TierHold() { tier_unpin(e, d); }
    } hold{e, d};
    DigestHold placing(e, d, "a running dm_cache_import is placing it");
    tier_pin(e, d);
    struct stat st;
    const bool placed = stat(dst.c_str(), &st) != 0;    // already in the disk tier: keep that copy, the staged one goes
    if (placed) {
        Blob b;
        b.digest = d; b.size = size;
        TierRes res;
        if (!tier_stage_to_blob(e, im.staged, size, sidecar_json(b).size(), &res))
            return fail(DM_ENOMEM, "no room under the disk-tier limit for the imported file");
        if (rename(im.staged.c_str(), dst.c_str()) != 0) {
            tier_release(e, res);
            return fail(DM_EIO, "could not move the imported copy into the disk tier");
        }
        im.staged.clear();
        if (!write_sidecar(dst + ".meta", b)) {
            unlink(dst.c_str());
            unlink((dst + ".meta").c_str());
            tier_release(e, res);
            return fail(DM_EIO, "could not write the imported blob's sidecar");
        }
        tier_placed(e, d, false, &res, true);
    }
    {
        std::lock_guard<std::mutex> g(e->mu);
        auto it = e->blobs.find(d);
        if (it == e->blobs.end()) {
            auto b = std::make_shared<Blob>();
            b->digest = d; b->size = size;
            b->on_disk = b->spill_done = true;
            e->blobs[d] = b;
        } else if (!it->second->on_disk) {
            it->second->on_disk = it->second->spill_done = true;
        }
    }
    if (placed) e->st_committed++;
    return DM_OK;
}

}  // namespace

static int cache_import_impl(dm_engine *e, const char *const *paths, const uint8_t *expect, const char *const *keys,
                             uint32_t n, uint32_t flags, uint8_t *digests_out, int32_t *status_out)
{
    if (!e || (n && (!paths || !digests_out || !status_out))) return fail(DM_EINVAL, "null argument");
    if (flags & ~DM_IMP_LINK) return fail(DM_EINVAL, "unknown dm_cache_import flag");
    for (uint32_t i = 0; i < n; ++i) {
        if (!paths[i]) return fail(DM_EINVAL, "null path");
        if (keys && keys[i] && !alias_key_ok(keys[i])) return fail(DM_EINVAL, "alias key must be 1..4096 bytes without control characters");
    }
    if (e->cas_dir.empty()) return fail(DM_ESTATE, "dm_cache_import needs a cas_dir");
    // staged copies of an import that was killed part way would otherwise stay for good on an engine that never
    // sweeps (one without DM_F_DISK_DIRECT)
    mkdirs(e->cas_dir + "/incoming/x");
    sweep_incoming(e->cas_dir + "/incoming");
    static const uint8_t kZero[32] = {0};
    std::vector<Check> work;
    std::vector<Import> imp;
    std::vector<uint32_t> slot_of;
    auto expected = [&](uint32_t i) { return expect ? expect + 32ull * i : kZero; };
    dedup(n, &slot_of,
          [&](uint32_t i, std::string *k) {                    // path and expected digest: a duplicate is imported once
              *k = paths[i];
              k->push_back('\0');
              k->append((const char *)expected(i), 32);
              return DM_OK;
          },
          [&](uint32_t i) {
              work.emplace_back();
              imp.emplace_back();
              work.back().known = memcmp(expected(i), kZero, 32) != 0;
              memcpy(work.back().d.b, expected(i), 32);
              imp.back().src = paths[i];
          });
    CheckRun run(e, work.size());
    run.run(work,
            [&](Check &c, int *fd, std::string *path) -> int {
                return import_prepare(e, run, flags, c, imp[&c - work.data()], fd, path);
            },
            [&](Check &c, int rc) -> int {
                Import &im = imp[&c - work.data()];
                if (rc == 1) rc = import_publish(e, c, im);
                if (!im.staged.empty()) { unlink(im.staged.c_str()); tier_unstage(e, im.staged); im.staged.clear(); }
                return rc;
            });
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t k = slot_of[i];
        status_out[i] = work[k].status;
        const bool has = work[k].status == DM_OK || work[k].status == DM_ECORRUPT;
        memcpy(digests_out + 32ull * i, has ? imp[k].got : kZero, 32);
        if (work[k].status == DM_OK && keys && keys[i]) dm_cache_alias_put(e, keys[i], imp[k].got);
    }
    return DM_OK;
}

// ---- exporting cached blobs to files (dm_cache_export) ----------------------------------------------------------
// The other half of an import.  Each blob is copied to a private file next to its destination - out of its HBM extent
// (held by a reader reference, without touching the LRU order) or, from the disk tier, the way an import stages its
// source - and that file is checked as an import checks its staged copy, with the digest as the expected value.  Only a
// file that hashed to its name is renamed over the destination: no byte leaves the cache unless the GPU hashed it.  The
// cache is only read.  A tier file whose copy fails its check stays where it is: deciding about it is dm_cache_verify's
// job, and dropping it from here would let a bad destination disk remove good blobs.

namespace {

constexpr StageTexts kExportTexts = {"could not copy the disk tier file to the staged file", "could not read the disk tier file",
                                     "could not write the staged file next to the destination"};
constexpr char kExportTag[] = ".dm-export-";
std::atomic<uint64_t> g_export_id{1};     // per process: engines of one process may export into the same directory

struct Export {
    const char *dest = nullptr;
    std::string staged;                   // the private copy, while it exists
    bool held = false;                    // hold_digest and tier_pin on the digest, from the source copy to the verdict
};

std::string dir_of(const char *path)      // up to and including the last '/', "" for a name in the working directory
{
    const char *slash = strrchr(path, '/');
    return slash ? std::string(path, (size_t)(slash - path) + 1) : std::string();
}

// Staged files are .<basename>.dm-export-<pid>-<id>.part in the destination's directory: remove those of processes that
// are gone (the rule sweep_incoming applies to incoming/), and leave every live process's alone.
void sweep_export_staging(const std::string &dir)
{
    DIR *d = opendir(dir.empty() ? "." : dir.c_str());
    if (!d) return;
    while (struct dirent *de = readdir(d)) {
        const char *name = de->d_name;
        const size_t n = strlen(name);
        if (name[0] != '.' || n < 5 || strcmp(name + n - 5, ".part") != 0) continue;
        const char *tag = nullptr;
        for (const char *p = strstr(name, kExportTag); p; p = strstr(p + 1, kExportTag)) tag = p;
        if (!tag) continue;
        const char *digits = tag + sizeof kExportTag - 1;
        char *end = nullptr;
        const long pid = strtol(digits, &end, 10);
        if (end == digits || *end != '-' || pid <= 0) continue;
        if (kill((pid_t)pid, 0) == 0 || errno == EPERM) continue;        // alive (EPERM: alive, another user's)
        unlink((dir + name).c_str());
    }
    closedir(d);
}

void export_release(dm_engine *e, const Check &c, Export &ex)
{
    if (!ex.staged.empty()) { unlink(ex.staged.c_str()); ex.staged.clear(); }
    if (ex.held) { tier_unpin(e, c.d); release_digest(e, c.d); ex.held = false; }
}

// Copy the blob to its staged file and open that file for its check (prepare of CheckRun::run).  Whatever it leaves
// held or staged is undone by export_release.
int export_prepare(dm_engine *e, const CheckRun &run, Check &c, Export &ex, int *fd, std::string *path)
{
    struct stat ds;
    if (stat(ex.dest, &ds) == 0 && S_ISDIR(ds.st_mode)) return fail(DM_EIO, "the destination is a directory");
    if (const int b = run.blocked()) return b;
    hold_digest(e, c.d, "a running dm_cache_export");
    tier_pin(e, c.d);                                    // the tier file is not a disk-tier victim while it is copied
    ex.held = true;
    std::shared_ptr<Blob> hbm;
    std::vector<Extent> ext;
    {
        std::lock_guard<std::mutex> g(e->mu);
        auto it = e->blobs.find(c.d);
        if (it != e->blobs.end() && it->second->in_hbm) {   // verified at ingest; the reference keeps the extent
            hbm = it->second;
            hbm->readers++;
            ext = hbm->extents;
        }
    }
    int src = -1;
    if (!hbm) {
        std::string side;
        const int rc = open_disk_copy(e, c.d, &src, &c.seen, &side, true);
        if (rc == DM_ECORRUPT)
            return note_err(e, 0, fail(DM_ECORRUPT, "the disk tier file is not the size its sidecar says: nothing was "
                                                     "exported, and the file is left to dm_cache_verify"));
        if (rc != DM_OK) return rc;
    }
    mkdirs(ex.dest);
    ex.staged = dir_of(ex.dest) + "." + (strrchr(ex.dest, '/') ? strrchr(ex.dest, '/') + 1 : ex.dest) + kExportTag +
                std::to_string((long)getpid()) + "-" + std::to_string(g_export_id.fetch_add(1)) + ".part";
    int rc = DM_OK;
    const int out = open(ex.staged.c_str(), O_CREAT | O_EXCL | O_WRONLY | O_CLOEXEC, 0644);
    if (out < 0) {
        ex.staged.clear();                               // not ours to unlink
        rc = fail(DM_EIO, "could not create the staged file next to the destination");
    }
    if (hbm) {
        if (out >= 0) {
            bool cuda_failed = false;
            const bool copied = d2h_to_fd(e, ext, hbm->size, out, &cuda_failed);
            const bool closed = close(out) == 0;
            if (cuda_failed) rc = fail(DM_ECUDA, "could not copy the blob out of HBM");
            else if (!copied || !closed) rc = fail(DM_EIO, kExportTexts.write);
        }
        std::vector<Extent> gone;
        { std::lock_guard<std::mutex> g(e->mu); gone = reader_gone(hbm.get()); }
        if (!gone.empty()) free_extents(e, gone);
    } else {
        if (out >= 0) rc = copy_into(src, out, kExportTexts);
        close(src);
    }
    if (rc == DM_OK) {
        *fd = open(ex.staged.c_str(), O_RDONLY | O_CLOEXEC);
        if (*fd < 0) rc = fail(DM_EIO, "could not open the staged file");
        else if (fstat(*fd, &c.seen) != 0) { close(*fd); rc = fail(DM_EIO, "could not stat the staged file"); }
    }
    if (rc != DM_OK) return rc;
    *path = ex.staged;
    return 1;
}

// The verdict of an export's check is due: rename the staged file over the destination when it hashed to its name.
int export_publish(dm_engine *e, Check &c, Export &ex)
{
    uint8_t got[32];
    int matched = 0;
    const int rc = check_finish(e, c.stream, got, &matched);
    if (rc != DM_OK) return rc;
    if (!matched)
        return note_err(e, 0, fail(DM_ECORRUPT, "the copy of the blob does not hash to its name: nothing was exported, "
                                                 "and the cache is left as it is (dm_cache_verify decides about the tier file)"));
    const bool sync = (e->cfg.flags & DM_F_DISK_SYNC) != 0;
    if (sync && !fsync_path(ex.staged.c_str())) return fail(DM_EIO, "could not fsync the staged file");
    if (rename(ex.staged.c_str(), ex.dest) != 0) return fail(DM_EIO, "could not rename the staged file over the destination");
    ex.staged.clear();
    const std::string dir = dir_of(ex.dest);
    if (sync && !fsync_path(dir.empty() ? "." : dir.c_str(), true))
        return fail(DM_EIO, "could not fsync the destination's directory");
    return DM_OK;
}

}  // namespace

static int cache_export_impl(dm_engine *e, const uint8_t *digests, const char *const *dest_paths, uint32_t n,
                             int32_t *status_out)
{
    if (!e || (n && (!digests || !dest_paths || !status_out))) return fail(DM_EINVAL, "null argument");
    std::vector<Check> work;
    std::vector<Export> exp;
    std::vector<uint32_t> slot_of;
    std::unordered_map<std::string, const uint8_t *> named;   // destination -> its digest: written once, by one digest
    const int bad = dedup(
        n, &slot_of,
        [&](uint32_t i, std::string *k) -> int {
            if (!dest_paths[i]) return fail(DM_EINVAL, "null path");
            const uint8_t *d = digests + 32ull * i;
            if (memcmp(named.emplace(dest_paths[i], d).first->second, d, 32) != 0)
                return fail(DM_EINVAL, "one destination named with two different digests");
            *k = dest_paths[i];
            return DM_OK;
        },
        [&](uint32_t i) {
            work.emplace_back();
            memcpy(work.back().d.b, digests + 32ull * i, 32);
            exp.emplace_back();
            exp.back().dest = dest_paths[i];
        });
    if (bad) return bad;
    {
        std::vector<std::string> dirs;
        for (const Export &ex : exp) dirs.push_back(dir_of(ex.dest));
        std::sort(dirs.begin(), dirs.end());
        dirs.erase(std::unique(dirs.begin(), dirs.end()), dirs.end());
        for (const std::string &dir : dirs) sweep_export_staging(dir);
    }
    // the check of a staged file reads it back through the ring's device mirror on the disk threads, which an engine
    // without a cas_dir has not started
    int ring_rc = DM_OK;
    if (!work.empty() && e->cas_dir.empty()) {
        ensure_disk_threads(e);
        ring_rc = ensure_dev_ring(e);
    }
    CheckRun run(e, work.size());
    run.run(work,
            [&](Check &c, int *fd, std::string *path) -> int {
                Export &ex = exp[&c - work.data()];
                const int rc = ring_rc != DM_OK ? ring_rc : export_prepare(e, run, c, ex, fd, path);
                if (rc != 1) export_release(e, c, ex);
                return rc;
            },
            [&](Check &c, int rc) -> int {
                Export &ex = exp[&c - work.data()];
                if (rc == 1) rc = export_publish(e, c, ex);
                export_release(e, c, ex);
                return rc;
            });
    for (uint32_t i = 0; i < n; ++i) status_out[i] = work[slot_of[i]].status;
    return DM_OK;
}

// ---- listing the disk tier (dm_cache_list) ----------------------------------------------------------------------
// Stateless: a page starts strictly after the last digest of the one before, so blobs may come and go between calls.
// Only the prefix directories from after[0] on are read, one at a time, each sorted on its own.
static int cache_list_impl(dm_engine *e, const uint8_t after[32], uint8_t *digests_out, uint64_t *sizes_out,
                           uint32_t cap, uint32_t *n_out)
{
    if (!e || !n_out || (cap && !digests_out)) return fail(DM_EINVAL, "null argument");
    *n_out = 0;
    if (e->cas_dir.empty()) return DM_OK;
    const std::string root = e->cas_dir + "/blobs/sha256/";
    uint32_t got = 0;
    std::vector<Digest> names;
    for (int p = after ? after[0] : 0; p < 256 && got < cap; ++p) {
        char aa[3];
        snprintf(aa, sizeof aa, "%02x", p);
        const std::string dir = root + aa + "/";
        DIR *d = opendir(dir.c_str());
        if (!d) continue;
        names.clear();
        while (struct dirent *de = readdir(d)) {
            Digest dg;
            if (!blob_name(de->d_name, aa, &dg)) continue;                  // .meta, .part and strays
            if (after && memcmp(dg.b, after, 32) <= 0) continue;
            names.push_back(dg);
        }
        closedir(d);
        std::sort(names.begin(), names.end(), [](const Digest &a, const Digest &b) { return memcmp(a.b, b.b, 32) < 0; });
        for (const Digest &dg : names) {
            if (got == cap) break;
            struct stat st;
            if (stat((dir + hex_of(dg.b, 32)).c_str(), &st) != 0 || !S_ISREG(st.st_mode)) continue;   // gone meanwhile
            memcpy(digests_out + 32ull * got, dg.b, 32);
            if (sizes_out) sizes_out[got] = (uint64_t)st.st_size;
            ++got;
        }
    }
    *n_out = got;
    return DM_OK;
}

// ---- disk-tier limit (dm_cache_set_disk_limit, dm_cache_disk_usage) ---------------------------------------------
// The bookkeeping is in engine_core.cu (struct DiskTier); this builds the index on the first limit and evicts down.
static int cache_set_disk_limit_impl(dm_engine *e, uint64_t limit_bytes)
{
    if (!e) return fail(DM_EINVAL, "null argument");
    if (e->cas_dir.empty()) return fail(DM_ESTATE, "dm_cache_set_disk_limit needs a disk tier (cas_dir)");
    std::lock_guard<std::mutex> g(e->tier_mu);
    DiskTier &T = e->tier;
    if (limit_bytes == 0) {                              // off: nothing is tracked, touched or reserved any more
        T.on = false;
        T.limit = 0;
        T.blobs.clear(); T.saved.clear(); T.order.clear(); T.staging.clear();
        T.blob_bytes = T.partial_bytes = T.staging_bytes = T.reserved_blob = T.reserved_partial = 0;
        e->tier_on.store(false, std::memory_order_release);
        return DM_OK;
    }
    if (!T.on) {
        mkdirs(e->cas_dir + "/incoming/x");
        tier_build(e);
        e->tier_on.store(true, std::memory_order_release);
    }
    T.limit = limit_bytes;
    tier_make_room(e, 0, true);                          // down to the limit, or to what is pinned
    return DM_OK;
}

static int cache_disk_usage_impl(dm_engine *e, dm_disk_usage *out)
{
    if (!e || !out) return fail(DM_EINVAL, "null argument");
    if (out->struct_size != sizeof(dm_disk_usage)) return fail(DM_EINVAL, "dm_disk_usage has the wrong struct_size");
    std::lock_guard<std::mutex> g(e->tier_mu);
    const DiskTier &T = e->tier;
    memset(out, 0, sizeof *out);
    out->struct_size = sizeof *out;
    out->evicted_files = T.evicted_files;
    out->evicted_bytes = T.evicted_bytes;
    out->refused = T.refused;
    if (!T.on) return DM_OK;
    out->limit_bytes = T.limit;
    out->blob_files = T.blobs.size();
    out->blob_bytes = T.blob_bytes + T.reserved_blob;
    out->staging_bytes = T.staging_bytes;
    out->partial_bytes = T.partial_bytes + T.reserved_partial;
    out->used_bytes = out->blob_bytes + out->staging_bytes + out->partial_bytes;
    return DM_OK;
}

// ---- exported wrappers: file the error text under the stream id (dm_error_detail) ----
int dm_cache_set_disk_limit(dm_engine *e, uint64_t limit_bytes) { return note_err(e, 0, cache_set_disk_limit_impl(e, limit_bytes)); }
int dm_cache_disk_usage(dm_engine *e, dm_disk_usage *out) { return note_err(e, 0, cache_disk_usage_impl(e, out)); }
int dm_cache_promote(dm_engine *e, const uint8_t *digests, uint32_t n, int32_t *status_out)
{
    return note_err(e, 0, cache_promote_impl(e, digests, n, status_out));
}
int dm_cache_verify(dm_engine *e, const uint8_t *digests, uint32_t n, int32_t *status_out)
{
    return note_err(e, 0, cache_verify_impl(e, digests, n, status_out));
}
int dm_cache_import(dm_engine *e, const char *const *paths, const uint8_t *expect, const char *const *keys, uint32_t n,
                    uint32_t flags, uint8_t *digests_out, int32_t *status_out)
{
    return note_err(e, 0, cache_import_impl(e, paths, expect, keys, n, flags, digests_out, status_out));
}
int dm_cache_export(dm_engine *e, const uint8_t *digests, const char *const *dest_paths, uint32_t n, int32_t *status_out)
{
    return note_err(e, 0, cache_export_impl(e, digests, dest_paths, n, status_out));
}
int dm_cache_list(dm_engine *e, const uint8_t after[32], uint8_t *digests_out, uint64_t *sizes_out, uint32_t cap,
                  uint32_t *n_out)
{
    return note_err(e, 0, cache_list_impl(e, after, digests_out, sizes_out, cap, n_out));
}
int dm_stream_suspend(dm_engine *e, uint64_t id, uint64_t *resume_from) { return note_err(e, id, stream_suspend_impl(e, id, resume_from)); }
int dm_stream_resume_saved(dm_engine *e, const uint8_t expect[32], uint64_t size_hint, uint64_t *id, uint64_t *resume_from)
{
    return note_err(e, 0, stream_resume_saved_impl(e, expect, size_hint, id, resume_from));
}
int dm_stream_write(dm_engine *e, uint64_t id, const void *buf, size_t len) { return note_err(e, id, stream_write_impl(e, id, buf, len)); }
int dm_stream_write_at(dm_engine *e, uint64_t id, uint64_t offset, const void *buf, size_t len) { return note_err(e, id, stream_write_at_impl(e, id, offset, buf, len)); }
int dm_stream_checkpoint(dm_engine *e, uint64_t id, dm_checkpoint *out) { return note_err(e, id, stream_checkpoint_impl(e, id, out)); }
int dm_stream_set_meta(dm_engine *e, uint64_t id, const char *key, const char *value) { return note_err(e, id, stream_set_meta_impl(e, id, key, value)); }
int dm_stream_acquire(dm_engine *e, uint64_t id, void **ptr, size_t *cap) { return note_err(e, id, stream_acquire_impl(e, id, ptr, cap)); }
int dm_stream_commit(dm_engine *e, uint64_t id, size_t len) { return note_err(e, id, stream_commit_impl(e, id, len)); }
int dm_stream_flush(dm_engine *e, uint64_t id) { return note_err(e, id, stream_flush_impl(e, id)); }
int dm_stream_finish(dm_engine *e, uint64_t id, uint8_t digest_out[32], int *matched) { return note_err(e, id, stream_finish_impl(e, id, digest_out, matched)); }
int dm_stream_abort(dm_engine *e, uint64_t id) { return note_err(e, id, stream_abort_impl(e, id)); }

}  // extern "C"
