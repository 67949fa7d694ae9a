// TEST INFRASTRUCTURE ONLY — see fake_cuda/cuda_runtime.h.  Asynchronous fake runtime (one worker thread per stream) + the three
// SHA-256 "kernel" launchers executed on the CPU by the oracle (oracle/sha256_oracle.c), honouring
// exactly the HashJob contract the real kernels implement (INIT / FINAL flags, state table, fused copy).
#include "fake_cuda/cuda_runtime.h"
#include "../../demodel_b200/csrc/sha256_kernels.cuh"
#include "../../demodel_b200/csrc/blobgen.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>

extern "C" {
#include "../../oracle/sha256_oracle.c"
}

// ---- asynchronous streams -----------------------------------------------------------------------
// Each stream is a worker thread draining a FIFO of closures; copies and "kernels" run there, later
// than the call that enqueued them, so ThreadSanitizer sees any host-side reuse of a buffer that is not
// ordered after the event guarding it as a data race — exactly the engine's lifetime rules.
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

// FAKE_CUDA_JITTER_US=n: every queued operation starts after a random 0..n us pause, so that the windows
// between "enqueued" and "executed" that real hardware has (and a fast CPU thread hides) are explored.
static unsigned jitter_us()
{
    static const unsigned j = [] { const char *v = getenv("FAKE_CUDA_JITTER_US"); return v ? (unsigned)atoi(v) : 0u; }();
    return j;
}

struct fakeStream {
    std::mutex mu;
    std::condition_variable cv;
    std::deque<std::function<void()>> q;
    bool stop = false, busy = false;
    uint64_t rng = (uint64_t)(uintptr_t)this;
    std::thread th;
    fakeStream() : th([this] { run(); }) {}
    void run()
    {
        for (;;) {
            std::function<void()> f;
            {
                std::unique_lock<std::mutex> g(mu);
                cv.wait(g, [&] { return stop || !q.empty(); });
                if (q.empty()) return;
                f = std::move(q.front());
                q.pop_front();
                busy = true;
            }
            if (const unsigned j = jitter_us()) {
                rng = rng * 6364136223846793005ull + 1442695040888963407ull;
                std::this_thread::sleep_for(std::chrono::microseconds((rng >> 33) % (j + 1)));
            }
            f();
            {
                std::lock_guard<std::mutex> g(mu);
                busy = false;
            }
            cv.notify_all();
        }
    }
    void push(std::function<void()> f)
    {
        { std::lock_guard<std::mutex> g(mu); q.push_back(std::move(f)); }
        cv.notify_all();
    }
    void drain()
    {
        std::unique_lock<std::mutex> g(mu);
        cv.wait(g, [&] { return q.empty() && !busy; });
    }
};
struct EvState {
    std::mutex mu;
    std::condition_variable cv;
    uint64_t recorded = 0, done = 0;      // generations: a wait targets the record current at the time of the call
};
// The handle may be destroyed while work that refers to the event is still queued (legal in CUDA:
// resources are released when that work completes), so queued closures share ownership of the state.
struct fakeEvent { std::shared_ptr<EvState> st = std::make_shared<EvState>(); };
static std::mutex g_reg_mu;
static std::vector<fakeStream *> g_streams;

// FAKE_CUDA_FAIL_PPM=n: each host-to-device copy and each kernel launch fails with probability n per million
// (returns an error, does nothing) - what a device fault looks like to the engine.
static bool inject_failure()
{
    static const unsigned ppm = [] { const char *v = getenv("FAKE_CUDA_FAIL_PPM"); return v ? (unsigned)atoi(v) : 0u; }();
    if (!ppm) return false;
    static std::atomic<uint64_t> seq{0x9e3779b97f4a7c15ull};
    uint64_t x = seq.fetch_add(0x9e3779b97f4a7c15ull);
    x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull; x ^= x >> 27; x *= 0x94d049bb133111ebull; x ^= x >> 31;
    return x % 1000000u < ppm;
}

static void on_stream(cudaStream_t s, std::function<void()> f)
{
    if (!s) { f(); return; }              // legacy stream: synchronous
    s->push(std::move(f));
}

extern "C" {
cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
cudaError_t cudaSetDevice(int) { return cudaSuccess; }
cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int) { memset(p, 0, sizeof *p); p->major = 9; p->minor = 0; p->multiProcessorCount = 132; return cudaSuccess; }
cudaError_t cudaDeviceSynchronize(void)
{
    std::vector<fakeStream *> all;
    { std::lock_guard<std::mutex> g(g_reg_mu); all = g_streams; }
    for (fakeStream *s : all) s->drain();
    return cudaSuccess;
}
cudaError_t cudaDeviceGetPCIBusId(char *buf, int len, int) { if (len > 0) buf[0] = 0; return cudaErrorInvalidValue; }   // no PCI topology on the rig
cudaError_t cudaMemGetInfo(size_t *f, size_t *t) { *f = *t = 1ull << 30; return cudaSuccess; }
const char *cudaGetErrorString(cudaError_t) { return "fake cuda error"; }
// The real runtime keeps a per-thread "last error" that cudaGetLastError returns and clears - and a query that says
// "not ready" counts: cudaEventQuery / cudaStreamQuery leave cudaErrorNotReady there.  A launch wrapper that ends in
// `return cudaGetLastError()` on a thread that polls events therefore reports a stale cudaErrorNotReady.
static thread_local cudaError_t tl_last_error = cudaSuccess;
cudaError_t cudaGetLastError(void) { const cudaError_t e = tl_last_error; tl_last_error = cudaSuccess; return e; }
// Allocation registries, to model what the real runtime does with PAGEABLE host memory:
//   cudaMemcpyAsync H2D  - the source is staged before the call returns (snapshot here), the device write is
//                          stream-ordered;
//   cudaMemcpyAsync D2H  - synchronous with respect to the host (enqueue, then wait);
//   cudaMemcpy      H2D  - returns after staging; the device write completes LATER and is not ordered with
//                          work on non-blocking streams (deferred on a hidden legacy stream here) - which is
//                          how the resume-state upload once raced with the first job.
// With pinned memory the copy touches the caller's buffer on the stream thread, so TSan sees reuse races.
static std::mutex g_alloc_mu;
static std::map<uintptr_t, size_t> g_pinned, g_device;
static void reg_add(std::map<uintptr_t, size_t> &m, void *p, size_t n) { std::lock_guard<std::mutex> g(g_alloc_mu); m[(uintptr_t)p] = n ? n : 1; }
static void reg_del(std::map<uintptr_t, size_t> &m, void *p) { std::lock_guard<std::mutex> g(g_alloc_mu); m.erase((uintptr_t)p); }
static bool reg_has(std::map<uintptr_t, size_t> &m, const void *p, size_t n)
{
    std::lock_guard<std::mutex> g(g_alloc_mu);
    auto it = m.upper_bound((uintptr_t)p);
    if (it == m.begin()) return false;
    --it;
    return (uintptr_t)p + n <= it->first + it->second;
}
[[noreturn]] static void misuse(const char *what)
{
    fprintf(stderr, "FAKE CUDA: %s\n", what);
    abort();
}

// FAKE_CUDA_FAIL_ALLOC_NTH=k: the k-th device / pinned allocation (and stream / event creation) of the process fails,
// to walk dm_engine_create's unwinding.
static bool alloc_should_fail()
{
    static const long nth = [] { const char *v = getenv("FAKE_CUDA_FAIL_ALLOC_NTH"); return v ? atol(v) : 0L; }();
    static std::atomic<long> count{0};
    return nth > 0 && ++count == nth;
}

cudaError_t cudaMalloc(void **p, size_t n)
{
    if (alloc_should_fail()) { *p = nullptr; return cudaErrorMemoryAllocation; }
    *p = malloc(n ? n : 1);
    if (!*p) return cudaErrorMemoryAllocation;
    reg_add(g_device, *p, n);
    return cudaSuccess;
}
cudaError_t cudaFree(void *p) { cudaDeviceSynchronize(); if (p) reg_del(g_device, p); free(p); return cudaSuccess; }   // implicit sync, as the real one
cudaError_t cudaHostAlloc(void **p, size_t n, unsigned)
{
    if (alloc_should_fail()) { *p = nullptr; return cudaErrorMemoryAllocation; }
    *p = calloc(1, n ? n : 1);
    if (!*p) return cudaErrorMemoryAllocation;
    reg_add(g_pinned, *p, n);
    return cudaSuccess;
}
cudaError_t cudaFreeHost(void *p) { cudaDeviceSynchronize(); if (p) reg_del(g_pinned, p); free(p); return cudaSuccess; }
cudaError_t cudaHostGetDevicePointer(void **dev, void *host, unsigned)
{
    if (!reg_has(g_pinned, host, 1)) misuse("cudaHostGetDevicePointer on memory that is not pinned");
    *dev = host;
    return cudaSuccess;
}
static fakeStream *legacy_stream()
{
    static fakeStream *ls = [] { auto *x = new fakeStream(); std::lock_guard<std::mutex> g(g_reg_mu); g_streams.push_back(x); return x; }();
    return ls;
}
cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind kind)
{
    if (kind == cudaMemcpyHostToDevice && n && !reg_has(g_pinned, s, n)) {
        auto snap = std::make_shared<std::vector<uint8_t>>((const uint8_t *)s, (const uint8_t *)s + n);
        legacy_stream()->push([d, snap] { memcpy(d, snap->data(), snap->size()); });
        return cudaSuccess;
    }
    cudaDeviceSynchronize();
    memcpy(d, s, n);
    return cudaSuccess;
}
cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind kind, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    if (kind == cudaMemcpyHostToDevice && inject_failure()) return cudaErrorUnknown;
    if (kind == cudaMemcpyDeviceToHost && getenv("FAKE_CUDA_FAIL_D2H") && inject_failure()) return cudaErrorUnknown;
    if (kind == cudaMemcpyHostToDevice && !reg_has(g_pinned, s, n)) {
        auto snap = std::make_shared<std::vector<uint8_t>>((const uint8_t *)s, (const uint8_t *)s + n);
        on_stream(st, [d, snap] { memcpy(d, snap->data(), snap->size()); });
        return cudaSuccess;
    }
    on_stream(st, [d, s, n] { memcpy(d, s, n); });
    if (kind == cudaMemcpyDeviceToHost && !reg_has(g_pinned, d, n) && st) st->drain();
    return cudaSuccess;
}
cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned)
{
    if (alloc_should_fail()) { *s = nullptr; return cudaErrorMemoryAllocation; }
    *s = new fakeStream();
    std::lock_guard<std::mutex> g(g_reg_mu);
    g_streams.push_back(*s);
    return cudaSuccess;
}
cudaError_t cudaStreamDestroy(cudaStream_t s)
{
    if (!s) return cudaSuccess;
    s->drain();
    { std::lock_guard<std::mutex> g(s->mu); s->stop = true; }
    s->cv.notify_all();
    s->th.join();
    { std::lock_guard<std::mutex> g(g_reg_mu); for (auto &x : g_streams) if (x == s) { x = g_streams.back(); g_streams.pop_back(); break; } }
    delete s;
    return cudaSuccess;
}
cudaError_t cudaStreamSynchronize(cudaStream_t s) { if (s) s->drain(); return cudaSuccess; }
cudaError_t cudaEventCreate(cudaEvent_t *e) { if (alloc_should_fail()) { *e = nullptr; return cudaErrorMemoryAllocation; } *e = new fakeEvent(); return cudaSuccess; }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { if (alloc_should_fail()) { *e = nullptr; return cudaErrorMemoryAllocation; } *e = new fakeEvent(); return cudaSuccess; }
cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
cudaError_t cudaEventRecord(cudaEvent_t ev, cudaStream_t s)
{
    std::shared_ptr<EvState> e = ev->st;
    uint64_t gen;
    { std::lock_guard<std::mutex> g(e->mu); gen = ++e->recorded; }
    on_stream(s, [e, gen] {
        { std::lock_guard<std::mutex> g(e->mu); if (e->done < gen) e->done = gen; }
        e->cv.notify_all();
    });
    return cudaSuccess;
}
cudaError_t cudaEventQuery(cudaEvent_t ev)
{
    std::lock_guard<std::mutex> g(ev->st->mu);
    if (ev->st->done >= ev->st->recorded) return cudaSuccess;
    tl_last_error = cudaErrorNotReady;
    return cudaErrorNotReady;
}
cudaError_t cudaEventSynchronize(cudaEvent_t ev)
{
    std::shared_ptr<EvState> e = ev->st;
    std::unique_lock<std::mutex> g(e->mu);
    const uint64_t gen = e->recorded;
    e->cv.wait(g, [&] { return e->done >= gen; });
    return cudaSuccess;
}
cudaError_t cudaStreamWaitEvent(cudaStream_t s, cudaEvent_t ev, unsigned)
{
    std::shared_ptr<EvState> e = ev->st;
    uint64_t gen;
    { std::lock_guard<std::mutex> g(e->mu); gen = e->recorded; }
    on_stream(s, [e, gen] {
        std::unique_lock<std::mutex> g(e->mu);
        e->cv.wait(g, [&] { return e->done >= gen; });
    });
    return cudaSuccess;
}
cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t, cudaEvent_t) { *ms = 0.001f; return cudaSuccess; }
}

namespace dm {

// One HashJob, the way every real kernel shape treats it.
static void run_job(const HashJob &jb, uint32_t *states, uint32_t *digests)
{
    // FAKE_CUDA_NULL_KERNEL=1: skip the hashing (digests are then meaningless) - for measuring the engine's HOST-side
    // cost per body on the CPU box (tools: tests/native/host_cost_probe.py), where the oracle would dominate
    static const char *null_mode = getenv("FAKE_CUDA_NULL_KERNEL");      // "2": not even the fused copy (bulk_cost_probe.py)
    static const bool null_kernel = null_mode != nullptr, null_copy = null_mode && null_mode[0] != '2';
    if (null_kernel) {
        if (null_copy && jb.nbytes && jb.dst) memcpy(jb.dst, jb.src, jb.nbytes);
        if (jb.flags & JOB_FINAL) {                     // a well-mixed stand-in (distinct per source address and length), not a hash
            uint32_t w[8];
            uint64_t x = (uint64_t)(uintptr_t)jb.src * 0x9E3779B97F4A7C15ull + jb.total_len;
            for (int i = 0; i < 8; i += 2) {
                x += 0x9E3779B97F4A7C15ull;
                uint64_t z = x;
                z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; z ^= z >> 31;
                w[i] = (uint32_t)z; w[i + 1] = (uint32_t)(z >> 32);
            }
            memcpy(digests + 8ull * jb.slot, w, 32);
        }
        return;
    }
    dmo_sha256_ctx c;
    if (jb.flags & JOB_INIT) dmo_sha256_init(&c);
    else {
        memcpy(c.h, states + 8ull * jb.slot, 32);
        c.nbuf = 0;
        c.nbytes = 0;
    }
    if (jb.nbytes) {
        if (jb.dst) memcpy(jb.dst, jb.src, jb.nbytes);
        if (jb.flags & JOB_FINAL) dmo_sha256_update(&c, jb.src, jb.nbytes);
        else dmo_sha256_update(&c, jb.src, jb.nbytes & ~63ull);      // non-final jobs are whole blocks by contract
    }
    if (jb.flags & JOB_FINAL) {
        c.nbytes = jb.total_len;                                     // padding carries the whole-blob length
        uint8_t out[32];
        dmo_sha256_final(&c, out);
        uint32_t w[8];
        for (int i = 0; i < 8; ++i) w[i] = ((uint32_t)out[4 * i] << 24) | ((uint32_t)out[4 * i + 1] << 16) | ((uint32_t)out[4 * i + 2] << 8) | out[4 * i + 3];
        memcpy(states + 8ull * jb.slot, w, 32);
        memcpy(digests + 8ull * jb.slot, w, 32);
    } else {
        memcpy(states + 8ull * jb.slot, c.h, 32);
    }
}

// the "kernel" runs later, on the stream's thread, reading the job table that an earlier copy on the
// same stream delivered
static cudaError_t run_all(const HashJob *jobs, uint32_t n, uint32_t *states, uint32_t *digests, cudaStream_t st)
{
    if (inject_failure()) return cudaErrorUnknown;
    on_stream(st, [jobs, n, states, digests] { for (uint32_t i = 0; i < n; ++i) run_job(jobs[i], states, digests); });
    return cudaGetLastError();                   // as the real launch wrappers end (sha256_kernels.cu)
}
cudaError_t launch_sha256_wide(const HashJob *j, uint32_t n, uint32_t *s, uint32_t *d, cudaStream_t st, int) { return run_all(j, n, s, d, st); }
cudaError_t launch_sha256_deep(const HashJob *j, uint32_t n, uint32_t *s, uint32_t *d, cudaStream_t st, int) { return run_all(j, n, s, d, st); }
cudaError_t launch_sha256_group(const HashJob *j, uint32_t n, uint32_t *s, uint32_t *d, cudaStream_t st, int, int) { return run_all(j, n, s, d, st); }

cudaError_t launch_synth_fill(uint64_t seed, uint64_t blob, uint64_t off, void *dst, size_t len, cudaStream_t st)
{
    on_stream(st, [=] { dmo_blob_fill(seed, blob, off, dst, len); });
    return cudaGetLastError();
}
cudaError_t launch_synth_fill_many(uint64_t seed, uint64_t first, void *base, const uint64_t *offs, const uint64_t *lens,
                                   uint32_t n, uint64_t, uint64_t, cudaStream_t st)
{
    on_stream(st, [=] { for (uint32_t i = 0; i < n; ++i) dmo_blob_fill(seed, first + i, 0, static_cast<uint8_t *>(base) + offs[i], lens[i]); });
    return cudaGetLastError();
}

}  // namespace dm
