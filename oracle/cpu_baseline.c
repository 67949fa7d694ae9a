/*
 * oracle/cpu_baseline.c — TEST / MEASUREMENT INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * The CPU arm of the benchmark: the hash-and-cache loop north_star attributes
 * to the reference ("Go io.Copy + crypto/sha256"), restated for this image.
 * The reference holds no such loop (SURVEY.md §0: the hooks at
 * demodel/cmd/demodel/start.go:197-204 only print) and Go is not
 * installed, so the stand-in is what that loop would be:
 *
 *     for each blob (one goroutine per connection -> one thread per blob):
 *         h := sha256.New()
 *         io.Copy(io.MultiWriter(h, cacheFile), resp.Body)   // 32 KiB reads
 *         h.Sum(nil) == expected
 *
 * with OpenSSL 3 EVP_sha256 standing in for Go's crypto/sha256 — both are
 * FIPS 180-4 and both dispatch to the SHA-NI instructions on amd64 when the
 * CPU has them, so per-core speed is comparable.  Every report that quotes a
 * number from here must say "OpenSSL stand-in for Go crypto/sha256".
 *
 * dmb_hash_and_cache(): `nthreads` workers pull blob indices from a shared
 * counter; each streams its blob in `chunk`-byte pieces from the source
 * buffer through EVP_DigestUpdate and memcpy()s the piece into the in-memory
 * cache region (the CAS write), exactly one read and one write per blob
 * byte.  Returns wall seconds; digests land in out[32*i].
 */
#define _GNU_SOURCE
#include <openssl/evp.h>
#include <pthread.h>
#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include <time.h>

typedef struct {
    const uint8_t *src;
    uint8_t *cache;              /* may be NULL: hash only */
    const uint64_t *offsets;     /* n+1 entries */
    uint32_t n;
    size_t chunk;
    uint8_t *out;
    volatile uint32_t next;
    int failed;
} dmb_job;

static void *dmb_worker(void *arg)
{
    dmb_job *j = (dmb_job *)arg;
    EVP_MD_CTX *ctx = EVP_MD_CTX_new();
    const EVP_MD *md = EVP_sha256();
    if (!ctx) { j->failed = 1; return NULL; }
    for (;;) {
        uint32_t i = __atomic_fetch_add(&j->next, 1u, __ATOMIC_RELAXED);
        if (i >= j->n) break;
        uint64_t off = j->offsets[i], end = j->offsets[i + 1];
        unsigned int dl = 0;
        if (EVP_DigestInit_ex(ctx, md, NULL) != 1) { j->failed = 1; break; }
        while (off < end) {
            size_t nb = (size_t)(end - off);
            if (nb > j->chunk) nb = j->chunk;
            EVP_DigestUpdate(ctx, j->src + off, nb);
            if (j->cache) memcpy(j->cache + off, j->src + off, nb);
            off += nb;
        }
        EVP_DigestFinal_ex(ctx, j->out + 32u * i, &dl);
    }
    EVP_MD_CTX_free(ctx);
    return NULL;
}

double dmb_hash_and_cache(const void *src, void *cache, const uint64_t *offsets, uint32_t n,
                          size_t chunk, int nthreads, uint8_t *out)
{
    dmb_job j;
    pthread_t th[1024];
    struct timespec t0, t1;
    if (nthreads < 1) nthreads = 1;
    if (nthreads > 1024) nthreads = 1024;
    j.src = (const uint8_t *)src; j.cache = (uint8_t *)cache; j.offsets = offsets; j.n = n;
    j.chunk = chunk ? chunk : 32768; j.out = out; j.next = 0; j.failed = 0;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    for (int t = 0; t < nthreads; ++t) pthread_create(&th[t], NULL, dmb_worker, &j);
    for (int t = 0; t < nthreads; ++t) pthread_join(th[t], NULL);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    if (j.failed) return -1.0;
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}

/* Same loop with the cache on a filesystem (BASELINE.md: "write the bytes to a tmpfs content-addressed
 * file"): each blob is streamed to <dir>/<index>.part in `chunk` writes and renamed to its hex digest. */
#include <fcntl.h>
#include <stdio.h>
#include <unistd.h>

typedef struct {
    dmb_job j;
    const char *dir;
} dmb_fjob;

static void *dmb_file_worker(void *arg)
{
    dmb_fjob *fj = (dmb_fjob *)arg;
    dmb_job *j = &fj->j;
    EVP_MD_CTX *ctx = EVP_MD_CTX_new();
    const EVP_MD *md = EVP_sha256();
    char tmp[4096], fin[4096];
    if (!ctx) { j->failed = 1; return NULL; }
    for (;;) {
        uint32_t i = __atomic_fetch_add(&j->next, 1u, __ATOMIC_RELAXED);
        if (i >= j->n) break;
        uint64_t off = j->offsets[i], end = j->offsets[i + 1];
        unsigned int dl = 0;
        snprintf(tmp, sizeof tmp, "%s/%u.part", fj->dir, i);
        int fd = open(tmp, O_CREAT | O_TRUNC | O_WRONLY, 0644);
        if (fd < 0 || EVP_DigestInit_ex(ctx, md, NULL) != 1) { j->failed = 1; break; }
        while (off < end) {
            size_t nb = (size_t)(end - off);
            if (nb > j->chunk) nb = j->chunk;
            EVP_DigestUpdate(ctx, j->src + off, nb);
            size_t w = 0;
            while (w < nb) {
                ssize_t r = write(fd, j->src + off + w, nb - w);
                if (r <= 0) { j->failed = 1; break; }
                w += (size_t)r;
            }
            off += nb;
        }
        close(fd);
        uint8_t *d = j->out + 32u * i;
        EVP_DigestFinal_ex(ctx, d, &dl);
        int k = snprintf(fin, sizeof fin, "%s/", fj->dir);
        for (int b = 0; b < 32; ++b) k += snprintf(fin + k, sizeof fin - (size_t)k, "%02x", d[b]);
        rename(tmp, fin);
    }
    EVP_MD_CTX_free(ctx);
    return NULL;
}

double dmb_hash_and_cache_files(const void *src, const char *dir, const uint64_t *offsets, uint32_t n,
                                size_t chunk, int nthreads, uint8_t *out)
{
    dmb_fjob fj;
    pthread_t th[1024];
    struct timespec t0, t1;
    if (nthreads < 1) nthreads = 1;
    if (nthreads > 1024) nthreads = 1024;
    fj.j.src = (const uint8_t *)src; fj.j.cache = NULL; fj.j.offsets = offsets; fj.j.n = n;
    fj.j.chunk = chunk ? chunk : 32768; fj.j.out = out; fj.j.next = 0; fj.j.failed = 0;
    fj.dir = dir;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    for (int t = 0; t < nthreads; ++t) pthread_create(&th[t], NULL, dmb_file_worker, &fj);
    for (int t = 0; t < nthreads; ++t) pthread_join(th[t], NULL);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    if (fj.j.failed) return -1.0;
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}

/* One-shot digest through OpenSSL: the second, independent oracle. */
int dmb_openssl_sha256(const void *data, size_t len, uint8_t out[32])
{
    unsigned int dl = 0;
    return EVP_Digest(data, len, out, &dl, EVP_sha256(), NULL) == 1 ? 0 : -1;
}
