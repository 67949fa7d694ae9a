/*
 * oracle/sha256_oracle.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the digest algorithm the hot path must reproduce.
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load this; nothing under demodel_b200/ does.
 *
 * What it restates.  BASELINE.json's north_star names Go's standard-library
 * crypto/sha256 (Go 1.24.3 per demodel/go.mod:3) as the reference
 * digest.  The reference repository itself has NO call site of it — the
 * response hook at demodel/cmd/demodel/start.go:201-204 only prints
 * and returns resp unchanged, and grep finds no sha256 import (SURVEY.md §0).
 * crypto/sha256 is an implementation of FIPS 180-4 SHA-256, so this file
 * restates FIPS 180-4 §4.1.2 (functions), §4.2.2 (constants), §5.1.1
 * (padding), §5.3.3 (initial hash value) and §6.2.2 (compression) directly,
 * with the streaming init/update/final shape of Go's hash.Hash
 * (Write / Sum) that an io.Copy-style loop would drive.
 *
 * Pinning.  The reference ships no golden vectors for this path ("parity
 * unpinned by the reference", SURVEY.md §8c).  The oracle is pinned instead
 * against the FIPS 180-4 / NIST CAVP known answers, against OpenSSL
 * EVP_sha256 and Python hashlib on the same bytes, and against the one
 * byte-level fixture the reference holds (CONTRIBUTING.md:76-99), see
 * tests/test_oracle.py and tests/golden/.
 *
 * Plain scalar C on purpose: it shares no code, table layout or loop
 * structure with the CUDA kernels it checks.
 */
#include <stdint.h>
#include <stddef.h>
#include <string.h>

typedef struct {
    uint32_t h[8];      /* FIPS 180-4 §6.2.1 working hash value H(i) */
    uint64_t nbytes;    /* message bytes absorbed so far */
    uint8_t  buf[64];   /* partial block */
    uint32_t nbuf;
} dmo_sha256_ctx;

/* FIPS 180-4 §4.2.2: first 32 bits of the fractional parts of the cube
 * roots of the first 64 primes. */
static const uint32_t K256[64] = {
    0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u,
    0x923f82a4u, 0xab1c5ed5u, 0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u,
    0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u, 0xe49b69c1u, 0xefbe4786u,
    0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau,
    0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u,
    0x06ca6351u, 0x14292967u, 0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u,
    0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u, 0xa2bfe8a1u, 0xa81a664bu,
    0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u,
    0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au,
    0x5b9cca4fu, 0x682e6ff3u, 0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u,
    0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u,
};

static uint32_t rotr32(uint32_t x, unsigned n) { return (x >> n) | (x << (32u - n)); }

/* FIPS 180-4 §6.2.2: one 512-bit block. */
static void dmo_compress(uint32_t h[8], const uint8_t blk[64])
{
    uint32_t w[64];
    for (int t = 0; t < 16; ++t)
        w[t] = ((uint32_t)blk[4 * t] << 24) | ((uint32_t)blk[4 * t + 1] << 16) |
               ((uint32_t)blk[4 * t + 2] << 8) | (uint32_t)blk[4 * t + 3];
    for (int t = 16; t < 64; ++t) {
        uint32_t s0 = rotr32(w[t - 15], 7) ^ rotr32(w[t - 15], 18) ^ (w[t - 15] >> 3);
        uint32_t s1 = rotr32(w[t - 2], 17) ^ rotr32(w[t - 2], 19) ^ (w[t - 2] >> 10);
        w[t] = s1 + w[t - 7] + s0 + w[t - 16];
    }
    uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
    for (int t = 0; t < 64; ++t) {
        uint32_t S1 = rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25);
        uint32_t ch = (e & f) ^ (~e & g);
        uint32_t t1 = hh + S1 + ch + K256[t] + w[t];
        uint32_t S0 = rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22);
        uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
        uint32_t t2 = S0 + mj;
        hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

/* FIPS 180-4 §5.3.3 */
void dmo_sha256_init(dmo_sha256_ctx *c)
{
    static const uint32_t iv[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au,
                                   0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
    memcpy(c->h, iv, sizeof iv);
    c->nbytes = 0;
    c->nbuf = 0;
}

/* hash.Hash.Write: absorb len bytes; any split of the message into calls
 * yields the same digest. */
void dmo_sha256_update(dmo_sha256_ctx *c, const void *data, size_t len)
{
    const uint8_t *p = (const uint8_t *)data;
    c->nbytes += len;
    if (c->nbuf) {
        size_t take = 64 - c->nbuf;
        if (take > len) take = len;
        memcpy(c->buf + c->nbuf, p, take);
        c->nbuf += (uint32_t)take; p += take; len -= take;
        if (c->nbuf == 64) { dmo_compress(c->h, c->buf); c->nbuf = 0; }
    }
    while (len >= 64) { dmo_compress(c->h, p); p += 64; len -= 64; }
    if (len) { memcpy(c->buf, p, len); c->nbuf = (uint32_t)len; }
}

/* hash.Hash.Sum: FIPS 180-4 §5.1.1 padding (0x80, zeros, 64-bit big-endian
 * bit length), then big-endian serialisation of H. */
void dmo_sha256_final(dmo_sha256_ctx *c, uint8_t out[32])
{
    uint64_t bits = c->nbytes * 8u;
    uint8_t pad[72];
    size_t npad = (c->nbuf < 56) ? (56 - c->nbuf) : (120 - c->nbuf);
    memset(pad, 0, sizeof pad);
    pad[0] = 0x80;
    for (int i = 0; i < 8; ++i) pad[npad + i] = (uint8_t)(bits >> (56 - 8 * i));
    uint64_t keep = c->nbytes;
    dmo_sha256_update(c, pad, npad + 8);
    c->nbytes = keep;
    for (int i = 0; i < 8; ++i) {
        out[4 * i] = (uint8_t)(c->h[i] >> 24); out[4 * i + 1] = (uint8_t)(c->h[i] >> 16);
        out[4 * i + 2] = (uint8_t)(c->h[i] >> 8); out[4 * i + 3] = (uint8_t)c->h[i];
    }
}

void dmo_sha256(const void *data, size_t len, uint8_t out[32])
{
    dmo_sha256_ctx c;
    dmo_sha256_init(&c);
    dmo_sha256_update(&c, data, len);
    dmo_sha256_final(&c, out);
}

/* Streaming in fixed-size pieces, the way an io.Copy loop (32 KiB buffer)
 * would feed hash.Hash. */
void dmo_sha256_chunked(const void *data, size_t len, size_t chunk, uint8_t out[32])
{
    dmo_sha256_ctx c;
    const uint8_t *p = (const uint8_t *)data;
    dmo_sha256_init(&c);
    if (chunk == 0) chunk = 32768;
    while (len) {
        size_t n = len < chunk ? len : chunk;
        dmo_sha256_update(&c, p, n);
        p += n; len -= n;
    }
    dmo_sha256_final(&c, out);
}

/* Many independent blobs packed back to back: offsets[i]..offsets[i+1]. */
void dmo_sha256_many(const void *base, const uint64_t *offsets, uint32_t n, uint8_t *out)
{
    const uint8_t *p = (const uint8_t *)base;
    for (uint32_t i = 0; i < n; ++i)
        dmo_sha256(p + offsets[i], (size_t)(offsets[i + 1] - offsets[i]), out + 32u * i);
}

unsigned dmo_ctx_size(void) { return (unsigned)sizeof(dmo_sha256_ctx); }

/* ------------------------------------------------------------------------
 * Synthetic blob bytes (SURVEY.md §8d): counter-based generator so that the
 * same blob can be produced on the host here and on the device by the
 * product's own generator (demodel_b200/csrc/blobgen.cuh) without shipping
 * bytes.  Byte j of blob b under seed s is byte (j & 7), little-endian, of
 *     splitmix64_finalise(s ^ (b * 0x9E3779B97F4A7C15) ^ ((j >> 3) * 0xD1B54A32D192ED03) + ...)
 * restated independently below; tests assert both generators agree.
 * ---------------------------------------------------------------------- */
static uint64_t dmo_mix64(uint64_t z)
{
    z ^= z >> 30; z *= 0xBF58476D1CE4E5B9ull;
    z ^= z >> 27; z *= 0x94D049BB133111EBull;
    z ^= z >> 31;
    return z;
}

uint64_t dmo_blob_word(uint64_t seed, uint64_t blob, uint64_t word_index)
{
    uint64_t k = dmo_mix64(seed + 0x9E3779B97F4A7C15ull * (blob + 1));
    return dmo_mix64(k + 0xD1B54A32D192ED03ull * (word_index + 1));
}

void dmo_blob_fill(uint64_t seed, uint64_t blob, uint64_t byte_off, void *dst, size_t len)
{
    uint8_t *p = (uint8_t *)dst;
    uint64_t j = byte_off;
    while (len) {
        uint64_t w = dmo_blob_word(seed, blob, j >> 3);
        unsigned sh = (unsigned)(j & 7);
        size_t n = 8 - sh;
        if (n > len) n = len;
        for (size_t i = 0; i < n; ++i) p[i] = (uint8_t)(w >> (8 * (sh + i)));
        p += n; j += n; len -= n;
    }
}
