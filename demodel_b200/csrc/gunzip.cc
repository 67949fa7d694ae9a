// dm_gunzip: inflate a gzip (RFC 1952) or zlib (RFC 1950) body - host code, no dependencies.
//
// Why it is on this path: registries answer manifest requests with `Content-Encoding: gzip`, and the one
// cached body the reference documents is exactly that (demodel/CONTRIBUTING.md:76-99 is the hexdump,
// :116 says the cache kept it encoded).  The manifest hook (dm_manifest_parse -> dm_manifest_prefetch) needs
// the JSON, so the tee inflates such a body first.  Blob bodies themselves (LFS files, OCI layers) are
// served identity-encoded and never come through here.
//
// DEFLATE (RFC 1951) decoder, table driven: every Huffman code set is expanded into a flat table indexed by
// the next `maxbits` input bits (LSB first, i.e. by the bit-reversed code), entry = symbol and code length.
// Input is untrusted: every read is bounds-checked, over-subscribed and incomplete code sets are rejected
// (except the single-code distance set RFC 1951 §3.2.7 allows), distances must lie inside what has been
// produced, and CRC-32 / Adler-32 and the stated length are verified.  Fuzzed under ASan/UBSan by
// tests/native/fuzz_gunzip.cc.
#include "../../include/demodel_b200.h"

#include <cstdint>
#include <cstring>
#include <vector>

namespace {

struct Bits {
    const uint8_t *p, *end;
    uint64_t acc = 0;
    int n = 0;
    bool fill(int need)            // make `need` (<= 32) bits available; false at end of input
    {
        while (n < need) {
            if (p == end) return false;
            acc |= (uint64_t)*p++ << n;
            n += 8;
        }
        return true;
    }
    bool get(int k, uint32_t *v)
    {
        if (!fill(k)) return false;
        *v = (uint32_t)(acc & ((1ull << k) - 1));
        acc >>= k; n -= k;
        return true;
    }
    void align() { acc >>= (n & 7); n -= (n & 7); }
};

struct Table {
    std::vector<uint16_t> e;       // (symbol << 4) | length, 0 = no code
    int maxbits = 0;
};

// Canonical Huffman (RFC 1951 §3.2.2) from code lengths.  Returns false for a set that is over-subscribed,
// or incomplete unless `allow_single` and it has at most one code.
bool build(Table &t, const uint8_t *len, int nsym, bool allow_single)
{
    int count[16] = {0};
    for (int i = 0; i < nsym; ++i) count[len[i]]++;
    count[0] = 0;
    int maxbits = 0, used = 0;
    for (int l = 1; l <= 15; ++l) if (count[l]) { maxbits = l; used += count[l]; }
    t.maxbits = maxbits ? maxbits : 1;
    t.e.assign((size_t)1 << t.maxbits, 0);
    if (used == 0) return allow_single;                     // no codes at all: legal only where none will be used
    long left = 1;                                           // Kraft sum check
    for (int l = 1; l <= 15; ++l) {
        left <<= 1;
        left -= count[l];
        if (left < 0) return false;
    }
    if (left > 0 && !(allow_single && used == 1)) return false;
    uint32_t next[16], code = 0;
    for (int l = 1; l <= 15; ++l) { code = (code + (uint32_t)count[l - 1]) << 1; next[l] = code; }
    for (int s = 0; s < nsym; ++s) {
        const int l = len[s];
        if (!l) continue;
        uint32_t c = next[l]++, r = 0;
        for (int b = 0; b < l; ++b) r |= ((c >> b) & 1u) << (l - 1 - b);     // the stream carries codes MSB first
        for (uint32_t k = r; k < t.e.size(); k += 1u << l) t.e[k] = (uint16_t)((s << 4) | l);
    }
    return true;
}

bool decode(Bits &in, const Table &t, int *sym)
{
    in.fill(t.maxbits);                                       // near the end fewer bits may be left: that is fine
    const uint16_t ent = t.e[(size_t)(in.acc & ((1ull << t.maxbits) - 1))];
    const int l = ent & 15;
    if (!l || l > in.n) return false;
    in.acc >>= l; in.n -= l;
    *sym = ent >> 4;
    return true;
}

const uint16_t kLenBase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
const uint8_t kLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
const uint16_t kDistBase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
                                4097, 6145, 8193, 12289, 16385, 24577};
const uint8_t kDistExtra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};

struct Out {
    uint8_t *dst;
    size_t cap, n = 0;       // n counts every byte produced; bytes past cap are dropped (the caller learns the size)
    void put(uint8_t b) { if (n < cap) dst[n] = b; ++n; }
};

// 0 ok, -1 malformed.  Once the output overflows `cap` a back-reference can no longer be resolved, so the
// decoder stops there and reports overflow through out.n > out.cap.
int inflate_blocks(Bits &in, Out &out)
{
    Table lit, dist;
    for (;;) {
        uint32_t final_blk, type;
        if (!in.get(1, &final_blk) || !in.get(2, &type)) return -1;
        if (type == 0) {
            in.align();
            uint32_t len, nlen;
            if (!in.get(16, &len) || !in.get(16, &nlen) || (len ^ 0xffffu) != nlen) return -1;
            for (uint32_t i = 0; i < len; ++i) {
                uint32_t b;
                if (!in.get(8, &b)) return -1;
                out.put((uint8_t)b);
            }
        } else if (type == 1 || type == 2) {
            uint8_t lens[320];
            if (type == 1) {                                  // RFC 1951 §3.2.6
                int i = 0;
                for (; i < 144; ++i) lens[i] = 8;
                for (; i < 256; ++i) lens[i] = 9;
                for (; i < 280; ++i) lens[i] = 7;
                for (; i < 288; ++i) lens[i] = 8;
                if (!build(lit, lens, 288, false)) return -1;
                for (i = 0; i < 32; ++i) lens[i] = 5;         // 30 and 31 are part of the code but never valid
                if (!build(dist, lens, 32, true)) return -1;
            } else {                                          // §3.2.7
                uint32_t hlit, hdist, hclen;
                if (!in.get(5, &hlit) || !in.get(5, &hdist) || !in.get(4, &hclen)) return -1;
                hlit += 257; hdist += 1; hclen += 4;
                if (hlit > 286 || hdist > 30) return -1;
                static const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
                uint8_t cl[19] = {0};
                for (uint32_t i = 0; i < hclen; ++i) {
                    uint32_t v;
                    if (!in.get(3, &v)) return -1;
                    cl[order[i]] = (uint8_t)v;
                }
                Table clt;
                if (!build(clt, cl, 19, false)) return -1;
                uint32_t i = 0;
                while (i < hlit + hdist) {
                    int sym;
                    if (!decode(in, clt, &sym)) return -1;
                    if (sym < 16) { lens[i++] = (uint8_t)sym; continue; }
                    uint32_t rep, prev = 0;
                    if (sym == 16) {
                        if (i == 0 || !in.get(2, &rep)) return -1;
                        prev = lens[i - 1]; rep += 3;
                    } else if (sym == 17) { if (!in.get(3, &rep)) return -1; rep += 3; }
                    else { if (!in.get(7, &rep)) return -1; rep += 11; }
                    if (i + rep > hlit + hdist) return -1;
                    while (rep--) lens[i++] = (uint8_t)prev;
                }
                if (lens[256] == 0) return -1;                // no end-of-block code
                if (!build(lit, lens, (int)hlit, true)) return -1;          // a lone end-of-block code is legal
                if (!build(dist, lens + hlit, (int)hdist, true)) return -1;
            }
            for (;;) {
                int sym;
                if (!decode(in, lit, &sym)) return -1;
                if (sym < 256) { out.put((uint8_t)sym); continue; }
                if (sym == 256) break;
                sym -= 257;
                if (sym >= 29) return -1;
                uint32_t extra;
                if (!in.get(kLenExtra[sym], &extra)) return -1;
                const uint32_t len = kLenBase[sym] + extra;
                int ds;
                if (!decode(in, dist, &ds) || ds >= 30) return -1;
                if (!in.get(kDistExtra[ds], &extra)) return -1;
                const size_t d = kDistBase[ds] + extra;
                if (d > out.n) return -1;                     // reaches before the start of the output
                if (out.n + len > out.cap) { out.n += len; return 0; }       // overflow: stop (see above)
                for (uint32_t k = 0; k < len; ++k) { out.dst[out.n] = out.dst[out.n - d]; ++out.n; }
            }
        } else return -1;
        if (out.n > out.cap) return 0;
        if (final_blk) return 0;
    }
}

uint32_t crc32_of(const uint8_t *p, size_t n)
{
    static uint32_t table[256];
    static bool ready = false;
    if (!ready) {
        for (uint32_t i = 0; i < 256; ++i) {
            uint32_t c = i;
            for (int k = 0; k < 8; ++k) c = (c & 1) ? 0xedb88320u ^ (c >> 1) : c >> 1;
            table[i] = c;
        }
        ready = true;
    }
    uint32_t c = 0xffffffffu;
    for (size_t i = 0; i < n; ++i) c = table[(c ^ p[i]) & 0xff] ^ (c >> 8);
    return ~c;
}

uint32_t adler32_of(const uint8_t *p, size_t n)
{
    uint32_t a = 1, b = 0;
    for (size_t i = 0; i < n; ++i) { a = (a + p[i]) % 65521u; b = (b + a) % 65521u; }
    return (b << 16) | a;
}

uint32_t le32(const uint8_t *p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }

}  // namespace

extern "C" int dm_gunzip(const void *src, size_t len, void *dst, size_t cap, size_t *out_len)
{
    if (out_len) *out_len = 0;
    if (!src || (!dst && cap) || len < 6) return DM_EINVAL;
    const uint8_t *p = static_cast<const uint8_t *>(src), *end = p + len;
    bool gz;
    if (p[0] == 0x1f && p[1] == 0x8b) {                       // RFC 1952 member header
        if (len < 18 || p[2] != 8 || (p[3] & 0xe0)) return DM_EINVAL;
        const uint8_t flg = p[3];
        p += 10;
        if (flg & 4) {                                        // FEXTRA
            if (end - p < 2) return DM_EINVAL;
            const size_t xl = (size_t)p[0] | (size_t)p[1] << 8;
            p += 2;
            if ((size_t)(end - p) < xl) return DM_EINVAL;
            p += xl;
        }
        for (int bit = 8; bit <= 16; bit <<= 1)               // FNAME, FCOMMENT: NUL-terminated
            if (flg & bit) {
                while (p < end && *p) ++p;
                if (p == end) return DM_EINVAL;
                ++p;
            }
        if (flg & 2) { if (end - p < 2) return DM_EINVAL; p += 2; }          // FHCRC
        if (end - p < 8) return DM_EINVAL;
        gz = true;
    } else if ((p[0] & 0x0f) == 8 && (((uint32_t)p[0] << 8) | p[1]) % 31 == 0 && !(p[1] & 0x20)) {   // RFC 1950, no preset dictionary
        p += 2;
        gz = false;
    } else return DM_EINVAL;
    const size_t trailer = gz ? 8 : 4;
    if ((size_t)(end - p) < trailer) return DM_EINVAL;
    Bits in{p, end - trailer};
    Out out{static_cast<uint8_t *>(dst), cap};
    if (inflate_blocks(in, out) != 0) return DM_EINVAL;
    if (out.n > cap) {                                        // too small: the gzip trailer says how much is needed
        if (out_len) *out_len = gz ? (size_t)le32(end - 4) : out.n;
        return DM_ENOMEM;
    }
    const uint8_t *t = end - trailer;
    if (gz) {
        if (le32(t) != crc32_of(out.dst, out.n) || le32(t + 4) != (uint32_t)out.n) return DM_EINVAL;
    } else {
        const uint32_t want = (uint32_t)t[0] << 24 | (uint32_t)t[1] << 16 | (uint32_t)t[2] << 8 | t[3];
        if (want != adler32_of(out.dst, out.n)) return DM_EINVAL;
    }
    if (out_len) *out_len = out.n;
    return DM_OK;
}
