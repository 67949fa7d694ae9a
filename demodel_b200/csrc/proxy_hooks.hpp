// Host half of the path, above the C-ABI: what the reference's two goproxy
// hooks become once the engine is wired in.  The reference is Go and this
// image has no Go toolchain, so the wrappers are written in C++ with the same
// shape the Go ones have in go/demodel_b200.go (io.ReadCloser semantics), and
// the parity tests drive these instead.
//
//   BodyTee    — installed by the OnResponse hook around resp.Body
//                (demodel/cmd/demodel/start.go:201-204 returns resp
//                unchanged today).  Read(p) reads from upstream, tees the
//                bytes into the engine, returns them to goproxy's copy loop;
//                at EOF it finishes the stream and records the verdict;
//                Close() before EOF aborts (client went away / upstream error).
//   HitReader  — the body of the *http.Response the OnRequest hook returns to
//                short-circuit upstream (start.go:197-200 returns req,nil
//                today).  Read(p) serves bytes from the CAS.
#pragma once
#include "../../include/demodel_b200.h"

#include <cstddef>
#include <cstdint>
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

namespace dm {

// ---- which blob does a request name?  (OnRequest, start.go:197-200, is handed a URL, not a digest) ----
// OCI / Ollama blob URLs carry the digest: /v2/<name>/blobs/sha256:<64 hex> (some mirrors write sha256-<hex>).
inline bool DigestFromURL(const char *url, uint8_t out[32])
{
    if (!url) return false;
    for (const char *p = url; (p = strstr(p, "sha256")) != nullptr; p += 6) {
        if (p[6] != ':' && p[6] != '-') continue;
        const char *h = p + 7;
        auto nib = [](char c) { return c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : c >= 'A' && c <= 'F' ? c - 'A' + 10 : -1; };
        int i = 0;
        for (; i < 64; ++i) if (nib(h[i]) < 0) break;
        if (i < 64 || nib(h[64]) >= 0) continue;                 // not exactly 64 hex digits
        for (i = 0; i < 32; ++i) out[i] = (uint8_t)(nib(h[2 * i]) << 4 | nib(h[2 * i + 1]));
        return true;
    }
    return false;
}
// HuggingFace resolve/ URLs (and anything else without a digest in it) go through the alias index that the
// tee fills when a body fetched under that URL verifies.
inline bool ResolveRequest(dm_engine *e, const char *url, uint8_t out[32])
{
    return DigestFromURL(url, out) || dm_cache_alias_get(e, url, out) == DM_OK;
}

// io.Reader: returns bytes read, 0 at EOF, <0 on error.
struct Upstream {
    virtual ~Upstream() {}
    virtual long Read(void *p, size_t n) = 0;
};

class BodyTee {
public:
    BodyTee(dm_engine *e, Upstream *up, const uint8_t *expect, uint64_t content_length)
        : e_(e), up_(up)
    {
        rc_ = dm_stream_open(e, expect, content_length, &id_);
        open_ = rc_ == DM_OK;
    }
    ~BodyTee() { Close(); }

    // Reads up to n bytes from upstream into p (goproxy's buffer) and tees them.
    long Read(void *p, size_t n)
    {
        if (rc_ != DM_OK) return rc_;
        if (eof_) return 0;
        const long got = up_->Read(p, n);
        if (got < 0) { Abort(); return got; }
        if (got == 0) return Finish() == DM_OK ? 0 : rc_;
        rc_ = dm_stream_write(e_, id_, p, (size_t)got);
        if (rc_ != DM_OK) { Abort(); return rc_; }
        return got;
    }

    // Zero-copy form: the upstream read lands directly in the pinned ring;
    // *view points at the bytes for the client-side write.  The window belongs
    // to the caller only between dm_stream_acquire and dm_stream_commit (after
    // the commit the engine may DMA the slab and hand it to another stream at
    // any time), so the commit is DEFERRED: the view stays valid until the next
    // call on this tee (ReadInPlace / Pump / Wait / Close), which commits it
    // first - the lifetime rule of a bufio.Reader.Peek slice.
    long ReadInPlace(const void **view, size_t max_n)
    {
        if (rc_ != DM_OK) return rc_;
        if (eof_) return 0;
        if (!CommitHeld()) return rc_;
        void *win = nullptr;
        size_t cap = 0;
        rc_ = dm_stream_acquire(e_, id_, &win, &cap);
        if (rc_ != DM_OK) { Abort(); return rc_; }
        const long got = up_->Read(win, cap < max_n ? cap : max_n);
        if (got <= 0) {
            rc_ = dm_stream_commit(e_, id_, 0);
            if (got < 0 || rc_ != DM_OK) { Abort(); return got < 0 ? got : rc_; }
            return Finish() == DM_OK ? 0 : rc_;
        }
        held_ = (size_t)got;                    // committed by the next call, after the caller has used *view
        has_held_ = true;
        *view = win;
        return got;
    }

    // Multiplexing drivers: Pump() moves one piece like Read()/ReadInPlace() but at EOF only
    // *starts* the final hash (dm_stream_flush); Wait() then collects the verdict.  A Go
    // goroutine would simply block in Read(); an OS thread playing many goroutines must not.
    long Pump(void *scratch, size_t n, bool in_place)
    {
        if (rc_ != DM_OK) return rc_;
        if (eof_ || flushed_) return 0;
        if (!CommitHeld()) return rc_;
        long got;
        if (in_place) {
            void *win = nullptr;
            size_t cap = 0;
            rc_ = dm_stream_acquire(e_, id_, &win, &cap);
            if (rc_ != DM_OK) { Abort(); return rc_; }
            got = up_->Read(win, cap < n ? cap : n);
            int rc2 = dm_stream_commit(e_, id_, got > 0 ? (size_t)got : 0);
            if (got >= 0 && rc2 != DM_OK) { rc_ = rc2; Abort(); return rc_; }
        } else {
            got = up_->Read(scratch, n);
            if (got > 0) {
                rc_ = dm_stream_write(e_, id_, scratch, (size_t)got);
                if (rc_ != DM_OK) { Abort(); return rc_; }
            }
        }
        if (got < 0) { Abort(); return got; }
        if (got == 0) {
            rc_ = dm_stream_flush(e_, id_);
            if (rc_ != DM_OK) { Abort(); return rc_; }
            flushed_ = true;
        }
        return got;
    }
    int Wait()
    {
        if (eof_) return rc_;
        if (!CommitHeld()) return rc_;
        return Finish();
    }

    // io.Closer: before EOF this is an abort; after EOF a no-op.
    int Close()
    {
        if (open_ && !eof_) Abort();
        return DM_OK;
    }

    // The request URL this body answers: kept in the sidecar, and - once the body has verified - entered in
    // the alias index so that the next request for the same URL is a hit even though it names no digest.
    void SetURL(const char *url)
    {
        if (!url || !open_) return;
        url_ = url;
        dm_stream_set_meta(e_, id_, "url", url);
    }

    bool done() const { return eof_; }
    bool matched() const { return matched_ != 0; }
    const uint8_t *digest() const { return digest_; }
    int status() const { return rc_; }

private:
    // Hand the window lent out by the last ReadInPlace back to the engine.
    bool CommitHeld()
    {
        if (!has_held_) return true;
        has_held_ = false;
        rc_ = dm_stream_commit(e_, id_, held_);
        if (rc_ != DM_OK) { Abort(); return false; }
        return true;
    }
    int Finish()
    {
        eof_ = true;
        open_ = false;
        rc_ = dm_stream_finish(e_, id_, digest_, &matched_);
        if (rc_ != DM_OK) dm_stream_abort(e_, id_);     // some failures leave the stream open; a released id just says so (ids are never reused)
        else if (matched_ && !url_.empty()) dm_cache_alias_put(e_, url_.c_str(), digest_);     // best effort
        return rc_;
    }
    void Abort()
    {
        if (open_) dm_stream_abort(e_, id_);
        open_ = false;
    }
    dm_engine *e_;
    Upstream *up_;
    uint64_t id_ = 0;
    int rc_ = DM_OK;
    bool open_ = false, eof_ = false, flushed_ = false, has_held_ = false;
    size_t held_ = 0;
    int matched_ = 0;
    uint8_t digest_[32] = {0};
    std::string url_;
};

// The OnResponse hook for MANIFEST responses (Content-Type application/vnd.oci.image.manifest.v1+json,
// application/vnd.docker.distribution.manifest.v2+json): the body passes through to the client unchanged
// while a copy is kept (manifests are a few KiB; capped at 4 MiB); at EOF it is inflated if the response
// carried Content-Encoding: gzip (the reference's documented cached body is one: CONTRIBUTING.md:76-99),
// parsed, and one pre-verified stream per layer that is not cached yet is opened (dm_manifest_prefetch),
// so each layer's extent is reserved and its digest known before the client asks for it.
class ManifestTee {
public:
    ManifestTee(dm_engine *e, Upstream *up, const char *content_encoding)
        : e_(e), up_(up), gzip_(content_encoding && (strcmp(content_encoding, "gzip") == 0 || strcmp(content_encoding, "x-gzip") == 0)),
          identity_(!content_encoding || !*content_encoding || strcmp(content_encoding, "identity") == 0) {}
    long Read(void *p, size_t n)
    {
        const long got = up_->Read(p, n);
        if (got > 0 && !overflow_) {
            if (body_.size() + (size_t)got > kMaxBody) { overflow_ = true; body_.clear(); }
            else body_.insert(body_.end(), static_cast<const uint8_t *>(p), static_cast<const uint8_t *>(p) + got);
        }
        if (got == 0 && !done_) { done_ = true; OnEOF(); }
        return got;
    }
    int status() const { return rc_; }                    // DM_OK, or why the manifest was not used (the body still passed through)
    const std::vector<dm_layer> &layers() const { return layers_; }
    const std::vector<uint64_t> &ids() const { return ids_; }      // stream ids opened by the prefetch (0 = hit / duplicate)
private:
    static constexpr size_t kMaxBody = 4u << 20;
    void OnEOF()
    {
        if (overflow_ || (!gzip_ && !identity_)) { rc_ = DM_EINVAL; return; }     // br / zstd / deflate: not handled, pass through
        std::vector<uint8_t> plain;
        const uint8_t *json = body_.data();
        size_t len = body_.size();
        if (gzip_) {
            size_t need = 0;
            plain.resize(std::max<size_t>(8 * body_.size(), 4096));
            rc_ = dm_gunzip(body_.data(), body_.size(), plain.data(), plain.size(), &need);
            if (rc_ == DM_ENOMEM && need && need <= 16 * kMaxBody) {
                plain.resize(need);
                rc_ = dm_gunzip(body_.data(), body_.size(), plain.data(), plain.size(), &need);
            }
            if (rc_ != DM_OK) return;
            json = plain.data(); len = need;
        }
        uint32_t n = 0;
        layers_.resize(64);
        rc_ = dm_manifest_parse(reinterpret_cast<const char *>(json), len, layers_.data(), (uint32_t)layers_.size(), &n);
        if (rc_ == DM_OK && n > layers_.size()) {
            layers_.resize(n);
            rc_ = dm_manifest_parse(reinterpret_cast<const char *>(json), len, layers_.data(), n, &n);
        }
        if (rc_ != DM_OK) { layers_.clear(); return; }
        layers_.resize(n);
        ids_.assign(n, 0);
        if (n) rc_ = dm_manifest_prefetch(e_, layers_.data(), n, ids_.data());
    }
    dm_engine *e_;
    Upstream *up_;
    bool gzip_, identity_, overflow_ = false, done_ = false;
    int rc_ = DM_OK;
    std::vector<uint8_t> body_;
    std::vector<dm_layer> layers_;
    std::vector<uint64_t> ids_;
};

class HitReader {
public:
    // Verified: Pool.HitVerified (dm_cache_open_verified): a disk-tier blob is served only as the GPU verifies it, and
    // Read returns DM_ECORRUPT / DM_EIO / DM_ECUDA instead of its last byte when it does not hash to its name.
    // VerifiedRing: Pool.HitVerifiedRing (dm_cache_open_verified_ring), the same promise without an HBM extent, for
    // blobs Verified answers with DM_ENOMEM or DM_ESTATE (rc()); its reads go forward only.
    // VerifiedRange: Pool.HitVerifiedRange (dm_cache_open_verified_range), VerifiedRing's promise for the bytes
    // [off, off + len) of a Range: request (len 0: to the end), served by a ring load shared with the blob's other range
    // readers.  Read starts at off and returns 0 at off + len; size() is still the whole blob's (Content-Range).
    enum Mode { Plain, Verified, VerifiedRing, VerifiedRange };
    HitReader(dm_engine *e, const uint8_t digest[32], Mode mode = Plain, uint64_t off = 0, uint64_t len = 0) : e_(e)
    {
        rc_ = mode == Verified       ? dm_cache_open_verified(e, digest, &id_, &size_)
              : mode == VerifiedRing  ? dm_cache_open_verified_ring(e, digest, &id_, &size_)
              : mode == VerifiedRange ? dm_cache_open_verified_range(e, digest, off, len, &id_, &size_)
                                      : dm_cache_open(e, digest, &id_, &size_);
        open_ = rc_ == DM_OK;
        if (mode == VerifiedRange) off_ = off;
    }
    // the bool form is Plain / Verified
    HitReader(dm_engine *e, const uint8_t digest[32], bool verified) : HitReader(e, digest, verified ? Verified : Plain) {}
    // By request URL: a digest in the URL (OCI) or the alias index (HuggingFace resolve/ URLs).
    HitReader(dm_engine *e, const char *url) : e_(e)
    {
        uint8_t d[32];
        rc_ = ResolveRequest(e, url, d) ? dm_cache_open(e, d, &id_, &size_) : (int)DM_ENOENT;
        open_ = rc_ == DM_OK;
    }
    uint64_t id() const { return id_; }
    uint64_t Release() { open_ = false; return id_; }      // hand the open reader to the caller (C-ABI drivers)
    ~HitReader() { Close(); }
    bool hit() const { return open_; }
    int rc() const { return rc_; }              // why it is not a hit: DM_ENOENT (a miss) or the open's error
    uint64_t size() const { return size_; }     // Content-Length of the synthesised response
    long Read(void *p, size_t n)
    {
        if (!open_) return rc_;
        size_t got = 0;
        rc_ = dm_cache_read(e_, id_, off_, p, n, &got);
        if (rc_ != DM_OK) return rc_;
        off_ += got;
        return (long)got;                       // 0 == io.EOF
    }
    int Close()
    {
        if (open_) dm_cache_close(e_, id_);
        open_ = false;
        return DM_OK;
    }
private:
    dm_engine *e_;
    uint64_t id_ = 0, size_ = 0, off_ = 0;
    int rc_ = DM_OK;
    bool open_ = false;
};

}  // namespace dm
