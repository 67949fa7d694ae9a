// Package b200 is the cgo binding of libdemodel_b200.so for demodel's proxy.
//
// NOT COMPILED IN THIS REPOSITORY'S CI: the build image has no Go toolchain
// (SURVEY.md §8c), so this file is source only.  Its C++ twin, which IS
// compiled and tested here, is demodel_b200/csrc/proxy_hooks.hpp; keep the
// two in step.
//
// Wiring (see INTEGRATION.md for the diff against cmd/demodel/start.go):
//
//	OnResponse (start.go:201-204)  resp.Body = b200.NewBodyTee(pool, resp.Body, oid, resp.ContentLength)
//	OnRequest  (start.go:197-200)  if r := pool.Hit(oid); r != nil { return req, hitResponse(req, r) }
//	start()    (start.go:167)      pool, err := b200.Open(b200.Config{...}); defer pool.Close()
package b200

/*
#cgo CFLAGS: -I${SRCDIR}/../include
#cgo LDFLAGS: -L${SRCDIR}/../demodel_b200 -ldemodel_b200 -Wl,-rpath,${SRCDIR}/../demodel_b200
#include <stdlib.h>
#include "demodel_b200.h"
*/
import "C"

import (
	"bytes"
	"errors"
	"fmt"
	"io"
	"sort"
	"unsafe"
)

// Error is a negative dm_err from the engine.
type Error struct {
	Code   int
	Detail string
}

func (e *Error) Error() string {
	return fmt.Sprintf("demodel_b200: %s (%d): %s", C.GoString(C.dm_strerror(C.int(e.Code))), e.Code, e.Detail)
}

// check turns a negative dm_err into an error.  The detail text is fetched with dm_error_detail(e, id), which
// files it under the stream / reader id (0 for calls that have none), NOT with the thread-local
// dm_last_error(): between the failing cgo call and this one the goroutine may have moved to another OS
// thread, whose "last error" belongs to some other connection.
func check(e *C.dm_engine, id C.uint64_t, rc C.int) error {
	if rc == C.DM_OK {
		return nil
	}
	var buf [512]C.char
	var n C.size_t
	C.dm_error_detail(e, id, &buf[0], C.size_t(len(buf)), &n)
	return &Error{Code: int(rc), Detail: C.GoString(&buf[0])}
}

// Config mirrors dm_config for one GPU.
type Config struct {
	HBMCacheBytes uint64 // 0 = half of free HBM
	RingBytes     uint64 // 0 = 256 MiB
	SlabBytes     uint32 // 0 = 1 MiB
	MaxStreams    uint32 // 0 = 65536
	CacheDir      string // "" = HBM tier only
	DiskSync      bool
	DiskDirect    bool // bodies too large for HBM (all bodies when HBM holds none) are cached on disk; needs CacheDir
	// DiskLimitBytes bounds the whole pool's disk tier (0 = no limit); each GPU's engine gets an equal share, since
	// dm_shard_of splits digests evenly.  Needs CacheDir; a value below the GPU count is refused (DM_EINVAL).
	DiskLimitBytes uint64
}

// Pool owns one engine per GPU and routes blobs by digest prefix
// (dm_shard_of): independent streams, no collective.
type Pool struct {
	engines []*C.dm_engine
}

// Open creates an engine on every visible GPU.  There is no CPU fallback:
// without a CUDA device this returns DM_ENODEV and the proxy should run
// without the cache path.
func Open(cfg Config) (*Pool, error) {
	n := int(C.dm_device_count())
	if n <= 0 {
		return nil, &Error{Code: int(C.DM_ENODEV), Detail: "no CUDA device"}
	}
	if cfg.DiskLimitBytes > 0 && cfg.DiskLimitBytes < uint64(n) {
		return nil, &Error{Code: int(C.DM_EINVAL), Detail: "DiskLimitBytes is smaller than one byte per GPU"}
	}
	p := &Pool{}
	for dev := 0; dev < n; dev++ {
		var c C.dm_config
		c.struct_size = C.uint32_t(unsafe.Sizeof(c))
		c.device = C.int32_t(dev)
		c.hbm_cas_bytes = C.uint64_t(cfg.HBMCacheBytes)
		c.ring_bytes = C.uint64_t(cfg.RingBytes)
		c.slab_bytes = C.uint32_t(cfg.SlabBytes)
		c.max_streams = C.uint32_t(cfg.MaxStreams)
		var dir *C.char
		if cfg.CacheDir != "" {
			dir = C.CString(fmt.Sprintf("%s/gpu%d", cfg.CacheDir, dev))
			defer C.free(unsafe.Pointer(dir))
		}
		c.cas_dir = dir
		if cfg.DiskSync {
			c.flags |= C.DM_F_DISK_SYNC
		}
		if cfg.DiskDirect {
			c.flags |= C.DM_F_DISK_DIRECT
		}
		var e *C.dm_engine
		if err := check(nil, 0, C.dm_engine_create(&c, &e)); err != nil {
			p.Close()
			return nil, err
		}
		p.engines = append(p.engines, e)
		if cfg.DiskLimitBytes > 0 {
			if err := check(e, 0, C.dm_cache_set_disk_limit(e, C.uint64_t(cfg.DiskLimitBytes/uint64(n)))); err != nil {
				p.Close()
				return nil, err
			}
		}
	}
	return p, nil
}

// DiskUsage mirrors dm_disk_usage for one GPU's engine.
type DiskUsage struct {
	LimitBytes, UsedBytes, BlobFiles, BlobBytes, StagingBytes, PartialBytes uint64
	EvictedFiles, EvictedBytes, Refused                                      uint64
}

// DiskUsage reports each engine's disk tier, in GPU order.
func (p *Pool) DiskUsage() []DiskUsage {
	out := make([]DiskUsage, len(p.engines))
	for i, e := range p.engines {
		var u C.dm_disk_usage
		u.struct_size = C.uint32_t(unsafe.Sizeof(u))
		if C.dm_cache_disk_usage(e, &u) != C.DM_OK {
			continue
		}
		out[i] = DiskUsage{uint64(u.limit_bytes), uint64(u.used_bytes), uint64(u.blob_files), uint64(u.blob_bytes),
			uint64(u.staging_bytes), uint64(u.partial_bytes), uint64(u.evicted_files), uint64(u.evicted_bytes), uint64(u.refused)}
	}
	return out
}

func (p *Pool) Close() {
	for _, e := range p.engines {
		C.dm_engine_destroy(e)
	}
	p.engines = nil
}

// engineFor picks the GPU that owns a digest; blobs with no known digest
// are homed by a hash of the URL computed by the caller.
func (p *Pool) engineFor(digest *[32]byte) *C.dm_engine {
	i := C.dm_shard_of((*C.uint8_t)(unsafe.Pointer(&digest[0])), C.uint32_t(len(p.engines)))
	return p.engines[int(i)]
}

// BodyTee is the io.ReadCloser the OnResponse hook installs around
// resp.Body: bytes flow to the client unchanged while the engine hashes them
// and lands them in the cache.
type BodyTee struct {
	e       *C.dm_engine
	up      io.ReadCloser
	id      C.uint64_t
	open    bool
	eof     bool
	url     string
	Digest  [32]byte
	Matched bool
}

// NewBodyTee opens a stream.  expect may be nil (digest unknown up front);
// home is then required to pick the GPU (e.g. a hash of the request URL).
func NewBodyTee(p *Pool, up io.ReadCloser, expect *[32]byte, home *[32]byte, contentLength int64) (*BodyTee, error) {
	key := expect
	if key == nil {
		key = home
	}
	t := &BodyTee{e: p.engineFor(key), up: up}
	var ex *C.uint8_t
	if expect != nil {
		ex = (*C.uint8_t)(unsafe.Pointer(&expect[0]))
	}
	hint := C.uint64_t(0)
	if contentLength > 0 {
		hint = C.uint64_t(contentLength)
	}
	if err := check(t.e, 0, C.dm_stream_open(t.e, ex, hint, &t.id)); err != nil {
		return nil, err
	}
	t.open = true
	return t, nil
}

// Read implements io.Reader for goproxy's copy loop.  dm_stream_write copies
// p before returning, so goproxy may reuse its buffer.
func (t *BodyTee) Read(p []byte) (int, error) {
	if t.eof {
		return 0, io.EOF
	}
	n, err := t.up.Read(p)
	if n > 0 {
		if werr := check(t.e, t.id, C.dm_stream_write(t.e, t.id, unsafe.Pointer(&p[0]), C.size_t(n))); werr != nil {
			t.abort()
			return n, werr
		}
	}
	if errors.Is(err, io.EOF) {
		return n, t.finish()
	}
	if err != nil {
		t.abort()
	}
	return n, err
}

// WriteTo is the zero-copy path (io.Copy prefers io.WriterTo): each upstream
// Read lands directly in a window of the engine's pinned ring.
func (t *BodyTee) WriteTo(w io.Writer) (int64, error) {
	var total int64
	for {
		var win unsafe.Pointer
		var capN C.size_t
		if err := check(t.e, t.id, C.dm_stream_acquire(t.e, t.id, &win, &capN)); err != nil {
			t.abort()
			return total, err
		}
		buf := unsafe.Slice((*byte)(win), int(capN))
		n, rerr := t.up.Read(buf)
		// The window is ours only until dm_stream_commit: afterwards the engine may DMA the slab and
		// hand it to another stream at any time.  So the client-side write happens BEFORE the commit.
		var werr error
		if n > 0 {
			var m int
			m, werr = w.Write(buf[:n])
			total += int64(m)
		}
		if err := check(t.e, t.id, C.dm_stream_commit(t.e, t.id, C.size_t(n))); err != nil {
			t.abort()
			return total, err
		}
		if werr != nil {
			t.abort()
			return total, werr
		}
		if errors.Is(rerr, io.EOF) {
			if ferr := t.finish(); ferr != io.EOF {
				return total, ferr
			}
			return total, nil
		}
		if rerr != nil {
			t.abort()
			return total, rerr
		}
	}
}

func (t *BodyTee) finish() error {
	t.eof = true
	t.open = false
	var m C.int
	if err := check(t.e, t.id, C.dm_stream_finish(t.e, t.id, (*C.uint8_t)(unsafe.Pointer(&t.Digest[0])), &m)); err != nil {
		C.dm_stream_abort(t.e, t.id) // some failures leave the stream open; a released id just says so (ids are never reused)
		return err
	}
	t.Matched = m != 0
	if t.Matched && t.url != "" { // best effort: the next request for this URL is a hit
		cu := C.CString(t.url)
		C.dm_cache_alias_put(t.e, cu, (*C.uint8_t)(unsafe.Pointer(&t.Digest[0])))
		C.free(unsafe.Pointer(cu))
	}
	return io.EOF
}

func (t *BodyTee) abort() {
	if t.open {
		C.dm_stream_abort(t.e, t.id)
		t.open = false
	}
}

// Close before EOF means the client went away or upstream failed.
func (t *BodyTee) Close() error {
	t.abort()
	return t.up.Close()
}

// HitReader is the body of the response the OnRequest hook synthesises on
// a cache hit.
type HitReader struct {
	e    *C.dm_engine
	id   C.uint64_t
	Size int64
	off  uint64
}

// Hit returns nil on a miss.
func (p *Pool) Hit(digest *[32]byte) *HitReader {
	e := p.engineFor(digest)
	var id, size C.uint64_t
	rc := C.dm_cache_open(e, (*C.uint8_t)(unsafe.Pointer(&digest[0])), &id, &size)
	if rc != C.DM_OK {
		return nil
	}
	return &HitReader{e: e, id: id, Size: int64(size)}
}

// HitVerified is Hit that never serves a disk-tier blob the GPU has not
// verified (dm_cache_open_verified).  A blob in HBM opens as with Hit; one on
// the disk tier only is loaded into HBM and hashed there while it is served
// from the loaded bytes.  Size is the blob's size (send it as Content-Length):
// the Read that would return the last byte waits for the verdict, and on a
// mismatch (DM_ECORRUPT), a failed read of the file (DM_EIO) or a failed copy
// or launch (DM_ECUDA) Read returns an *Error instead, so net/http cuts the
// response short and the client never receives a whole body that does not
// hash to its name.  nil on a miss, and when the blob cannot be loaded
// (DM_ENOMEM: larger than the arena, no room, no stream slot to spare;
// DM_ESTATE: a pool without an HBM tier); Hit still serves those, unverified,
// for a caller that accepts that, and HitVerifiedRing serves them verified.
func (p *Pool) HitVerified(digest *[32]byte) *HitReader {
	r, _ := p.HitVerifiedErr(digest)
	return r
}

// HitVerifiedErr is HitVerified that also says why a blob could not be
// opened: (nil, nil) on a miss, (nil, *Error) otherwise.  An *Error with Code
// DM_ENOMEM or DM_ESTATE means the blob is cached but cannot be loaded into
// HBM: serve it with HitVerifiedRing.
func (p *Pool) HitVerifiedErr(digest *[32]byte) (*HitReader, error) {
	e := p.engineFor(digest)
	var id, size C.uint64_t
	rc := C.dm_cache_open_verified(e, (*C.uint8_t)(unsafe.Pointer(&digest[0])), &id, &size)
	if rc == C.DM_ENOENT {
		return nil, nil
	}
	if err := check(e, 0, rc); err != nil {
		return nil, err
	}
	return &HitReader{e: e, id: id, Size: int64(size)}, nil
}

// HitVerifiedRing is a verified hit that takes no HBM extent
// (dm_cache_open_verified_ring): for blobs larger than the arena, an arena
// with no room, and pools without an HBM tier.  A blob in HBM opens as with
// Hit.  One on the disk tier only is read through the engine's pinned ring,
// hashed on the GPU, and served from the same ring slabs; nothing is placed
// in HBM, so every such hit hashes the blob again.  Size and the last-byte
// rule are HitVerified's: the Read that would return the last byte waits for
// the verdict and returns an *Error (DM_ECORRUPT, DM_EIO, DM_ECUDA) instead
// on a failure.  Reads go forward only, which io.Copy does.  (nil, nil) on a
// miss; DM_ENOMEM when ring loads already hold their share of the ring or no
// stream slot is to spare: retry, or serve with Hit.
func (p *Pool) HitVerifiedRing(digest *[32]byte) (*HitReader, error) {
	e := p.engineFor(digest)
	var id, size C.uint64_t
	rc := C.dm_cache_open_verified_ring(e, (*C.uint8_t)(unsafe.Pointer(&digest[0])), &id, &size)
	if rc == C.DM_ENOENT {
		return nil, nil
	}
	if err := check(e, 0, rc); err != nil {
		return nil, err
	}
	return &HitReader{e: e, id: id, Size: int64(size)}, nil
}

// HitVerifiedRange is a verified hit on bytes [off, off+length) of a blob
// (dm_cache_open_verified_range; length 0: to the end), for a `Range:`
// request.  A blob in HBM opens as with Hit, limited to the range.  A
// disk-only blob is served from a shared ring load: every range reader of the
// blob that the load can still serve attaches to it, so N parallel parts of
// one blob read and hash the file once instead of N times.  Size is the whole
// blob's size (for Content-Range); Read starts at off and returns io.EOF at
// off+length, and the Read that would return the blob's last byte waits for
// the verdict as HitVerifiedRing's does.  (nil, nil) on a miss; DM_ERANGE when
// the range is not within the blob; DM_ENOMEM only when a new load was needed
// and ring loads already hold their share of the ring or no stream slot is to
// spare.
func (p *Pool) HitVerifiedRange(digest *[32]byte, off, length uint64) (*HitReader, error) {
	e := p.engineFor(digest)
	var id, size C.uint64_t
	rc := C.dm_cache_open_verified_range(e, (*C.uint8_t)(unsafe.Pointer(&digest[0])), C.uint64_t(off), C.uint64_t(length), &id, &size)
	if rc == C.DM_ENOENT {
		return nil, nil
	}
	if err := check(e, 0, rc); err != nil {
		return nil, err
	}
	return &HitReader{e: e, id: id, Size: int64(size), off: off}, nil
}

func (r *HitReader) Read(p []byte) (int, error) {
	if len(p) == 0 {
		return 0, nil
	}
	var n C.size_t
	if err := check(r.e, r.id, C.dm_cache_read(r.e, r.id, C.uint64_t(r.off), unsafe.Pointer(&p[0]), C.size_t(len(p)), &n)); err != nil {
		return 0, err
	}
	if n == 0 {
		return 0, io.EOF
	}
	r.off += uint64(n)
	return int(n), nil
}

func (r *HitReader) Close() error {
	return check(r.e, r.id, C.dm_cache_close(r.e, r.id))
}

// ---- Range parts, checkpoint / resume, manifest prefetch (source only, see header note) ----

// WriteAt feeds one piece of a `Range:` response into the stream that owns the
// blob; parts may arrive in any order (dm_stream_write_at).
func (t *BodyTee) WriteAt(p []byte, off int64) (int, error) {
	if len(p) == 0 {
		return 0, nil
	}
	if err := check(t.e, t.id, C.dm_stream_write_at(t.e, t.id, C.uint64_t(off), unsafe.Pointer(&p[0]), C.size_t(len(p)))); err != nil {
		return 0, err
	}
	return len(p), nil
}

// Checkpoint is the SHA-256 mid-state of an interrupted download.
type Checkpoint struct {
	H     [8]uint32
	Bytes uint64
}

// Checkpoint waits until every whole block received in order is hashed.
func (t *BodyTee) Checkpoint() (Checkpoint, error) {
	var ck C.dm_checkpoint
	if err := check(t.e, t.id, C.dm_stream_checkpoint(t.e, t.id, &ck)); err != nil {
		return Checkpoint{}, err
	}
	out := Checkpoint{Bytes: uint64(ck.bytes)}
	for i := range out.H {
		out.H[i] = uint32(ck.h[i])
	}
	return out, nil
}

// Resume continues a blob from a checkpoint when the client retries with
// `Range: bytes=<ck.Bytes>-`.
func Resume(p *Pool, up io.ReadCloser, ck Checkpoint, expect *[32]byte, contentLength int64) (*BodyTee, error) {
	t := &BodyTee{e: p.engineFor(expect), up: up}
	var c C.dm_checkpoint
	for i := range ck.H {
		c.h[i] = C.uint32_t(ck.H[i])
	}
	c.bytes = C.uint64_t(ck.Bytes)
	c.abi = C.DM_ABI_VERSION
	if err := check(t.e, 0, C.dm_stream_resume(t.e, &c, (*C.uint8_t)(unsafe.Pointer(&expect[0])), C.uint64_t(contentLength), &t.id)); err != nil {
		return nil, err
	}
	t.open = true
	return t, nil
}

// Layer is one descriptor of an OCI / Ollama manifest.
type Layer struct {
	Digest    [32]byte
	Size      uint64
	MediaType string
	StreamID  uint64 // set by ManifestTee: the stream pre-opened for this layer (0 = cached already)
}

// ParseManifest lists config + layers of a manifest body (the shape of the
// reference's cached fixture, CONTRIBUTING.md:128-153).
func ParseManifest(body []byte) ([]Layer, error) {
	if len(body) == 0 {
		return nil, &Error{Code: int(C.DM_EINVAL), Detail: "empty manifest"}
	}
	var n C.uint32_t
	raw := make([]C.dm_layer, 64)
	if err := check(nil, 0, C.dm_manifest_parse((*C.char)(unsafe.Pointer(&body[0])), C.size_t(len(body)), &raw[0], 64, &n)); err != nil {
		return nil, err
	}
	if int(n) > len(raw) {
		n = C.uint32_t(len(raw))
	}
	out := make([]Layer, int(n))
	for i := range out {
		copy(out[i].Digest[:], C.GoBytes(unsafe.Pointer(&raw[i].digest[0]), 32))
		out[i].Size = uint64(raw[i].size)
		out[i].MediaType = C.GoString(&raw[i].media_type[0])
	}
	return out, nil
}

// SetMeta records a response header to replay when the blob is served from
// the cache (stored in the sidecar on the disk tier).
func (t *BodyTee) SetMeta(key, value string) error {
	k, v := C.CString(key), C.CString(value)
	defer C.free(unsafe.Pointer(k))
	defer C.free(unsafe.Pointer(v))
	return check(t.e, t.id, C.dm_stream_set_meta(t.e, t.id, k, v))
}

// Meta returns the blob's sidecar JSON ({"digest","size","encoding","headers":{...}}).
func (r *HitReader) Meta() (string, error) {
	var n C.size_t
	if err := check(r.e, r.id, C.dm_cache_meta(r.e, r.id, nil, 0, &n)); err != nil {
		return "", err
	}
	buf := make([]byte, int(n)+1)
	if err := check(r.e, r.id, C.dm_cache_meta(r.e, r.id, (*C.char)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)), &n)); err != nil {
		return "", err
	}
	return string(buf[:int(n)]), nil
}

// Follow attaches to a body another connection is ingesting right now
// (request coalescing); nil if nothing is in flight for this digest, or if the
// stream retains nothing to serve (verify-only).  Reads block until the bytes
// have arrived - in HBM, or in the file of a disk-backed body (DM_F_DISK_DIRECT),
// served as its writes complete - and the read at EOF waits for the verdict,
// which for a disk-backed body means until the GPU has hashed the whole file.
// An aborted, corrupt or suspended body makes Read return an *Error with
// DM_ESTATE; after a suspend, Follow again once the download is resumed.
func (p *Pool) Follow(digest *[32]byte) *HitReader {
	e := p.engineFor(digest)
	var id, size C.uint64_t
	if C.dm_cache_follow(e, (*C.uint8_t)(unsafe.Pointer(&digest[0])), &id, &size) != C.DM_OK {
		return nil
	}
	return &HitReader{e: e, id: id, Size: int64(size)} // Size 0 = unknown: send chunked
}

// Promote brings cached blobs back into HBM (dm_cache_promote): each disk copy is loaded and verified on the GPU
// that owns its digest, the engines in parallel.  It blocks until every blob has a status: 0 (DM_OK, in HBM now)
// or a negative dm_err - DM_ENOENT, DM_ENOMEM, DM_EIO, DM_ECUDA, or DM_ECORRUPT when the disk copy did not hash to
// its name and was removed.  Run it in a goroutine after start-up; hits are served from disk meanwhile.
func (p *Pool) Promote(digests [][32]byte) ([]int, error) {
	status := make([]int, len(digests))
	byEngine := make(map[*C.dm_engine][]int)
	for i := range digests {
		e := p.engineFor(&digests[i])
		byEngine[e] = append(byEngine[e], i)
	}
	errs := make(chan error, len(byEngine))
	for e, idx := range byEngine {
		go func(e *C.dm_engine, idx []int) {
			buf := make([][32]byte, len(idx))
			for k, i := range idx {
				buf[k] = digests[i]
			}
			st := make([]C.int32_t, len(idx))
			err := check(e, 0, C.dm_cache_promote(e, (*C.uint8_t)(unsafe.Pointer(&buf[0][0])), C.uint32_t(len(idx)), &st[0]))
			for k, i := range idx {
				status[i] = int(st[k])
			}
			errs <- err
		}(e, idx)
	}
	var first error
	for range byEngine {
		if err := <-errs; err != nil && first == nil {
			first = err
		}
	}
	return status, first
}

// Verify checks disk-tier copies in place (dm_cache_verify): each file is hashed on the GPU that owns its digest,
// the engines in parallel, without loading anything into HBM or evicting anything there.  It blocks until every blob
// has a status: 0 (DM_OK) or a negative dm_err - DM_ENOENT, DM_EIO, DM_ECUDA, DM_ENOMEM (no stream slot to spare),
// or DM_ECORRUPT when the file did not hash to its name and was removed.  For a background scrub of the whole tier,
// page through List and pass each page to Verify.
func (p *Pool) Verify(digests [][32]byte) ([]int, error) {
	status := make([]int, len(digests))
	byEngine := make(map[*C.dm_engine][]int)
	for i := range digests {
		e := p.engineFor(&digests[i])
		byEngine[e] = append(byEngine[e], i)
	}
	errs := make(chan error, len(byEngine))
	for e, idx := range byEngine {
		go func(e *C.dm_engine, idx []int) {
			buf := make([][32]byte, len(idx))
			for k, i := range idx {
				buf[k] = digests[i]
			}
			st := make([]C.int32_t, len(idx))
			err := check(e, 0, C.dm_cache_verify(e, (*C.uint8_t)(unsafe.Pointer(&buf[0][0])), C.uint32_t(len(idx)), &st[0]))
			for k, i := range idx {
				status[i] = int(st[k])
			}
			errs <- err
		}(e, idx)
	}
	var first error
	for range byEngine {
		if err := <-errs; err != nil && first == nil {
			first = err
		}
	}
	return status, first
}

// ImportFile is one file for Pool.Import.
type ImportFile struct {
	Path   string    // a regular file; symlinks are followed
	Digest *[32]byte // its SHA-256 when the layout names it (an Ollama blob, a HuggingFace LFS blob), else nil
	Key    string    // a URL to enter in the alias index once the file is cached ("" for none)
}

// Import seeds the disk tier from files already on the host (dm_cache_import): each file is staged under
// <CacheDir>/incoming/, hashed on the GPU and renamed into the tier, the engines in parallel.  A file with a known
// digest goes to the engine that owns that digest; a file without one goes to engine 0, with its key, as a body
// whose digest is unknown is homed by its URL and found by HitURL on every engine.  link hard-links files into the
// cache where it can instead of copying them.  It blocks until every file has a status: 0 (DM_OK, in the disk tier
// now, digests[i] its SHA-256) or a negative dm_err - DM_ECORRUPT (it does not hash to Digest; digests[i] is what it
// hashed to), DM_ENOENT, DM_EINVAL (not a regular file), DM_EIO, DM_ECUDA or DM_ENOMEM.  Sources are never modified.
func (p *Pool) Import(files []ImportFile, link bool) ([]int, [][32]byte, error) {
	status := make([]int, len(files))
	digests := make([][32]byte, len(files))
	byEngine := make(map[*C.dm_engine][]int)
	for i := range files {
		e := p.engines[0]
		if files[i].Digest != nil {
			e = p.engineFor(files[i].Digest)
		}
		byEngine[e] = append(byEngine[e], i)
	}
	var flags C.uint32_t
	if link {
		flags = C.DM_IMP_LINK
	}
	errs := make(chan error, len(byEngine))
	for e, idx := range byEngine {
		go func(e *C.dm_engine, idx []int) {
			paths := make([]*C.char, len(idx)) // C strings: a Go slice of C pointers may be passed to C
			keys := make([]*C.char, len(idx))
			expect := make([][32]byte, len(idx))
			for k, i := range idx {
				paths[k] = C.CString(files[i].Path)
				if files[i].Key != "" {
					keys[k] = C.CString(files[i].Key)
				}
				if files[i].Digest != nil {
					expect[k] = *files[i].Digest
				}
			}
			out := make([][32]byte, len(idx))
			st := make([]C.int32_t, len(idx))
			err := check(e, 0, C.dm_cache_import(e, (**C.char)(unsafe.Pointer(&paths[0])), (*C.uint8_t)(unsafe.Pointer(&expect[0][0])),
				(**C.char)(unsafe.Pointer(&keys[0])), C.uint32_t(len(idx)), flags, (*C.uint8_t)(unsafe.Pointer(&out[0][0])), &st[0]))
			for k, i := range idx {
				status[i] = int(st[k])
				digests[i] = out[k]
				C.free(unsafe.Pointer(paths[k]))
				if keys[k] != nil {
					C.free(unsafe.Pointer(keys[k]))
				}
			}
			errs <- err
		}(e, idx)
	}
	var first error
	for range byEngine {
		if err := <-errs; err != nil && first == nil {
			first = err
		}
	}
	return status, digests, first
}

// ExportFile is one blob for Pool.Export.
type ExportFile struct {
	Digest [32]byte // the cached blob
	Path   string   // the file to write; missing parent directories are created
}

// Export writes cached blobs to files (dm_cache_export): each blob is copied out of HBM or its disk-tier file into a
// private file next to Path, hashed on the GPU that owns its digest and renamed over Path only when it hashed to
// Digest, the engines in parallel.  The cache is only read.  It blocks until every file has a status: 0 (DM_OK) or a
// negative dm_err - DM_ENOENT (not cached), DM_ECORRUPT (the copy did not hash to its name: nothing written, the tier
// file is left to Verify), DM_EIO, DM_ECUDA or DM_ENOMEM.  One Path given two different digests is refused before
// anything is done (DM_EINVAL).
func (p *Pool) Export(files []ExportFile) ([]int, error) {
	status := make([]int, len(files))
	byEngine := make(map[*C.dm_engine][]int)
	seen := make(map[string][32]byte, len(files))
	for i := range files {
		if d, ok := seen[files[i].Path]; ok && d != files[i].Digest {
			return nil, &Error{Code: int(C.DM_EINVAL), Detail: "one destination named with two different digests: " + files[i].Path}
		}
		seen[files[i].Path] = files[i].Digest
		e := p.engineFor(&files[i].Digest)
		byEngine[e] = append(byEngine[e], i)
	}
	errs := make(chan error, len(byEngine))
	for e, idx := range byEngine {
		go func(e *C.dm_engine, idx []int) {
			paths := make([]*C.char, len(idx)) // C strings: a Go slice of C pointers may be passed to C
			digests := make([][32]byte, len(idx))
			for k, i := range idx {
				paths[k] = C.CString(files[i].Path)
				digests[k] = files[i].Digest
			}
			st := make([]C.int32_t, len(idx))
			err := check(e, 0, C.dm_cache_export(e, (*C.uint8_t)(unsafe.Pointer(&digests[0][0])),
				(**C.char)(unsafe.Pointer(&paths[0])), C.uint32_t(len(idx)), &st[0]))
			for k, i := range idx {
				status[i] = int(st[k])
				C.free(unsafe.Pointer(paths[k]))
			}
			errs <- err
		}(e, idx)
	}
	var first error
	for range byEngine {
		if err := <-errs; err != nil && first == nil {
			first = err
		}
	}
	return status, first
}

// List returns up to limit blobs of the disk tier of every engine (dm_cache_list), merged in ascending digest order,
// strictly after `after` (nil: from the start), with their sizes.  Fewer than limit entries means the listing is
// complete; the next page starts after the last digest returned.
func (p *Pool) List(after *[32]byte, limit int) ([][32]byte, []uint64, error) {
	if limit <= 0 {
		return nil, nil, nil
	}
	var from *C.uint8_t
	if after != nil {
		from = (*C.uint8_t)(unsafe.Pointer(&after[0]))
	}
	type entry struct {
		d    [32]byte
		size uint64
	}
	var all []entry
	for _, e := range p.engines {
		digs := make([][32]byte, limit)
		sizes := make([]C.uint64_t, limit)
		var n C.uint32_t
		if err := check(e, 0, C.dm_cache_list(e, from, (*C.uint8_t)(unsafe.Pointer(&digs[0][0])), &sizes[0], C.uint32_t(limit), &n)); err != nil {
			return nil, nil, err
		}
		for k := 0; k < int(n); k++ {
			all = append(all, entry{digs[k], uint64(sizes[k])})
		}
	}
	sort.Slice(all, func(a, b int) bool { return bytes.Compare(all[a].d[:], all[b].d[:]) < 0 })
	if len(all) > limit {
		all = all[:limit]
	}
	digests := make([][32]byte, len(all))
	sizes := make([]uint64, len(all))
	for k, x := range all {
		digests[k], sizes[k] = x.d, x.size
	}
	return digests, sizes, nil
}

// Remove deletes blobs from the cache (dm_cache_remove) on the engine that owns each digest, the engines in
// parallel.  aliases also deletes every alias naming a removed digest on that engine; partial also deletes a download
// of it saved by Suspend.  It blocks until every blob has a status: 0 (DM_OK) or a negative dm_err - DM_ENOENT (on
// neither tier), DM_ESTATE (something is placing or loading it right now and nothing of it was removed: retry later)
// or DM_EIO.  Open HitReaders keep reading what they opened.  Aliases of a blob imported without a known digest live
// on engine 0 (see Import): delete those with AliasDel.
func (p *Pool) Remove(digests [][32]byte, aliases, partial bool) ([]int, error) {
	status := make([]int, len(digests))
	byEngine := make(map[*C.dm_engine][]int)
	for i := range digests {
		e := p.engineFor(&digests[i])
		byEngine[e] = append(byEngine[e], i)
	}
	var flags C.uint32_t
	if aliases {
		flags |= C.DM_RM_ALIASES
	}
	if partial {
		flags |= C.DM_RM_PARTIAL
	}
	errs := make(chan error, len(byEngine))
	for e, idx := range byEngine {
		go func(e *C.dm_engine, idx []int) {
			buf := make([][32]byte, len(idx))
			for k, i := range idx {
				buf[k] = digests[i]
			}
			st := make([]C.int32_t, len(idx))
			err := check(e, 0, C.dm_cache_remove(e, (*C.uint8_t)(unsafe.Pointer(&buf[0][0])), C.uint32_t(len(idx)), flags, &st[0]))
			for k, i := range idx {
				status[i] = int(st[k])
			}
			errs <- err
		}(e, idx)
	}
	var first error
	for range byEngine {
		if err := <-errs; err != nil && first == nil {
			first = err
		}
	}
	return status, first
}

// AliasDel deletes an alias (dm_cache_alias_del) on every engine: an alias lives on the engine that verified its
// body, and Import puts the aliases of files of unknown digest on engine 0.  It reports whether any engine had it.
func (p *Pool) AliasDel(key string) (bool, error) {
	ck := C.CString(key)
	defer C.free(unsafe.Pointer(ck))
	found := false
	for _, e := range p.engines {
		rc := C.dm_cache_alias_del(e, ck)
		if rc == C.DM_OK {
			found = true
		} else if rc != C.DM_ENOENT {
			return found, check(e, 0, rc)
		}
	}
	return found, nil
}

// Alias is one entry of AliasList.
type Alias struct {
	Key    string
	Digest [32]byte
}

// AliasList returns up to limit aliases whose keys start with prefix, strictly after `after` ("" for the start),
// merged across the engines in ascending byte order of the keys (dm_cache_alias_list).  Fewer than limit entries
// means the listing is complete; the next page starts after the last key returned.  A key present on two engines is
// listed once, with the digest of the lowest-numbered engine.
func (p *Pool) AliasList(prefix, after string, limit int) ([]Alias, error) {
	if limit <= 0 {
		return nil, nil
	}
	cp := C.CString(prefix)
	defer C.free(unsafe.Pointer(cp))
	var ca *C.char
	if after != "" {
		ca = C.CString(after)
		defer C.free(unsafe.Pointer(ca))
	}
	const keyBytes = 1 << 20 // a key is at most 4096 bytes, so every page holds at least one
	keys := (*[keyBytes]byte)(C.malloc(keyBytes))
	defer C.free(unsafe.Pointer(keys))
	var all []Alias
	seen := make(map[string]bool)
	for _, e := range p.engines {
		digs := make([][32]byte, limit)
		from := ca
		for got := 0; got < limit; {
			var n C.uint32_t
			var more C.int
			if err := check(e, 0, C.dm_cache_alias_list(e, cp, from, (*C.char)(unsafe.Pointer(&keys[0])), keyBytes,
				(*C.uint8_t)(unsafe.Pointer(&digs[0][0])), C.uint32_t(limit-got), &n, &more)); err != nil {
				return nil, err
			}
			pos, last := 0, ""
			for k := 0; k < int(n); k++ {
				end := bytes.IndexByte(keys[pos:], 0) + pos
				last = string(keys[pos:end])
				if !seen[last] {
					seen[last] = true
					all = append(all, Alias{last, digs[k]})
				}
				pos = end + 1
			}
			got += int(n)
			if more == 0 || n == 0 {
				break
			}
			if from != ca {
				C.free(unsafe.Pointer(from))
			}
			from = C.CString(last)
		}
		if from != ca {
			C.free(unsafe.Pointer(from))
		}
	}
	sort.Slice(all, func(a, b int) bool { return all[a].Key < all[b].Key })
	if len(all) > limit {
		all = all[:limit]
	}
	return all, nil
}

// ---- requests are URLs, not digests (start.go:197-200) ------------------------------------------------------

// SetURL records the request URL with the body: it goes into the sidecar, and once the body has verified the
// pair URL -> digest is entered in the alias index (dm_cache_alias_put), so the next request for a URL that
// names no digest (HuggingFace resolve/...) is a hit.  Call it right after NewBodyTee.
func (t *BodyTee) SetURL(url string) {
	t.url = url
	_ = t.SetMeta("url", url)
}

// HitURL answers the OnRequest hook: a digest in the URL (OCI `sha256:<hex>`), else the alias index.
func (p *Pool) HitURL(url string) *HitReader {
	cu := C.CString(url)
	defer C.free(unsafe.Pointer(cu))
	for _, e := range p.engines { // the alias lives on the engine that ingested the body
		var id, size C.uint64_t
		if C.dm_proxy_request(e, cu, &id, &size) == C.DM_OK {
			return &HitReader{e: e, id: id, Size: int64(size)}
		}
	}
	return nil
}

// Suspend saves an interrupted download (mid-state + bytes so far) under <CacheDir>/partial and closes the
// stream; the proxy re-requests upstream with `Range: bytes=<returned offset>-`.  Call it from Close() when the
// upstream connection drops, and for every open tee on a graceful shutdown.
func (t *BodyTee) Suspend() (uint64, error) {
	var off C.uint64_t
	if err := check(t.e, t.id, C.dm_stream_suspend(t.e, t.id, &off)); err != nil {
		return 0, err
	}
	t.open = false
	return uint64(off), nil
}

// ResumeSaved continues a download saved by Suspend - in this process or a previous one.  nil, 0 when nothing is
// saved for the digest.
func ResumeSaved(p *Pool, up io.ReadCloser, expect *[32]byte, contentLength int64) (*BodyTee, uint64) {
	t := &BodyTee{e: p.engineFor(expect), up: up}
	var off C.uint64_t
	if C.dm_stream_resume_saved(t.e, (*C.uint8_t)(unsafe.Pointer(&expect[0])), C.uint64_t(contentLength), &t.id, &off) != C.DM_OK {
		return nil, 0
	}
	t.open = true
	return t, uint64(off)
}

// Gunzip inflates a `Content-Encoding: gzip` manifest body (the reference's documented cached body is one,
// CONTRIBUTING.md:76-99) for ParseManifest.  compress/gzip would do as well on the Go side; this keeps the
// hook's behaviour identical to the C++ twin (ManifestTee in proxy_hooks.hpp).
func Gunzip(body []byte) ([]byte, error) {
	if len(body) == 0 {
		return nil, &Error{Code: int(C.DM_EINVAL), Detail: "empty body"}
	}
	out := make([]byte, 8*len(body)+4096)
	var n C.size_t
	rc := C.dm_gunzip(unsafe.Pointer(&body[0]), C.size_t(len(body)), unsafe.Pointer(&out[0]), C.size_t(len(out)), &n)
	if rc == C.DM_ENOMEM && n > 0 {
		out = make([]byte, int(n))
		rc = C.dm_gunzip(unsafe.Pointer(&body[0]), C.size_t(len(body)), unsafe.Pointer(&out[0]), C.size_t(len(out)), &n)
	}
	if rc != C.DM_OK {
		return nil, &Error{Code: int(rc), Detail: "not a gzip / zlib stream"}
	}
	return out[:int(n)], nil
}

// ManifestTee is the OnResponse hook's body for a MANIFEST response (Content-Type
// application/vnd.oci.image.manifest.v1+json or application/vnd.docker.distribution.manifest.v2+json): the bytes
// pass through to the client unchanged while a copy is kept (capped at 4 MiB); at EOF the copy is inflated if the
// response was gzip-encoded, parsed, and one pre-verified stream per layer not yet cached is opened
// (dm_manifest_prefetch).  The C++ twin of the same name is in proxy_hooks.hpp.
type ManifestTee struct {
	pool     *Pool
	up       io.ReadCloser
	encoding string
	body     []byte
	overflow bool
	done     bool
	Layers   []Layer
	Err      error // why the manifest was not used; the body still passed through
}

func NewManifestTee(p *Pool, up io.ReadCloser, contentEncoding string) *ManifestTee {
	return &ManifestTee{pool: p, up: up, encoding: contentEncoding}
}

func (m *ManifestTee) Read(p []byte) (int, error) {
	n, err := m.up.Read(p)
	if n > 0 && !m.overflow {
		if len(m.body)+n > 4<<20 {
			m.overflow, m.body = true, nil
		} else {
			m.body = append(m.body, p[:n]...)
		}
	}
	if errors.Is(err, io.EOF) && !m.done {
		m.done = true
		m.onEOF()
	}
	return n, err
}

func (m *ManifestTee) Close() error { return m.up.Close() }

func (m *ManifestTee) onEOF() {
	if m.overflow {
		m.Err = &Error{Code: int(C.DM_EINVAL), Detail: "manifest larger than 4 MiB"}
		return
	}
	plain := m.body
	switch m.encoding {
	case "", "identity":
	case "gzip", "x-gzip":
		if plain, m.Err = Gunzip(m.body); m.Err != nil {
			return
		}
	default: // br, zstd, deflate: not decoded here; the body passed through untouched
		m.Err = &Error{Code: int(C.DM_EINVAL), Detail: "unsupported Content-Encoding " + m.encoding}
		return
	}
	if m.Layers, m.Err = ParseManifest(plain); m.Err != nil {
		return
	}
	for i := range m.Layers { // one engine per GPU: each layer is prefetched on the GPU that owns its digest
		l := &m.Layers[i]
		var raw C.dm_layer
		for k := 0; k < 32; k++ {
			raw.digest[k] = C.uint8_t(l.Digest[k])
		}
		raw.size = C.uint64_t(l.Size)
		var id C.uint64_t
		e := m.pool.engineFor(&l.Digest)
		if err := check(e, 0, C.dm_manifest_prefetch(e, &raw, 1, &id)); err != nil && m.Err == nil {
			m.Err = err
		}
		l.StreamID = uint64(id) // 0: already cached (or a duplicate)
	}
}
