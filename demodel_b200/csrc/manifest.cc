// OCI / Ollama image-manifest awareness (SURVEY.md §8f-4): the manifest names
// every layer blob with its sha256 digest and size *before* the bodies are
// requested, so the proxy can pre-open one verified stream per layer.
//
// Manifest shape: demodel/CONTRIBUTING.md:128-153 (the decoded body of
// the reference's one cached fixture) — {"config": {descriptor}, "layers":
// [{descriptor}, ...]} with descriptor = {"mediaType", "digest": "sha256:<hex>",
// "size"}.  The parser below is a small JSON walker that collects every object
// carrying both a sha256 "digest" and a numeric "size", in document order, and
// tolerates nested annotations/platform objects and unknown keys.
#include "../../include/demodel_b200.h"

#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

namespace {

struct Walker {
    const char *p, *end;
    std::vector<dm_layer> found;
    bool ok = true;

    void ws() { while (p < end && (*p == ' ' || *p == '\n' || *p == '\t' || *p == '\r')) ++p; }

    bool string(std::string *out)
    {
        if (p >= end || *p != '"') return ok = false;
        ++p;
        std::string s;
        while (p < end && *p != '"') {
            if (*p == '\\') {
                if (++p >= end) return ok = false;
                switch (*p) {
                case 'n': s += '\n'; break; case 't': s += '\t'; break; case 'r': s += '\r'; break;
                case 'b': s += '\b'; break; case 'f': s += '\f'; break;
                case 'u': if (end - p < 5) return ok = false; s += '?'; p += 4; break;   // not needed for digests
                default: s += *p;
                }
                ++p;
            } else s += *p++;
        }
        if (p >= end) return ok = false;
        ++p;
        if (out) *out = std::move(s);
        return true;
    }

    bool number(uint64_t *out, bool *integral)
    {
        const char *q = p;
        uint64_t v = 0;
        bool intg = true, any = false;
        if (q < end && *q == '-') { intg = false; ++q; }
        while (q < end && ((*q >= '0' && *q <= '9') || *q == '.' || *q == 'e' || *q == 'E' || *q == '+' || *q == '-')) {
            if (*q >= '0' && *q <= '9') { if (intg) v = v * 10 + (uint64_t)(*q - '0'); any = true; }
            else intg = false;
            ++q;
        }
        if (!any) return ok = false;
        p = q;
        if (out) *out = v;
        if (integral) *integral = intg;
        return true;
    }

    bool value(int depth)
    {
        if (depth > 64) return ok = false;
        ws();
        if (p >= end) return ok = false;
        if (*p == '{') return object(depth);
        if (*p == '[') {
            ++p; ws();
            if (p < end && *p == ']') { ++p; return true; }
            for (;;) {
                if (!value(depth + 1)) return false;
                ws();
                if (p < end && *p == ',') { ++p; continue; }
                if (p < end && *p == ']') { ++p; return true; }
                return ok = false;
            }
        }
        if (*p == '"') return string(nullptr);
        if (!strncmp(p, "true", (size_t)std::min<long>(4, end - p)) && end - p >= 4) { p += 4; return true; }
        if (!strncmp(p, "false", (size_t)std::min<long>(5, end - p)) && end - p >= 5) { p += 5; return true; }
        if (!strncmp(p, "null", (size_t)std::min<long>(4, end - p)) && end - p >= 4) { p += 4; return true; }
        return number(nullptr, nullptr);
    }

    bool object(int depth)
    {
        ++p;   // '{'
        std::string digest, media;
        uint64_t size = 0;
        bool have_size = false;
        const size_t slot = found.size();      // a descriptor is recorded before its nested objects
        found.emplace_back();
        bool is_desc = false;
        ws();
        if (p < end && *p == '}') { ++p; found.erase(found.begin() + (long)slot); return true; }
        for (;;) {
            ws();
            std::string key;
            if (!string(&key)) return false;
            ws();
            if (p >= end || *p != ':') return ok = false;
            ++p; ws();
            if (key == "digest" && p < end && *p == '"') { if (!string(&digest)) return false; }
            else if (key == "mediaType" && p < end && *p == '"') { if (!string(&media)) return false; }
            else if (key == "size" && p < end && *p != '"' && *p != '{' && *p != '[') {
                bool intg = false;
                if (!number(&size, &intg)) return false;
                have_size = intg;
            } else if (!value(depth + 1)) return false;
            ws();
            if (p < end && *p == ',') { ++p; continue; }
            if (p < end && *p == '}') { ++p; break; }
            return ok = false;
        }
        if (have_size && digest.size() == 7 + 64 && digest.compare(0, 7, "sha256:") == 0) {
            dm_layer L;
            memset(&L, 0, sizeof L);
            is_desc = true;
            for (int i = 0; i < 32 && is_desc; ++i) {
                auto hx = [](char c) { return c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10
                                              : c >= 'A' && c <= 'F' ? c - 'A' + 10 : -1; };
                const int hi = hx(digest[7 + 2 * i]), lo = hx(digest[8 + 2 * i]);
                if (hi < 0 || lo < 0) { is_desc = false; break; }
                L.digest[i] = (uint8_t)((hi << 4) | lo);
            }
            L.size = size;
            strncpy(L.media_type, media.c_str(), sizeof L.media_type - 1);
            if (is_desc) found[slot] = L;
        }
        if (!is_desc) found.erase(found.begin() + (long)slot);
        return true;
    }
};

}  // namespace

extern "C" int dm_manifest_parse(const char *json, size_t len, dm_layer *out, uint32_t max_layers, uint32_t *n_layers)
{
    if (!json || !n_layers || (!out && max_layers)) return DM_EINVAL;
    Walker w{json, json + len, {}, true};
    if (!w.value(0) || !w.ok) return DM_EINVAL;
    w.ws();
    if (w.p != w.end) return DM_EINVAL;
    *n_layers = (uint32_t)w.found.size();
    for (uint32_t i = 0; i < w.found.size() && i < max_layers; ++i) out[i] = w.found[i];
    return DM_OK;
}

extern "C" int dm_manifest_prefetch(dm_engine *e, const dm_layer *layers, uint32_t n, uint64_t *ids)
{
    if (!e || (!layers && n) || (!ids && n)) return DM_EINVAL;
    for (uint32_t i = 0; i < n; ++i) ids[i] = 0;
    for (uint32_t i = 0; i < n; ++i) {
        uint64_t have = 0;
        if (dm_cache_contains(e, layers[i].digest, &have) == DM_OK && have == layers[i].size) continue;   // hit: nothing to fetch
        bool dup = false;                      // the same blob listed twice: one stream is enough
        for (uint32_t k = 0; k < i && !dup; ++k) dup = memcmp(layers[k].digest, layers[i].digest, 32) == 0;
        if (dup) continue;
        int rc = dm_stream_open(e, layers[i].digest, layers[i].size, &ids[i]);
        if (rc != DM_OK) {
            for (uint32_t k = 0; k < i; ++k) if (ids[k]) { dm_stream_abort(e, ids[k]); ids[k] = 0; }
            return rc;
        }
    }
    return DM_OK;
}
