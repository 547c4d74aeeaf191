// CRAM 3.x compression-header reader (host): the data-series and tag encoding maps of a container, i.e. the
// table that says which codec (EXTERNAL / HUFFMAN / BYTE_ARRAY_LEN / BYTE_ARRAY_STOP / BETA / ...) and which
// external block feeds every data series.  This is the first step of cram_decode_slice's record loop
// (SURVEY.md §8f row 1): a device record decoder needs exactly this table to turn the blocks that
// hgpu_cram_uncompress_blocks_host left in HBM into per-series cursors.
//
// Follows cram_decode_compression_header (cram/cram_decode.c:144-538: preservation map :165-344, record
// encoding map :346-493, tag encoding map :495-535) and the *_decode_init parsers of cram/cram_codecs.c
// (external :459, huffman :2814, byte_array_len :3427, byte_array_stop :3682, beta :1143, subexp :2509,
// gamma :2581).  The text it can emit is cram_describe_encodings' (cram/cram_external.c:476-494, one
// "\tKEY\tCODEC(...)\n" line per series), which is what tests/test_cram_header.py compares with the
// compiled reference on every container of every CRAM fixture.  Input is the UNCOMPRESSED payload of the
// compression-header block (content type 1); CRAM 4.0's codecs are reported as "?".
#include "hgpu_internal.h"
#include <new>
#include <string>
#include <vector>
#include <algorithm>
#include <stdio.h>
#include <string.h>

namespace {

enum { E_NULL = 0, E_EXTERNAL = 1, E_GOLOMB = 2, E_HUFFMAN = 3, E_BYTE_ARRAY_LEN = 4, E_BYTE_ARRAY_STOP = 5, E_BETA = 6,
       E_SUBEXP = 7, E_GOLOMB_RICE = 8, E_GAMMA = 9 };

struct Rd {
    const uint8_t *p, *e;
    bool err = false;
    int32_t itf8()                                                   // itf8_get, cram/cram_io.c
    {
        if (p >= e) { err = true; return 0; }
        const uint8_t c = *p;
        int n = c < 0x80 ? 0 : c < 0xc0 ? 1 : c < 0xe0 ? 2 : c < 0xf0 ? 3 : 4;
        if (e - p < n + 1) { err = true; p = e; return 0; }
        uint32_t v;
        switch (n) {
        case 0: v = c; break;
        case 1: v = ((c & 0x3fu) << 8) | p[1]; break;
        case 2: v = ((c & 0x1fu) << 16) | (p[1] << 8) | p[2]; break;
        case 3: v = ((c & 0x0fu) << 24) | (p[1] << 16) | (p[2] << 8) | p[3]; break;
        default: v = ((c & 0x0fu) << 28) | (p[1] << 20) | (p[2] << 12) | (p[3] << 4) | (p[4] & 0x0f); break;
        }
        p += n + 1;
        return (int32_t)v;
    }
};

struct Codec { std::string text; int32_t id[2] = {-1, -1}; };

// one encoding: `size` parameter bytes at r.p.  false = the reference's decoder_init would fail.
bool parse_codec(int32_t encoding, const uint8_t *data, int32_t size, int depth, Codec &out)
{
    Rd r{data, data + size};
    char buf[96];
    switch (encoding) {
    case E_EXTERNAL: {
        if (size < 1) return false;
        const int32_t id = r.itf8();
        if (r.err || r.p != r.e) return false;
        snprintf(buf, sizeof buf, "EXTERNAL(id=%d)", id);
        out.text = buf; out.id[0] = id;
        return true; }
    case E_HUFFMAN: {
        const int32_t n = r.itf8();
        if (r.err || n < 0 || n > size) return false;
        std::vector<std::pair<int32_t, int64_t>> codes((size_t)n);      // (length, symbol)
        for (int32_t i = 0; i < n; i++) codes[(size_t)i].second = r.itf8();
        if (r.err || r.itf8() != n) return false;
        if (n == 0) { out.text = "?"; return true; }                    // the NULL huffman stream (:2885-2890) has no describe method
        int32_t max_len = 0;
        for (int32_t i = 0; i < n; i++) {
            const int32_t l = r.itf8();
            if (r.err || l < 0) return false;
            codes[(size_t)i].first = l;
            if (l > max_len) max_len = l;
        }
        if (n && (r.p != r.e || max_len >= n || max_len > 31)) return false;
        std::sort(codes.begin(), codes.end());                          // by bit length, then symbol (code_sort :2622)
        out.text = "HUFFMAN(codes={";
        for (int32_t i = 0; i < n; i++) { snprintf(buf, sizeof buf, "%s%lld", i ? "," : "", (long long)codes[(size_t)i].second); out.text += buf; }
        out.text += "},lengths={";
        for (int32_t i = 0; i < n; i++) { snprintf(buf, sizeof buf, "%s%d", i ? "," : "", codes[(size_t)i].first); out.text += buf; }
        out.text += "})";
        return true; }
    case E_BYTE_ARRAY_LEN: {
        if (depth > 4) return false;
        Codec sub[2];
        for (int k = 0; k < 2; k++) {
            const int32_t enc = r.itf8(), sz = r.itf8();
            if (r.err || sz < 0 || r.e - r.p < sz) return false;
            if (!parse_codec(enc, r.p, sz, depth + 1, sub[k])) return false;
            r.p += sz;
        }
        out.text = "BYTE_ARRAY_LEN(len_codec={" + sub[0].text + "},val_codec={" + sub[1].text + "}";   // no ')' there either (:3412-3424)
        out.id[0] = sub[0].id[0]; out.id[1] = sub[1].id[0];
        return true; }
    case E_BYTE_ARRAY_STOP: {
        if (size < 2) return false;
        const int stop = *r.p++;
        const int32_t id = r.itf8();
        if (r.err) return false;
        snprintf(buf, sizeof buf, "BYTE_ARRAY_STOP(stop=%d,id=%d)", stop, id);
        out.text = buf; out.id[0] = id;
        return true; }
    case E_BETA: {
        const int32_t off = r.itf8();
        const int32_t nbits = r.p < r.e ? r.itf8() : -1;
        if (r.err || r.p != r.e || nbits < 0 || nbits > 32) return false;
        snprintf(buf, sizeof buf, "BETA(offset=%d, nbits=%d)", off, nbits);
        out.text = buf;
        return true; }
    case E_SUBEXP: {
        const int32_t off = r.itf8(), k = r.itf8();
        if (r.err || r.p != r.e || k < 0) return false;
        snprintf(buf, sizeof buf, "SUBEXP(offset=%d,k=%d)", off, k);
        out.text = buf;
        return true; }
    case E_GAMMA: {
        const int32_t off = r.itf8();
        if (r.err || r.p != r.e) return false;
        snprintf(buf, sizeof buf, "GAMMA(offset=%d)", off);
        out.text = buf;
        return true; }
    case E_GOLOMB: case E_GOLOMB_RICE:
        out.text = "?";                                                  // these codecs have no describe method there
        return true;
    default:
        return false;                                                    // cram_decoder_init: "Unimplemented codec"
    }
}

// data series the reference knows (:389-461), in its DS enum order (the order cram_codec_iter walks them)
const char *const k_series[] = {"RN", "QS", "IN", "SC", "BF", "CF", "AP", "RG", "MQ", "NS", "MF", "TS", "NP", "NF", "RL", "FN", "FC", "FP",
                                "DL", "BA", "BS", "TL", "RI", "RS", "PD", "HC", "BB", "QQ", "TN", "TC"};

}  // namespace

static long hgpu_cram_parse_compression_header_impl(const uint8_t *hdr, uint32_t len, int major_version,
        hgpu_cram_series *series, long cap, char *text, size_t text_cap)
{
    if (!hdr || major_version != 3) { hgpu_set_error("compression header: CRAM 3.x only"); return -1; }
    Rd r{hdr, hdr + len};
    // preservation map: its byte size lets us step over it (RN / AP / RR / SM / TD do not change the encodings)
    const int32_t psz = r.itf8();
    if (r.err || psz < 0 || r.e - r.p < psz) { hgpu_set_error("compression header: preservation map"); return -1; }
    r.p += psz;
    struct Entry { uint32_t key; int32_t encoding; Codec c; };
    std::vector<Entry> out;
    // record encoding map (:346-493)
    {
        const int32_t msz = r.itf8();
        const uint8_t *start = r.p;
        const int32_t cnt = r.itf8();
        if (r.err || msz < 0 || cnt < 0) { hgpu_set_error("compression header: record encoding map"); return -1; }
        std::vector<Entry> seen;
        for (int32_t i = 0; i < cnt; i++) {
            if (r.e - r.p < 4) { hgpu_set_error("compression header: truncated record encoding map"); return -1; }
            const uint32_t key = (uint32_t)r.p[0] << 8 | r.p[1];
            r.p += 2;
            const int32_t enc = r.itf8(), sz = r.itf8();
            if (r.err) return -1;
            if (enc == E_NULL) continue;
            if (sz < 0 || r.e - r.p < sz) { hgpu_set_error("compression header: encoding runs past the block"); return -1; }
            const char ks[3] = {(char)(key >> 8), (char)key, 0};
            bool known = false;
            for (const char *s : k_series) if (!strcmp(s, ks)) known = true;
            if (known) {
                Entry e{key, enc, Codec()};
                if (!parse_codec(enc, r.p, sz, 0, e.c)) { hgpu_set_error("compression header: codec of %s", ks); return -1; }
                bool replaced = false;
                for (Entry &o : seen) if (o.key == key) { o = e; replaced = true; }      // "defined more than once": the later wins
                if (!replaced) seen.push_back(e);
            }
            r.p += sz;
        }
        if (r.p - start != msz) { hgpu_set_error("compression header: record encoding map size"); return -1; }
        for (const char *s : k_series)
            for (const Entry &e : seen) if (e.key == ((uint32_t)(uint8_t)s[0] << 8 | (uint8_t)s[1])) out.push_back(e);
    }
    // tag encoding map (:495-535): key = tag[0] << 16 | tag[1] << 8 | type
    {
        const int32_t msz = r.itf8();
        const uint8_t *start = r.p;
        const int32_t cnt = r.itf8();
        if (r.err || msz < 0 || cnt < 0) { hgpu_set_error("compression header: tag encoding map"); return -1; }
        for (int32_t i = 0; i < cnt; i++) {
            if (r.e - r.p < 6) { hgpu_set_error("compression header: truncated tag encoding map"); return -1; }
            const uint32_t key = (uint32_t)r.itf8();
            const int32_t enc = r.itf8(), sz = r.itf8();
            if (r.err || sz < 0 || r.e - r.p < sz) { hgpu_set_error("compression header: tag encoding runs past the block"); return -1; }
            Entry e{key, enc, Codec()};
            if (!parse_codec(enc, r.p, sz, 0, e.c)) { hgpu_set_error("compression header: codec of a tag"); return -1; }
            out.push_back(e);
            r.p += sz;
        }
        if (r.p - start != msz) { hgpu_set_error("compression header: tag encoding map size"); return -1; }
    }
    std::string t;
    for (size_t i = 0; i < out.size(); i++) {
        const Entry &e = out[i];
        if (series && (long)i < cap) {
            series[i].key = e.key; series[i].encoding = e.encoding;
            series[i].id[0] = e.c.id[0]; series[i].id[1] = e.c.id[1];
        }
        char ks[4] = {0, 0, 0, 0};
        int k = 0;
        if (e.key >> 16) ks[k++] = (char)(e.key >> 16);
        ks[k++] = (char)(e.key >> 8); ks[k++] = (char)e.key;
        t += "\t"; t += ks; t += "\t"; t += e.c.text; t += "\n";
    }
    if (text && text_cap) {
        const size_t n = t.size() < text_cap - 1 ? t.size() : text_cap - 1;
        memcpy(text, t.data(), n);
        text[n] = 0;
    }
    return (long)out.size();
}

extern "C" long hgpu_cram_parse_compression_header(const uint8_t *hdr, uint32_t len, int major_version,
        hgpu_cram_series *series, long cap, char *text, size_t text_cap)
{
    return hgpu_abi_call([&] { return hgpu_cram_parse_compression_header_impl(hdr, len, major_version, series, cap, text, text_cap); }, -1, -1);
}
