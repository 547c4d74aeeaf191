// Host-side walk of a CRAM 3.x file image down to its blocks — the container/block framing of
// cram_read_container (cram/cram_io.c:3760-3900) and cram_read_block (:1414-1483), so that the
// payloads of every entropy-coded block can be handed to the batch decoders in one launch
// (what cram_decode_slice does block by block through cram_uncompress_block, cram_io.c:1576).
// Pure framing: ITF8/LTF8 integers, no decompression, no CRC.
#include "hgpu_internal.h"
#include <string.h>
#include <stdlib.h>

namespace {

// ITF8 (cram_io.c:138-200): 1-5 bytes, length in the leading ones of the first byte
int itf8(const uint8_t *p, const uint8_t *end, int32_t *v)
{
    if (p >= end) return 0;
    uint8_t b = p[0];
    int n = b < 0x80 ? 1 : b < 0xc0 ? 2 : b < 0xe0 ? 3 : b < 0xf0 ? 4 : 5;
    if (end - p < n) return 0;
    uint32_t u;
    switch (n) {
    case 1: u = b; break;
    case 2: u = ((b & 0x3fu) << 8) | p[1]; break;
    case 3: u = ((b & 0x1fu) << 16) | (p[1] << 8) | p[2]; break;
    case 4: u = ((b & 0x0fu) << 24) | (p[1] << 16) | (p[2] << 8) | p[3]; break;
    default: u = ((b & 0x0fu) << 28) | (p[1] << 20) | (p[2] << 12) | (p[3] << 4) | (p[4] & 0x0f); break;
    }
    *v = (int32_t)u;
    return n;
}

// LTF8 (cram_io.c:~400): 1-9 bytes; only the length matters here
int ltf8_len(const uint8_t *p, const uint8_t *end)
{
    if (p >= end) return 0;
    uint8_t b = p[0];
    int n = b < 0x80 ? 1 : b < 0xc0 ? 2 : b < 0xe0 ? 3 : b < 0xf0 ? 4 : b < 0xf8 ? 5 : b < 0xfc ? 6 : b < 0xfe ? 7 : b < 0xff ? 8 : 9;
    return end - p < n ? 0 : n;
}

} // namespace

extern "C" long hgpu_cram_scan_blocks(const uint8_t *file, uint64_t len, hgpu_cram_block *blocks, long cap,
                                      int *major, int *minor)
{
    if (!file || len < 26 || memcmp(file, "CRAM", 4) != 0) { hgpu_set_error("not a CRAM file"); return -1; }
    int maj = file[4], min = file[5];
    if (major) *major = maj;
    if (minor) *minor = min;
    if (maj != 3) { hgpu_set_error("CRAM major version %d not supported (3.x only)", maj); return -1; }
    const uint8_t *end = file + len, *p = file + 26;
    long n = 0;
    uint32_t container = 0;
    while (p < end) {
        if (end - p < 4) { hgpu_set_error("truncated container header"); return -1; }
        int32_t clen = (int32_t)(p[0] | p[1] << 8 | p[2] << 16 | (uint32_t)p[3] << 24), v, nblk, nland;
        p += 4;
        int k;
        for (int f = 0; f < 4; f++) { if (!(k = itf8(p, end, &v))) { hgpu_set_error("truncated or malformed CRAM container/block header"); return -1; } p += k; }       // ref id, start, span, n records
        if (!(k = ltf8_len(p, end))) { hgpu_set_error("truncated or malformed CRAM container/block header"); return -1; } p += k;                                          // record counter
        if (!(k = ltf8_len(p, end))) { hgpu_set_error("truncated or malformed CRAM container/block header"); return -1; } p += k;                                          // bases
        if (!(k = itf8(p, end, &nblk))) { hgpu_set_error("truncated or malformed CRAM container/block header"); return -1; } p += k;
        if (!(k = itf8(p, end, &nland))) { hgpu_set_error("truncated or malformed CRAM container/block header"); return -1; } p += k;
        for (int f = 0; f < nland; f++) { if (!(k = itf8(p, end, &v))) { hgpu_set_error("truncated or malformed CRAM container/block header"); return -1; } p += k; }
        if (end - p < 4) { hgpu_set_error("truncated or malformed CRAM container/block header"); return -1; }
        p += 4;                                                                                  // container CRC32
        if (clen < 0 || (uint64_t)(end - p) < (uint64_t)clen) { hgpu_set_error("container %u runs past the file", container); return -1; }
        const uint8_t *cend = p + clen;
        while (p < cend) {
            if (cend - p < 2) { hgpu_set_error("truncated or malformed CRAM container/block header"); return -1; }
            hgpu_cram_block b;
            const uint8_t *hdr = p;
            b.method = p[0]; b.content_type = p[1]; b.container = container;
            p += 2;
            int32_t cs, us;
            if (!(k = itf8(p, cend, &b.content_id))) { hgpu_set_error("truncated or malformed CRAM container/block header"); return -1; } p += k;
            if (!(k = itf8(p, cend, &cs))) { hgpu_set_error("truncated or malformed CRAM container/block header"); return -1; } p += k;
            if (!(k = itf8(p, cend, &us))) { hgpu_set_error("truncated or malformed CRAM container/block header"); return -1; } p += k;
            if (cs < 0 || us < 0 || (uint64_t)(cend - p) < (uint64_t)cs + 4) { hgpu_set_error("block runs past its container"); return -1; }
            b.data_off = (uint64_t)(p - file);
            b.hdr_len = (uint16_t)(p - hdr);
            b.comp_size = (uint32_t)cs; b.uncomp_size = (uint32_t)us;
            if (blocks && n < cap) blocks[n] = b;
            n++;
            p += cs + 4;                                                                         // payload + block CRC32
        }
        container++;
    }
    return n;
}

// =============================================================================================
// cram_write_block (cram/cram_io.c:1511-1563) for a batch: the framing is host bytes (method, content type,
// ITF8 content id / sizes, payload), the CRC-32 over header + payload of EVERY block comes from one device
// launch over the assembled image (crc32_batch_kernel, the check side of hgpu_cram_uncompress_blocks_host).
// =============================================================================================
namespace {
int itf8_put(uint8_t *p, int32_t v)                       // itf8_put (cram/cram_io.h), CRAM 3.x varint_put32
{
    const uint32_t u = (uint32_t)v;
    if (u < 0x80u) { p[0] = (uint8_t)u; return 1; }
    if (u < 0x4000u) { p[0] = (uint8_t)(0x80 | (u >> 8)); p[1] = (uint8_t)u; return 2; }
    if (u < 0x200000u) { p[0] = (uint8_t)(0xc0 | (u >> 16)); p[1] = (uint8_t)(u >> 8); p[2] = (uint8_t)u; return 3; }
    if (u < 0x10000000u) { p[0] = (uint8_t)(0xe0 | (u >> 24)); p[1] = (uint8_t)(u >> 16); p[2] = (uint8_t)(u >> 8); p[3] = (uint8_t)u; return 4; }
    p[0] = (uint8_t)(0xf0 | ((u >> 28) & 0xff)); p[1] = (uint8_t)(u >> 20); p[2] = (uint8_t)(u >> 12); p[3] = (uint8_t)(u >> 4); p[4] = (uint8_t)(u & 0x0f);
    return 5;
}
}

// blocks[i]: method, content_type, content_id, comp_size, uncomp_size are read (RAW blocks carry uncomp_size bytes,
// :1527-1530); payload[i] -> the block's bytes.  Writes the blocks back to back into out (cap bytes); out_off[i] (may be
// NULL) receives each block's offset, *out_len the total.  Returns HGPU_OK, HGPU_ERR_ARG (a RAW block whose sizes
// differ: the reference asserts), HGPU_ERR_NOMEM (cap too small; *out_len = bytes needed).
extern "C" int hgpu_cram_write_blocks_host(hgpu_ctx *ctx, const hgpu_cram_block *blocks, const uint8_t *const *payload, uint32_t n,
                                           uint8_t *out, uint64_t cap, uint64_t *out_off, uint64_t *out_len)
{
    if (!ctx || !out_len || (n && (!blocks || !payload))) { hgpu_set_error("bad argument"); return HGPU_ERR_ARG; }
    uint64_t need = 0;
    for (uint32_t i = 0; i < n; i++) {
        const hgpu_cram_block &b = blocks[i];
        if (b.method == 0 && b.comp_size != b.uncomp_size) { hgpu_set_error("block %u: RAW with comp_size != uncomp_size", i); return HGPU_ERR_ARG; }
        need += 2 + 15 + (uint64_t)(b.method == 0 ? b.uncomp_size : b.comp_size) + 4;
    }
    if (!out || cap < need) { *out_len = need; hgpu_set_error("output buffer too small"); return HGPU_ERR_NOMEM; }
    if (n == 0) { *out_len = 0; return HGPU_OK; }
    if (hgpu_check(cudaSetDevice(ctx->device), "cudaSetDevice")) return HGPU_ERR_CUDA;
    // ---- framing
    uint64_t p = 0;
    uint64_t *coff = nullptr;
    uint32_t *clen = nullptr, *crc = nullptr;
    coff = (uint64_t *)malloc((size_t)n * 8); clen = (uint32_t *)malloc((size_t)n * 4); crc = (uint32_t *)malloc((size_t)n * 4);
    if (!coff || !clen || !crc) { free(coff); free(clen); free(crc); hgpu_set_error("out of host memory"); return HGPU_ERR_NOMEM; }
    for (uint32_t i = 0; i < n; i++) {
        const hgpu_cram_block &b = blocks[i];
        const uint32_t dl = b.method == 0 ? b.uncomp_size : b.comp_size;
        if (out_off) out_off[i] = p;
        coff[i] = p;
        uint8_t *q = out + p;
        q[0] = b.method; q[1] = b.content_type;
        int k = 2;
        k += itf8_put(q + k, b.content_id);
        k += itf8_put(q + k, (int32_t)b.comp_size);
        k += itf8_put(q + k, (int32_t)b.uncomp_size);
        if (dl) memcpy(q + k, payload[i], dl);
        clen[i] = (uint32_t)k + dl;
        p += (uint64_t)k + dl + 4;
    }
    // ---- one CRC launch over the image
    StageLayout L;
    const auto s_img = L.seg(p + 8), s_coff = L.seg((size_t)n * 8), s_clen = L.seg((size_t)n * 4), s_crc = L.seg((size_t)n * 4);
    int rc = hgpu_stage_ensure(ctx, L);
    cudaStream_t s = ctx->stream;
    if (!rc && (hgpu_h2d(L.at(s_img), out, p, s) || hgpu_h2d(L.at(s_coff), coff, (size_t)n * 8, s) ||
                hgpu_h2d(L.at(s_clen), clen, (size_t)n * 4, s))) rc = HGPU_ERR_CUDA;
    if (!rc) rc = hgpu_launch_crc32_batch(ctx, L.at(s_img), L.at<uint64_t>(s_coff), L.at<uint32_t>(s_clen), n, L.at<uint32_t>(s_crc), s);
    if (!rc && (hgpu_d2h(crc, L.at(s_crc), (size_t)n * 4, s) || hgpu_check(cudaStreamSynchronize(s), "sync"))) rc = HGPU_ERR_CUDA;
    if (!rc) for (uint32_t i = 0; i < n; i++) {
        uint8_t *q = out + coff[i] + clen[i];
        q[0] = (uint8_t)crc[i]; q[1] = (uint8_t)(crc[i] >> 8); q[2] = (uint8_t)(crc[i] >> 16); q[3] = (uint8_t)(crc[i] >> 24);
    }
    free(coff); free(clen); free(crc);
    *out_len = p;
    return rc;
}
