// cram_uncompress_block (cram/cram_io.c:1576-1754) for every block of a CRAM 3.x file image at once.
//
// The reference uncompresses a slice's blocks one at a time on a CPU thread (cram_decode_slice,
// cram/cram_decode.c:619-627 -> cram_uncompress_block).  Here the whole block list from
// hgpu_cram_scan_blocks goes to the device: one upload of the file image, one CRC-32 launch over every
// block's header+payload (:1585-1592), one batch launch per entropy codec (method 4 rANS 4x8, 5 rANS
// Nx16, 6 adaptive arithmetic, 8 tok3 names), one download of all payloads.  RAW blocks are host copies.
// Method 7 (fqzcomp) blocks go through hgpu_fqz_decode_batch_host.  GZIP blocks (whole gzip members of any size) take
// gzip_inflate_kernel; BZIP2 / LZMA blocks are reported HGPU_CRAM_UNSUPPORTED and stay with the host library.
#include "hgpu_internal.h"
#include <vector>
#include <string.h>

// Size fields of a CRAM block are untrusted.  A block that claims more than this is refused on its own
// (HGPU_CRAM_ERR_DECODE, what the reference's cram_uncompress_block returns when its malloc fails); blocks above
// BIG_BLOCK are launched one at a time so that their scratch (3 x size per resident CTA) is sized for one CTA.
static const uint32_t MAX_BLOCK = 1u << 30, BIG_BLOCK = 16u << 20;

static int cram_uncompress_impl(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len,
        const hgpu_cram_block *blocks, uint32_t n, uint8_t *out, const uint64_t *out_off,
        uint32_t *got_len, int32_t *status)
{
    if (!ctx || (n && (!file || !blocks || !out || !out_off || !got_len || !status))) { hgpu_set_error("bad argument"); return HGPU_ERR_ARG; }
    if (n == 0) return HGPU_OK;
    if (hgpu_check(cudaSetDevice(ctx->device), "cudaSetDevice")) return HGPU_ERR_CUDA;

    // ---- sort the blocks by codec
    std::vector<uint32_t> idx[9];
    uint64_t out_lo = ~0ull, out_hi = 0;
    for (uint32_t i = 0; i < n; i++) {
        const hgpu_cram_block &b = blocks[i];
        got_len[i] = 0;
        if (b.data_off < b.hdr_len || b.data_off + (uint64_t)b.comp_size + 4 > file_len) { hgpu_set_error("block %u lies outside the file image", i); return HGPU_ERR_ARG; }
        status[i] = b.method <= 8 ? HGPU_OK : HGPU_CRAM_ERR_DECODE;           // default: -1 (cram_io.c:1749)
        if (b.uncomp_size > MAX_BLOCK) { status[i] = HGPU_CRAM_ERR_DECODE; continue; }
        if (b.method <= 8) idx[b.method].push_back(i);
        if (b.uncomp_size && (b.method == 1 || b.method == 4 || b.method == 5 || b.method == 6)) {
            if (out_off[i] < out_lo) out_lo = out_off[i];
            if (out_off[i] + b.uncomp_size > out_hi) out_hi = out_off[i] + b.uncomp_size;
        }
    }
    if (out_lo > out_hi) out_lo = out_hi = 0;
    const uint64_t out_span = out_hi - out_lo;

    // ---- tok3 name blocks (their own host entry point; it uses the staging buffer, so it goes first)
    std::vector<uint8_t> tok_out;
    std::vector<uint64_t> t_in_off, t_out_off;
    std::vector<uint32_t> t_in_len, t_cap, t_got;
    std::vector<int32_t> t_st;
    {
        uint64_t acc = 0;
        for (uint32_t i : idx[8]) {
            const hgpu_cram_block &b = blocks[i];
            if (b.uncomp_size == 0) continue;
            uint32_t cap = hgpu_tok3_out_bound(file + b.data_off, b.comp_size);
            if (cap < 1024) cap = 1024;
            if (cap > b.uncomp_size + 1024u) cap = b.uncomp_size + 1024u;     // the block header bounds what the stream may claim
            t_in_off.push_back(b.data_off); t_in_len.push_back(b.comp_size);
            t_out_off.push_back(acc); t_cap.push_back(cap);
            acc += cap;
        }
        if (!t_in_off.empty()) {
            tok_out.resize(acc);
            t_got.resize(t_in_off.size()); t_st.resize(t_in_off.size());
            int rc = hgpu_tok3_decode_batch_host(ctx, file, t_in_off.data(), t_in_len.data(), (uint32_t)t_in_off.size(),
                                                 tok_out.data(), t_out_off.data(), t_cap.data(), t_got.data(), t_st.data());
            if (rc) return rc;
        }
    }

    // ---- fqzcomp quality blocks (same arrangement: own entry point, own use of the staging buffer)
    std::vector<uint64_t> f_in_off, f_out_off;
    std::vector<uint32_t> f_in_len, f_cap, f_got;
    std::vector<int32_t> f_st;
    std::vector<uint8_t> fqz_out;                                             // copied into place after the big download below
    {
        uint64_t acc = 0;
        for (uint32_t i : idx[7]) {
            const hgpu_cram_block &b = blocks[i];
            if (b.uncomp_size == 0) continue;
            f_in_off.push_back(b.data_off); f_in_len.push_back(b.comp_size);
            f_out_off.push_back(acc); f_cap.push_back(b.uncomp_size);
            acc += ((uint64_t)b.uncomp_size + 15) & ~(uint64_t)15;
        }
        if (!f_in_off.empty()) {
            fqz_out.resize(acc);
            f_got.resize(f_in_off.size()); f_st.resize(f_in_off.size());
            int rc = hgpu_fqz_decode_batch_host(ctx, file, f_in_off.data(), f_in_len.data(), (uint32_t)f_in_off.size(),
                                                fqz_out.data(), f_out_off.data(), f_cap.data(), f_got.data(), f_st.data());
            if (rc) return rc;
        }
    }

    // ---- device staging: file image, the output span (same layout as the caller's), job arrays
    std::vector<uint32_t> order;                                              // job order: 4x8, Nx16, arith
    uint32_t big5 = 0, big6 = 0;                                              // blocks launched on their own, at the end of their group
    for (int m : {4, 5, 6}) {
        for (uint32_t i : idx[m]) if (blocks[i].uncomp_size && (m == 4 || blocks[i].uncomp_size <= BIG_BLOCK)) order.push_back(i);
        if (m != 4) for (uint32_t i : idx[m]) if (blocks[i].uncomp_size > BIG_BLOCK) { order.push_back(i); (m == 5 ? big5 : big6)++; }
    }
    // GZIP blocks (method 1, zlib_mem_inflate cram_io.c:1068-1157): whole gzip members of any size, one warp each
    uint32_t n1 = 0;
    for (uint32_t i : idx[1]) if (blocks[i].uncomp_size && blocks[i].comp_size >= 18) { order.push_back(i); n1++; }
    const uint32_t nj = (uint32_t)order.size();
    uint32_t n4 = 0, n5 = 0, n6 = 0, max5 = 0, max6 = 0;
    std::vector<uint64_t> jio(nj), joo(nj), coff(n);
    std::vector<uint32_t> jil(nj), jol(nj), clen(n);
    for (uint32_t k = 0; k < nj; k++) {
        const hgpu_cram_block &b = blocks[order[k]];
        jio[k] = b.data_off; jil[k] = b.comp_size; joo[k] = out_off[order[k]] - out_lo; jol[k] = b.uncomp_size;
        if (b.method == 1) continue;
        if (b.method == 4) n4++;
        else if (b.method == 5) { n5++; if (b.uncomp_size > max5 && b.uncomp_size <= BIG_BLOCK) max5 = b.uncomp_size; }
        else { n6++; if (b.uncomp_size > max6 && b.uncomp_size <= BIG_BLOCK) max6 = b.uncomp_size; }
    }
    for (uint32_t i = 0; i < n; i++) { coff[i] = blocks[i].data_off - blocks[i].hdr_len; clen[i] = blocks[i].hdr_len + blocks[i].comp_size; }
    StageLayout L;
    const auto s_file = L.seg(file_len + 8), s_out = L.seg(out_span + 8), s_jio = L.seg((size_t)nj * 8), s_joo = L.seg((size_t)nj * 8),
               s_jil = L.seg((size_t)nj * 4), s_jol = L.seg((size_t)nj * 4), s_got = L.seg((size_t)nj * 4), s_st = L.seg((size_t)nj * 4),
               s_coff = L.seg((size_t)n * 8), s_clen = L.seg((size_t)n * 4), s_crc = L.seg((size_t)n * 4);
    int rc = hgpu_stage_ensure(ctx, L);
    if (rc) return rc;
    cudaStream_t s = ctx->stream;
    if (hgpu_h2d(L.at(s_file), file, file_len, s) || hgpu_h2d(L.at(s_coff), coff.data(), (size_t)n * 8, s) ||
        hgpu_h2d(L.at(s_clen), clen.data(), (size_t)n * 4, s) || hgpu_h2d(L.at(s_jio), jio.data(), (size_t)nj * 8, s) ||
        hgpu_h2d(L.at(s_joo), joo.data(), (size_t)nj * 8, s) || hgpu_h2d(L.at(s_jil), jil.data(), (size_t)nj * 4, s) ||
        hgpu_h2d(L.at(s_jol), jol.data(), (size_t)nj * 4, s)) return HGPU_ERR_CUDA;
    uint8_t *d_file = L.at(s_file), *d_out = L.at(s_out);
    rc = hgpu_launch_crc32_batch(ctx, d_file, L.at<uint64_t>(s_coff), L.at<uint32_t>(s_clen), n, L.at<uint32_t>(s_crc), s);
    if (rc) return rc;
    const uint64_t *d_jio = L.at<uint64_t>(s_jio), *d_joo = L.at<uint64_t>(s_joo);
    const uint32_t *d_jil = L.at<uint32_t>(s_jil), *d_jol = L.at<uint32_t>(s_jol);
    uint32_t *d_got = L.at<uint32_t>(s_got);
    int32_t *d_st = L.at<int32_t>(s_st);
    if (n4) {
        rc = hgpu_rans4x8_decode_batch_dev(ctx, d_file, d_jio, d_jil, n4, d_out, d_joo, d_jol, d_got, d_st, s);
        if (rc) return rc;
    }
    std::vector<uint32_t> nomem;                                              // big blocks whose own scratch could not be had
    if (n5 - big5) {
        rc = hgpu_launch_rans_nx16(ctx, d_file, d_jio + n4, d_jil + n4, n5 - big5, d_out, d_joo + n4, d_jol + n4,
                                   d_got + n4, d_st + n4, max5, s);
        if (rc) return rc;
    }
    for (uint32_t k = n4 + n5 - big5; k < n4 + n5; k++) {
        rc = hgpu_launch_rans_nx16(ctx, d_file, d_jio + k, d_jil + k, 1, d_out, d_joo + k, d_jol + k, d_got + k, d_st + k, jol[k], s);
        if (rc == HGPU_ERR_NOMEM) nomem.push_back(k); else if (rc) return rc;
    }
    if (n6 - big6) {
        rc = hgpu_arith_decode_batch_dev(ctx, d_file, d_jio + n4 + n5, d_jil + n4 + n5, n6 - big6, d_out, d_joo + n4 + n5,
                                         d_jol + n4 + n5, d_got + n4 + n5, d_st + n4 + n5, max6, s);
        if (rc) return rc;
    }
    for (uint32_t k = n4 + n5 + n6 - big6; k < n4 + n5 + n6; k++) {
        rc = hgpu_arith_decode_batch_dev(ctx, d_file, d_jio + k, d_jil + k, 1, d_out, d_joo + k, d_jol + k, d_got + k, d_st + k, jol[k], s);
        if (rc == HGPU_ERR_NOMEM) nomem.push_back(k); else if (rc) return rc;
    }
    if (n1) {
        const uint32_t k0 = n4 + n5 + n6;
        rc = hgpu_launch_gzip_inflate(ctx, d_file, d_jio + k0, d_jil + k0, n1, d_out, d_joo + k0, d_jol + k0, d_got + k0, d_st + k0, s);
        if (rc) return rc;
    }
    std::vector<uint32_t> jgot(nj), crc(n);
    std::vector<int32_t> jst(nj);
    if (hgpu_d2h(out + out_lo, d_out, out_span, s) || hgpu_d2h(jgot.data(), d_got, (size_t)nj * 4, s) ||
        hgpu_d2h(jst.data(), d_st, (size_t)nj * 4, s) || hgpu_d2h(crc.data(), L.at(s_crc), (size_t)n * 4, s)) return HGPU_ERR_CUDA;
    if (hgpu_check(cudaStreamSynchronize(s), "sync")) return HGPU_ERR_CUDA;

    for (uint32_t k : nomem) jst[k] = HGPU_CRAM_ERR_DECODE;                    // never launched: its status word is stale
    // ---- results, in the reference's order of checks: CRC first, then the codec, then the size
    for (uint32_t k = 0; k < nj; k++) {
        const uint32_t i = order[k];
        // a gzip member the device decoder declines (a deflate block beyond its match-record limit, a zlib wrapper) goes back
        // to the host library rather than being called corrupt
        if (blocks[i].method == 1 && (jst[k] == HGPU_BGZF_ERR_ZLIB || jst[k] == HGPU_BGZF_ERR_HEADER || jst[k] == HGPU_BGZF_ERR_SPACE)) status[i] = HGPU_CRAM_UNSUPPORTED;
        else if (jst[k] != HGPU_OK || jgot[k] != blocks[i].uncomp_size) status[i] = HGPU_CRAM_ERR_DECODE;   // usize != usize2
        else { got_len[i] = jgot[k]; status[i] = HGPU_OK; }
    }
    for (uint32_t i : idx[0]) {                                               // RAW: the payload is the data
        const hgpu_cram_block &b = blocks[i];
        const uint32_t m = b.comp_size < b.uncomp_size ? b.comp_size : b.uncomp_size;
        memcpy(out + out_off[i], file + b.data_off, m);
        got_len[i] = m;
    }
    for (int m : {2, 3}) for (uint32_t i : idx[m]) status[i] = blocks[i].uncomp_size ? HGPU_CRAM_UNSUPPORTED : HGPU_OK;
    for (uint32_t i : idx[1]) if (blocks[i].uncomp_size && blocks[i].comp_size < 18) status[i] = HGPU_CRAM_UNSUPPORTED;
    {
        size_t t = 0;
        for (uint32_t i : idx[7]) {
            if (blocks[i].uncomp_size == 0) continue;
            if (f_st[t] != HGPU_OK) status[i] = HGPU_CRAM_ERR_DECODE;
            else { memcpy(out + out_off[i], fqz_out.data() + f_out_off[t], f_got[t]); got_len[i] = f_got[t]; }
            t++;
        }
    }
    {
        size_t t = 0;
        for (uint32_t i : idx[8]) {
            const hgpu_cram_block &b = blocks[i];
            if (b.uncomp_size == 0) continue;
            if (t_st[t] != HGPU_OK) status[i] = HGPU_CRAM_ERR_DECODE;
            else if (t_got[t] > b.uncomp_size) status[i] = HGPU_CRAM_ERR_SPACE;  // the reference adopts the new size; the slot cannot
            else { memcpy(out + out_off[i], tok_out.data() + t_out_off[t], t_got[t]); got_len[i] = t_got[t]; }
            t++;
        }
    }
    for (uint32_t i = 0; i < n; i++) {
        const hgpu_cram_block &b = blocks[i];
        const uint8_t *c = file + b.data_off + b.comp_size;
        const uint32_t want = c[0] | c[1] << 8 | c[2] << 16 | (uint32_t)c[3] << 24;
        if (crc[i] != want) { status[i] = HGPU_CRAM_ERR_CRC; got_len[i] = 0; }
    }
    return HGPU_OK;
}

extern "C" int hgpu_cram_uncompress_blocks_host(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len,
        const hgpu_cram_block *blocks, uint32_t n, uint8_t *out, const uint64_t *out_off,
        uint32_t *got_len, int32_t *status)
{
    return hgpu_abi_call([&] { return cram_uncompress_impl(ctx, file, file_len, blocks, n, out, out_off, got_len, status); });
}
