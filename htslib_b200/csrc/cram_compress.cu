// hgpu_cram_compress_blocks_host — the method trial of cram_compress_block2 / cram_compress_block3
// (cram/cram_io.c:1912-2308: "try every method the mask allows, keep the smallest") for a whole batch of blocks, with
// cram_compress_by_method's mapping from methods to codec calls (:1697-1897) and cram_write_block's framing (:1511-1563).
//
// Stateless form: the reference amortises the trial over many slices with cram_metrics (trial every N-th block, then
// reuse the winner); here every block is tried with every allowed method in the same launches, because the candidates
// of all blocks are one job list per codec — three launches (rANS 4x8, rANS Nx16, adaptive arithmetic) whatever the
// number of blocks and methods.  The winner of a block is the smallest stream; RAW when nothing is smaller than the
// data (cram_compress_block3 :2283-2298).  Not tried here (left in the mask, ignored): GZIP / GZIP_RLE / GZIP_1 / BZIP2 /
// LZMA (the device deflate writes BGZF members, not one zlib stream), FQZ (needs the slice's record lengths:
// hgpu_fqz_encode_batch_host), TOK3 / TOKA (hgpu_tok3_encode_batch_host).
#include "hgpu_internal.h"
#include <vector>
#include <string.h>

namespace {

// enum cram_block_method_int, cram/cram_structs.h:215-266
enum { M_RAW = 0, M_RANS0 = 4, M_RANS_PR0 = 5, M_ARITH_PR0 = 6, M_RANS1 = 16, M_RANS_PR1 = 17, M_RANS_PR193 = 23, M_ARITH_PR1 = 25, M_ARITH_PR193 = 31 };
const int k_methmap[7] = {1, 64, 9, 128, 129, 192, 193};               // cram_io.c:1854, :1875

struct Cand { uint32_t block; int method; int codec; uint32_t order; uint32_t cap; };   // codec: 0 rANS 4x8, 1 rANS Nx16, 2 arith
inline size_t up16(size_t x) { return (x + 15) & ~(size_t)15; }

int compress_impl(hgpu_ctx *ctx, const uint8_t *const *payload, const uint32_t *payload_len, const uint32_t *method_mask,
                  const int32_t *content_id, const uint8_t *content_type, uint32_t n, uint8_t *out, uint64_t cap, uint64_t *out_off,
                  uint64_t *out_len, int32_t *chosen)
{
    if (!ctx || !payload || !payload_len || !method_mask || !content_id || !content_type || !out_len) { hgpu_set_error("cram compress: null argument"); return HGPU_ERR_ARG; }
    if (n == 0) { *out_len = 0; return HGPU_OK; }
    if (hgpu_check(cudaSetDevice(ctx->device), "cudaSetDevice")) return HGPU_ERR_CUDA;
    std::vector<Cand> cand;
    std::vector<uint64_t> in_off((size_t)n + 1, 0);
    uint32_t max_in = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (payload_len[i] && !payload[i]) { hgpu_set_error("cram compress: block %u has no payload", i); return HGPU_ERR_ARG; }
        in_off[i + 1] = in_off[i] + up16(payload_len[i]);
        if (payload_len[i] > max_in) max_in = payload_len[i];
        if (payload_len[i] == 0) continue;                                // cram_compress_block3 :1925-1931: nothing to do
        const uint32_t mask = method_mask[i], sz = payload_len[i];
        for (int m = 0; m < 32; m++) {
            if (!(mask & (1u << m))) continue;
            if (m == M_RANS0 || m == M_RANS1) cand.push_back({i, m, 0, m == M_RANS0 ? 0u : 1u, hgpu_rans4x8_compress_bound(sz)});
            else if (m == M_RANS_PR0 || (m >= M_RANS_PR1 && m <= M_RANS_PR193)) {
                uint32_t order = m == M_RANS_PR0 ? 0u : (uint32_t)k_methmap[m - M_RANS_PR1];
                if (sz >= 50000 && !(order & 8)) order |= 4;              // RANS_ORDER_SIMD_AUTO (rANS_static4x16pr.c:1234-1237)
                cand.push_back({i, m, 1, order, hgpu_rans_nx16_compress_bound(sz, (int)order)});
            } else if (m == M_ARITH_PR0 || (m >= M_ARITH_PR1 && m <= M_ARITH_PR193)) {
                uint32_t order = m == M_ARITH_PR0 ? 0u : (uint32_t)k_methmap[m - M_ARITH_PR1];
                if (order == 9) continue;                                  // X4 stripe: this encoder writes it unstriped, the plain order-1 candidate covers it
                cand.push_back({i, m, 2, order, hgpu_arith_compress_bound(sz, (int)order)});
            }
        }
    }
    const size_t nc = cand.size();
    // device image: [payloads | candidate outputs | job arrays]
    std::vector<uint64_t> c_in((size_t)nc + 1), c_out((size_t)nc + 1);
    std::vector<uint32_t> c_len((size_t)nc + 1), c_ord((size_t)nc + 1), c_cap((size_t)nc + 1);
    size_t out_bytes = 0;
    std::vector<size_t> order_idx[3];
    for (size_t k = 0; k < nc; k++) order_idx[cand[k].codec].push_back(k);
    size_t pos = 0;
    std::vector<size_t> slot(nc);                                          // job index of candidate k inside its codec's list
    std::vector<size_t> first(4, 0);
    for (int c = 0; c < 3; c++) {
        first[c] = pos;
        for (size_t k : order_idx[c]) {
            slot[k] = pos;
            c_in[pos] = in_off[cand[k].block]; c_len[pos] = payload_len[cand[k].block]; c_ord[pos] = cand[k].order; c_cap[pos] = cand[k].cap;
            c_out[pos] = out_bytes; out_bytes += up16((size_t)cand[k].cap + 16);
            pos++;
        }
    }
    first[3] = pos;
    StageLayout L;
    const auto s_in = L.seg(in_off[n] + 64), s_out = L.seg(out_bytes + 64), s_cin = L.seg((nc + 1) * 8), s_cout = L.seg((nc + 1) * 8),
               s_len = L.seg((nc + 1) * 4), s_ord = L.seg((nc + 1) * 4), s_cap = L.seg((nc + 1) * 4), s_got = L.seg((nc + 1) * 4),
               s_st = L.seg((nc + 1) * 4);
    int rc = hgpu_stage_ensure(ctx, L);
    if (rc) return rc;
    cudaStream_t st = ctx->stream;
    uint8_t *d_in = L.at(s_in), *d_out = L.at(s_out);
    for (uint32_t i = 0; i < n; i++)
        if (hgpu_h2d(d_in + in_off[i], payload[i], payload_len[i], st)) return HGPU_ERR_CUDA;
    uint64_t *d_cin = L.at<uint64_t>(s_cin), *d_cout = L.at<uint64_t>(s_cout);
    uint32_t *d_len = L.at<uint32_t>(s_len), *d_ord = L.at<uint32_t>(s_ord), *d_cap = L.at<uint32_t>(s_cap), *d_got = L.at<uint32_t>(s_got);
    int32_t *d_st = L.at<int32_t>(s_st);
    std::vector<uint32_t> got((size_t)nc + 1, 0);
    std::vector<int32_t> stt((size_t)nc + 1, 0);
    if (nc) {
        if (hgpu_h2d(d_cin, c_in.data(), nc * 8, st) || hgpu_h2d(d_cout, c_out.data(), nc * 8, st) || hgpu_h2d(d_len, c_len.data(), nc * 4, st) ||
            hgpu_h2d(d_ord, c_ord.data(), nc * 4, st) || hgpu_h2d(d_cap, c_cap.data(), nc * 4, st)) return HGPU_ERR_CUDA;
        for (int c = 0; c < 3; c++) {
            const size_t f = first[c], m = first[c + 1] - first[c];
            if (!m) continue;
            if (c == 0) rc = hgpu_rans4x8_encode_batch_dev(ctx, d_in, d_cin + f, d_len + f, d_ord + f, (uint32_t)m, d_out, d_cout + f, d_cap + f, d_got + f, d_st + f, st);
            else if (c == 1) rc = hgpu_rans_nx16_encode_batch_dev(ctx, d_in, d_cin + f, d_len + f, d_ord + f, (uint32_t)m, d_out, d_cout + f, d_cap + f, d_got + f, d_st + f, st);
            else rc = hgpu_arith_encode_batch_dev(ctx, d_in, d_cin + f, d_len + f, d_ord + f, (uint32_t)m, d_out, d_cout + f, d_cap + f, d_got + f, d_st + f, max_in, st);
            if (rc) return rc;
        }
        if (hgpu_d2h(got.data(), d_got, nc * 4, st) || hgpu_d2h(stt.data(), d_st, nc * 4, st) ||
            hgpu_check(cudaStreamSynchronize(st), "cram compress")) return HGPU_ERR_CUDA;
    }
    // winners
    std::vector<long> best((size_t)n, -1);
    for (size_t k = 0; k < nc; k++) {
        const size_t j = slot[k];
        if (stt[j] != HGPU_OK || got[j] == 0) continue;                    // "this method lost" (cram_io.c:2083-2087)
        const uint32_t b = cand[k].block;
        const uint32_t cur = best[b] < 0 ? payload_len[b] : got[slot[(size_t)best[b]]];
        if (got[j] < cur) best[b] = (long)k;
    }
    std::vector<std::vector<uint8_t>> comp((size_t)n);
    std::vector<hgpu_cram_block> blk((size_t)n);
    std::vector<const uint8_t *> pay((size_t)n);
    for (uint32_t i = 0; i < n; i++) {
        memset(&blk[i], 0, sizeof(hgpu_cram_block));
        blk[i].content_id = content_id[i]; blk[i].content_type = content_type[i]; blk[i].uncomp_size = payload_len[i];
        if (best[i] < 0) { blk[i].method = M_RAW; blk[i].comp_size = payload_len[i]; pay[i] = payload[i]; if (chosen) chosen[i] = M_RAW; continue; }
        const Cand &c = cand[(size_t)best[i]];
        const size_t j = slot[(size_t)best[i]];
        comp[i].resize(got[j]);
        if (hgpu_d2h(comp[i].data(), d_out + c_out[j], got[j], st)) return HGPU_ERR_CUDA;
        blk[i].method = (uint8_t)(c.codec == 0 ? 4 : c.codec == 1 ? 5 : 6);   // the externalised method (cram_structs.h:219-230)
        blk[i].comp_size = got[j];
        pay[i] = comp[i].data();
        if (chosen) chosen[i] = c.method;
    }
    if (hgpu_check(cudaStreamSynchronize(st), "cram compress D2H")) return HGPU_ERR_CUDA;
    return hgpu_cram_write_blocks_host(ctx, blk.data(), pay.data(), n, out, cap, out_off, out_len);
}

}  // namespace

extern "C" int hgpu_cram_compress_blocks_host(hgpu_ctx *ctx, const uint8_t *const *payload, const uint32_t *payload_len,
        const uint32_t *method_mask, const int32_t *content_id, const uint8_t *content_type, uint32_t n,
        uint8_t *out, uint64_t cap, uint64_t *out_off, uint64_t *out_len, int32_t *chosen)
{
    return hgpu_abi_call([&] { return compress_impl(ctx, payload, payload_len, method_mask, content_id, content_type, n, out, cap, out_off, out_len, chosen); },
                         HGPU_ERR_NOMEM, HGPU_ERR_NOMEM);
}
