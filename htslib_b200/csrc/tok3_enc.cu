// CRAM 3.1 read-name tokeniser ("tok3", block method 8) — ENCODE side.
//
// Stands where tok3_encode_names stands (htscodecs/htscodecs/tokenise_name3.c:1451-1665, encode_name
// :697-1021, compress :1268-1417) as called from cram_compress_by_method (cram/cram_io.c:1885-1899),
// for a batch of name blocks.  Like the rANS Nx16 encoder of this library it is NOT the reference's
// byte stream: the bar is that the reference's tok3_decode_names (and this library's decoder) rebuild the
// names exactly, at a stated size ratio (tests/test_gpu_tok3_enc.py).  What differs by design:
//   * every name is diffed against the one before it (dist 1; identical -> N_DUP).  The reference searches
//     a trie for the best earlier name; the format does not require it.
//   * tokens come from the text alone: letter runs (N_ALPHA), digit runs of up to 9 starting with '0'
//     (N_DIGITS0 + N_DZLEN) or not (N_DIGITS), any other byte (N_CHAR); against the previous name's token
//     at the same position they become N_MATCH, N_DDELTA / N_DDELTA0 (0 < delta < 256) or stay literal.
//   * each token stream is entropy-coded by this library's rANS Nx16 encoder: order 0, order 1 and the reference's level-3
//     transform choices for its type (PACK / RLE / 4-way STRIPE, compress() :1299-1313), all tried, smallest kept.
// Work split: tok3_tokenise_kernel<0> counts the bytes of every (position, type) stream, one THREAD per
// block (a name's tokens depend on the previous name's, a serial chain); the host lays the streams out;
// tok3_tokenise_kernel<1> writes them; one rANS encode launch covers all streams of all blocks; the
// host writes the descriptor framing (ttype byte, varint length, stream) the decoder walks (:1706-1806).
#include "tok3_internal.h"
#include <vector>
#include <string.h>

namespace {

constexpr uint32_t NSTREAM = TOK_MAX * 16;

struct EncMeta { uint32_t nreads, max_tok, ulen; int32_t status; };

__device__ __forceinline__ bool is_alpha(uint32_t c) { c |= 32; return c >= 'a' && c <= 'z'; }
__device__ __forceinline__ bool is_digit(uint32_t c) { return c >= '0' && c <= '9'; }

template <int PASS>
__global__ void __launch_bounds__(32) tok3_tokenise_kernel(const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len, uint32_t n,
        uint32_t *cnt, const uint32_t *soff, uint8_t *arena, const uint64_t *arena_off, EncMeta *meta)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n) return;
    const uint8_t *blob = in + in_off[b];
    const uint32_t blen = in_len[b];
    uint32_t *C = cnt + (size_t)b * NSTREAM;                        // PASS 0: byte counts; PASS 1: write cursors
    const uint32_t *SO = soff + (size_t)b * NSTREAM;
    uint8_t *A = PASS ? arena + arena_off[b] : nullptr;

    auto put1 = [&](uint32_t k, uint32_t t, uint32_t v) {
        const uint32_t id = k * 16 + t;
        if (PASS) A[SO[id] + C[id]] = (uint8_t)v;
        C[id] += 1;
    };
    auto put4 = [&](uint32_t k, uint32_t t, uint32_t v) {
        const uint32_t id = k * 16 + t;
        if (PASS) { uint8_t *d = A + SO[id] + C[id]; d[0] = (uint8_t)v; d[1] = (uint8_t)(v >> 8); d[2] = (uint8_t)(v >> 16); d[3] = (uint8_t)(v >> 24); }
        C[id] += 4;
    };
    auto puts = [&](uint32_t k, uint32_t t, const uint8_t *s, uint32_t l) {   // string + NUL
        const uint32_t id = k * 16 + t;
        if (PASS) { uint8_t *d = A + SO[id] + C[id]; for (uint32_t i = 0; i < l; i++) d[i] = s[i]; d[l] = 0; }
        C[id] += l + 1;
    };

    // token lists of the previous and the current name: type, numeric value, text range
    uint8_t ty[2][TOK_MAX];
    uint32_t val[2][TOK_MAX];
    uint16_t ts[2][TOK_MAX], tl[2][TOK_MAX];
    uint32_t pn = 0, prev_ntok = 0, prev_start = 0, prev_len = 0, cur = 0;
    bool have_prev = false;
    uint32_t nreads = 0, max_tok = 1, ulen = 0;
    int status = 0;

    uint32_t p = 0;
    while (p < blen) {
        uint32_t q = p;
        while (q < blen && blob[q] > '\n') q++;                      // names end in NUL or LF (:1460-1462)
        if (q >= blen) break;                                        // an unterminated tail is left out (:1471-1477)
        const uint8_t *nm = blob + p;
        const uint32_t len = q - p;
        if (len > 65535) { status = -1; break; }
        bool same = have_prev && len == prev_len;
        if (same) for (uint32_t i = 0; i < len; i++) if (nm[i] != blob[prev_start + i]) { same = false; break; }
        if (same) {                                                  // exact duplicate of the previous name
            put1(0, T_TYPE, T_DUP);
            put4(0, T_DUP, 1);
        } else {
            put1(0, T_TYPE, T_DIFF);
            put4(0, T_DIFF, have_prev ? 1u : 0u);
            cur = pn ^ 1;
            uint32_t k = 1, i = 0;
            while (i < len) {
                if (k >= (uint32_t)TOK_MAX - 1) { status = -1; break; }       // more token positions than the format has (:991-995)
                const uint32_t c = nm[i];
                uint32_t j = i + 1, type, v = 0;
                if (is_alpha(c)) { type = T_ALPHA; while (j < len && is_alpha(nm[j])) j++; }
                else if (is_digit(c)) {
                    type = c == '0' ? T_DIGITS0 : T_DIGITS;
                    v = c - '0';
                    while (j < len && is_digit(nm[j]) && j - i < 9) { v = v * 10 + (nm[j] - '0'); j++; }
                } else type = T_CHAR;
                const uint32_t l = j - i;
                const bool hp = have_prev && k < prev_ntok;
                const uint32_t ptype = hp ? ty[pn][k] : 255u;
                bool match = false;
                if (type == T_ALPHA) {
                    if (ptype == T_ALPHA && tl[pn][k] == l) {
                        match = true;
                        const uint8_t *o = blob + prev_start + ts[pn][k];
                        for (uint32_t x = 0; x < l; x++) if (o[x] != nm[i + x]) { match = false; break; }
                    }
                    if (match) put1(k, T_TYPE, T_MATCH);
                    else { put1(k, T_TYPE, T_ALPHA); puts(k, T_ALPHA, nm + i, l); }
                } else if (type == T_CHAR) {
                    if (ptype == T_CHAR && val[pn][k] == c) put1(k, T_TYPE, T_MATCH);
                    else { put1(k, T_TYPE, T_CHAR); put1(k, T_CHAR, c); }
                    v = c;
                } else if (type == T_DIGITS0) {
                    const bool cmp = ptype == T_DIGITS0 && tl[pn][k] == l;
                    const uint32_t d = v - val[pn][k];
                    if (cmp && d == 0) put1(k, T_TYPE, T_MATCH);
                    else if (cmp && v > val[pn][k] && d < 256) { put1(k, T_TYPE, T_DDELTA0); put1(k, T_DDELTA0, d); }
                    else { put1(k, T_TYPE, T_DIGITS0); put4(k, T_DIGITS0, v); put1(k, T_DZLEN, l); }
                } else {
                    const bool cmp = ptype == T_DIGITS;
                    const uint32_t d = v - val[pn][k];
                    if (cmp && d == 0) put1(k, T_TYPE, T_MATCH);
                    else if (cmp && v > val[pn][k] && d < 256) { put1(k, T_TYPE, T_DDELTA); put1(k, T_DDELTA, d); }
                    else { put1(k, T_TYPE, T_DIGITS); put4(k, T_DIGITS, v); }
                }
                ty[cur][k] = (uint8_t)type; val[cur][k] = v; ts[cur][k] = (uint16_t)i; tl[cur][k] = (uint16_t)l;
                i = j; k++;
            }
            if (status) break;
            put1(k, T_TYPE, T_END);
            if (k + 1 > max_tok) max_tok = k + 1;
            prev_ntok = k; pn = cur;
            have_prev = true;
        }
        prev_start = p; prev_len = len;                              // a duplicate has the same text, so either copy serves
        nreads++;
        ulen += len + 1;
        p = q + 1;
    }
    if (nreads == 0) status = -1;                                    // create_context refuses an empty block (:172-174)
    if (!PASS) { EncMeta m; m.nreads = nreads; m.max_tok = max_tok; m.ulen = ulen; m.status = status; meta[b] = m; }
}

int put_varint(uint8_t *p, uint32_t v)                               // var_put_u32, varint.h:206
{
    int n = 1;
    while (n < 5 && (v >> (7 * n))) n++;
    for (int k = n - 1; k >= 0; k--) *p++ = (uint8_t)(((v >> (7 * k)) & 0x7f) | (k ? 0x80 : 0));
    return n;
}

}  // namespace

extern "C" uint32_t hgpu_tok3_compress_bound(uint32_t in_len)
{
    const uint64_t b = 14ull * in_len + 32768;
    return b > 0xffffffffull ? 0xffffffffu : (uint32_t)b;
}

static int hgpu_tok3_encode_batch_host_impl(hgpu_ctx *ctx, const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len,
        uint32_t n, uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap, uint32_t *out_len, int32_t *status)
{
    if (!ctx || (n && (!in || !in_off || !in_len || !out || !out_off || !out_cap || !out_len || !status))) {
        hgpu_set_error("bad argument");
        return HGPU_ERR_ARG;
    }
    if (n == 0) return HGPU_OK;
    if (hgpu_check(cudaSetDevice(ctx->device), "cudaSetDevice")) return HGPU_ERR_CUDA;
    cudaStream_t s = ctx->stream;

    // ---- pass 0: sizes of every (position, type) stream
    const uint64_t in_end = hgpu_slots_end(in_off, in_len, n);
    StageLayout L;
    const auto s_in = L.seg(in_end + 8), s_ioff = L.seg((size_t)n * 8), s_ilen = L.seg((size_t)n * 4), s_cnt = L.seg((size_t)n * NSTREAM * 4),
               s_soff = L.seg((size_t)n * NSTREAM * 4), s_meta = L.seg((size_t)n * sizeof(EncMeta)), s_aoff = L.seg((size_t)n * 8);
    const size_t fixed_end = L.total;
    // the stream arena (each stream 16-byte aligned) is sized from the counts of pass 0, which does not touch it
    std::vector<uint64_t> aoff(n, 0);
    StageLayout arena;                             // one 256-byte-aligned region per block
    int rc = hgpu_stage_ensure(ctx, L);
    if (rc) return rc;
    if (hgpu_h2d(L.at(s_in), in, in_end, s) || hgpu_h2d(L.at(s_ioff), in_off, (size_t)n * 8, s) || hgpu_h2d(L.at(s_ilen), in_len, (size_t)n * 4, s) ||
        hgpu_memset(L.at(s_cnt), 0, (size_t)n * NSTREAM * 4, s)) return HGPU_ERR_CUDA;
    tok3_tokenise_kernel<0><<<(n + 31) / 32, 32, 0, s>>>(L.at(s_in), L.at<uint64_t>(s_ioff), L.at<uint32_t>(s_ilen), n, L.at<uint32_t>(s_cnt),
                                                         L.at<uint32_t>(s_soff), L.base + fixed_end, L.at<uint64_t>(s_aoff), L.at<EncMeta>(s_meta));
    if (hgpu_check(cudaGetLastError(), "tok3_tokenise_kernel<0>")) return HGPU_ERR_CUDA;
    hgpu_count_launch();
    std::vector<uint32_t> cnt((size_t)n * NSTREAM), soff((size_t)n * NSTREAM, 0);
    std::vector<EncMeta> meta(n);
    if (hgpu_d2h(cnt.data(), L.at(s_cnt), cnt.size() * 4, s) || hgpu_d2h(meta.data(), L.at(s_meta), (size_t)n * sizeof(EncMeta), s)) return HGPU_ERR_CUDA;
    if (hgpu_check(cudaStreamSynchronize(s), "sync")) return HGPU_ERR_CUDA;

    // ---- layout + the entropy-coder job list: each stream once with order 0, streams of >= 64 bytes also with order 1
    struct StreamRef { uint32_t block, id, job0, njobs; };
    std::vector<StreamRef> streams;
    std::vector<uint64_t> jio, joo;
    std::vector<uint32_t> jil, jord, jcap;
    uint64_t comp_bytes = 0;
    for (uint32_t b = 0; b < n; b++) {
        aoff[b] = arena.total;
        if (meta[b].status) continue;
        uint32_t o = 0;
        for (uint32_t id = 0; id < meta[b].max_tok * 16 && id < NSTREAM; id++) {
            const uint32_t c = cnt[(size_t)b * NSTREAM + id];
            if (!c) continue;
            soff[(size_t)b * NSTREAM + id] = o;
            // candidate orders: 0, 1 (>= 64 bytes), and what the reference tries for this stream type at CRAM's level 3
            // (compress(), tokenise_name3.c:1299-1313: PACK / RLE for the type and alphabet streams, 4-way STRIPE for the
            // 32-bit integer streams); the smallest stream wins below
            static const int k_l3[13][2] = {{192, -1}, {129, -1}, {-1, -1}, {136, -1}, {-1, -1}, {200, -1}, {136, -1}, {200, -1}, {-1, -1}, {128, -1}, {-1, -1}, {-1, -1}, {-1, -1}};
            uint32_t ords[4], no = 0;
            ords[no++] = 0;
            if (c >= 64) ords[no++] = 1;
            const uint32_t ty = id & 15;
            if (ty < 13 && c >= 16)
                for (int q = 0; q < 2; q++) { const int m = k_l3[ty][q]; if (m > 1 && (!(m & 8) || c % 4 == 0)) ords[no++] = (uint32_t)m; }
            StreamRef r{b, id, (uint32_t)jio.size(), no};
            for (uint32_t k = 0; k < r.njobs; k++) {
                jio.push_back(fixed_end + aoff[b] + o);                          // relative to the input's region (at 0), the encoder's d_in
                jil.push_back(c); jord.push_back(ords[k]);
                const uint32_t cap = c + 256;                                    // every level of the coder falls back to CAT, so c + framing is enough
                joo.push_back(comp_bytes); jcap.push_back(cap);
                comp_bytes += (cap + 15) & ~15u;
            }
            streams.push_back(r);
            o += (c + 15) & ~15u;
        }
        arena.seg((size_t)o + 16);
    }
    const uint32_t nj = (uint32_t)jio.size();
    // second part of the staging layout, behind the arena: job arrays and the compressed streams
    L.seg(arena.total + 64);
    const auto s_jio = L.seg((size_t)nj * 8), s_joo = L.seg((size_t)nj * 8), s_jil = L.seg((size_t)nj * 4), s_jord = L.seg((size_t)nj * 4),
               s_jcap = L.seg((size_t)nj * 4), s_jlen = L.seg((size_t)nj * 4), s_jst = L.seg((size_t)nj * 4), s_comp = L.seg(comp_bytes + 64);
    // growing the staging buffer moves it: the arena is rebuilt by pass 1 anyway, but the input has to be uploaded again
    bool moved = false;
    rc = hgpu_stage_ensure(ctx, L, &moved);
    if (rc) return rc;
    if (moved && (hgpu_h2d(L.at(s_in), in, in_end, s) || hgpu_h2d(L.at(s_ioff), in_off, (size_t)n * 8, s) ||
                  hgpu_h2d(L.at(s_ilen), in_len, (size_t)n * 4, s))) return HGPU_ERR_CUDA;
    if (hgpu_h2d(L.at(s_aoff), aoff.data(), (size_t)n * 8, s) || hgpu_memset(L.at(s_cnt), 0, (size_t)n * NSTREAM * 4, s) ||
        hgpu_h2d(L.at(s_soff), soff.data(), soff.size() * 4, s)) return HGPU_ERR_CUDA;
    tok3_tokenise_kernel<1><<<(n + 31) / 32, 32, 0, s>>>(L.at(s_in), L.at<uint64_t>(s_ioff), L.at<uint32_t>(s_ilen), n, L.at<uint32_t>(s_cnt),
                                                         L.at<uint32_t>(s_soff), L.base + fixed_end, L.at<uint64_t>(s_aoff), L.at<EncMeta>(s_meta));
    if (hgpu_check(cudaGetLastError(), "tok3_tokenise_kernel<1>")) return HGPU_ERR_CUDA;
    hgpu_count_launch();
    std::vector<uint32_t> jlen(nj);
    std::vector<int32_t> jst(nj);
    std::vector<uint8_t> comp(comp_bytes + 64);
    if (nj) {
        if (hgpu_h2d(L.at(s_jio), jio.data(), (size_t)nj * 8, s) || hgpu_h2d(L.at(s_joo), joo.data(), (size_t)nj * 8, s) ||
            hgpu_h2d(L.at(s_jil), jil.data(), (size_t)nj * 4, s) || hgpu_h2d(L.at(s_jord), jord.data(), (size_t)nj * 4, s) ||
            hgpu_h2d(L.at(s_jcap), jcap.data(), (size_t)nj * 4, s)) return HGPU_ERR_CUDA;
        rc = hgpu_rans_nx16_encode_batch_dev(ctx, L.at(s_in), L.at<uint64_t>(s_jio), L.at<uint32_t>(s_jil), L.at<uint32_t>(s_jord), nj,
                                             L.at(s_comp), L.at<uint64_t>(s_joo), L.at<uint32_t>(s_jcap), L.at<uint32_t>(s_jlen),
                                             L.at<int32_t>(s_jst), s);
        if (rc) return rc;
        if (hgpu_d2h(jlen.data(), L.at(s_jlen), (size_t)nj * 4, s) || hgpu_d2h(jst.data(), L.at(s_jst), (size_t)nj * 4, s) ||
            hgpu_d2h(comp.data(), L.at(s_comp), comp_bytes, s)) return HGPU_ERR_CUDA;
    }
    if (hgpu_check(cudaStreamSynchronize(s), "sync")) return HGPU_ERR_CUDA;

    // ---- framing (tok3_decode_names walks exactly this, :1706-1806): header, then per stream ttype, varint size, bytes
    std::vector<uint32_t> wp(n, 0);
    std::vector<int> last_tok(n, -1);
    for (uint32_t b = 0; b < n; b++) {
        status[b] = HGPU_TOK3_ERR; out_len[b] = 0;
        if (meta[b].status || out_cap[b] < 9) continue;
        uint8_t *o = out + out_off[b];
        const uint32_t ul = meta[b].ulen, nr = meta[b].nreads;
        o[0] = (uint8_t)ul; o[1] = (uint8_t)(ul >> 8); o[2] = (uint8_t)(ul >> 16); o[3] = (uint8_t)(ul >> 24);
        o[4] = (uint8_t)nr; o[5] = (uint8_t)(nr >> 8); o[6] = (uint8_t)(nr >> 16); o[7] = (uint8_t)(nr >> 24);
        o[8] = 0;                                                    // use_arith = 0: rANS Nx16 sub-streams
        wp[b] = 9;
        status[b] = HGPU_OK;
    }
    for (const StreamRef &r : streams) {                             // streams are in (block, position, type) order
        const uint32_t b = r.block;
        if (status[b] != HGPU_OK) continue;
        uint32_t best = 0xffffffffu, bj = 0;
        for (uint32_t k = 0; k < r.njobs; k++)
            if (jst[r.job0 + k] == 0 && jlen[r.job0 + k] && jlen[r.job0 + k] < best) { best = jlen[r.job0 + k]; bj = r.job0 + k; }
        if (best == 0xffffffffu || (uint64_t)wp[b] + 6 + best > out_cap[b]) { status[b] = HGPU_TOK3_ERR; continue; }
        uint8_t *o = out + out_off[b] + wp[b];
        const int tnum = (int)(r.id >> 4);
        *o++ = (uint8_t)((r.id & 15) | (tnum != last_tok[b] ? 128 : 0));   // bit 7: first stream of a new token position
        last_tok[b] = tnum;
        o += put_varint(o, best);
        memcpy(o, comp.data() + joo[bj], best);
        wp[b] = (uint32_t)(o + best - (out + out_off[b]));
    }
    for (uint32_t b = 0; b < n; b++) out_len[b] = status[b] == HGPU_OK ? wp[b] : 0;
    return HGPU_OK;
}

extern "C" int hgpu_tok3_encode_batch_host(hgpu_ctx *ctx, const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len,
        uint32_t n, uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap, uint32_t *out_len, int32_t *status)
{
    return hgpu_abi_call([&] { return hgpu_tok3_encode_batch_host_impl(ctx, in, in_off, in_len, n, out, out_off, out_cap, out_len, status); });
}
