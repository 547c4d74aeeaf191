// CRAM 3.1 read-name tokeniser ("tok3", block method 8) — decode side.
//
// Replaces tok3_decode_names (htscodecs/htscodecs/tokenise_name3.c:1679-1834) as called from
// cram_uncompress_block (cram/cram_io.c:1753-1765) for a BATCH of name blocks:
//   host   : walks each block's descriptor framing (ttype byte, dup links, varint sizes) and turns the
//            compressed token streams of all blocks into one job list;
//   device : the existing rANS-Nx16 / adaptive-arithmetic batch decoders expand every token stream
//            into an arena, then tok3_names_kernel (tok3_names.cu) rebuilds the names, one warp per block.
//
// Layout per block in HBM: a descriptor table of max_tok*16 {offset,len,synth} entries into the stream
// arena; a history table (nreads+1) x max_tok of {value, type|aux} so that any earlier name can be the
// reference of a later one (decode_name :1023-1210 keeps the same per-name token history); a name
// table {offset, ntok, history row}.  A duplicate name aliases its source's history row.
#include "tok3_internal.h"
#include <vector>
#include <string.h>
#include <stdlib.h>
#include <mutex>

namespace {

float g_tok3_ms[2];
struct Job { uint64_t in_off; uint32_t in_len; uint64_t out_off; uint32_t out_len; };

}  // namespace

extern "C" uint32_t hgpu_tok3_out_bound(const uint8_t *in, uint32_t len)
{
    if (!in || len < 9) return 0;
    uint32_t ulen = in[0] | in[1] << 8 | in[2] << 16 | (uint32_t)in[3] << 24;
    if ((int32_t)ulen < 0 || ulen >= 0x7fffffffu - 1024) return 0;
    return ulen + 1024;
}

static int hgpu_tok3_decode_batch_host_impl(hgpu_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
        const uint32_t *in_len, uint32_t n, uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
        uint32_t *out_len, int32_t *status)
{
    if (!ctx || (n && (!in || !in_off || !in_len || !out || !out_off || !out_cap || !out_len || !status))) {
        hgpu_set_error("bad argument");
        return HGPU_ERR_ARG;
    }
    if (n == 0) return HGPU_OK;
    if (hgpu_check(cudaSetDevice(ctx->device), "cudaSetDevice")) return HGPU_ERR_CUDA;

    // ---- host: descriptor framing of every block (tok3_decode_names :1679-1806)
    std::vector<Tok3Block> blocks(n);
    std::vector<Tok3Desc> descs;
    std::vector<Job> rjobs, ajobs;                 // rANS-Nx16 / adaptive arithmetic
    std::vector<uint32_t> rjob_block_first(n, 0), ajob_block_first(n, 0);
    uint64_t arena = 0, hist = 0, names = 0;
    const uint64_t in_end = hgpu_slots_end(in_off, in_len, n), out_end = hgpu_slots_end(out_off, out_cap, n);
    uint32_t max_stream = 0, max_ndesc = 16;
    for (uint32_t b = 0; b < n; b++) {
        Tok3Block &B = blocks[b];
        memset(&B, 0, sizeof(B));
        B.out_off = out_off[b]; B.out_cap = out_cap[b];
        B.host_status = HGPU_TOK3_ERR;
        const uint8_t *p = in + in_off[b];
        const uint32_t sz = in_len[b];
        if (sz < 9) continue;
        uint32_t ulen = p[0] | p[1] << 8 | p[2] << 16 | (uint32_t)p[3] << 24;
        if ((int32_t)ulen < 0 || ulen >= 0x7fffffffu - 1024) continue;
        int32_t nreads = (int32_t)(p[4] | p[5] << 8 | p[6] << 16 | (uint32_t)p[7] << 24);
        const int use_arith = p[8];
        if (nreads <= 0 || nreads > 10000000) continue;                       // create_context :172-187
        std::vector<Job> &jobs = use_arith ? ajobs : rjobs;
        const size_t job_mark = jobs.size(), desc_mark = descs.size();
        const uint64_t arena_mark = arena;
        descs.resize(desc_mark + 16, Tok3Desc{0, 0, 0});
        std::vector<uint8_t> present(TOK_MAX * 16, 0);                        // desc[i].buf != NULL
        uint32_t o = 9;
        int tnum = -1;
        bool ok = true, limit = false;
        while (ok && o < sz) {
            const uint8_t tt = p[o++];
            const bool dup = tt & 64;
            int j = 0;
            if (dup) {
                if (o + 2 > sz) { ok = false; break; }
                j = (p[o] << 4) + p[o + 1]; o += 2;
            }
            if (tt & 128) {
                if (++tnum >= TOK_MAX) { ok = false; break; }
                descs.resize(desc_mark + (size_t)(tnum + 1) * 16, Tok3Desc{0, 0, 0});
                for (int k = 0; k < 16; k++) { descs[desc_mark + (tnum << 4) + k] = Tok3Desc{0, 0, 0}; present[(tnum << 4) + k] = 0; }
            }
            if ((tt & 15) != 0 && (tt & 128)) {
                descs[desc_mark + (tnum << 4)] = Tok3Desc{0, (uint32_t)nreads, 0x100u | (tt & 15u)};
                present[tnum << 4] = 1;
            }
            if (tnum < 0) { ok = false; break; }
            const int i = (tnum << 4) | (tt & 15);
            if (dup) {
                if (j >= i || !present[j]) { ok = false; break; }
                descs[desc_mark + i] = descs[desc_mark + j];
                present[i] = 1;
                continue;
            }
            const uint8_t *s = p + o, *e = p + sz;
            uint32_t clen, usz;
            const int nb = hgpu_var_get_u32(s, e, &clen);
            hgpu_var_get_u32(s + nb + 1 <= e ? s + nb + 1 : e, e, &usz);
            if ((int32_t)usz < 0 || usz >= 0x7fffffffu) { ok = false; break; }
            // No encoder writes a token stream longer than 4 bytes per name (integers) or two per name
            // byte (strings + NUL); beyond that the reference would still malloc(usz) and decode, this
            // implementation refuses instead of sizing device arenas from a corrupt field.
            if ((uint64_t)usz > 4ull * (uint64_t)nreads + 2ull * ulen + 1024) { ok = false; limit = true; break; }
            if ((uint64_t)o + nb > sz) { ok = false; break; }                 // nothing left for the sub-decoder
            Job jb;
            jb.in_off = in_off[b] + o + nb;
            jb.in_len = sz - o - nb;                                          // the sub-decoder is handed the rest of the block (:1436)
            jb.out_off = arena;
            jb.out_len = usz;
            jobs.push_back(jb);
            descs[desc_mark + i] = Tok3Desc{arena, usz, 0};
            present[i] = 1;
            arena += ((uint64_t)usz + 15) & ~(uint64_t)15;
            if (usz > max_stream) max_stream = usz;
            if ((uint64_t)o + clen + nb > 0xffffffffull) { ok = false; break; }
            o += clen + nb;
        }
        if (!ok) {                                                            // drop what this block queued
            jobs.resize(job_mark); descs.resize(desc_mark); arena = arena_mark;
            if (limit) B.host_status = HGPU_TOK3_ERR_LIMIT;
            continue;
        }
        B.host_status = HGPU_OK;
        B.desc_base = (uint32_t)desc_mark;
        B.max_tok = (uint32_t)(tnum + 1 > 1 ? tnum + 1 : 1);
        if (B.max_tok * 16 > max_ndesc) max_ndesc = B.max_tok * 16;
        B.nreads = (uint32_t)nreads;
        B.ulen = ulen;
        B.job0 = (uint32_t)job_mark | (use_arith ? 0x80000000u : 0);          // rebased below
        B.njobs = (uint32_t)(jobs.size() - job_mark);
        B.hist_off = hist; hist += (uint64_t)(nreads + 1) * B.max_tok;
        B.name_off = names; names += (uint64_t)nreads + 1;
    }
    const uint32_t nr = (uint32_t)rjobs.size(), na = (uint32_t)ajobs.size(), nj = nr + na;
    for (uint32_t b = 0; b < n; b++) {
        Tok3Block &B = blocks[b];
        if (B.host_status) continue;
        B.job0 = (B.job0 & 0x80000000u) ? (B.job0 & 0x7fffffffu) + nr : B.job0;
    }
    if (descs.empty()) descs.push_back(Tok3Desc{0, 0, 0});

    // ---- device layout in the staging buffer
    StageLayout L;
    const auto s_in = L.seg(in_end + 8), s_arena = L.seg(arena + 16), s_out = L.seg(out_end), s_hist = L.seg(hist * 8),
               s_names = L.seg(names * 16), s_blocks = L.seg((size_t)n * sizeof(Tok3Block)), s_descs = L.seg(descs.size() * sizeof(Tok3Desc)),
               s_jio = L.seg((size_t)nj * 8), s_joo = L.seg((size_t)nj * 8), s_jil = L.seg((size_t)nj * 4), s_jol = L.seg((size_t)nj * 4),
               s_jgot = L.seg((size_t)nj * 4), s_jst = L.seg((size_t)nj * 4), s_olen = L.seg((size_t)n * 4), s_st = L.seg((size_t)n * 4),
               s_order = L.seg((size_t)n * 4);
    int rc = hgpu_stage_ensure(ctx, L);
    if (rc) return rc;
    // blocks with at most 16 token positions (every Illumina-style block) share a warp in pairs; the rest,
    // and the blocks the framing walk already rejected (their status still has to be written), take the
    // general kernel.  order[] = [paired blocks ..., general blocks ...]
    std::vector<uint32_t> order(n);
    uint32_t n16 = 0, max_ndesc_gen = 16;
    const bool h16_ok = arena < (1ull << 36) - 4096;                 // its shared-memory descriptors hold offsets in 16-byte units
    for (uint32_t b = 0; b < n; b++)
        if (h16_ok && blocks[b].host_status == HGPU_OK && blocks[b].max_tok <= TOK3_H16_MAX_TOK) order[n16++] = b;
    {
        uint32_t g = n16;
        for (uint32_t b = 0; b < n; b++)
            if (!(h16_ok && blocks[b].host_status == HGPU_OK && blocks[b].max_tok <= TOK3_H16_MAX_TOK)) {
                order[g++] = b;
                if (blocks[b].host_status == HGPU_OK && blocks[b].max_tok * 16 > max_ndesc_gen) max_ndesc_gen = blocks[b].max_tok * 16;
            }
    }
    (void)max_ndesc;
    cudaStream_t s = ctx->stream;
    std::vector<uint64_t> jio(nj), joo(nj);
    std::vector<uint32_t> jil(nj), jol(nj);
    for (uint32_t k = 0; k < nj; k++) {
        const Job &jb = k < nr ? rjobs[k] : ajobs[k - nr];
        jio[k] = jb.in_off; joo[k] = jb.out_off; jil[k] = jb.in_len; jol[k] = jb.out_len;
    }
    if (hgpu_h2d(L.at(s_in), in, in_end, s) || hgpu_h2d(L.at(s_blocks), blocks.data(), (size_t)n * sizeof(Tok3Block), s) ||
        hgpu_h2d(L.at(s_descs), descs.data(), descs.size() * sizeof(Tok3Desc), s) || hgpu_h2d(L.at(s_jio), jio.data(), (size_t)nj * 8, s) ||
        hgpu_h2d(L.at(s_joo), joo.data(), (size_t)nj * 8, s) || hgpu_h2d(L.at(s_jil), jil.data(), (size_t)nj * 4, s) ||
        hgpu_h2d(L.at(s_jol), jol.data(), (size_t)nj * 4, s)) return HGPU_ERR_CUDA;
    const uint64_t *d_jio = L.at<uint64_t>(s_jio), *d_joo = L.at<uint64_t>(s_joo);
    const uint32_t *d_jil = L.at<uint32_t>(s_jil), *d_jol = L.at<uint32_t>(s_jol);
    uint32_t *d_jgot = L.at<uint32_t>(s_jgot);
    int32_t *d_jst = L.at<int32_t>(s_jst);
    uint8_t *d_in = L.at(s_in), *d_arena = L.at(s_arena);
    uint2 *d_hist = L.at<uint2>(s_hist);
    uint4 *d_names = L.at<uint4>(s_names);
    struct Events {                                                  // released on every return path
        cudaEvent_t e[3] = {nullptr, nullptr, nullptr};
        ~Events() { for (cudaEvent_t x : e) if (x) cudaEventDestroy(x); }
    } evs;
    cudaEvent_t *tev = evs.e;
    for (int k = 0; k < 3; k++) if (hgpu_check(cudaEventCreate(&tev[k]), "event")) return HGPU_ERR_CUDA;
    cudaEventRecord(tev[0], s);
    if (nr) {
        rc = hgpu_launch_rans_nx16(ctx, d_in, d_jio, d_jil, nr, d_arena, d_joo, d_jol, d_jgot, d_jst, max_stream, s);
        if (rc) return rc;
    }
    if (na) {
        rc = hgpu_arith_decode_batch_dev(ctx, d_in, d_jio + nr, d_jil + nr, na, d_arena, d_joo + nr, d_jol + nr,
                                         d_jgot + nr, d_jst + nr, max_stream, s);
        if (rc) return rc;
    }
    cudaEventRecord(tev[1], s);
    if (hgpu_h2d(L.at(s_order), order.data(), (size_t)n * 4, s)) return HGPU_ERR_CUDA;
    const uint32_t *d_order = L.at<uint32_t>(s_order);
    rc = hgpu_launch_tok3_names_h16(ctx, L.at<Tok3Block>(s_blocks), d_order, n16, L.at<Tok3Desc>(s_descs), d_arena, d_jst, d_jgot, d_jol,
                                    d_hist, d_names, L.at(s_out), L.at<uint32_t>(s_olen), L.at<int32_t>(s_st), s);
    if (rc) return rc;
    rc = hgpu_launch_tok3_names(ctx, L.at<Tok3Block>(s_blocks), d_order + n16, n - n16, max_ndesc_gen, L.at<Tok3Desc>(s_descs), d_arena,
                                d_jst, d_jgot, d_jol, d_hist, d_names, L.at(s_out), L.at<uint32_t>(s_olen), L.at<int32_t>(s_st), s);
    if (rc) return rc;
    cudaEventRecord(tev[2], s);
    if (hgpu_d2h(out_len, L.at(s_olen), (size_t)n * 4, s) || hgpu_d2h(status, L.at(s_st), (size_t)n * 4, s) ||
        hgpu_d2h(out, L.at(s_out), out_end, s)) return HGPU_ERR_CUDA;
    if (hgpu_check(cudaStreamSynchronize(s), "sync")) return HGPU_ERR_CUDA;
    cudaEventElapsedTime(&g_tok3_ms[0], tev[0], tev[1]);
    cudaEventElapsedTime(&g_tok3_ms[1], tev[1], tev[2]);
    return HGPU_OK;
}

extern "C" int hgpu_tok3_decode_batch_host(hgpu_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
        const uint32_t *in_len, uint32_t n, uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
        uint32_t *out_len, int32_t *status)
{
    return hgpu_abi_call([&] { return hgpu_tok3_decode_batch_host_impl(ctx, in, in_off, in_len, n, out, out_off, out_cap, out_len, status); });
}

// device time of the last hgpu_tok3_decode_batch_host call: [0] token-stream entropy decode, [1] name rebuild
extern "C" void hgpu_tok3_last_ms(float *ms2) { ms2[0] = g_tok3_ms[0]; ms2[1] = g_tok3_ms[1]; }

// Drop-in for the reference symbol (tokenise_name3.h:59): one block, malloc'd result, NULL on failure.
extern "C" uint8_t *tok3_decode_names(uint8_t *in, uint32_t sz, uint32_t *out_len)
{
    if (!in || !out_len) return nullptr;
    uint32_t cap = hgpu_tok3_out_bound(in, sz);
    if (!cap) return nullptr;
    ShimLock lock;
    hgpu_ctx *g_tok3_ctx = hgpu_shim_ctx();
    if (!g_tok3_ctx) return nullptr;
    uint8_t *out = (uint8_t *)malloc(cap);
    if (!out) return nullptr;
    uint64_t ioff = 0, ooff = 0;
    uint32_t got = 0;
    int32_t st = 0;
    int rc = hgpu_tok3_decode_batch_host(g_tok3_ctx, in, &ioff, &sz, 1, out, &ooff, &cap, &got, &st);
    if (rc != HGPU_OK || st != HGPU_OK) { free(out); return nullptr; }
    *out_len = got;
    return out;
}
