// fqzcomp quality codec ("FQZ", CRAM 3.1 block method 7) — ENCODE side.
//
// Stands where fqz_compress stands (htscodecs/htscodecs/fqzcomp_qual.c:1615 -> compress_block_fqz2f
// :1004-1239) as called from cram_compress_by_method (cram/cram_io.c:1804-1825), for a batch of quality
// blocks.  The bar is the decoder's: the reference's fqz_decompress (and this library's) must return the
// input; the bytes are this encoder's own where the reference's parameter search is not reproduced:
//   * one parameter block, no selector (the reference may split READ1/READ2 or by average quality,
//     fqz_qual_stats :392-672); qualities are stored in their original orientation (CRAM >= 3.1);
//   * the strategy rows (strat_opts :195-202), the context bits rows 0 and 1 set aside for a selector
//     (:601-622, applied by the reference even where it then keeps no selector), the size / alphabet
//     adjustments (:805-833), the quality map for <= 8 symbols, fixed-length detection, the position and delta tables and the
//     duplicate-record flag (a record equal to the previous one costs one symbol) are the reference's.
// Work split: the host reads each block once (histogram, lengths, duplicates) and writes the parameter
// block (fqz_store_parameters :674-733, store_array :102-144); the device initialises the 65 536 models
// per stream with coalesced stores and runs one range ENCODER per thread (compress_new_read :930-1002,
// fqz_update_ctx :344-386, RC_Encode / RC_ShiftLow c_range_coder.h:77-146, SIMPLE_MODEL_encodeSymbol
// c_simple_model.h:112-133) — the same sequential machine as the decoder, so streams are the parallel axis.
#include "hgpu_internal.h"
#include <new>
#include <vector>
#include <string.h>
#include <math.h>

namespace {

constexpr uint32_t TOP = 1u << 24, THRES = 255u * TOP;
constexpr uint32_t MAX_FREQ = (1u << 16) - 17;
constexpr uint32_t STEP = 16;
constexpr uint32_t CTX_SIZE = 1u << 16;
constexpr int PFLAG_DO_DEDUP = 2, PFLAG_DO_LEN = 4, PFLAG_HAVE_QMAP = 16, PFLAG_HAVE_PTAB = 32, PFLAG_HAVE_DTAB = 64;

struct EncParam {                                  // what the symbol loop needs of fqz_param
    uint32_t context, qmask, qshift, qloc, sloc, fixed_len, do_dedup, nsym;   // nsym: model symbols (gp.max_sym + 1)
    uint32_t ptab[1024];                           // already shifted by ploc (:1051-1058)
    uint32_t dtab[256];                            // already shifted by dloc
    uint8_t  qmap[256];                            // quality value -> model symbol
};

struct EncStream {
    uint64_t in_off, out_off, model_off, rec_off;  // rec_off: first record length of this stream in rec_len[]
    uint32_t in_len, out_cap, nrec, hdr_len;       // hdr_len: size varint + parameter block, already in `out`
    int32_t  host_status;
};

struct RCE { uint8_t *p, *begin, *end; uint32_t low, range, ffnum, carry, cache; int err; };

__device__ __forceinline__ void rc_shift_low(RCE &rc)                    // RC_ShiftLowCheck :77-101
{
    if (rc.low < THRES || rc.carry) {
        if (rc.ffnum >= (uint32_t)(rc.end - rc.p)) { rc.err = -1; return; }
        *rc.p++ = (uint8_t)(rc.cache + rc.carry);
        while (rc.ffnum) { *rc.p++ = (uint8_t)(rc.carry - 1); rc.ffnum--; }
        rc.cache = rc.low >> 24;
        rc.carry = 0;
    } else {
        rc.ffnum++;
    }
    rc.low <<= 8;
}

// compact model words as in fqzcomp.cu: [0] TotFreq, [1] sentinel, [2..2+nsym) Freq | Symbol << 16, zero terminator, terminal
__device__ void model_init(uint32_t *m, uint32_t nsym)
{
    m[0] = nsym; m[1] = MAX_FREQ;
    for (uint32_t i = 0; i < nsym; i++) m[2 + i] = 1u | i << 16;
    m[2 + nsym] = 0; m[3 + nsym] = MAX_FREQ;
}

__device__ void model_encode(uint32_t *m, RCE &rc, uint32_t sym)         // SIMPLE_MODEL_encodeSymbol :112-133
{
    uint32_t *s = m + 2;
    uint32_t acc = 0;
    while ((*s >> 16) != sym) { acc += *s & 0xffffu; s++; }
    const uint32_t f = *s & 0xffffu, tot = m[0];
    const uint32_t tmp = rc.low;
    rc.range /= tot;
    rc.low += acc * rc.range;
    rc.range *= f;
    rc.carry += rc.low < tmp;
    while (rc.range < TOP) { rc.range <<= 8; rc_shift_low(rc); }
    *s += STEP;
    m[0] = tot + STEP;
    if (m[0] > MAX_FREQ) {
        uint32_t t = 0;
        for (uint32_t *q = m + 2; *q & 0xffffu; q++) {
            uint32_t g = *q & 0xffffu;
            g -= g >> 1;
            *q = (*q & 0xffff0000u) | g;
            t += g;
        }
        m[0] = t;
    }
    const uint32_t cur = *s, prev = s[-1];
    if ((cur & 0xffffu) > (prev & 0xffffu)) { *s = prev; s[-1] = cur; }
}

__global__ void fqz_enc_init_models_kernel(const EncStream *streams, const EncParam *params, uint32_t *models)
{
    const EncStream &S = streams[blockIdx.y];
    if (S.host_status) return;
    const uint32_t nsym = params[blockIdx.y].nsym, stride = nsym + 4;
    const uint64_t total = (uint64_t)CTX_SIZE * stride;
    uint32_t *m = models + S.model_off;
    for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < total; w += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t slot = (uint32_t)(w % stride);
        uint32_t v;
        if (slot == 0) v = nsym;
        else if (slot == 1 || slot == stride - 1) v = MAX_FREQ;
        else if (slot == stride - 2) v = 0;
        else v = 1u | (slot - 2) << 16;
        m[w] = v;
    }
}

// the symbol loop of compress_block_fqz2f (:1100-1190) with compress_new_read (:930-1002)
__global__ void fqz_encode_kernel(const EncStream *streams, const EncParam *params, uint32_t first, uint32_t n, const uint8_t *in,
                                  const uint32_t *rec_len, uint32_t *models, uint8_t *out, uint32_t *out_len, int32_t *status)
{
    const uint32_t t = first + blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const EncStream &S = streams[t];
    if (S.host_status) { status[t] = S.host_status; out_len[t] = 0; return; }
    const EncParam *pm = params + t;
    const uint32_t stride = pm->nsym + 4;
    uint32_t *qual = models + S.model_off;
    uint32_t *small = qual + (uint64_t)CTX_SIZE * stride;          // len[4] (256 symbols each), dup (2)
    uint32_t *m_len = small, *m_dup = small + 4 * 260;
    for (int k = 0; k < 4; k++) model_init(m_len + k * 260, 256);
    model_init(m_dup, 2);
    const uint8_t *src = in + S.in_off;
    const uint32_t *L = rec_len + S.rec_off;
    uint8_t *o = out + S.out_off;
    RCE rc;
    rc.p = rc.begin = o + S.hdr_len; rc.end = o + S.out_cap;
    rc.range = 0xffffffffu; rc.low = 0; rc.ffnum = 0; rc.carry = 0; rc.cache = 0; rc.err = 0;

    uint32_t qctx = 0, p = 0, delta = 0, prevq = 0, first_len = 1, last_len = 0, last = 0, rec = 0;
    bool fail = false;
    for (uint32_t i = 0; i < S.in_len; i++) {
        if (p == 0) {
            if (rec >= S.nrec || L[rec] == 0) { fail = true; break; }
            const uint32_t len = L[rec];
            if (!pm->fixed_len || first_len) {
                model_encode(m_len, rc, len & 0xff);
                model_encode(m_len + 260, rc, (len >> 8) & 0xff);
                model_encode(m_len + 520, rc, (len >> 16) & 0xff);
                model_encode(m_len + 780, rc, (len >> 24) & 0xff);
                first_len = 0;
            }
            rec++;
            p = len; delta = 0; qctx = 0; prevq = 0;
            last = pm->context;
            if (pm->do_dedup) {
                bool same = i && len == last_len && (uint64_t)i + len <= S.in_len;
                if (same) for (uint32_t k = 0; k < len; k++) if (src[i - last_len + k] != src[i + k]) { same = false; break; }
                if (same) {
                    model_encode(m_dup, rc, 1);
                    i += len - 1;                                   // the loop's i++ steps over the last byte
                    p = 0;
                    continue;
                }
                model_encode(m_dup, rc, 0);
                last_len = len;
            }
        }
        const uint32_t qm = pm->qmap[src[i]];
        model_encode(qual + (uint64_t)last * stride, rc, qm);
        // fqz_update_ctx (:344-386); qtab is the identity in this encoder
        qctx = (qctx << pm->qshift) + qm;
        uint32_t c = (qctx & pm->qmask) << pm->qloc;
        c += pm->ptab[p < 1023 ? p : 1023];
        c += pm->dtab[delta < 255 ? delta : 255];
        delta += prevq != qm;
        prevq = qm;
        p--;
        last = c & (CTX_SIZE - 1);
        if (rc.err) { fail = true; break; }
    }
    if (!fail) { for (int k = 0; k < 5; k++) rc_shift_low(rc); if (rc.err) fail = true; }   // RC_FinishEncode
    status[t] = fail ? HGPU_FQZ_ERR : HGPU_OK;
    out_len[t] = fail ? 0 : (uint32_t)(rc.p - o);
}

int put_varint(uint8_t *p, uint32_t v)                               // var_put_u32, varint.h:206
{
    int n = 1;
    while (n < 5 && (v >> (7 * n))) n++;
    for (int k = n - 1; k >= 0; k--) *p++ = (uint8_t)(((v >> (7 * k)) & 0x7f) | (k ? 0x80 : 0));
    return n;
}

// store_array (:102-144): run lengths of each value, then a run-length code over those
int store_array(uint8_t *out, const uint32_t *array, int size)
{
    uint8_t tmp[2048];
    int i, j, k;
    for (i = j = k = 0; i < size; j++) {
        int run_len = i;
        while (i < size && array[i] == (uint32_t)j) i++;
        run_len = i - run_len;
        int r;
        do { r = run_len < 255 ? run_len : 255; tmp[k++] = (uint8_t)r; run_len -= r; } while (r == 255);
    }
    int last = -1;
    for (i = j = 0; j < k; i++) {
        out[i] = tmp[j++];
        if (out[i] == last) {
            int n = j;
            while (j < k && tmp[j] == last) j++;
            out[++i] = (uint8_t)(j - n);
        } else {
            last = out[i];
        }
    }
    return i;
}

const int strat_opts[4][12] = {                                      // :195-201 (qb qs pb ps db ds ql sl pl dl r2 qa)
    {10, 5, 4, -1, 2, 1, 0, 14, 10, 14, 0, -1},
    {8, 5, 7, 0, 0, 0, 0, 14, 8, 14, 1, -1},
    {12, 6, 2, 0, 2, 3, 0, 9, 12, 14, 0, 0},
    {12, 6, 0, 0, 0, 0, 0, 12, 0, 0, 0, 0},
};

}  // namespace

// (num_records * len_sz + in_size) * 1.1 + 10000, the reference's own allocation (:1040-1047), with len_sz 4.25
extern "C" uint32_t hgpu_fqz_compress_bound(uint32_t in_len, uint32_t nrec)
{
    const double b = ((double)nrec * 4.25 + in_len) * 1.1 + 10000 + 2048;
    return b > 4294967295.0 ? 0xffffffffu : (uint32_t)b;
}

static int hgpu_fqz_encode_batch_host_impl(hgpu_ctx *ctx, const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len,
        const uint32_t *rec_len, const uint64_t *rec_off, const uint32_t *nrec, uint32_t n, int strat,
        uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap, uint32_t *out_len, int32_t *status)
{
    if (!ctx || (n && (!in || !in_off || !in_len || !rec_len || !rec_off || !nrec || !out || !out_off || !out_cap || !out_len || !status))) {
        hgpu_set_error("bad argument");
        return HGPU_ERR_ARG;
    }
    if (n == 0) return HGPU_OK;
    if (strat < 0) strat = 0;
    if (strat > 3) strat = 3;
    if (hgpu_check(cudaSetDevice(ctx->device), "cudaSetDevice")) return HGPU_ERR_CUDA;

    // ---- host: parameters of every stream (fqz_pick_parameters :736-924 without the selector search)
    std::vector<EncStream> streams(n);
    std::vector<EncParam> params(n);
    const uint64_t MODEL_BUDGET = 6ull << 30;
    std::vector<uint32_t> wave_first(1, 0u);                              // first stream of every wave
    uint64_t model_words = 0 /* largest wave */, wave_words = 0;
    const uint64_t in_end = hgpu_slots_end(in_off, in_len, n), out_end = hgpu_slots_end(out_off, out_cap, n),
                   rec_end = hgpu_slots_end(rec_off, nrec, n);
    for (uint32_t s = 0; s < n; s++) {
        EncStream &S = streams[s];
        EncParam &P = params[s];
        memset(&S, 0, sizeof(S)); memset(&P, 0, sizeof(P));
        S.in_off = in_off[s]; S.in_len = in_len[s]; S.out_off = out_off[s]; S.out_cap = out_cap[s];
        S.rec_off = rec_off[s]; S.nrec = nrec[s];
        S.host_status = HGPU_FQZ_ERR;
        const uint8_t *q = in + in_off[s];
        const uint32_t *L = rec_len + rec_off[s];
        const uint32_t size = in_len[s];
        uint64_t tl = 0;
        bool ok = nrec[s] > 0 && size > 0;
        for (uint32_t r = 0; ok && r < nrec[s]; r++) { if (L[r] == 0) ok = false; tl += L[r]; }
        if (!ok || tl != size || out_cap[s] < 4096) continue;            // lengths must tile the block
        uint32_t qhist[256] = {0};
        for (uint32_t i = 0; i < size; i++) qhist[q[i]]++;
        uint32_t nsym = 0, max_sym = 0;
        for (int i = 0; i < 256; i++) if (qhist[i]) { max_sym = (uint32_t)i; nsym++; }
        // duplicates of the previous record (:436-446, :469)
        uint64_t dups = 0, pos = 0;
        for (uint32_t r = 0; r < nrec[s]; r++) {
            if (r && L[r] == L[r - 1] && memcmp(q + pos - L[r - 1], q + pos, L[r]) == 0) dups++;
            pos += L[r];
        }
        const bool do_dedup = ((uint64_t)nrec[s] + 1) / (dups + 1) < 500;
        bool fixed_len = true;
        for (uint32_t r = 1; r < nrec[s]; r++) if (L[r] != L[0]) { fixed_len = false; break; }
        int qbits = strat_opts[strat][0], qshift = strat_opts[strat][1], pbits = strat_opts[strat][2], pshift = strat_opts[strat][3],
            dbits = strat_opts[strat][4], dshift = strat_opts[strat][5];
        int qloc = strat_opts[strat][6], sloc = strat_opts[strat][7], ploc = strat_opts[strat][8], dloc = strat_opts[strat][9];
        if (strat_opts[strat][11] == -1) {                                 // qa -1 frees context bits for a selector (:601-622),
            if (pbits > 0 && dbits > 0) { sloc = dloc - 1; pbits--; dbits--; dloc++; }   // whether or not one is kept
            else if (dbits >= 2) { sloc = dloc; dbits -= 2; dloc += 2; }
            else if (qbits >= 2) { qbits -= 2; ploc -= 2; sloc = 16 - 2 - strat_opts[strat][10]; if (qbits == 6 && qshift == 5) qbits--; }
        }
        const bool store_qmap = nsym <= 8 && nsym * 2 < max_sym;
        if (pshift < 0) { double v = log((double)L[0] / (1 << pbits)) / log(2.0) + .5; pshift = v > 0 ? (int)v : 0; }
        if (nsym <= 4) { qshift = 2; if (size < 5000000) { pbits = 2; pshift = 5; } }
        else if (nsym <= 8) { if (qbits > 9) qbits = 9; qshift = 3; if (size < 5000000) qbits = 6; }
        if (size < 300000) { qbits = qshift; dbits = 2; }
        int dsqr[64] = {0, 1, 1, 1, 2, 2, 2, 2, 2, 3, 3, 3, 3, 3, 3, 3, 4, 4, 4, 4, 4, 4, 4, 4, 4, 5, 5, 5, 5, 5, 5, 5,
                        5, 5, 5, 5, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7};
        for (int i = 0; i < 64; i++) if (dsqr[i] > (1 << dbits) - 1) dsqr[i] = (1 << dbits) - 1;
        uint32_t sym_max;                                                 // pm->max_sym as stored
        if (store_qmap) {
            uint32_t j = 0;
            for (int i = 0; i < 256; i++) P.qmap[i] = qhist[i] ? (uint8_t)j++ : 0;
            sym_max = nsym;
        } else {
            for (int i = 0; i < 256; i++) P.qmap[i] = (uint8_t)i;
            sym_max = max_sym;
        }
        uint32_t ptab[1024], dtab[256];
        for (int i = 0; i < 1024; i++) { int v = i >> pshift; ptab[i] = pbits ? (uint32_t)(v < (1 << pbits) - 1 ? v : (1 << pbits) - 1) : 0; }
        for (int i = 0; i < 256; i++) { int v = i >> dshift; dtab[i] = dbits ? (uint32_t)dsqr[v < 63 ? v : 63] : 0; }
        const uint32_t pflags = (dbits ? PFLAG_HAVE_DTAB : 0) | (pbits ? PFLAG_HAVE_PTAB : 0) | (fixed_len ? PFLAG_DO_LEN : 0) |
                                (do_dedup ? PFLAG_DO_DEDUP : 0) | (store_qmap ? PFLAG_HAVE_QMAP : 0);
        // header: size, global block (:710-733), parameter block (:674-707)
        uint8_t *o = out + out_off[s];
        uint32_t k = (uint32_t)put_varint(o, size);
        o[k++] = 5;                                                       // FQZ_VERS
        o[k++] = 0;                                                       // gflags: one block, no selector table, original orientation
        o[k++] = 0; o[k++] = 0;                                           // starting context
        o[k++] = (uint8_t)pflags;
        o[k++] = (uint8_t)sym_max;
        o[k++] = (uint8_t)(qbits << 4 | qshift);
        o[k++] = (uint8_t)(qloc << 4 | sloc);
        o[k++] = (uint8_t)(ploc << 4 | dloc);
        if (store_qmap) for (int i = 0; i < 256; i++) if (qhist[i]) o[k++] = (uint8_t)i;
        if (pbits) k += (uint32_t)store_array(o + k, ptab, 1024);
        if (dbits) k += (uint32_t)store_array(o + k, dtab, 256);
        S.hdr_len = k;
        P.context = 0; P.qmask = (1u << qbits) - 1; P.qshift = (uint32_t)qshift; P.qloc = (uint32_t)qloc; P.sloc = (uint32_t)sloc;
        P.fixed_len = fixed_len; P.do_dedup = do_dedup; P.nsym = sym_max + 1;
        for (int i = 0; i < 1024; i++) P.ptab[i] = ptab[i] << ploc;
        for (int i = 0; i < 256; i++) P.dtab[i] = dtab[i] << dloc;
        // model arenas per WAVE, as the decoder hands them out (fqzcomp.cu): a wave's arenas fit MODEL_BUDGET (one
        // stream alone may exceed it) and the next wave reuses the memory
        const uint64_t words = (uint64_t)CTX_SIZE * (P.nsym + 4) + 4 * 260 + 6 + 16;
        if (wave_words && (wave_words + words) * 4 > MODEL_BUDGET) { wave_first.push_back(s); wave_words = 0; }
        S.model_off = wave_words;
        wave_words += words;
        if (wave_words > model_words) model_words = wave_words;
        S.host_status = HGPU_OK;
    }
    wave_first.push_back(n);

    StageLayout L;
    const auto s_in = L.seg(in_end + 8), s_out = L.seg(out_end + 8), s_rec = L.seg(rec_end * 4 + 8), s_streams = L.seg((size_t)n * sizeof(EncStream)),
               s_params = L.seg((size_t)n * sizeof(EncParam)), s_olen = L.seg((size_t)n * 4), s_st = L.seg((size_t)n * 4),
               s_models = L.seg(model_words * 4 + 16);
    int rc = hgpu_stage_ensure(ctx, L);
    if (rc) return rc;
    cudaStream_t st = ctx->stream;
    const EncStream *d_streams = L.at<EncStream>(s_streams);
    const EncParam *d_params = L.at<EncParam>(s_params);
    if (hgpu_h2d(L.at(s_in), in, in_end, st) || hgpu_h2d(L.at(s_out), out, out_end, st) /* the headers */ ||
        hgpu_h2d(L.at(s_rec), rec_len, rec_end * 4, st) || hgpu_h2d(L.at(s_streams), streams.data(), (size_t)n * sizeof(EncStream), st) ||
        hgpu_h2d(L.at(s_params), params.data(), (size_t)n * sizeof(EncParam), st)) return HGPU_ERR_CUDA;
    for (size_t w = 0; w + 1 < wave_first.size(); w++) {                 // waves run back to back on one stream: the arena is reused
        const uint32_t w0 = wave_first[w], wend = wave_first[w + 1];
        if (w0 == wend) continue;
        for (uint32_t first = w0; first < wend; first += 65535u) {       // gridDim.y limit
            const uint32_t cnt = wend - first < 65535u ? wend - first : 65535u;
            fqz_enc_init_models_kernel<<<dim3(64, cnt), 256, 0, st>>>(d_streams + first, d_params + first, L.at<uint32_t>(s_models));
            if (hgpu_check(cudaGetLastError(), "fqz_enc_init_models_kernel")) return HGPU_ERR_CUDA;
            hgpu_count_launch();
        }
        fqz_encode_kernel<<<(wend - w0 + 31) / 32, 32, 0, st>>>(d_streams, d_params, w0, wend, L.at(s_in), L.at<uint32_t>(s_rec),
                                                                L.at<uint32_t>(s_models), L.at(s_out), L.at<uint32_t>(s_olen), L.at<int32_t>(s_st));
        if (hgpu_check(cudaGetLastError(), "fqz_encode_kernel")) return HGPU_ERR_CUDA;
        hgpu_count_launch();
    }
    if (hgpu_d2h(out_len, L.at(s_olen), (size_t)n * 4, st) || hgpu_d2h(status, L.at(s_st), (size_t)n * 4, st) ||
        hgpu_d2h(out, L.at(s_out), out_end, st)) return HGPU_ERR_CUDA;
    if (hgpu_check(cudaStreamSynchronize(st), "sync")) return HGPU_ERR_CUDA;
    return HGPU_OK;
}

extern "C" int hgpu_fqz_encode_batch_host(hgpu_ctx *ctx, const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len,
        const uint32_t *rec_len, const uint64_t *rec_off, const uint32_t *nrec, uint32_t n, int strat,
        uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap, uint32_t *out_len, int32_t *status)
{
    return hgpu_abi_call([&] {
        return hgpu_fqz_encode_batch_host_impl(ctx, in, in_off, in_len, rec_len, rec_off, nrec, n, strat, out, out_off, out_cap, out_len, status);
    });
}
