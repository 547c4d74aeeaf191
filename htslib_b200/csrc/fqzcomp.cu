// fqzcomp quality codec ("FQZ", CRAM 3.1 block method 7) — decode side.
//
// Replaces fqz_decompress -> uncompress_block_fqz2f (htscodecs/htscodecs/fqzcomp_qual.c:1626, :1456-1613)
// as called from cram_uncompress_block (cram/cram_io.c:1684-1695), for a batch of quality blocks.
//   host   : reads the parameter blocks of every stream (fqz_read_parameters :1325-1379,
//            fqz_read_parameters1 :1241-1322, read_array :146-190) — a few hundred bytes of tables;
//   device : fqz_init_models_kernel fills the 65 536 adaptive models of every stream with coalesced
//            stores (fqz_create_models :320-338 does this serially per block; it is most of the
//            reference's per-block cost on short blocks), then fqz_decode_kernel runs one range coder
//            per THREAD.  The coder is strictly sequential (one 32-bit range/code pair, the model it
//            reads is updated after every symbol), so streams are the only parallel axis — the same
//            shape as arith_dynamic.cu.
// Models are stored compactly: the reference's SIMPLE_MODEL(256) always holds 256 symbol slots, of
// which only max_sym+1 are live (the rest have frequency 0 and sit behind the live ones for ever);
// here a model is tot, sentinel, max_sym+1 live slots, the zero terminator and the terminal, which
// is the same machine (c_simple_model.h:85-169) in (max_sym+5)*4 bytes instead of 1040.
#include "hgpu_internal.h"
#include <new>
#include <vector>
#include <string.h>
#include <stdlib.h>
#include <mutex>

namespace {

constexpr uint32_t TOP = 1u << 24;
constexpr uint32_t MAX_FREQ = (1u << 16) - 17;
constexpr uint32_t STEP = 16;
constexpr uint32_t CTX_SIZE = 1u << 16;            // fqzcomp_qual.c:73-74
constexpr int GFLAG_MULTI_PARAM = 1, GFLAG_HAVE_STAB = 2, GFLAG_DO_REV = 4;
constexpr int PFLAG_DO_DEDUP = 2, PFLAG_DO_LEN = 4, PFLAG_DO_SEL = 8, PFLAG_HAVE_QMAP = 16,
              PFLAG_HAVE_PTAB = 32, PFLAG_HAVE_DTAB = 64, PFLAG_HAVE_QTAB = 128;

struct FqzParam {                                  // fqz_param, fqzcomp_qual.h:90-122 (decoder fields)
    uint32_t context, qmask, qshift, qloc, sloc;
    uint32_t do_sel, fixed_len, do_dedup;
    uint16_t qtab[256];
    uint32_t ptab[1024];                           // already shifted by ploc (:1489-1496)
    uint32_t dtab[256];                            // already shifted by dloc
    uint8_t  qmap[256];
};

struct FqzStream {
    uint64_t in_off;                               // the whole stream (for bounds) ...
    uint32_t in_len, payload;                      // ... and where the range coder's bytes start
    uint64_t out_off, model_off, flag_off;         // model_off in u32 words; flag_off: per-output-byte record marks (DO_REV)
    uint32_t out_cap, ulen;
    uint32_t nparam, gflags, max_sel, nsym;        // nsym = gp.max_sym + 1
    uint32_t param0;                               // first FqzParam of this stream
    int32_t  host_status;
    uint16_t stab[256];
};

struct RC { const uint8_t *p, *end; uint32_t range, code; int err; };

__device__ __forceinline__ void rc_start(RC &rc, const uint8_t *p, const uint8_t *end)     // c_range_coder.h:62-76
{
    rc.range = 0xffffffffu; rc.code = 0; rc.err = 0; rc.p = p; rc.end = end;
    if (p + 5 > end) { rc.p = end; return; }
    for (int i = 0; i < 5; i++) rc.code = (rc.code << 8) | *rc.p++;
}

// model words: [0] TotFreq, [1] sentinel, [2 .. 2+nsym) symbols, [2+nsym] zero terminator, [3+nsym] terminal;
// a slot is Freq | Symbol << 16
__device__ __forceinline__ uint32_t model_words(uint32_t nsym) { return nsym + 4; }

__device__ void model_init(uint32_t *m, uint32_t nsym)
{
    m[0] = nsym;
    m[1] = MAX_FREQ;
    for (uint32_t i = 0; i < nsym; i++) m[2 + i] = 1u | i << 16;
    m[2 + nsym] = 0;
    m[3 + nsym] = MAX_FREQ;
}

// SIMPLE_MODEL_decodeSymbol, c_simple_model.h:135-169 (RC_GetFreq / RC_Decode c_range_coder.h:147-164)
__device__ uint32_t model_decode(uint32_t *m, uint32_t nsym, RC &rc)
{
    const uint32_t tot = m[0];
    const uint32_t freq = (tot && rc.range >= tot) ? rc.code / (rc.range /= tot) : 0;
    if (freq > MAX_FREQ) return 0;
    uint32_t *s = m + 2;
    uint32_t acc = 0, f;
    for (;;) { f = *s & 0xffffu; acc += f; if (acc > freq) break; s++; }
    if ((uint32_t)(s - (m + 2)) > nsym) return 0;
    acc -= f;
    rc.code -= acc * rc.range;
    rc.range *= f;
    while (rc.range < TOP) {
        if (rc.p >= rc.end) { rc.err = -1; break; }
        rc.code = (rc.code << 8) + *rc.p++;
        rc.range <<= 8;
    }
    *s += STEP;                                                   // Freq is the low half; it cannot carry (<= 65535)
    m[0] = tot + STEP;
    if (m[0] > MAX_FREQ) {                                        // normalize: halve until the zero terminator
        uint32_t t = 0;
        for (uint32_t *q = m + 2; *q & 0xffffu; q++) {
            uint32_t g = *q & 0xffffu;
            g -= g >> 1;
            *q = (*q & 0xffff0000u) | g;
            t += g;
        }
        m[0] = t;
    }
    const uint32_t cur = *s, prev = s[-1];                        // s[-1] of the first slot is the sentinel
    if ((cur & 0xffffu) > (prev & 0xffffu)) { *s = prev; s[-1] = cur; }
    return cur >> 16;
}

// every quality model of every stream: word w of a stream's block is slot (w mod stride) of model (w / stride)
__global__ void fqz_init_models_kernel(const FqzStream *streams, uint32_t *models)
{
    const FqzStream &S = streams[blockIdx.y];
    if (S.host_status) return;
    const uint32_t stride = S.nsym + 4;
    const uint64_t total = (uint64_t)CTX_SIZE * stride;
    uint32_t *m = models + S.model_off;
    for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < total; w += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t slot = (uint32_t)(w % stride);
        uint32_t v;
        if (slot == 0) v = S.nsym;
        else if (slot == 1 || slot == stride - 1) v = MAX_FREQ;
        else if (slot == stride - 2) v = 0;
        else v = 1u | (slot - 2) << 16;
        m[w] = v;
    }
}

// uncompress_block_fqz2f (:1456-1613) with decompress_new_read (:1381-1453) and fqz_update_ctx (:344-386)
__global__ void fqz_decode_kernel(const FqzStream *streams, uint32_t n, const FqzParam *params, const uint8_t *in,
                                  uint32_t *models, uint8_t *flags, uint8_t *out, uint32_t *got_len, int32_t *status)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const FqzStream &S = streams[t];
    if (S.host_status) { status[t] = S.host_status; got_len[t] = 0; return; }
    const uint32_t len = S.ulen;
    int rc_status = HGPU_FQZ_ERR;
    uint32_t produced = 0;
    do {
        if (len > S.out_cap) break;
        const uint32_t stride = S.nsym + 4;
        uint32_t *qual = models + S.model_off;
        uint32_t *small = qual + (uint64_t)CTX_SIZE * stride;      // len[4] (256), revcomp (2), dup (2), sel (max_sel+1)
        uint32_t *m_len = small, *m_rev = small + 4 * 260, *m_dup = m_rev + 6, *m_sel = m_dup + 6;
        for (int k = 0; k < 4; k++) model_init(m_len + k * 260, 256);
        model_init(m_rev, 2);
        model_init(m_dup, 2);
        if (S.max_sel > 0) model_init(m_sel, S.max_sel + 1);
        const FqzParam *P = params + S.param0;
        const FqzParam *pm0 = P;                                    // the main loop keeps using block 0 (pm is passed by value, :1541)
        const uint8_t *src = in + S.in_off;
        uint8_t *o = out + S.out_off;
        uint8_t *fl = flags + S.flag_off;
        const bool do_rev = S.gflags & GFLAG_DO_REV;
        RC rc;
        rc_start(rc, src + S.payload, src + S.in_len);

        uint32_t qctx = 0, p = 0, delta = 0, prevq = 0, sel = 0, first_len = 1, last_len = 0, last = 0;
        bool fail = false;
        uint32_t i = 0;
        while (i < len) {
            if (p == 0) {
                // ---- decompress_new_read
                sel = pm0->do_sel ? model_decode(m_sel, S.max_sel + 1, rc) : 0;
                const uint32_t x = (S.gflags & GFLAG_HAVE_STAB) ? S.stab[sel < 255 ? sel : 255] : sel;
                if (x >= S.nparam) { fail = true; break; }
                const FqzParam *pm = P + x;
                uint32_t rl = last_len;
                if (!pm->fixed_len || first_len) {
                    rl = model_decode(m_len, 256, rc);
                    rl |= model_decode(m_len + 260, 256, rc) << 8;
                    rl |= model_decode(m_len + 520, 256, rc) << 16;
                    rl |= model_decode(m_len + 780, 256, rc) << 24;
                    first_len = 0;
                    last_len = rl;
                }
                if (rl > len - i || rl == 0) { fail = true; break; }
                uint32_t rev = 0;
                if (do_rev) rev = model_decode(m_rev, 2, rc);
                if (do_rev) fl[i] = (uint8_t)(1u | rev << 1);       // record start (+ reversed) mark for the final pass
                if (pm->do_dedup && model_decode(m_dup, 2, rc)) {   // duplicate of the bytes just before it (:1420-1432)
                    if (rl > i) { fail = true; break; }
                    for (uint32_t k = 0; k < rl; k++) o[i + k] = o[i - rl + k];
                    i += rl;
                    p = 0;
                    continue;
                }
                p = rl; delta = 0; prevq = 0; qctx = 0;
                last = pm->context;
            }
            do {
                const uint32_t Q = model_decode(qual + (uint64_t)last * stride, S.nsym, rc);
                // ---- fqz_update_ctx
                qctx = (qctx << pm0->qshift) + pm0->qtab[Q & 255];
                uint32_t c = (qctx & pm0->qmask) << pm0->qloc;
                c += pm0->ptab[p < 1023 ? p : 1023];
                c += pm0->dtab[delta < 255 ? delta : 255];
                c += sel << pm0->sloc;
                delta += prevq != Q;
                prevq = Q;
                p--;
                last = c & (CTX_SIZE - 1);
                o[i++] = pm0->qmap[Q & 255];
            } while (p != 0 && i < len);
        }
        if (fail) break;
        if (do_rev) {                                               // :1566-1580, records in order, each reversed in place
            uint32_t a = 0;
            while (a < len) {
                uint32_t b = a + 1;
                while (b < len && !(fl[b] & 1)) b++;
                if (fl[a] & 2) for (uint32_t I = a, J = b - 1; I < J; I++, J--) { uint8_t c = o[I]; o[I] = o[J]; o[J] = c; }
                a = b;
            }
        }
        if (rc.err < 0) break;                                      // RC_FinishDecode
        rc_status = HGPU_OK;
        produced = len;
    } while (0);
    status[t] = rc_status;
    got_len[t] = produced;
}

// read_array (:146-190): two levels of run-length coding -> array[0..size) of run indices.  Bytes used or -1.
int h_read_array(const uint8_t *in, size_t in_size, uint32_t *array, int size)
{
    uint8_t R[1024];
    int i, j, z, last = -1;
    if (size > 1024) size = 1024;
    for (i = j = z = 0; z < size && (size_t)i < in_size; i++) {
        const int run = in[i];
        R[j++] = (uint8_t)run;
        z += run;
        if (run == last) {
            if ((size_t)i + 1 >= in_size) return -1;
            int copy = in[++i];
            z += run * copy;
            while (copy-- && z <= size && j < 1024) R[j++] = (uint8_t)run;
        }
        if (j >= 1024) return -1;
        last = run;
    }
    const int nb = i, r_max = j;
    for (i = j = z = 0; j < size; i++) {
        int run_len = 0, part;
        if (z >= r_max) return -1;
        do { part = R[z++]; run_len += part; } while (part == 255 && z < r_max);
        if (part == 255) return -1;
        while (run_len && j < size) { run_len--; array[j++] = (uint32_t)i; }
    }
    return nb;
}

// fqz_read_parameters1 (:1241-1322).  Bytes used or -1.
int h_read_param(FqzParam &pm, uint32_t &max_sym, const uint8_t *in, size_t in_size)
{
    if (in_size < 7) return -1;
    size_t k = 0;
    uint32_t tmp[1024];
    pm.context = in[0] | in[1] << 8; k = 2;
    const uint32_t pflags = in[k++];
    pm.do_sel = pflags & PFLAG_DO_SEL; pm.fixed_len = pflags & PFLAG_DO_LEN; pm.do_dedup = pflags & PFLAG_DO_DEDUP;
    max_sym = in[k++];
    const uint32_t qbits = in[k] >> 4;
    pm.qmask = (1u << qbits) - 1; pm.qshift = in[k++] & 15;
    pm.qloc = in[k] >> 4; pm.sloc = in[k++] & 15;
    const uint32_t ploc = in[k] >> 4, dloc = in[k++] & 15;
    if (pflags & PFLAG_HAVE_QMAP) {
        memset(pm.qmap, 0xff, 256);                                  // unset entries are INT_MAX there: 0xff once stored as a byte
        if (k + max_sym > in_size) return -1;
        for (uint32_t i = 0; i < max_sym; i++) pm.qmap[i] = in[k++];
    } else {
        for (int i = 0; i < 256; i++) pm.qmap[i] = (uint8_t)i;
    }
    for (int i = 0; i < 256; i++) pm.qtab[i] = (uint16_t)i;
    if (qbits && (pflags & PFLAG_HAVE_QTAB)) {
        int used = h_read_array(in + k, in_size - k, tmp, 256);
        if (used < 0) return -1;
        k += used;
        for (int i = 0; i < 256; i++) pm.qtab[i] = (uint16_t)tmp[i];
    }
    memset(pm.ptab, 0, sizeof(pm.ptab));
    if (pflags & PFLAG_HAVE_PTAB) {
        int used = h_read_array(in + k, in_size - k, pm.ptab, 1024);
        if (used < 0) return -1;
        k += used;
    }
    memset(pm.dtab, 0, sizeof(pm.dtab));
    if (pflags & PFLAG_HAVE_DTAB) {
        int used = h_read_array(in + k, in_size - k, pm.dtab, 256);
        if (used < 0) return -1;
        k += used;
    }
    for (int i = 0; i < 1024; i++) pm.ptab[i] <<= ploc;              // :1489-1496
    for (int i = 0; i < 256; i++) pm.dtab[i] <<= dloc;
    return (int)k;
}

}  // namespace

// One batch of fqzcomp streams, HOST buffers.  out_cap[i]: the block's uncomp_size; status HGPU_OK / HGPU_FQZ_ERR.
static int hgpu_fqz_decode_batch_host_impl(hgpu_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
        const uint32_t *in_len, uint32_t n, uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
        uint32_t *got_len, int32_t *status)
{
    if (!ctx || (n && (!in || !in_off || !in_len || !out || !out_off || !out_cap || !got_len || !status))) {
        hgpu_set_error("bad argument");
        return HGPU_ERR_ARG;
    }
    if (n == 0) return HGPU_OK;
    if (hgpu_check(cudaSetDevice(ctx->device), "cudaSetDevice")) return HGPU_ERR_CUDA;

    std::vector<FqzStream> streams(n);
    std::vector<FqzParam> params;
    const uint64_t MODEL_BUDGET = 6ull << 30;
    std::vector<uint32_t> wave_first(1, 0u);                                  // first stream of every wave
    uint64_t model_words_total = 0 /* largest wave */, wave_words = 0, flag_bytes = 0;
    const uint64_t in_end = hgpu_slots_end(in_off, in_len, n), out_end = hgpu_slots_end(out_off, out_cap, n);
    for (uint32_t s = 0; s < n; s++) {
        FqzStream &S = streams[s];
        memset(&S, 0, sizeof(S));
        S.in_off = in_off[s]; S.in_len = in_len[s]; S.out_off = out_off[s]; S.out_cap = out_cap[s];
        S.host_status = HGPU_FQZ_ERR;
        const uint8_t *p = in + in_off[s], *e = p + in_len[s];
        uint32_t ulen;
        size_t k = (size_t)hgpu_var_get_u32(p, e, &ulen);
        // fqz_read_parameters (:1325-1379)
        if ((size_t)in_len[s] < k || in_len[s] - k < 10) continue;
        const uint8_t *q = p + k;
        const size_t qn = in_len[s] - k;
        size_t j = 0;
        if (q[j++] != 5) continue;                                       // FQZ_VERS
        const uint32_t gflags = q[j++];
        const int nparam = (gflags & GFLAG_MULTI_PARAM) ? q[j++] : 1;
        if (nparam <= 0) continue;
        uint32_t max_sel = nparam > 1 ? (uint32_t)nparam : 0;
        uint32_t stab[256];
        if (gflags & GFLAG_HAVE_STAB) {
            max_sel = q[j++];
            int used = h_read_array(q + j, qn - j, stab, 256);
            if (used < 0) continue;
            j += used;
        } else {
            for (int i = 0; i < 256; i++) stab[i] = i < nparam ? (uint32_t)i : (uint32_t)nparam - 1;
        }
        const size_t pmark = params.size();
        params.resize(pmark + nparam);
        uint32_t gmax = 0;
        bool ok = true;
        for (int i = 0; i < nparam && ok; i++) {
            uint32_t ms = 0;
            int used = j <= qn ? h_read_param(params[pmark + i], ms, q + j, qn - j) : -1;
            if (used < 0 || (params[pmark + i].do_sel && max_sel == 0)) { ok = false; break; }
            j += used;
            if (ms > gmax) gmax = ms;
        }
        if (!ok) { params.resize(pmark); continue; }
        S.ulen = ulen; S.payload = (uint32_t)(k + j);
        S.nparam = (uint32_t)nparam; S.gflags = gflags; S.max_sel = max_sel; S.nsym = gmax + 1;
        S.param0 = (uint32_t)pmark;
        for (int i = 0; i < 256; i++) S.stab[i] = (uint16_t)stab[i];
        // Model arenas are handed out per WAVE: a 65 536-context arena is 11 MB at 40 symbols and 68 MB at 256, so an
        // archive-profile file with thousands of quality blocks would ask for hundreds of GB at once.  Streams are
        // decoded in waves whose arenas fit MODEL_BUDGET (one stream alone may exceed it); a wave reuses the arena.
        const uint64_t words = (uint64_t)CTX_SIZE * (S.nsym + 4) + 4 * 260 + 6 + 6 + (max_sel + 1 + 4) + 8;
        if (wave_words && (wave_words + words) * 4 > MODEL_BUDGET) { wave_first.push_back(s); wave_words = 0; }
        S.model_off = wave_words;
        wave_words += words;
        if (wave_words > model_words_total) model_words_total = wave_words;
        S.flag_off = flag_bytes;
        if (gflags & GFLAG_DO_REV) flag_bytes += ((uint64_t)ulen + 16) & ~(uint64_t)15;
        S.host_status = HGPU_OK;
    }
    if (params.empty()) params.resize(1);

    StageLayout L;
    const auto s_in = L.seg(in_end + 8), s_out = L.seg(out_end + 8), s_streams = L.seg((size_t)n * sizeof(FqzStream)),
               s_params = L.seg(params.size() * sizeof(FqzParam)), s_flags = L.seg(flag_bytes + 16), s_got = L.seg((size_t)n * 4),
               s_st = L.seg((size_t)n * 4), s_models = L.seg(model_words_total * 4 + 16);
    int rc = hgpu_stage_ensure(ctx, L);
    if (rc) return rc;
    cudaStream_t st = ctx->stream;
    const FqzStream *d_streams = L.at<FqzStream>(s_streams);
    if (hgpu_h2d(L.at(s_in), in, in_end, st) || hgpu_h2d(L.at(s_streams), streams.data(), (size_t)n * sizeof(FqzStream), st) ||
        hgpu_h2d(L.at(s_params), params.data(), params.size() * sizeof(FqzParam), st) || hgpu_memset(L.at(s_flags), 0, flag_bytes, st)) return HGPU_ERR_CUDA;
    wave_first.push_back(n);
    for (size_t w = 0; w + 1 < wave_first.size(); w++) {                      // waves run back to back on one stream: the arena is reused
        const uint32_t w0 = wave_first[w], wn = wave_first[w + 1] - w0;
        if (!wn) continue;
        for (uint32_t first = 0; first < wn; first += 65535u) {               // gridDim.y limit
            const uint32_t cnt = wn - first < 65535u ? wn - first : 65535u;
            fqz_init_models_kernel<<<dim3(64, cnt), 256, 0, st>>>(d_streams + w0 + first, L.at<uint32_t>(s_models));
            if (hgpu_check(cudaGetLastError(), "fqz_init_models_kernel")) return HGPU_ERR_CUDA;
            hgpu_count_launch();
        }
        fqz_decode_kernel<<<(wn + 31) / 32, 32, 0, st>>>(d_streams + w0, wn, L.at<FqzParam>(s_params), L.at(s_in), L.at<uint32_t>(s_models),
                                                        L.at(s_flags), L.at(s_out), L.at<uint32_t>(s_got) + w0, L.at<int32_t>(s_st) + w0);
        if (hgpu_check(cudaGetLastError(), "fqz_decode_kernel")) return HGPU_ERR_CUDA;
        hgpu_count_launch();
    }
    if (hgpu_d2h(got_len, L.at(s_got), (size_t)n * 4, st) || hgpu_d2h(status, L.at(s_st), (size_t)n * 4, st) ||
        hgpu_d2h(out, L.at(s_out), out_end, st)) return HGPU_ERR_CUDA;
    if (hgpu_check(cudaStreamSynchronize(st), "sync")) return HGPU_ERR_CUDA;
    return HGPU_OK;
}

extern "C" int hgpu_fqz_decode_batch_host(hgpu_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
        const uint32_t *in_len, uint32_t n, uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
        uint32_t *got_len, int32_t *status)
{
    return hgpu_abi_call([&] { return hgpu_fqz_decode_batch_host_impl(ctx, in, in_off, in_len, n, out, out_off, out_cap, got_len, status); });
}

// Drop-in for the reference symbol (fqzcomp_qual.h): malloc'd result or NULL.  lengths/nlengths as in the
// reference are not filled (cram_uncompress_block passes NULL, 0).
extern "C" char *fqz_decompress(char *in, size_t comp_size, size_t *uncomp_size, int *lengths, int nlengths)
{
    (void)lengths; (void)nlengths;
    if (!in || !uncomp_size || comp_size > 0xffffffffull) return nullptr;
    uint32_t ulen = 0;
    hgpu_var_get_u32((const uint8_t *)in, (const uint8_t *)in + comp_size, &ulen);
    ShimLock lock;
    hgpu_ctx *g_fqz_ctx = hgpu_shim_ctx();
    if (!g_fqz_ctx) return nullptr;
    uint8_t *out = (uint8_t *)malloc(ulen ? ulen : 1);
    if (!out) return nullptr;
    uint64_t ioff = 0, ooff = 0;
    uint32_t ilen = (uint32_t)comp_size, got = 0;
    int32_t st = 0;
    int rc = hgpu_fqz_decode_batch_host(g_fqz_ctx, (const uint8_t *)in, &ioff, &ilen, 1, out, &ooff, &ulen, &got, &st);
    if (rc != HGPU_OK || st != HGPU_OK) { free(out); return nullptr; }
    *uncomp_size = got;
    return (char *)out;
}
