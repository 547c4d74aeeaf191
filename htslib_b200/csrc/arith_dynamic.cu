// Adaptive arithmetic coder ("ARITH_PR", CRAM 3.1 block method 6) decoder for sm_90a.
//
// Replaces arith_uncompress_to and the bodies behind it (htscodecs arith_dynamic.c:1033-1278,
// :137-165 O0, :227-272 O1, :520-580 O0_RLE, :660-728 O1_RLE; range coder c_range_coder.h:62-166;
// adaptive model c_simple_model.h:85-171).  The coder is strictly sequential — one range-coder
// state, the model is updated after every symbol — so the unit of parallelism is the STREAM: one
// thread per stream, thousands of streams per launch (SURVEY.md §7 "hard parts").  PACK, STRIPE,
// CAT and NOSZ wrappers are handled in the same thread.  X_EXT (bzip2 payload) is rejected, as the
// reference itself does when built without libbz2 (:1218-1226).
//
// Model layout follows the reference bit for bit, because the approximate sort order of the
// symbol array (swap-with-previous after each update, halving at 65519) is part of the format.
// Parity: golden streams htscodecs/tests/dat/arith/* and the compiled reference (oracle/_ref) on
// seeded inputs; the CPU restatement oracle/orc_arith.c is pinned on the same fixtures.
#include "hgpu_internal.h"

namespace {

constexpr uint32_t TOP = 1u << 24;
constexpr uint32_t MAX_FREQ = (1u << 16) - 17;
constexpr int STEP = 16;
constexpr int NS = 258;                 // large enough for both the byte (256) and run (258) models
constexpr int MAX_RUN = 4;

struct SymFreq { uint16_t freq, sym; };
struct Model {                          // SIMPLE_MODEL(NSYM,_), c_simple_model.h:74-79
    uint32_t tot;
    SymFreq sentinel, F[NS + 1], terminal;
};

struct RC {                             // decoder half of RangeCoder
    const uint8_t *p, *end;
    uint32_t range, code;
    int err;
};

__device__ void model_init(Model *m, int nsym, int max_sym)
{
    for (int i = 0; i < nsym; i++) { m->F[i].sym = (uint16_t)i; m->F[i].freq = i < max_sym ? 1 : 0; }
    m->tot = (uint32_t)max_sym;
    m->sentinel.sym = 0; m->sentinel.freq = (uint16_t)MAX_FREQ;
    m->F[nsym].freq = 0;                                    // terminates the normalise loop
    m->F[nsym].sym = 0;
    // the reference's `terminal` sits right behind F[NSYM]; with one struct for both model sizes
    // F[nsym+1] plays that role for the 256-symbol models
    if (nsym < NS) { m->F[nsym + 1].freq = (uint16_t)MAX_FREQ; m->F[nsym + 1].sym = 0; }
    m->terminal.sym = 0; m->terminal.freq = (uint16_t)MAX_FREQ;
}

__device__ void rc_start(RC *rc, const uint8_t *p, const uint8_t *end)
{
    rc->range = 0xffffffffu; rc->code = 0; rc->err = 0; rc->p = p; rc->end = end;
    if (p + 5 > end) { rc->p = end; return; }
    for (int i = 0; i < 5; i++) rc->code = (rc->code << 8) | *rc->p++;
}

// SIMPLE_MODEL_decodeSymbol, c_simple_model.h:135-169
__device__ uint16_t model_decode(Model *m, int nsym, RC *rc)
{
    SymFreq *s = m->F;
    uint32_t tot = m->tot;
    uint32_t freq = (tot && rc->range >= tot) ? rc->code / (rc->range /= tot) : 0;     // RC_GetFreq
    if (freq > MAX_FREQ) return 0;
    uint32_t acc = 0;
    for (acc = 0; (acc += s->freq) <= freq; s++)
        ;
    if (s - m->F > nsym) return 0;
    acc -= s->freq;
    // RC_Decode
    rc->code -= acc * rc->range;
    rc->range *= s->freq;
    while (rc->range < TOP) {
        if (rc->p >= rc->end) { rc->err = -1; break; }
        rc->code = (rc->code << 8) + *rc->p++;
        rc->range <<= 8;
    }
    s->freq += STEP;
    m->tot += STEP;
    if (m->tot > MAX_FREQ) {                                // normalise: halve until a zero frequency
        uint32_t t = 0;
        for (SymFreq *q = m->F; q->freq; q++) { q->freq -= q->freq >> 1; t += q->freq; }
        m->tot = t;
    }
    SymFreq *prev = s == m->F ? &m->sentinel : s - 1;
    if (s->freq > prev->freq) {
        SymFreq t = *s; *s = *prev; *prev = t;
        return t.sym;
    }
    return s->sym;
}

struct ThreadScratch {
    Model *byte_model;   // [256]
    Model *run_model;    // [258]
    uint8_t *tmp, *planes;
    uint32_t max_out;
};

__device__ int vget(const uint8_t *p, const uint8_t *end, uint32_t &v)      // var_get_u32, varint.h:267
{
    const uint8_t *s = p;
    uint32_t acc = 0;
    uint8_t c;
    if (end - p >= 6) {
        int budget = 5;
        do { c = *p++; acc = (acc << 7) | (c & 0x7f); } while ((c & 0x80) && budget-- > 0);
    } else {
        if (p >= end) { v = 0; return 0; }
        do { c = *p++; acc = (acc << 7) | (c & 0x7f); } while ((c & 0x80) && p < end);
    }
    v = acc;
    return (int)(p - s);
}

__device__ int body(const ThreadScratch &ts, const uint8_t *in, uint32_t in_size, uint8_t *out, uint32_t out_sz,
                    int order, bool rle)
{
    if (in_size == 0) return -1;
    const int m = in[0] ? in[0] : 256;
    RC rc;
    Model *bm = ts.byte_model, *rm = ts.run_model;
    const int nctx = order == 1 ? 256 : 1;
    for (int i = 0; i < nctx; i++) model_init(&bm[i], 256, m);
    if (rle) for (int i = 0; i < NS; i++) model_init(&rm[i], NS, MAX_RUN);
    rc_start(&rc, in + 1, in + in_size);
    uint32_t last = 0;
    for (uint32_t i = 0; i < out_sz; i++) {
        uint32_t c = model_decode(&bm[order == 1 ? last : 0], 256, &rc);
        out[i] = (uint8_t)c;
        last = c & 0xff;
        if (rle) {
            uint32_t run = 0, r;
            uint32_t rctx = last;
            do {
                r = model_decode(&rm[rctx], NS, &rc);
                if (rctx == last) rctx = 256;
                else rctx += (rctx < (uint32_t)NS - 1);
                run += r;
            } while (r == (uint32_t)MAX_RUN - 1 && run < out_sz);
            while (run-- && i + 1 < out_sz) out[++i] = (uint8_t)last;
        }
    }
    return rc.err < 0 ? -1 : 0;
}

__device__ int unpack_meta(const uint8_t *d, uint32_t len, uint8_t *map, int &per_byte)   // pack.c:161-196
{
    if (!len) return 0;
    uint32_t n = d[0] ? d[0] : 256, j = 1, c = 0;
    if (n <= 1) per_byte = 0;
    else if (n <= 2) per_byte = 8;
    else if (n <= 4) per_byte = 4;
    else if (n <= 16) per_byte = 2;
    else { per_byte = 1; return 1; }
    if (len <= 1) return 0;
    do { map[c++] = d[j++]; } while (c < n && j < len);
    return c < n ? 0 : (int)j;
}

__device__ int decode_plain(const ThreadScratch &ts, const uint8_t *in, uint32_t in_size, uint8_t *out,
                            uint32_t out_cap, uint32_t &out_size)
{
    const uint8_t *end = in + in_size;
    int fmt = *in++; in_size--;
    const bool do_pack = fmt & 0x80, do_rle = fmt & 0x40, do_cat = fmt & 0x20, no_size = fmt & 0x10, do_ext = fmt & 0x04;
    const int order = fmt & 3;
    uint32_t osz;
    if (!no_size) { int s = vget(in, end, osz); in += s; in_size -= s; } else osz = out_cap;
    if (osz >= 0x7fffffffu || out_cap < osz || osz > ts.max_out) return -1;
    out_size = osz;
    uint32_t t1_size = osz;
    uint8_t *t1 = do_pack ? ts.tmp : out;
    uint8_t map[16];
    for (int k = 0; k < 16; k++) map[k] = 0;
    int per_byte = 0;
    uint64_t unpacked = 0;
    if (do_pack) {
        int mlen = unpack_meta(in, in_size, map, per_byte);
        if (!mlen) return -1;
        unpacked = osz;
        in += mlen; in_size -= mlen;
        uint32_t psz;
        int s = vget(in, end, psz);
        in += s; in_size -= s;
        if (psz > t1_size) return -1;
        t1_size = psz;
    }
    if (in_size) {
        if (do_cat) {
            if (t1_size > in_size || t1_size > out_size) return -1;
            for (uint32_t i = 0; i < t1_size; i++) t1[i] = in[i];
        } else if (do_ext) return -1;                        // bzip2 payload: not supported (reference without libbz2 errors too)
        else if (body(ts, in, in_size, t1, t1_size, order, do_rle)) return -1;
    } else
        t1_size = 0;
    if (do_pack) {
        if (per_byte == 1) unpacked = t1_size;
        // hts_unpack, pack.c:207-330
        if (per_byte == 1) { for (uint32_t i = 0; i < t1_size; i++) out[i] = t1[i]; }
        else if (per_byte == 0) { for (uint64_t i = 0; i < unpacked; i++) out[i] = map[0]; }
        else {
            int bits = per_byte == 8 ? 1 : per_byte == 4 ? 2 : 4;
            if ((unpacked + per_byte - 1) / per_byte > t1_size) return -1;
            for (uint64_t i = 0; i < unpacked; i++)
                out[i] = map[(t1[i / per_byte] >> (bits * (i % per_byte))) & ((1 << bits) - 1)];
        }
        out_size = (uint32_t)unpacked;
    } else
        out_size = t1_size;
    return 0;
}

__device__ int decode_stream(const ThreadScratch &ts, const uint8_t *in, uint32_t in_size, uint8_t *out,
                             uint32_t out_cap, uint32_t &out_size)
{
    if (in_size == 0) return -1;
    if (!(in[0] & 0x08)) return decode_plain(ts, in, in_size, out, out_cap, out_size);
    // STRIPE (:1041-1116)
    const uint8_t *end = in + in_size;
    uint32_t ulen, off = 1;
    off += vget(in + off, end, ulen);
    if (off >= in_size) return -1;
    uint32_t n = in[off++];
    if (n < 1 || ulen != out_cap || ulen > ts.max_out) return -1;
    uint64_t ctot = 0;
    uint32_t off2 = off;
    for (uint32_t k = 0; k < n; k++) {
        uint32_t cl;
        off2 += vget(in + off2, end, cl);
        ctot += cl;
        if (off2 > in_size || cl > in_size || cl < 1) return -1;
    }
    if (off2 + ctot > in_size) return -1;
    in_size = (uint32_t)(off2 + ctot);
    uint32_t data = off2, idx = 0;
    for (uint32_t k = 0; k < n; k++) {
        uint32_t cl;
        off += vget(in + off, end, cl);
        uint32_t ul = ulen / n + ((ulen % n) > k), got = 0;
        if (in_size <= data || (in[data] & 0x08)) return -1;         // nested stripes are never written
        if (decode_plain(ts, in + data, in_size - data, ts.planes + idx, ul, got) || got != ul) return -1;
        data += cl; idx += ul;
    }
    const uint32_t q = ulen / n, r = ulen % n;
    for (uint32_t j = 0; j < ulen; j++) {                            // unstripe, utils.h:79-138
        uint32_t k = j % n, i = j / n;
        out[j] = ts.planes[k * q + (k < r ? k : r) + i];
    }
    out_size = ulen;
    return 0;
}

__global__ void __launch_bounds__(32)
arith_decode_kernel(const uint8_t *__restrict__ in, const uint64_t *__restrict__ in_off,
                    const uint32_t *__restrict__ in_len, uint32_t n, uint8_t *out,
                    const uint64_t *__restrict__ out_off, const uint32_t *__restrict__ out_len,
                    uint32_t *got_len, int32_t *status, uint8_t *scratch, size_t per_thread, uint32_t max_out,
                    uint32_t *counter)
{
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint8_t *base = scratch + tid * per_thread;
    ThreadScratch ts;
    ts.byte_model = reinterpret_cast<Model *>(base);
    ts.run_model = ts.byte_model + 256;
    size_t mo = ((size_t)max_out + 15) & ~(size_t)15;
    ts.tmp = reinterpret_cast<uint8_t *>(ts.run_model + NS);
    ts.planes = ts.tmp + mo;
    ts.max_out = max_out;
    for (;;) {
        uint32_t job = atomicAdd(counter, 1u);
        if (job >= n) break;
        uint32_t got = 0;
        int rc = decode_stream(ts, in + in_off[job], in_len[job], out + out_off[job], out_len[job], got);
        status[job] = rc ? -1 : 0;
        got_len[job] = rc ? 0 : got;
    }
}

} // namespace

extern "C" int hgpu_arith_decode_batch_dev(hgpu_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
        const uint32_t *d_in_len, uint32_t n, uint8_t *d_out, const uint64_t *d_out_off, const uint32_t *d_out_len,
        uint32_t *d_got_len, int32_t *d_status, uint32_t max_out_len, void *stream)
{
    if (!ctx) { hgpu_set_error("null context"); return HGPU_ERR_ARG; }
    if (n == 0) return HGPU_OK;
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    uint32_t threads = n < 2048u ? n : 2048u;
    uint32_t grid = (threads + 31) / 32;
    size_t mo = ((size_t)max_out_len + 15) & ~(size_t)15;
    size_t per_thread = (sizeof(Model) * (256 + NS) + 2 * mo + 255) & ~(size_t)255;
    int rc = hgpu_ensure_scratch(ctx, per_thread * grid * 32);
    if (rc) return rc;
    uint32_t *counter = hgpu_take_counter(ctx, st);
    if (!counter) return HGPU_ERR_CUDA;
    arith_decode_kernel<<<grid, 32, 0, st>>>(d_in, d_in_off, d_in_len, n, d_out, d_out_off, d_out_len, d_got_len,
                                             d_status, ctx->d_scratch, per_thread, max_out_len, counter);
    hgpu_count_launch();
    return hgpu_check(cudaGetLastError(), "arith launch");
}
