// Adaptive arithmetic coder ("ARITH_PR", CRAM 3.1 block method 6) ENCODER for sm_90a.
//
// Stands where arith_compress_to stands (htscodecs/htscodecs/arith_dynamic.c:730-1026) with the bodies
// behind it: arith_compress_O0 :98-136, _O1 :172-222, _O0_RLE :441-519, _O1_RLE :572-658, hts_pack
// (pack.c:56-146), the range coder's encode half (c_range_coder.h:51-146) and the adaptive model
// (c_simple_model.h:85-133).  Like the decoder the coder is sequential — one range/low pair with carry
// propagation, a model updated per symbol — so the unit of parallelism is the stream: one THREAD per
// stream.  Because every step is deterministic the output is byte-identical to the reference encoder's
// for the same `order` flags (tests/test_gpu_arith_enc.py pins exactly that), including the CAT
// fallback when entropy coding does not pay and the PACK bit being dropped for > 16 symbols.
// X_STRIPE (a brute-force trial of sub-encodings per byte plane) is not produced: the flag is cleared
// and the stream is coded unstriped, which any arith_uncompress_to reads.  X_EXT (bzip2) is rejected.
#include "hgpu_internal.h"

namespace {

constexpr uint32_t TOP = 1u << 24;
constexpr uint32_t THRES = 255u * TOP;
constexpr uint32_t MAX_FREQ = (1u << 16) - 17;
constexpr int STEP = 16;
constexpr int NS = 258;
constexpr int MAX_RUN = 4;
constexpr int X_PACK = 0x80, X_RLE = 0x40, X_CAT = 0x20, X_NOSZ = 0x10, X_STRIPE = 0x08, X_EXT = 0x04;

struct SymFreq { uint16_t freq, sym; };
struct Model { uint32_t tot; SymFreq sentinel, F[NS + 1], terminal; };   // SIMPLE_MODEL(NSYM,_), c_simple_model.h:74-79

struct RCE {                                       // encoder half of RangeCoder (c_range_coder.h:29-36)
    uint8_t *p, *begin, *end;
    uint32_t low, range, ffnum, carry, cache;
    int err;
};

__device__ void model_init(Model *m, int nsym, int max_sym)
{
    for (int i = 0; i < nsym; i++) { m->F[i].sym = (uint16_t)i; m->F[i].freq = i < max_sym ? 1 : 0; }
    m->tot = (uint32_t)max_sym;
    m->sentinel.sym = 0; m->sentinel.freq = (uint16_t)MAX_FREQ;
    m->F[nsym].freq = 0; m->F[nsym].sym = 0;
}

__device__ __forceinline__ void rc_shift_low(RCE &rc)                    // RC_ShiftLowCheck :77-101
{
    if (rc.low < THRES || rc.carry) {
        if (rc.end && rc.ffnum >= (uint32_t)(rc.end - rc.p)) { rc.err = -1; return; }
        *rc.p++ = (uint8_t)(rc.cache + rc.carry);
        while (rc.ffnum) { *rc.p++ = (uint8_t)(rc.carry - 1); rc.ffnum--; }
        rc.cache = rc.low >> 24;
        rc.carry = 0;
    } else {
        rc.ffnum++;
    }
    rc.low <<= 8;
}

__device__ void model_encode(Model *m, RCE &rc, uint32_t sym)           // SIMPLE_MODEL_encodeSymbol :112-133
{
    SymFreq *s = m->F;
    uint32_t acc = 0;
    while (s->sym != sym) acc += (s++)->freq;
    // RC_Encode :133-146
    const uint32_t tmp = rc.low;
    rc.range /= m->tot;
    rc.low += acc * rc.range;
    rc.range *= s->freq;
    rc.carry += rc.low < tmp;
    while (rc.range < TOP) { rc.range <<= 8; rc_shift_low(rc); }
    s->freq += STEP;
    m->tot += STEP;
    if (m->tot > MAX_FREQ) {
        uint32_t t = 0;
        for (SymFreq *q = m->F; q->freq; q++) { q->freq -= q->freq >> 1; t += q->freq; }
        m->tot = t;
    }
    SymFreq *prev = s == m->F ? &m->sentinel : s - 1;
    if (s->freq > prev->freq) { SymFreq t = *s; *s = *prev; *prev = t; }
}

__device__ int vput(uint8_t *p, const uint8_t *end, uint32_t v)          // var_put_u32, varint.h:206-263
{
    int n = v < (1u << 7) ? 1 : v < (1u << 14) ? 2 : v < (1u << 21) ? 3 : v < (1u << 28) ? 4 : 5;
    if (end && end - p < n) return 0;
    for (int k = n - 1; k >= 0; k--) *p++ = (uint8_t)(((v >> (7 * k)) & 0x7f) | (k ? 0x80 : 0));
    return n;
}

// the four entropy coders; out[0] = max symbol + 1 (256 wraps to 0), then the range coder's bytes.
// Returns bytes written, or -1.
__device__ int encode_body(Model *bm, Model *rm, const uint8_t *in, uint32_t n, uint8_t *out, uint32_t cap, int order, bool rle)
{
    if (cap < 1) return -1;
    uint32_t mx = 0;
    for (uint32_t i = 0; i < n; i++) if (mx < in[i]) mx = in[i];
    mx++;
    out[0] = (uint8_t)mx;
    const int nctx = order ? 256 : 1;
    for (int i = 0; i < nctx; i++) model_init(&bm[i], 256, (int)mx);
    if (rle) for (int i = 0; i < NS; i++) model_init(&rm[i], NS, MAX_RUN);
    RCE rc;
    rc.p = rc.begin = out + 1; rc.end = out + cap;
    rc.range = 0xffffffffu; rc.low = 0; rc.ffnum = 0; rc.carry = 0; rc.cache = 0; rc.err = 0;
    uint32_t last = 0;
    if (!rle) {
        for (uint32_t i = 0; i < n; i++) {
            model_encode(&bm[order ? last : 0], rc, in[i]);
            last = in[i];
            if (rc.err) return -1;
        }
    } else {
        for (uint32_t i = 0; i < n;) {
            model_encode(&bm[order ? last : 0], rc, in[i]);
            int run = 0;
            last = in[i++];
            while (i < n && in[i] == last) { run++; i++; }
            uint32_t rctx = last;
            do {
                const int c = run < MAX_RUN ? run : MAX_RUN - 1;
                model_encode(&rm[rctx], rc, (uint32_t)c);
                run -= c;
                if (rctx == last) rctx = 256;
                else rctx += (rctx < (uint32_t)NS - 1);
                if (c == MAX_RUN - 1 && run == 0) model_encode(&rm[rctx], rc, 0);
            } while (run);
            if (rc.err) return -1;
        }
    }
    for (int k = 0; k < 5; k++) rc_shift_low(rc);                         // RC_FinishEncode
    if (rc.err) return -1;
    return (int)(rc.p - rc.begin) + 1;
}

// hts_pack (pack.c:56-146): meta into `meta`, packed bytes into `pk`.  Returns false when > 16 symbols.
__device__ bool pack(const uint8_t *in, uint32_t n, uint8_t *meta, uint32_t &meta_len, uint8_t *pk, uint32_t &pk_len)
{
    uint32_t present[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (uint32_t i = 0; i < n; i++) present[in[i] >> 5] |= 1u << (in[i] & 31);
    uint8_t code[256];
    int ns = 0;
    for (int i = 0; i < 256; i++)
        if (present[i >> 5] >> (i & 31) & 1) { code[i] = (uint8_t)ns++; if (ns <= 16) meta[ns] = (uint8_t)i; }
    meta[0] = (uint8_t)ns;
    if (ns > 16) return false;
    meta_len = (uint32_t)ns + 1;
    const int per = ns > 4 ? 2 : ns > 2 ? 4 : ns > 1 ? 8 : 0;
    uint32_t j = 0;
    if (per) {
        const int bits = 8 / per;
        for (uint32_t i = 0; i < n; i += per) {
            uint32_t v = 0;
            for (int k = 0; k < per && i + k < n; k++) v |= (uint32_t)code[in[i + k]] << (bits * k);
            pk[j++] = (uint8_t)v;
        }
    }
    pk_len = j;
    return true;
}

// arith_compress_to (:730-1026) without the STRIPE arm.  Returns the stream length or -1.
__device__ int encode_stream(Model *bm, Model *rm, uint8_t *pkbuf, const uint8_t *in, uint32_t in_size, uint8_t *out, uint32_t out_cap, int order)
{
    if (out_cap == 0) return -1;
    const uint8_t *out_end = out + out_cap;
    order &= ~X_STRIPE;
    order &= 0xff;
    if (order & X_CAT) {
        out[0] = X_CAT;
        const int k = vput(out + 1, out_end, in_size);
        const uint32_t meta = 1 + (uint32_t)k;
        if (!k || (uint64_t)meta + in_size > out_cap) return -1;
        for (uint32_t i = 0; i < in_size; i++) out[meta + i] = in[i];
        return (int)(meta + in_size);
    }
    if (order & X_EXT) return -1;
    bool do_pack = order & X_PACK;
    const bool do_rle = order & X_RLE;
    const int no_size = order & X_NOSZ;
    out[0] = (uint8_t)order;
    uint32_t meta = 1;
    if (!no_size) meta += (uint32_t)vput(out + 1, out_end, in_size);
    int ord = order & 3;
    uint32_t avail = out_cap;
    if (do_pack && in_size) {
        if (meta + 256 > out_cap) return -1;
        uint32_t ml = 0, pl = 0;
        if (!pack(in, in_size, out + meta, ml, pkbuf, pl)) {
            out[0] &= ~X_PACK;
            do_pack = false;
        } else {
            in = pkbuf; in_size = pl;
            meta += ml;
            const int sz = vput(out + meta, out_end, in_size);
            meta += (uint32_t)sz;
            avail -= (uint32_t)sz;
        }
    } else if (do_pack) {
        out[0] &= ~X_PACK;
    }
    if (do_rle && !in_size) out[0] &= ~X_RLE;
    if (avail < meta) return -1;
    avail -= meta;
    if (ord && in_size < 8) { out[0] &= ~3; ord = 0; }
    // each coder first checks that its worst case fits (arith_compress_bound(in_size, 0) - 5, :77-86)
    const uint32_t bound = (uint32_t)(1.05 * in_size + 257 * 3 + 4);
    const int o1 = do_rle ? ord != 0 : ord == 1;                          // the dispatch at :976-990, as written there
    int got = bound > avail ? -1 : encode_body(bm, rm, in, in_size, out + meta, avail, o1, do_rle);
    if (got < 0) return -1;
    uint32_t body = (uint32_t)got;
    if (body >= in_size) {                                                // no gain: store, keep e.g. PACK (:1003-1016)
        out[0] &= ~(3 | X_EXT);
        out[0] |= X_CAT | no_size;
        if ((uint64_t)meta + in_size > out_cap) return -1;
        for (uint32_t i = 0; i < in_size; i++) out[meta + i] = in[i];
        body = in_size;
    }
    return (int)(body + meta);
}

__global__ void __launch_bounds__(32)
arith_encode_kernel(const uint8_t *__restrict__ in, const uint64_t *__restrict__ in_off, const uint32_t *__restrict__ in_len,
                    const uint32_t *__restrict__ order, uint32_t n, uint8_t *out, const uint64_t *__restrict__ out_off,
                    const uint32_t *__restrict__ out_cap, uint32_t *out_len, int32_t *status, uint8_t *scratch,
                    size_t per_thread, uint32_t *counter)
{
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint8_t *base = scratch + tid * per_thread;
    Model *bm = reinterpret_cast<Model *>(base), *rm = bm + 256;
    uint8_t *pk = reinterpret_cast<uint8_t *>(rm + NS);
    for (;;) {
        const uint32_t job = atomicAdd(counter, 1u);
        if (job >= n) break;
        const int got = encode_stream(bm, rm, pk, in + in_off[job], in_len[job], out + out_off[job], out_cap[job], (int)order[job]);
        status[job] = got < 0 ? -1 : 0;
        out_len[job] = got < 0 ? 0 : (uint32_t)got;
    }
}

}  // namespace

// arith_compress_bound (:77-86)
extern "C" uint32_t hgpu_arith_compress_bound(uint32_t size, int order)
{
    int N = (order >> 8) & 0xff;
    if (!N) N = 4;
    return (uint32_t)((order == 0 ? 1.05 * size + 257 * 3 + 4 : 1.05 * size + 257 * 257 * 3 + 4 + 257 * 3 + 4) + 5 +
                      ((order & X_PACK) ? 1 : 0) + ((order & X_RLE) ? 1 + 257 * 3 + 4 : 0) + ((order & X_STRIPE) ? 7 + 5 * N : 0));
}

extern "C" int hgpu_arith_encode_batch_dev(hgpu_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
        const uint32_t *d_in_len, const uint32_t *d_order, uint32_t n, uint8_t *d_out, const uint64_t *d_out_off,
        const uint32_t *d_out_cap, uint32_t *d_out_len, int32_t *d_status, uint32_t max_in_len, void *stream)
{
    if (!ctx) { hgpu_set_error("null context"); return HGPU_ERR_ARG; }
    if (n == 0) return HGPU_OK;
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    const uint32_t threads = n < 2048u ? n : 2048u;
    const uint32_t grid = (threads + 31) / 32;
    const size_t mi = ((size_t)max_in_len + 16 + 15) & ~(size_t)15;
    const size_t per_thread = (sizeof(Model) * (256 + NS) + mi + 255) & ~(size_t)255;
    int rc = hgpu_ensure_scratch(ctx, per_thread * grid * 32);
    if (rc) return rc;
    uint32_t *counter = hgpu_take_counter(ctx, st);
    if (!counter) return HGPU_ERR_CUDA;
    arith_encode_kernel<<<grid, 32, 0, st>>>(d_in, d_in_off, d_in_len, d_order, n, d_out, d_out_off, d_out_cap, d_out_len,
                                             d_status, ctx->d_scratch, per_thread, counter);
    hgpu_count_launch();
    return hgpu_check(cudaGetLastError(), "arith encode launch");
}
