// Reference-named entry points of the libhtscodecs link seam (SURVEY.md §8b tier B1) that are thin
// wrappers over this library's batch kernels: one stream per call, the reference's signatures, malloc
// ownership and NULL-on-error convention (rANS_static.h:40-43, rANS_static4x16.h:41-64,
// arith_dynamic.h:40-55, tokenise_name3.h:49-58, fqzcomp_qual.h:152-167).  With `-lhtsgpu` ahead of
// `-lhtscodecs` (htslib's --with-external-htscodecs build) cram/cram_io.c:1666-1747 and :1834-1899 call
// these unchanged.  Each is a batch of one — H2D, one launch, D2H on the process-wide shim context —
// correct, not fast; the batch entry points are the fast path.  The decoders that already had shims
// (rans_uncompress_to_4x16, tok3_decode_names, fqz_decompress) live next to their host code.
#include "hgpu_internal.h"
#include <stdlib.h>
#include <string.h>
#include <vector>

namespace {

enum Kind { DEC_R4X8, DEC_ARITH, ENC_R4X8, ENC_ARITH, ENC_NX16 };

// one stream through a device batch entry point: host in -> host out (cap bytes).  Returns the length or -1.
long one_stream(Kind kind, const uint8_t *in, uint32_t in_size, uint8_t *out, uint32_t cap, uint32_t order)
{
    ShimLock lock;
    hgpu_ctx *ctx = hgpu_shim_ctx();
    if (!ctx) return -1;
    if (cudaSetDevice(ctx->device) != cudaSuccess) return -1;
    StageLayout L;
    const auto s_in = L.seg((size_t)in_size + 16), s_out = L.seg((size_t)cap + 16), s_off = L.seg(16) /* {in_off, out_off} */,
               s_w = L.seg(16) /* {in_len, out_cap, order, got} */, s_st = L.seg(4);
    if (hgpu_stage_ensure(ctx, L)) return -1;
    uint8_t *d_in = L.at(s_in), *d_out = L.at(s_out);
    uint64_t *d_off = L.at<uint64_t>(s_off);
    uint32_t *d_w = L.at<uint32_t>(s_w);
    int32_t *d_st = L.at<int32_t>(s_st);
    const uint64_t offs[2] = {0, 0};
    const uint32_t w[4] = {in_size, cap, order, 0};
    cudaStream_t s = ctx->stream;
    if (hgpu_h2d(d_in, in, in_size, s) || hgpu_h2d(d_off, offs, sizeof(offs), s) || hgpu_h2d(d_w, w, sizeof(w), s)) return -1;
    int rc;
    switch (kind) {
    case DEC_R4X8:  rc = hgpu_rans4x8_decode_batch_dev(ctx, d_in, d_off, d_w, 1, d_out, d_off + 1, d_w + 1, d_w + 3, d_st, s); break;
    case DEC_ARITH: rc = hgpu_arith_decode_batch_dev(ctx, d_in, d_off, d_w, 1, d_out, d_off + 1, d_w + 1, d_w + 3, d_st, cap, s); break;
    case ENC_R4X8:  rc = hgpu_rans4x8_encode_batch_dev(ctx, d_in, d_off, d_w, d_w + 2, 1, d_out, d_off + 1, d_w + 1, d_w + 3, d_st, s); break;
    case ENC_ARITH: rc = hgpu_arith_encode_batch_dev(ctx, d_in, d_off, d_w, d_w + 2, 1, d_out, d_off + 1, d_w + 1, d_w + 3, d_st, in_size, s); break;
    default:        rc = hgpu_rans_nx16_encode_batch_dev(ctx, d_in, d_off, d_w, d_w + 2, 1, d_out, d_off + 1, d_w + 1, d_w + 3, d_st, s); break;
    }
    if (rc) return -1;
    uint32_t got = 0;
    int32_t st = 0;
    if (hgpu_d2h(&got, d_w + 3, 4, s) || hgpu_d2h(&st, d_st, 4, s)) return -1;
    if (cudaStreamSynchronize(s) != cudaSuccess) return -1;
    if (st != HGPU_OK || got > cap) return -1;
    if (got && cudaMemcpy(out, d_out, got, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    return (long)got;
}

}  // namespace

extern "C" {

// ---- rANS 4x8 (CRAM 3.0 method 4), rANS_static.c:829-850
unsigned char *rans_uncompress(unsigned char *in, unsigned int in_size, unsigned int *out_size)
{
    if (!in || !out_size || in_size < 9) return nullptr;
    const unsigned int ulen = in[5] | in[6] << 8 | in[7] << 16 | (unsigned int)in[8] << 24;   // the stream's own size field (:606-612)
    if (ulen >= 0x7fffffffu) return nullptr;
    unsigned char *out = (unsigned char *)malloc(ulen ? ulen : 1);
    if (!out) return nullptr;
    const long got = one_stream(DEC_R4X8, in, in_size, out, ulen, 0);
    if (got < 0) { free(out); return nullptr; }
    *out_size = (unsigned int)got;
    return out;
}

unsigned char *rans_compress(unsigned char *in, unsigned int in_size, unsigned int *out_size, int order)
{
    if ((!in && in_size) || !out_size || in_size > 0x7fffffffu) { if (out_size) *out_size = 0; return nullptr; }
    const uint32_t cap = hgpu_rans4x8_compress_bound(in_size);
    unsigned char *out = (unsigned char *)malloc(cap);
    if (!out) return nullptr;
    const long got = one_stream(ENC_R4X8, in, in_size, out, cap, order ? 1u : 0u);
    if (got < 0) { free(out); return nullptr; }
    *out_size = (unsigned int)got;
    return out;
}

// ---- adaptive arithmetic coder (method 6), arith_dynamic.c:730-1031, :1033-1283
unsigned int arith_compress_bound(unsigned int size, int order) { return hgpu_arith_compress_bound(size, order); }

unsigned char *arith_uncompress_to(unsigned char *in, unsigned int in_size, unsigned char *out, unsigned int *out_size)
{
    if (!in || in_size == 0 || !out_size) return nullptr;
    unsigned int ulen = 0;
    const bool sized = (in[0] & 0x08) || !(in[0] & 0x10);               // STRIPE always carries the size; otherwise unless NOSZ
    if (sized) hgpu_var_get_u32_bounded(in + 1, in + in_size, &ulen);
    unsigned char *alloc = nullptr;
    if (!out) {
        if (!sized || ulen >= 0x7fffffffu) return nullptr;              // "Need one or the other" (:1148-1149)
        alloc = out = (unsigned char *)malloc(ulen ? ulen : 1);
        if (!out) return nullptr;
        *out_size = ulen;
    }
    const long got = one_stream(DEC_ARITH, in, in_size, out, *out_size, 0);
    if (got < 0) { free(alloc); return nullptr; }
    *out_size = (unsigned int)got;
    return out;
}

unsigned char *arith_uncompress(unsigned char *in, unsigned int in_size, unsigned int *out_size)
{
    return arith_uncompress_to(in, in_size, nullptr, out_size);
}

unsigned char *arith_compress_to(unsigned char *in, unsigned int in_size, unsigned char *out, unsigned int *out_size, int order)
{
    if ((!in && in_size) || !out_size || in_size > 0x7fffffffu || (out && *out_size == 0)) { if (out_size) *out_size = 0; return nullptr; }
    unsigned char *alloc = nullptr;
    if (!out) {
        *out_size = hgpu_arith_compress_bound(in_size, order);
        alloc = out = (unsigned char *)malloc(*out_size);
        if (!out) { *out_size = 0; return nullptr; }
    }
    const long got = one_stream(ENC_ARITH, in, in_size, out, *out_size, (uint32_t)order);
    if (got < 0) { free(alloc); *out_size = 0; return nullptr; }
    *out_size = (unsigned int)got;
    return out;
}

unsigned char *arith_compress(unsigned char *in, unsigned int in_size, unsigned int *out_size, int order)
{
    return arith_compress_to(in, in_size, nullptr, out_size, order);
}

// ---- rANS Nx16 encode (method 5), rANS_static4x16pr.c:1203-1584: every bit of `order` means what it means there
// (PACK / RLE / STRIPE / CAT / X32 / STRIPE_NO0 in rans_nx16_encode_kernel, SIMD_AUTO here, :1234-1237).
unsigned int rans_compress_bound_4x16(unsigned int size, int order) { return hgpu_rans_nx16_compress_bound(size, order); }

unsigned char *rans_compress_to_4x16(unsigned char *in, unsigned int in_size, unsigned char *out, unsigned int *out_size, int order)
{
    if ((!in && in_size) || !out_size || in_size > 0x7fffffffu) { if (out_size) *out_size = 0; return nullptr; }
    unsigned char *alloc = nullptr;
    if (!out) {
        *out_size = hgpu_rans_nx16_compress_bound(in_size, order);
        alloc = out = (unsigned char *)malloc(*out_size);
        if (!out) { *out_size = 0; return nullptr; }
    }
    uint32_t ord = (uint32_t)order & 0x1ffffu;
    if ((order & (1 << 17)) && in_size >= 50000 && !(order & 8)) ord |= 4;          // RANS_ORDER_SIMD_AUTO
    const long got = one_stream(ENC_NX16, in, in_size, out, *out_size, ord);
    if (got <= 0) { free(alloc); *out_size = 0; return nullptr; }
    *out_size = (unsigned int)got;
    return out;
}

unsigned char *rans_compress_4x16(unsigned char *in, unsigned int in_size, unsigned int *out_size, int order)
{
    return rans_compress_to_4x16(in, in_size, nullptr, out_size, order);
}

void rans_set_cpu(int opts) { (void)opts; }                              // selects SIMD variants in the reference; nothing to select here

// ---- tok3 encode (method 8), tokenise_name3.c:1451-1665.  level and use_arith are accepted and ignored
// (one tokenisation, rANS sub-streams).  *last_start_p: offset just past the last complete name (:1476-1484).
uint8_t *tok3_encode_names(char *blk, int len, int level, int use_arith, int *out_len, int *last_start_p)
{
    (void)level; (void)use_arith;
    if (!blk || len <= 0 || !out_len) { if (out_len) *out_len = 0; return nullptr; }
    int last_start = 0;
    for (int i = 0; i < len; i++) if ((unsigned char)blk[i] <= '\n') last_start = i + 1;
    if (last_start_p) *last_start_p = last_start;
    uint32_t cap = hgpu_tok3_compress_bound((uint32_t)len), ilen = (uint32_t)len, got = 0;
    uint8_t *out = (uint8_t *)malloc(cap);
    if (!out) { *out_len = 0; return nullptr; }
    uint64_t ioff = 0, ooff = 0;
    int32_t st = 0;
    int rc;
    {
        ShimLock lock;
        hgpu_ctx *ctx = hgpu_shim_ctx();
        rc = ctx ? hgpu_tok3_encode_batch_host(ctx, (const uint8_t *)blk, &ioff, &ilen, 1, out, &ooff, &cap, &got, &st) : -1;
    }
    if (rc != HGPU_OK || st != HGPU_OK) { free(out); *out_len = 0; return nullptr; }
    *out_len = (int)got;
    return out;
}

// ---- fqzcomp encode (method 7), fqzcomp_qual.c:1615-1624.  vers >= 4 only (CRAM 3.1 stores qualities in their
// original orientation; the 3.0 layout with per-record reversal is not produced) and no caller-supplied parameters.
typedef struct { int num_records; uint32_t *len; uint32_t *flags; } hgpu_fqz_slice;   // fqz_slice, fqzcomp_qual.h:59-63
char *fqz_compress(int vers, void *slice, char *in, size_t uncomp_size, size_t *comp_size, int strat, void *gp)
{
    const hgpu_fqz_slice *s = (const hgpu_fqz_slice *)slice;
    if (comp_size) *comp_size = 0;
    if (!s || !in || !comp_size || gp || vers < 4 || uncomp_size == 0 || uncomp_size > 0x7fffffffu || s->num_records <= 0) return nullptr;
    // the reference clips / extends the record lengths so that they tile the block (:787-795)
    std::vector<uint32_t> lens((size_t)s->num_records);
    uint64_t tl = 0;
    uint32_t nrec = 0;
    for (int i = 0; i < s->num_records && tl < uncomp_size; i++) {
        uint32_t l = s->len[i];
        if (tl + l > uncomp_size) l = (uint32_t)(uncomp_size - tl);
        if (l == 0) break;
        lens[nrec++] = l; tl += l;
    }
    if (nrec == 0) return nullptr;
    if (tl < uncomp_size) lens[nrec - 1] += (uint32_t)(uncomp_size - tl);
    uint32_t ilen = (uint32_t)uncomp_size, cap = hgpu_fqz_compress_bound(ilen, nrec), got = 0;
    char *out = (char *)malloc(cap);
    if (!out) return nullptr;
    uint64_t ioff = 0, ooff = 0, roff = 0;
    int32_t st = 0;
    int rc;
    {
        ShimLock lock;
        hgpu_ctx *ctx = hgpu_shim_ctx();
        rc = ctx ? hgpu_fqz_encode_batch_host(ctx, (const uint8_t *)in, &ioff, &ilen, lens.data(), &roff, &nrec, 1, strat,
                                              (uint8_t *)out, &ooff, &cap, &got, &st) : -1;
    }
    if (rc != HGPU_OK || st != HGPU_OK) { free(out); return nullptr; }
    *comp_size = got;
    return out;
}

}  // extern "C"
