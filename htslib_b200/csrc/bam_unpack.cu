// BAM record unpack for sm_90a: the data movement of bam_read1 (htslib sam.c:784-860) plus the
// 4-bit SEQ expand and QUAL+33 of sam_format1_append (sam.c:4324-4404; nibble2base,
// sam_internal.h:63-118; add33, sam.c:4317-4322), over an inflated BAM record stream that is
// already resident in device memory (the output of the BGZF inflate kernel).
//
// Three steps, all on the device:
//  1. record index.  Records are a length-prefixed chain (block_size, sam.c:793-799), serial by
//     nature.  The caller passes candidate record starts (the BGZF block boundaries: htslib's
//     writer does not split records across blocks when it can avoid it, bgzf_flush_try sam.c:888),
//     one thread walks the chain of each segment speculatively, a fix-up pass re-walks only the
//     segments whose guessed start was not where the previous segment ended, a prefix sum of the
//     per-segment counts gives every record its global index.
//  2. layout: per-record l_data / l_qseq -> exclusive prefix sums (offsets of the SoA blobs).
//  3. unpack: one warp per record: bam1_core_t exactly as bam_read1 leaves it (l_extranul
//     padding, recomputed bin, CIGAR/qlen check), the bam1_t::data bytes, ASCII bases, QUAL+33.
#include "hgpu_internal.h"

namespace {

constexpr uint64_t BROKEN = ~0ull;

__device__ __forceinline__ uint32_t ld32(const uint8_t *p)
{
    return p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24;
}

// walk records from `pos` while pos < end; returns count (or BROKEN) and the exit position
__device__ uint64_t walk(const uint8_t *st, uint64_t len, uint64_t pos, uint64_t end, uint64_t &exitp,
                         uint64_t *emit, uint64_t emit_cap, uint64_t emit_base)
{
    uint64_t n = 0;
    while (pos < end) {
        if (len - pos < 4) { exitp = pos; return BROKEN; }
        int32_t bl = (int32_t)ld32(st + pos);
        if (bl < 32 || pos + 4 + (uint64_t)bl > len) { exitp = pos; return BROKEN; }
        if (emit && emit_base + n < emit_cap) emit[emit_base + n] = pos;
        n++;
        pos += 4 + (uint64_t)bl;
    }
    exitp = pos;
    return n;
}

__global__ void bam_seg_scan_kernel(const uint8_t *st, uint64_t len, const uint64_t *hint, uint64_t nseg,
                                    uint64_t *seg_start, uint64_t *seg_cnt, uint64_t *seg_exit)
{
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nseg) return;
    uint64_t s = hint ? hint[i] : 0, e = (hint && i + 1 < nseg) ? hint[i + 1] : len;
    if (s > len) s = len;
    if (e > len) e = len;
    uint64_t ex;
    seg_start[i] = s;
    seg_cnt[i] = walk(st, len, s, e, ex, nullptr, 0, 0);
    seg_exit[i] = ex;
}

// single CTA: make the chain consistent, then exclusive-scan the counts
__global__ void __launch_bounds__(1024)
bam_seg_fix_kernel(const uint8_t *st, uint64_t len, const uint64_t *hint, uint64_t nseg, uint64_t *seg_start,
                   uint64_t *seg_cnt, uint64_t *seg_exit, uint64_t *seg_base, uint64_t *n_rec)
{
    __shared__ uint64_t part[1024];
    __shared__ int again;
    const uint32_t t = threadIdx.x;
    for (;;) {
        if (t == 0) again = 0;
        __syncthreads();
        // phase A: who starts in the wrong place?
        for (uint64_t base = 0; base < nseg; base += 1024) {
            uint64_t i = base + t;
            bool fix = false;
            uint64_t want = 0;
            if (i >= 1 && i < nseg) {
                uint64_t pe = seg_exit[i - 1];
                // a broken predecessor leaves its exit where it stopped; successors keep their guess
                if (seg_cnt[i - 1] != BROKEN && pe != seg_start[i]) { fix = true; want = pe; }
            }
            __syncthreads();
            if (fix) {
                uint64_t e = i + 1 < nseg ? hint[i + 1] : len, ex;
                if (e > len) e = len;
                seg_start[i] = want;
                seg_cnt[i] = walk(st, len, want, e, ex, nullptr, 0, 0);
                seg_exit[i] = ex;
                again = 1;
            }
            __syncthreads();
        }
        if (!again) break;
        __syncthreads();
    }
    // exclusive scan of counts (chunked over the CTA)
    const uint64_t per = (nseg + 1023) / 1024;
    uint64_t lo = (uint64_t)t * per, hi = lo + per < nseg ? lo + per : nseg, sum = 0;
    bool broken = false;
    for (uint64_t i = lo; i < hi; i++) { uint64_t c = seg_cnt[i]; if (c == BROKEN) broken = true; else sum += c; }
    part[t] = sum;
    __syncthreads();
    if (__syncthreads_or(broken)) { if (t == 0) *n_rec = BROKEN; return; }
    if (t == 0) {
        uint64_t run = 0;
        for (int k = 0; k < 1024; k++) { uint64_t v = part[k]; part[k] = run; run += v; }
        *n_rec = run;
    }
    __syncthreads();
    uint64_t run = part[t];
    for (uint64_t i = lo; i < hi; i++) { seg_base[i] = run; run += seg_cnt[i]; }
}

__global__ void bam_seg_emit_kernel(const uint8_t *st, uint64_t len, const uint64_t *hint, uint64_t nseg,
                                    const uint64_t *seg_start, const uint64_t *seg_base, uint64_t *rec_off,
                                    uint64_t rec_cap)
{
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nseg) return;
    uint64_t e = (hint && i + 1 < nseg) ? hint[i + 1] : len, ex;
    if (e > len) e = len;
    walk(st, len, seg_start[i], e, ex, rec_off, rec_cap, seg_base[i]);
}

// ---------------------------------------------------------------------------------------------
// sizes + generic u64 exclusive scan (three passes, 1024-element tiles)
// ---------------------------------------------------------------------------------------------
struct RecGeom { int32_t bl; uint32_t qn, xn, n_cigar, lq; bool ok, missing_nul; uint32_t l_data; };

// the validity rules of bam_read1 (sam.c:799, :824-828) and fixup_missing_qname_nul (:763-778)
__device__ __forceinline__ RecGeom geom(const uint8_t *rec)
{
    RecGeom g;
    g.bl = (int32_t)ld32(rec);
    g.qn = rec[12];
    g.n_cigar = ld32(rec + 16) & 0xffffu;
    int32_t lq = (int32_t)ld32(rec + 20);
    g.lq = (uint32_t)lq;
    g.xn = (g.qn & 3) ? 4 - (g.qn & 3) : 0;
    uint64_t nl = (uint64_t)(uint32_t)(g.bl - 32) + g.xn;
    g.ok = !(g.bl < 32 || nl > 0x7fffffffull || lq < 0 || g.qn < 1);
    if (g.ok && ((uint64_t)g.n_cigar << 2) + g.qn + g.xn + (((uint64_t)g.lq + 1) >> 1) + (uint64_t)g.lq > nl) g.ok = false;
    g.missing_nul = g.ok && rec[36 + g.qn - 1] != 0;
    if (g.missing_nul && g.xn == 0) nl += 4;
    g.l_data = g.ok ? (uint32_t)nl : 0;
    if (!g.ok) g.lq = 0;
    return g;
}

__global__ void bam_sizes_kernel(const uint8_t *st, const uint64_t *rec_off, uint64_t n, uint64_t *data_sz, uint64_t *seq_sz)
{
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    if (i == n) { data_sz[n] = 0; seq_sz[n] = 0; return; }
    RecGeom g = geom(st + rec_off[i]);
    data_sz[i] = g.l_data;
    seq_sz[i] = g.lq;
}

constexpr int TILE = 1024;

__global__ void __launch_bounds__(256) scan_tiles_reduce(const uint64_t *a, const uint64_t *b, uint64_t n, uint64_t *ta, uint64_t *tb)
{
    __shared__ uint64_t sa[256], sb[256];
    uint64_t base = (uint64_t)blockIdx.x * TILE, va = 0, vb = 0;
    for (int k = 0; k < 4; k++) { uint64_t i = base + threadIdx.x + 256 * k; if (i < n) { va += a[i]; vb += b[i]; } }
    sa[threadIdx.x] = va; sb[threadIdx.x] = vb;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) { sa[threadIdx.x] += sa[threadIdx.x + s]; sb[threadIdx.x] += sb[threadIdx.x + s]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { ta[blockIdx.x] = sa[0]; tb[blockIdx.x] = sb[0]; }
}

__global__ void __launch_bounds__(1024) scan_tile_sums(uint64_t *ta, uint64_t *tb, uint64_t nt)
{
    __shared__ uint64_t pa[1024], pb[1024];
    const uint32_t t = threadIdx.x;
    const uint64_t per = (nt + 1023) / 1024;
    uint64_t lo = (uint64_t)t * per, hi = lo + per < nt ? lo + per : nt, sa = 0, sb = 0;
    for (uint64_t i = lo; i < hi; i++) { sa += ta[i]; sb += tb[i]; }
    pa[t] = sa; pb[t] = sb;
    __syncthreads();
    if (t == 0) {
        uint64_t ra = 0, rb = 0;
        for (int k = 0; k < 1024; k++) { uint64_t x = pa[k], y = pb[k]; pa[k] = ra; pb[k] = rb; ra += x; rb += y; }
    }
    __syncthreads();
    uint64_t ra = pa[t], rb = pb[t];
    for (uint64_t i = lo; i < hi; i++) { uint64_t x = ta[i], y = tb[i]; ta[i] = ra; tb[i] = rb; ra += x; rb += y; }
}

__global__ void __launch_bounds__(256) scan_tiles_apply(uint64_t *a, uint64_t *b, uint64_t n, const uint64_t *ta, const uint64_t *tb)
{
    // one warp-shuffle scan per 1024-element tile: 256 threads x 4 consecutive elements
    __shared__ uint64_t wa[8], wb[8];
    uint64_t base = (uint64_t)blockIdx.x * TILE + (uint64_t)threadIdx.x * 4;
    uint64_t xa[4], xb[4], sa = 0, sb = 0;
    for (int k = 0; k < 4; k++) { uint64_t i = base + k; xa[k] = i < n ? a[i] : 0; xb[k] = i < n ? b[i] : 0; sa += xa[k]; sb += xb[k]; }
    uint64_t ia = sa, ib = sb;
    const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int d = 1; d < 32; d <<= 1) {
        uint64_t ya = __shfl_up_sync(0xffffffffu, ia, d), yb = __shfl_up_sync(0xffffffffu, ib, d);
        if (lane >= (uint32_t)d) { ia += ya; ib += yb; }
    }
    if (lane == 31) { wa[w] = ia; wb[w] = ib; }
    __syncthreads();
    uint64_t oa = ta[blockIdx.x], ob = tb[blockIdx.x];
    for (uint32_t k = 0; k < w; k++) { oa += wa[k]; ob += wb[k]; }
    uint64_t ra = oa + ia - sa, rb = ob + ib - sb;
    for (int k = 0; k < 4; k++) { uint64_t i = base + k; if (i < n) { a[i] = ra; b[i] = rb; } ra += xa[k]; rb += xb[k]; }
}

// ---------------------------------------------------------------------------------------------
// unpack: one warp per record
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint8_t nt16(uint32_t k)
{
    // "=ACMGRSVTWYHKDBN" (seq_nt16_str, hts.c:260) as two 64-bit immediates
    const uint64_t a = ((uint64_t)'=') | ((uint64_t)'A' << 8) | ((uint64_t)'C' << 16) | ((uint64_t)'M' << 24) |
                       ((uint64_t)'G' << 32) | ((uint64_t)'R' << 40) | ((uint64_t)'S' << 48) | ((uint64_t)'V' << 56);
    const uint64_t b = ((uint64_t)'T') | ((uint64_t)'W' << 8) | ((uint64_t)'Y' << 16) | ((uint64_t)'H' << 24) |
                       ((uint64_t)'K' << 32) | ((uint64_t)'D' << 40) | ((uint64_t)'B' << 48) | ((uint64_t)'N' << 56);
    return (uint8_t)(((k & 8) ? b : a) >> (8 * (k & 7)));
}

__device__ __forceinline__ int reg2bin(int64_t beg, int64_t end)       // hts_reg2bin(beg,end,14,5), hts.h:1516
{
    --end;
    if (beg >> 14 == end >> 14) return 4681 + (int)(beg >> 14);
    if (beg >> 17 == end >> 17) return 585 + (int)(beg >> 17);
    if (beg >> 20 == end >> 20) return 73 + (int)(beg >> 20);
    if (beg >> 23 == end >> 23) return 9 + (int)(beg >> 23);
    if (beg >> 26 == end >> 26) return 1 + (int)(beg >> 26);
    return 0;
}

__global__ void __launch_bounds__(256)
bam_unpack_kernel(const uint8_t *st, const uint64_t *rec_off, uint64_t n, hgpu_bam1_core *core, uint8_t *data,
                  const uint64_t *data_off, uint8_t *seq, uint8_t *qual, const uint64_t *seq_off, int32_t *status)
{
    const uint32_t lane = threadIdx.x & 31;
    uint64_t r = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (r >= n) return;
    const uint8_t *rec = st + rec_off[r];
    RecGeom g = geom(rec);
    if (!g.ok) {
        if (lane == 0) {
            if (status) status[r] = -4;
            if (core) { hgpu_bam1_core z = {}; core[r] = z; }
        }
        return;
    }
    const uint8_t *x = rec + 4, *body = rec + 36;
    hgpu_bam1_core c;
    c.tid = (int32_t)ld32(x);
    c.pos = (int32_t)ld32(x + 4);
    uint32_t x2 = ld32(x + 8), x3 = ld32(x + 12);
    c.bin = (uint16_t)(x2 >> 16);
    c.qual = (x2 >> 8) & 0xff;
    c.flag = (uint16_t)(x3 >> 16);
    c.n_cigar = x3 & 0xffff;
    c.l_qseq = (int32_t)g.lq;
    c.mtid = (int32_t)ld32(x + 20);
    c.mpos = (int32_t)ld32(x + 24);
    c.isize = (int32_t)ld32(x + 28);
    uint32_t xn = g.xn, lqn = g.qn;
    if (g.missing_nul) { xn = xn ? xn - 1 : 3; lqn++; }
    c.l_extranul = (uint8_t)xn;
    c.l_qname = (uint16_t)(lqn + xn);
    const uint32_t rest = (uint32_t)(g.bl - 32) - g.qn;
    if (data) {
        uint8_t *o = data + data_off[r];
        for (uint32_t i = lane; i < g.qn; i += 32) o[i] = body[i];
        if (lane < (g.missing_nul ? 1u : 0u) + xn) o[g.qn + lane] = 0;
        const uint8_t *from = body + g.qn;
        uint8_t *to = o + lqn + xn;
        for (uint32_t i = lane; i < rest; i += 32) to[i] = from[i];
    }
    const uint8_t *cig = body + g.qn, *sq = cig + 4 * (size_t)c.n_cigar, *ql = sq + ((g.lq + 1) >> 1);
    int st_code = 0;
    if (c.n_cigar > 0) {
        int64_t rlen = 0, qlen = 0;
        for (uint32_t k = lane; k < c.n_cigar; k += 32) {
            uint32_t op = ld32(cig + 4 * (size_t)k);
            uint32_t type = (0x3C1A7u >> ((op & 0xf) << 1)) & 3;
            if (type & 1) qlen += op >> 4;
            if (type & 2) rlen += op >> 4;
        }
        for (int d = 16; d > 0; d >>= 1) {
            rlen += __shfl_xor_sync(0xffffffffu, rlen, d);
            qlen += __shfl_xor_sync(0xffffffffu, qlen, d);
        }
        if (ld32(cig) == (4u | (g.lq << 4)) && c.tid >= 0 && c.pos >= 0) st_code = 1;   // bam_tag2cigar's trigger, sam.c:685-692
        if ((c.flag & 4) || rlen == 0) rlen = 1;
        c.bin = (uint16_t)reg2bin(c.pos, c.pos + rlen);
        if (g.lq > 0 && !(c.flag & 4) && qlen != (int64_t)g.lq) st_code = -4;
    }
    if (lane == 0) {
        if (core) core[r] = c;
        if (status) status[r] = st_code;
    }
    if (seq) {
        uint8_t *o = seq + seq_off[r];
        for (uint32_t i = lane; i < g.lq; i += 32) o[i] = nt16((sq[i >> 1] >> ((~i & 1) << 2)) & 0xf);
    }
    if (qual) {
        uint8_t *o = qual + seq_off[r];
        const bool absent = g.lq && ql[0] == 0xff;
        for (uint32_t i = lane; i < g.lq; i += 32) o[i] = absent ? ql[i] : (uint8_t)(ql[i] + 33);
    }
}

} // namespace

extern "C" int hgpu_bam_index_records_dev(hgpu_ctx *ctx, const uint8_t *d_stream, uint64_t len,
                                          const uint64_t *d_hint_off, uint64_t n_hint, uint64_t *d_rec_off,
                                          uint64_t rec_cap, uint64_t *d_n_rec, void *stream)
{
    if (!ctx || !d_stream || !d_n_rec) { hgpu_set_error("bad argument"); return HGPU_ERR_ARG; }
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    uint64_t nseg = d_hint_off && n_hint ? n_hint : 1;
    int rc = hgpu_ensure_bam(ctx, nseg * 4 * sizeof(uint64_t));
    if (rc) return rc;
    uint64_t *seg_start = (uint64_t *)ctx->d_bam, *seg_cnt = seg_start + nseg, *seg_exit = seg_cnt + nseg, *seg_base = seg_exit + nseg;
    const uint64_t *hint = nseg > 1 || (d_hint_off && n_hint) ? d_hint_off : nullptr;
    unsigned blocks = (unsigned)((nseg + 127) / 128);
    bam_seg_scan_kernel<<<blocks, 128, 0, st>>>(d_stream, len, hint, nseg, seg_start, seg_cnt, seg_exit);
    bam_seg_fix_kernel<<<1, 1024, 0, st>>>(d_stream, len, hint, nseg, seg_start, seg_cnt, seg_exit, seg_base, d_n_rec);
    if (d_rec_off)
        bam_seg_emit_kernel<<<blocks, 128, 0, st>>>(d_stream, len, hint, nseg, seg_start, seg_base, d_rec_off, rec_cap);
    hgpu_count_launch(d_rec_off ? 3 : 2);
    return hgpu_check(cudaGetLastError(), "bam index launch");
}

extern "C" int hgpu_bam_layout_dev(hgpu_ctx *ctx, const uint8_t *d_stream, uint64_t len, const uint64_t *d_rec_off,
                                   uint64_t n, uint64_t *d_data_off, uint64_t *d_seq_off, void *stream)
{
    (void)len;
    if (!ctx || !d_stream || !d_data_off || !d_seq_off) { hgpu_set_error("bad argument"); return HGPU_ERR_ARG; }
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    uint64_t m = n + 1, nt = (m + TILE - 1) / TILE;
    int rc = hgpu_ensure_bam(ctx, nt * 2 * sizeof(uint64_t) + 64);
    if (rc) return rc;
    uint64_t *ta = (uint64_t *)ctx->d_bam, *tb = ta + nt;
    bam_sizes_kernel<<<(unsigned)((m + 255) / 256), 256, 0, st>>>(d_stream, d_rec_off, n, d_data_off, d_seq_off);
    scan_tiles_reduce<<<(unsigned)nt, 256, 0, st>>>(d_data_off, d_seq_off, m, ta, tb);
    scan_tile_sums<<<1, 1024, 0, st>>>(ta, tb, nt);
    scan_tiles_apply<<<(unsigned)nt, 256, 0, st>>>(d_data_off, d_seq_off, m, ta, tb);
    hgpu_count_launch(4);
    return hgpu_check(cudaGetLastError(), "bam layout launch");
}

extern "C" int hgpu_bam_unpack_dev(hgpu_ctx *ctx, const uint8_t *d_stream, uint64_t len, const uint64_t *d_rec_off,
                                   uint64_t n, hgpu_bam1_core *d_core, uint8_t *d_data, const uint64_t *d_data_off,
                                   uint8_t *d_seq, uint8_t *d_qual, const uint64_t *d_seq_off, int32_t *d_status,
                                   void *stream)
{
    (void)len;
    if (!ctx || !d_stream || !d_rec_off) { hgpu_set_error("bad argument"); return HGPU_ERR_ARG; }
    if ((d_data && !d_data_off) || ((d_seq || d_qual) && !d_seq_off)) { hgpu_set_error("offsets missing"); return HGPU_ERR_ARG; }
    if (n == 0) return HGPU_OK;
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    uint64_t blocks = (n * 32 + 255) / 256;
    bam_unpack_kernel<<<(unsigned)blocks, 256, 0, st>>>(d_stream, d_rec_off, n, d_core, d_data, d_data_off, d_seq, d_qual,
                                                       d_seq_off, d_status);
    hgpu_count_launch();
    return hgpu_check(cudaGetLastError(), "bam unpack launch");
}

// =============================================================================================
// BAM record PACK — the inverse data movement, bam_write1 (sam.c:862-928): bam1_core_t + data ->
// block_size, 32-byte little-endian core, qname without the padding NULs, the rest verbatim.
// Records with more than 65535 CIGAR operations need the CG-tag rewrite (:899-925): they are
// flagged (status 1) and given zero bytes; qname > 254 / positions beyond INT_MAX -> status -1.
// =============================================================================================
namespace {

__global__ void bam_pack_sizes_kernel(const hgpu_bam1_core *core, const uint64_t *data_off, uint64_t n,
                                      uint64_t *out_sz, uint64_t *dummy)
{
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    uint64_t sz = 0;
    if (i < n) {
        hgpu_bam1_core c = core[i];
        uint32_t l_data = (uint32_t)(data_off[i + 1] - data_off[i]);
        bool bad = (uint32_t)c.l_qname - c.l_extranul > 255u || c.n_cigar > 0xffffu || c.pos > 0x7fffffffLL ||
                   c.mpos > 0x7fffffffLL || c.isize < -0x80000000LL || c.isize > 0x7fffffffLL;
        sz = bad ? 0 : 4ull + l_data - c.l_extranul + 32;
    }
    out_sz[i] = sz;
    dummy[i] = 0;
}

__global__ void __launch_bounds__(256)
bam_pack_kernel(const hgpu_bam1_core *core, const uint8_t *data, const uint64_t *data_off, uint64_t n,
                uint8_t *out, const uint64_t *out_off, int32_t *status)
{
    const uint32_t lane = threadIdx.x & 31;
    uint64_t r = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (r >= n) return;
    hgpu_bam1_core c = core[r];
    const uint8_t *d = data + data_off[r];
    const uint32_t l_data = (uint32_t)(data_off[r + 1] - data_off[r]);
    const uint32_t qn = (uint32_t)c.l_qname - c.l_extranul;
    int st = 0;
    if (qn > 255u || c.pos > 0x7fffffffLL || c.mpos > 0x7fffffffLL || c.isize < -0x80000000LL || c.isize > 0x7fffffffLL) st = -1;
    else if (c.n_cigar > 0xffffu) st = 1;
    if (lane == 0 && status) status[r] = st;
    if (st) return;
    uint8_t *o = out + out_off[r];
    const uint32_t block_len = l_data - c.l_extranul + 32;
    if (lane < 9) {
        uint32_t v;
        switch (lane) {
        case 0: v = block_len; break;
        case 1: v = (uint32_t)c.tid; break;
        case 2: v = (uint32_t)c.pos; break;
        case 3: v = (uint32_t)c.bin << 16 | (uint32_t)c.qual << 8 | qn; break;
        case 4: v = (uint32_t)c.flag << 16 | (c.n_cigar & 0xffffu); break;
        case 5: v = (uint32_t)c.l_qseq; break;
        case 6: v = (uint32_t)c.mtid; break;
        case 7: v = (uint32_t)c.mpos; break;
        default: v = (uint32_t)c.isize; break;
        }
        uint8_t *p = o + 4 * lane;
        p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24);
    }
    for (uint32_t i = lane; i < qn; i += 32) o[36 + i] = d[i];
    const uint32_t rest = l_data - c.l_qname;
    const uint8_t *from = d + c.l_qname;
    uint8_t *to = o + 36 + qn;
    for (uint32_t i = lane; i < rest; i += 32) to[i] = from[i];
}

} // namespace

// d_out_off: n+1 entries, filled here (exclusive prefix sums of the record sizes); pass d_out = NULL
// to only compute the layout.
extern "C" int hgpu_bam_pack_dev(hgpu_ctx *ctx, const hgpu_bam1_core *d_core, const uint8_t *d_data,
                                 const uint64_t *d_data_off, uint64_t n, uint8_t *d_out, uint64_t *d_out_off,
                                 int32_t *d_status, void *stream)
{
    if (!ctx || !d_core || !d_data_off || !d_out_off) { hgpu_set_error("bad argument"); return HGPU_ERR_ARG; }
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    if (!d_out) {
        uint64_t m = n + 1, nt = (m + TILE - 1) / TILE;
        int rc = hgpu_ensure_bam(ctx, (nt * 2 + m) * sizeof(uint64_t) + 64);
        if (rc) return rc;
        uint64_t *ta = (uint64_t *)ctx->d_bam, *tb = ta + nt, *dummy = tb + nt;
        bam_pack_sizes_kernel<<<(unsigned)((m + 255) / 256), 256, 0, st>>>(d_core, d_data_off, n, d_out_off, dummy);
        scan_tiles_reduce<<<(unsigned)nt, 256, 0, st>>>(d_out_off, dummy, m, ta, tb);
        scan_tile_sums<<<1, 1024, 0, st>>>(ta, tb, nt);
        scan_tiles_apply<<<(unsigned)nt, 256, 0, st>>>(d_out_off, dummy, m, ta, tb);
        hgpu_count_launch(4);
        return hgpu_check(cudaGetLastError(), "bam pack layout launch");
    }
    if (n == 0) return HGPU_OK;
    if (!d_data) { hgpu_set_error("bad argument"); return HGPU_ERR_ARG; }
    uint64_t blocks = (n * 32 + 255) / 256;
    bam_pack_kernel<<<(unsigned)blocks, 256, 0, st>>>(d_core, d_data, d_data_off, n, d_out, d_out_off, d_status);
    hgpu_count_launch();
    return hgpu_check(cudaGetLastError(), "bam pack launch");
}

// =============================================================================================
// SAM text — sam_format1_append (sam.c:4324-4404) + the '\n' sam_write1 adds, for n unpacked records.
// One walker per record formats into `out` at the record's offset; the same walker run with a null
// sink is the size pass (its sizes are prefix-summed into out_off).  Fields exactly as the
// reference prints them: QNAME (without the padding NULs), FLAG, RNAME / '*', POS+1, MAPQ,
// CIGAR ("<len><op>" per operation, BAM_CIGAR_STR "MIDNSHP=XB??????", or '*'), RNEXT ('*', '=' or the
// name), PNEXT+1, TLEN, SEQ (seq_nt16_str "=ACMGRSVTWYHKDBN", high nibble first, sam_internal.h:63-118)
// or '*', QUAL+33 or '*' when qual[0] == 0xff (sam.c:4370), then the aux fields TAG:TYPE:VALUE
// (sam_format_aux1, htslib/sam.h:1463-1630): A, c/C/s/S/i/I -> 'i', Z, H, B arrays of integers.
// Floating-point values ('f', 'd', B:f) are printed by the reference with printf("%g") / kputd;
// records that carry one are flagged status 1 and left to the host (zero bytes), so is a record
// with corrupted aux data (status -1, the reference returns -1 there).
// =============================================================================================
namespace {

struct Sink {
    uint8_t *p;            // null: count only
    uint64_t n;
    __device__ __forceinline__ void put(uint32_t c) { if (p) p[n] = (uint8_t)c; n++; }
    __device__ __forceinline__ void puts(const uint8_t *s, uint32_t l) { if (p) for (uint32_t i = 0; i < l; i++) p[n + i] = s[i]; n += l; }
    __device__ void putu(uint64_t v)
    {
        uint8_t b[20];
        int k = 0;
        do { b[k++] = (uint8_t)('0' + v % 10); v /= 10; } while (v);
        if (p) for (int i = 0; i < k; i++) p[n + i] = b[k - 1 - i];
        n += k;
    }
    __device__ void puti(int64_t v) { if (v < 0) { put('-'); putu((uint64_t)0 - (uint64_t)v); } else putu((uint64_t)v); }
};

__device__ int sam_format_record(const hgpu_bam1_core &c, const uint8_t *d, uint32_t l_data, const uint8_t *names,
                                 const uint64_t *name_off, int32_t n_targets, Sink &o)
{
    if (c.l_qname == 0) return -1;
    const uint32_t cig_off = c.l_qname, seq_off = cig_off + 4u * c.n_cigar, qual_off = seq_off + ((uint32_t)c.l_qseq + 1u) / 2u,
                   aux_off = qual_off + (uint32_t)c.l_qseq;
    if (c.l_qseq < 0 || aux_off > l_data || c.tid >= n_targets || c.mtid >= n_targets) return -1;
    o.puts(d, (uint32_t)c.l_qname - 1u - c.l_extranul); o.put('\t');
    o.putu(c.flag); o.put('\t');
    if (c.tid >= 0) { o.puts(names + name_off[c.tid], (uint32_t)(name_off[c.tid + 1] - name_off[c.tid])); o.put('\t'); }
    else { o.put('*'); o.put('\t'); }
    o.puti(c.pos + 1); o.put('\t');
    o.putu(c.qual); o.put('\t');
    if (c.n_cigar) {
        for (uint32_t i = 0; i < c.n_cigar; i++) {
            const uint8_t *q = d + cig_off + 4u * i;
            const uint32_t v = q[0] | q[1] << 8 | q[2] << 16 | (uint32_t)q[3] << 24;
            o.putu(v >> 4);
            o.put("MIDNSHP=XB??????"[v & 15]);
        }
    } else o.put('*');
    o.put('\t');
    if (c.mtid < 0) { o.put('*'); o.put('\t'); }
    else if (c.mtid == c.tid) { o.put('='); o.put('\t'); }
    else { o.puts(names + name_off[c.mtid], (uint32_t)(name_off[c.mtid + 1] - name_off[c.mtid])); o.put('\t'); }
    o.puti(c.mpos + 1); o.put('\t');
    o.puti(c.isize); o.put('\t');
    if (c.l_qseq) {
        const uint8_t *s = d + seq_off, *q = d + qual_off;
        if (o.p) for (int32_t i = 0; i < c.l_qseq; i++) o.p[o.n + i] = "=ACMGRSVTWYHKDBN"[(s[i >> 1] >> ((~i & 1) << 2)) & 15];
        o.n += (uint32_t)c.l_qseq;
        o.put('\t');
        if (q[0] == 0xff) o.put('*');
        else { if (o.p) for (int32_t i = 0; i < c.l_qseq; i++) o.p[o.n + i] = (uint8_t)(q[i] + 33); o.n += (uint32_t)c.l_qseq; }
    } else { o.put('*'); o.put('\t'); o.put('*'); }
    const uint8_t *s = d + aux_off, *end = d + l_data;
    while (end - s >= 4) {
        o.put('\t');
        o.put(s[0]); o.put(s[1]); o.put(':');
        const uint8_t type = s[2];
        s += 3;
        auto le = [&](int nb) { uint64_t v = 0; for (int k = 0; k < nb; k++) v |= (uint64_t)s[k] << (8 * k); return v; };
        if (type == 'C') { o.put('i'); o.put(':'); o.putu(s[0]); s += 1; }
        else if (type == 'c') { o.put('i'); o.put(':'); o.puti((int8_t)s[0]); s += 1; }
        else if (type == 'S') { if (end - s < 2) return -1; o.put('i'); o.put(':'); o.putu(le(2)); s += 2; }
        else if (type == 's') { if (end - s < 2) return -1; o.put('i'); o.put(':'); o.puti((int16_t)le(2)); s += 2; }
        else if (type == 'I') { if (end - s < 4) return -1; o.put('i'); o.put(':'); o.putu(le(4)); s += 4; }
        else if (type == 'i') { if (end - s < 4) return -1; o.put('i'); o.put(':'); o.puti((int32_t)le(4)); s += 4; }
        else if (type == 'A') { o.put('A'); o.put(':'); o.put(s[0]); s += 1; }
        else if (type == 'f' || type == 'd') return 1;
        else if (type == 'Z' || type == 'H') {
            o.put(type); o.put(':');
            while (s < end && *s) o.put(*s++);
            if (s >= end) return -1;
            s++;
        } else if (type == 'B') {
            const uint8_t sub = *s++;
            int sz = (sub == 'A' || sub == 'c' || sub == 'C') ? 1 : (sub == 's' || sub == 'S') ? 2 : (sub == 'i' || sub == 'I' || sub == 'f') ? 4 : 0;
            if (sz == 0 || end - s < 4) return -1;
            const uint32_t cnt = (uint32_t)le(4);
            s += 4;
            if ((size_t)(end - s) / (size_t)sz < cnt) return -1;
            if (sub == 'f') return 1;
            if (sub == 'A') return -1;                               // sam_format_aux1's second switch has no 'A'
            o.put('B'); o.put(':'); o.put(sub);
            for (uint32_t i = 0; i < cnt; i++) {
                o.put(',');
                const uint64_t v = le(sz);
                if (sub == 'c') o.puti((int8_t)v); else if (sub == 's') o.puti((int16_t)v); else if (sub == 'i') o.puti((int32_t)v); else o.putu(v);
                s += sz;
            }
        } else return -1;
    }
    o.put('\n');
    return 0;
}

__global__ void sam_format_kernel(const hgpu_bam1_core *core, const uint8_t *data, const uint64_t *data_off, uint64_t n,
                                  const uint8_t *names, const uint64_t *name_off, int32_t n_targets,
                                  uint8_t *out, uint64_t *out_off, uint64_t *dummy, int32_t *status)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    if (i == n) { if (!out) { out_off[n] = 0; dummy[n] = 0; } return; }
    const hgpu_bam1_core c = core[i];
    const uint32_t l_data = (uint32_t)(data_off[i + 1] - data_off[i]);
    Sink o;
    o.p = out ? out + out_off[i] : nullptr;
    o.n = 0;
    if (out && out_off[i + 1] == out_off[i]) return;                 // flagged by the size pass: no bytes
    const int rc = sam_format_record(c, data + data_off[i], l_data, names, name_off, n_targets, o);
    if (!out) { out_off[i] = rc == 0 ? o.n : 0; dummy[i] = 0; if (status) status[i] = rc; }
}

}  // namespace

// d_out == NULL: fills d_out_off[0..n] (exclusive prefix sums of the line lengths; total = last entry) and d_status.
// d_out != NULL: writes the lines.  d_names / d_name_off[0..n_targets]: the @SQ names of the header, back to back.
extern "C" int hgpu_sam_format_dev(hgpu_ctx *ctx, const hgpu_bam1_core *d_core, const uint8_t *d_data, const uint64_t *d_data_off,
                                   uint64_t n, const uint8_t *d_names, const uint64_t *d_name_off, int32_t n_targets,
                                   uint8_t *d_out, uint64_t *d_out_off, int32_t *d_status, void *stream)
{
    if (!ctx || !d_core || !d_data || !d_data_off || !d_out_off || (n_targets > 0 && (!d_names || !d_name_off))) { hgpu_set_error("bad argument"); return HGPU_ERR_ARG; }
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    const uint64_t m = n + 1, nt = (m + TILE - 1) / TILE;
    if (!d_out) {
        int rc = hgpu_ensure_bam(ctx, (nt * 2 + m) * sizeof(uint64_t) + 64);
        if (rc) return rc;
        uint64_t *ta = (uint64_t *)ctx->d_bam, *tb = ta + nt, *dummy = tb + nt;
        sam_format_kernel<<<(unsigned)((m + 127) / 128), 128, 0, st>>>(d_core, d_data, d_data_off, n, d_names, d_name_off, n_targets, nullptr, d_out_off, dummy, d_status);
        scan_tiles_reduce<<<(unsigned)nt, 256, 0, st>>>(d_out_off, dummy, m, ta, tb);
        scan_tile_sums<<<1, 1024, 0, st>>>(ta, tb, nt);
        scan_tiles_apply<<<(unsigned)nt, 256, 0, st>>>(d_out_off, dummy, m, ta, tb);
        hgpu_count_launch(4);
        return hgpu_check(cudaGetLastError(), "sam format layout launch");
    }
    if (n == 0) return HGPU_OK;
    sam_format_kernel<<<(unsigned)((m + 127) / 128), 128, 0, st>>>(d_core, d_data, d_data_off, n, d_names, d_name_off, n_targets, d_out, d_out_off, nullptr, nullptr);
    hgpu_count_launch();
    return hgpu_check(cudaGetLastError(), "sam format launch");
}
